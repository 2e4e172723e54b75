"""Host-side checks of the sharded full sort (streaming.sort.init_sharded_sort_state), no GPU needed: choose_splitters against a
brute-force restatement and the balance bound of DESIGN.md, the argument checks, PhysicalSort's plumbing, the C header, and the
collective refusal of a rank that would receive too many rows on a gloo world of 2."""

import math
import os
import socket

import numpy as np
import pytest

from bodo_b200 import _lib
from bodo_b200._lib import B200Error
from bodo_b200.physical import OperatorResult, PhysicalSort
from bodo_b200.streaming import sort as S
from bodo_b200.table import ArrTypes, Column, CTypes, Table

COLS = ["a", "b", "c"]


# ---- choose_splitters: a model of P ranks whose rows are one-key records (class, word, rank, position) ----
def rank_rows(keys_per_rank):
    """Every rank's sorted rows as record tuples (class 0 for NA, 1 otherwise; word; rank; sorted position)."""
    out = []
    for r, keys in enumerate(keys_per_rank):
        ks = sorted(keys, key=lambda k: (k is not None, 0 if k is None else k))  # NA first, then ascending
        out.append([(0 if k is None else 1, 0 if k is None else k, r, i) for i, k in enumerate(ks)])
    return out


def samples(rows, s):
    """The sample records and weights of one rank: positions floor(i n / s') for s' = min(s, n)."""
    n = len(rows)
    m = min(s, n)
    q = [i * n // m for i in range(m)] + [n] if m else [0]
    return [rows[q[i]] for i in range(m)], [q[i + 1] - q[i] for i in range(m)]


def brute_splitters(recs, weights, P):
    """Splitter k: the first record in tuple order whose exclusive cumulative weight is >= k N / P (None: +inf)."""
    pairs = sorted(zip(recs, weights))
    total = sum(weights)
    out = []
    for k in range(1, P):
        acc, pick = 0, None
        for t, w in pairs:
            if acc * P >= k * total:
                pick = t
                break
            acc += w
        out.append(pick)
    return out


def gather(rows, s):
    recs, ws = [], []
    for rr in rows:
        r, w = samples(rr, s)
        recs += r
        ws += w
    return recs, ws


def receive_counts(rows, spl, P):
    """Rows each rank receives: those whose tuple lies in [splitter k, splitter k + 1), by brute force over every row."""
    every = [t for rr in rows for t in rr]
    bounds = [0] + [len(every) if t is None else sum(1 for x in every if x < t) for t in spl] + [len(every)]
    return [bounds[k + 1] - bounds[k] for k in range(P)]


def check_model(keys_per_rank, P, s):
    rows = rank_rows(keys_per_rank)
    recs, ws = gather(rows, s)
    arr = np.array(recs, dtype=np.uint64).reshape(len(recs), 4)
    got = S.choose_splitters(arr, ws, P)
    exp = brute_splitters(recs, ws, P)
    finite = [t for t in exp if t is not None]
    assert exp[len(finite):] == [None] * (P - 1 - len(finite))  # once +inf, the later splitters are +inf too
    assert [tuple(int(x) for x in row) for row in got] == finite
    recv = receive_counts(rows, exp, P)
    N = sum(len(k) for k in keys_per_rank)
    G = sum(math.ceil(len(k) / min(s, len(k))) for k in keys_per_rank if len(k))
    assert sum(recv) == N
    assert all(c < math.ceil(N / P) + 2 * G for c in recv), (recv, N, G)
    # the same records in another order give the same splitters
    perm = np.random.default_rng(len(recs)).permutation(len(recs))
    again = S.choose_splitters(arr[perm], np.asarray(ws)[perm], P)
    np.testing.assert_array_equal(again, got)
    return got, recv


@pytest.mark.parametrize("P", [2, 3, 4, 8])
@pytest.mark.parametrize("s", [1, 3, 16])
def test_choose_splitters_random_keys(P, s):
    rng = np.random.default_rng(P * 100 + s)
    keys = [[int(x) for x in rng.integers(0, 1000, int(rng.integers(0, 300)))] for _ in range(P)]
    check_model(keys, P, s)


@pytest.mark.parametrize("P", [2, 3, 5, 8])
@pytest.mark.parametrize("s", [2, 16])
def test_choose_splitters_tie_heavy(P, s):
    rng = np.random.default_rng(7 + P * s)
    cases = [
        [[5] * 200 for _ in range(P)],  # every key equal: ties are split by (rank, position)
        [[5 if rng.random() < 0.9 else int(rng.integers(0, 9)) for _ in range(150)] for _ in range(P)],  # one value holds 90 %
        [[None if rng.random() < 0.3 else int(rng.integers(0, 3)) for _ in range(100)] for _ in range(P)],  # NA and 3 values
        [list(range(r * 100, r * 100 + 100)) for r in range(P)],  # already range-partitioned
        [list(range((P - 1 - r) * 100, (P - r) * 100)) for r in range(P)],  # range-partitioned, reversed
        [list(rng.integers(0, 50, 400)) if r == P // 2 else [] for r in range(P)],  # one rank holds every row
    ]
    for keys in cases:
        check_model([[None if k is None else int(k) for k in ks] for ks in keys], P, s)


def test_choose_splitters_infinite_splitters():
    """One rank of 10 rows and 2 samples (weights 5, 5) over 4 ranks: splitters 1 and 2 are the second sample, 3 is +inf."""
    recs = np.array([[1, 0, 0, 0], [1, 7, 0, 5]], dtype=np.uint64)
    got = S.choose_splitters(recs, [5, 5], 4)
    np.testing.assert_array_equal(got, recs[[1, 1]])
    assert S.choose_splitters(np.zeros((0, 4), np.uint64), [], 3).shape == (0, 4)  # no rows anywhere: every splitter +inf
    assert S.choose_splitters(recs, [5, 5], 1).shape == (0, 4)
    with pytest.raises(B200Error, match="at least one rank"):
        S.choose_splitters(recs, [5, 5], 0)


def test_choose_splitters_compares_every_word_unsigned():
    """Records are compared as uint64 words, most significant first: a word with the top bit set sorts last."""
    recs = np.array([[1, 1 << 63, 0, 0], [1, 1, 1, 0], [0, 1 << 63, 1, 1]], dtype=np.uint64)
    got = S.choose_splitters(recs, [1, 1, 1], 3)
    np.testing.assert_array_equal(got, recs[[1, 0]])


# ---- init_sharded_sort_state: argument checks and plumbing ----
def init(**kw):
    args = dict(operator_id=-1, by=["a"], asc=[True], na_position=["last"], col_names=COLS)
    args.update(kw)
    return S.init_sharded_sort_state(**args)


def test_sharded_state_is_lazy_and_keeps_the_key_plan():
    st = init(by=["c", "a"], asc=[False, True], na_position=["first", "last"], output_batch_size=100)
    assert st.local.handle is None and st.merged is None and not st.done
    assert st.local.phys == [2, 0, 1] and st.local.out_names == ["c", "a", "b"]
    assert st.local.full and st.output_batch_size == 100


@pytest.mark.parametrize("kw,msg", [
    (dict(by=[], asc=[], na_position=[]), "1 to 4 sort keys"),
    (dict(by=["a", "b", "c", "a", "b"], asc=True, na_position="last"), "1 to 4 sort keys"),
    (dict(by=["a", "b"], asc=[True]), "one entry per sort key"),
    (dict(by=["zz"]), "must be distinct columns"),
    (dict(by=["a", "a"], asc=True, na_position="last"), "must be distinct columns"),
    (dict(na_position="middle"), "na_position"),
    (dict(output_batch_size=0), "output_batch_size must be positive"),
    (dict(output_batch_size=-5), "output_batch_size must be positive"),
])
def test_sharded_sort_argument_checks(kw, msg):
    with pytest.raises(B200Error, match=msg):
        init(**kw)


def test_sharded_produce_before_consume_raises():
    with pytest.raises(B200Error, match="before the last batch"):
        S.produce_output_batch(init())


def test_physical_sort_full_parallel_builds_the_sharded_state(monkeypatch):
    seen = []
    monkeypatch.setattr(S.ShardedSortState, "consume", lambda self, table, is_last: seen.append((table.n_rows, is_last)) or True)
    t = Table([Column(np.arange(4, dtype=np.int64), None, CTypes.INT64, ArrTypes.NUMPY, 4)], ["k"])
    op = PhysicalSort(["k"], False, "first", full=True, parallel=True, output_batch_size=64)
    assert op.ConsumeBatch(t, OperatorResult.FINISHED) == OperatorResult.FINISHED
    assert isinstance(op.state, S.ShardedSortState) and seen == [(4, True)]
    assert op.state.local.asc == [False] and op.state.local.na_last == [False] and op.state.output_batch_size == 64
    # the top-k keeps its own parallel form
    op2 = PhysicalSort(["k"], limit=3, parallel=True)
    monkeypatch.setattr(S.SortState, "_ensure", lambda self, *a: None)
    monkeypatch.setattr(S.SortState, "_consume", lambda self, *a: True)
    op2.ConsumeBatch(t, OperatorResult.NEED_MORE_INPUT)
    assert type(op2.state) is S.SortState


def test_abi_declares_the_sharded_sort_entries():
    syms = _lib.declared_symbols()
    for s in ("b200_sort_state_init_runs", "b200_sort_sample", "b200_sort_count_below"):
        assert s in syms
    assert S.MAX_SHARDED_RECEIVE_ROWS == S.MAX_FULL_SORT_ROWS == 1 << 31
    assert S.SAMPLES_PER_RANK == 4096


# ---- the collective refusal, on a gloo world of 2 ----
def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _agree_worker(rank, world, port, q):
    import torch
    import torch.distributed as dist

    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        res = []
        sends = {0: [3, 8], 1: [2, 4]}
        for cap in (10, 13):  # lowered caps: rank 1 receives 8 + 4 = 12 rows
            S.MAX_SHARDED_RECEIVE_ROWS = cap
            try:
                res.append(S.agree_receive_rows(sends[rank], torch.device("cpu")).tolist())
            except B200Error as e:
                res.append(str(e))
        q.put((rank, res))
    finally:
        dist.destroy_process_group()


@pytest.mark.timeout(300)
def test_receive_cap_is_refused_on_every_rank():
    """A rank that would receive MAX_SHARDED_RECEIVE_ROWS rows or more makes every rank raise the same error after one all_reduce;
    under the cap every rank gets the same count matrix."""
    import torch.multiprocessing as mp

    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_agree_worker, args=(r, 2, port, q)) for r in range(2)]
    for p in procs:
        p.start()
    res = dict(q.get(timeout=240) for _ in range(2))
    for p in procs:
        p.join(timeout=60)
    assert res[0][0] == res[1][0]
    assert "rank 1 would receive 12 rows" in res[0][0] and "cap of 10 rows" in res[0][0]
    assert res[0][1] == res[1][1] == [[3, 8], [2, 4]]
