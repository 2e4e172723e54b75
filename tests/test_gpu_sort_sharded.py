"""The sharded full sort (streaming.sort.init_sharded_sort_state) on one GPU, with R ranks simulated as lock-step threads of this
process (tests/test_gpu_join_sharded.py's LockstepGroup), and the merge form it receives into (b200_sort_state_init_runs).

Every rank runs the API exactly as a process per GPU would: the local sort, the all-gathered samples, the splitter search, the
agreed count matrix, the all-to-all-v of the sorted slices with per-destination bitmaps, and the merge of the received runs.
The reference is tests/test_gpu_sort.py's oracle_perm over the rank inputs concatenated in rank order: the ranks' outputs, in
rank order, must be the input rows at that permutation, bit for bit on every column (data bytes and validity).  Each rank's
row count is held to the balance bound of DESIGN.md: fewer than ceil(N / R) + 2 G rows, G = sum over ranks with rows of
ceil(n_r / min(SAMPLES_PER_RANK, n_r))."""

import math
import os
import socket

import numpy as np
import pytest
import torch

from bodo_b200 import _lib
from bodo_b200._lib import B200Error
from bodo_b200.streaming import sort as S
from bodo_b200.table import ArrTypes, Column, CTypes, Table, np_dtype_of
from tests.helpers import table_to_device
from tests.test_gpu_join_sharded import LockstepGroup
from tests.test_gpu_sort import KEY_TYPES, batches_of, col_mask, make_column, oracle_perm

pytestmark = pytest.mark.gpu
RS = (2, 3, 4, 8)
WIDTHS = [CTypes.BOOL, CTypes.INT16, CTypes.FLOAT32, CTypes.INT64]  # payloads of 1, 2, 4 and 8 bytes


@pytest.fixture
def lockstep(monkeypatch):
    return lambda n: LockstepGroup(n).install(monkeypatch)


@pytest.fixture(autouse=True)
def _return_device_memory():
    yield
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    _lib.lib().b200_pool_trim(torch.cuda.current_device(), 0)


def concat_host(parts):
    cols = []
    for ci in range(parts[0].n_cols):
        cs = [p.columns[ci] for p in parts]
        data = np.concatenate([c.values_numpy() for c in cs])
        v = None
        if cs[0].arr_type != ArrTypes.NUMPY:
            v = np.packbits(np.concatenate([col_mask(c) for c in cs]), bitorder="little")
        cols.append(Column(np.ascontiguousarray(data), v, cs[0].c_type, cs[0].arr_type, len(data)))
    return Table(cols, list(parts[0].names))


def run_sharded(pg, parts, by, asc, nap, sizes=(1 << 30,), empty_every=0, output_batch_size=32768):
    """Per rank: ([(values, mask, first output column)] per column, output batch sizes)."""
    def rank_fn(r):
        st = S.init_sharded_sort_state(-1, by, asc, nap, parts[r].names, output_batch_size=output_batch_size)
        bs = batches_of(parts[r], list(sizes), empty_every)
        for i, b in enumerate(bs):
            S.sort_build_consume_batch(st, table_to_device(b), i == len(bs) - 1)
        outs = []
        while True:
            out, last = S.produce_output_batch(st)
            outs.append(out)
            if last:
                break
        res = [(np.concatenate([o.columns[c].values_numpy() for o in outs]), np.concatenate([col_mask(o.columns[c]) for o in outs]),
                outs[0].columns[c]) for c in range(parts[r].n_cols)]
        S.delete_stream_sort_state(st)
        return res, [o.n_rows for o in outs]
    return pg.run(rank_fn)


def check(pg, parts, by, asc, nap, samples=None, **kw):
    """Runs the sharded sort and checks it against the oracle and the balance bound; returns each rank's row count."""
    R = pg.n
    glob = concat_host(parts)
    perm = oracle_perm(glob, by, asc, nap)
    got = run_sharded(pg, parts, by, asc, nap, **kw)
    counts = [len(g[0][0][0]) for g in got]
    for ci, c in enumerate(glob.columns):
        vals = np.concatenate([g[0][ci][0] for g in got])
        mask = np.concatenate([g[0][ci][1] for g in got])
        for g in got:
            oc = g[0][ci][2]
            assert oc.c_type == c.c_type and oc.arr_type == c.arr_type and (oc.validity is None) == (c.arr_type == ArrTypes.NUMPY)
        exp = c.values_numpy()[perm]
        assert vals.dtype == np_dtype_of(c.c_type) and len(vals) == len(perm)
        np.testing.assert_array_equal(vals.view(np.uint8), exp.view(np.uint8))
        np.testing.assert_array_equal(mask, col_mask(c)[perm])
    obs = kw.get("output_batch_size", 32768)
    for (res, sizes), n in zip(got, counts):
        assert sum(sizes) == n and (sizes == [0] if n == 0 else all(0 < x <= -(-obs // 32) * 32 for x in sizes)), sizes
    s = S.SAMPLES_PER_RANK if samples is None else samples
    N = glob.n_rows
    G = sum(math.ceil(p.n_rows / min(s, p.n_rows)) for p in parts if p.n_rows)
    assert N == 0 or all(c < math.ceil(N / R) + 2 * G for c in counts), (counts, N, G)
    return counts, got


def table(rng, n, key_types, nullable=True, payload=(CTypes.INT64,), small=True, na_frac=0.15):
    cols = [make_column(ct, n, rng, nullable, na_frac=na_frac, small=small) for ct in key_types]
    cols += [make_column(ct, n, rng, j % 2 == 1, small=False) for j, ct in enumerate(payload)]
    return Table(cols, [f"k{j}" for j in range(len(key_types))] + [f"p{j}" for j in range(len(payload))])


def split(rng, R, n, key_types, **kw):
    sizes = rng.multinomial(n, [1 / R] * R)
    return [table(rng, int(m), key_types, **kw) for m in sizes]


# ---- keys: every key type, numpy and nullable, both directions and NA placements ----
@pytest.mark.parametrize("ct", KEY_TYPES)
@pytest.mark.parametrize("nullable", [False, True])
def test_key_types(gpu_lib, lockstep, ct, nullable):
    rng = np.random.default_rng(ct * 2 + nullable)
    R = RS[(ct + nullable) % len(RS)]
    parts = split(rng, R, 6000, [ct], nullable=nullable)
    for asc in (True, False):
        for nap in ("first", "last"):
            check(lockstep(R), parts, ["k0"], [asc], [nap], sizes=(700,), empty_every=3)
    wide = split(rng, R, 5000, [ct], nullable=nullable, small=False)
    check(lockstep(R), wide, ["k0"], [False], ["first"], sizes=(333,))


@pytest.mark.parametrize("n_keys", [1, 2, 3, 4])
@pytest.mark.parametrize("R", RS)
def test_multi_key_mixed_directions_and_payload_widths(gpu_lib, lockstep, n_keys, R):
    rng = np.random.default_rng(50 + 10 * n_keys + R)
    types = [CTypes.INT32, CTypes.FLOAT64, CTypes.DATETIME, CTypes.UINT16][:n_keys]
    parts = split(rng, R, 20_000, types, payload=WIDTHS, na_frac=0.1)
    asc = [j % 2 == 0 for j in range(n_keys)]
    nap = ["first" if j % 3 == 1 else "last" for j in range(n_keys)]
    check(lockstep(R), parts, [f"k{j}" for j in range(n_keys)], asc, nap, sizes=(4096, 1000), output_batch_size=1000)
    # keys need not be the leading columns
    rev = [p.select(list(range(p.n_cols))[::-1]) for p in parts]
    check(lockstep(R), rev, [f"k{j}" for j in range(n_keys)][::-1], asc[::-1], nap[::-1], output_batch_size=77)


# ---- skew ----
def _i64_parts(values_per_rank):
    return [Table([Column(np.ascontiguousarray(v, dtype=np.int64), None, CTypes.INT64, ArrTypes.NUMPY, len(v)),
                   Column(np.arange(len(v), dtype=np.int64) + 1000 * r, None, CTypes.INT64, ArrTypes.NUMPY, len(v))], ["k", "p"])
            for r, v in enumerate(values_per_rank)]


@pytest.mark.parametrize("R", RS)
@pytest.mark.parametrize("samples", [None, 16])
def test_skew(gpu_lib, lockstep, monkeypatch, R, samples):
    if samples is not None:
        monkeypatch.setattr(S, "SAMPLES_PER_RANK", samples)
    rng = np.random.default_rng(R + (samples or 0))
    n = 30_000
    cases = {
        "all equal": [np.full(n // R, 7) for _ in range(R)],
        "one value holds 90 %": [np.where(rng.random(n // R) < 0.9, 42, rng.integers(-1000, 1000, n // R)) for _ in range(R)],
        "range-partitioned": [np.arange(r * (n // R), (r + 1) * (n // R)) for r in range(R)],
        "range-partitioned, reversed": [np.arange((R - 1 - r) * (n // R), (R - r) * (n // R)) for r in range(R)],
        "one rank holds every row": [rng.integers(0, 100, n) if r == R - 1 else np.zeros(0) for r in range(R)],
        "every rank empty": [np.zeros(0) for _ in range(R)],
        "fewer rows than samples": [rng.integers(0, 5, int(rng.integers(0, 12))) for _ in range(R)],
    }
    for name, vals in cases.items():
        counts, _ = check(lockstep(R), _i64_parts(vals), ["k"], [True], ["last"], samples=samples, sizes=(5000,))
        if name == "all equal":
            assert min(counts) > 0  # ties are split by (rank, position)


def test_determinism_across_runs_and_batch_splits(gpu_lib, lockstep):
    rng = np.random.default_rng(9)
    R = 3
    parts = split(rng, R, 50_000, [CTypes.FLOAT64, CTypes.INT8], payload=WIDTHS)
    by = ["k0", "k1"]
    a = run_sharded(lockstep(R), parts, by, [True, False], ["last", "first"], sizes=(1 << 30,))
    b = run_sharded(lockstep(R), parts, by, [True, False], ["last", "first"], sizes=(999, 4096), empty_every=2)
    for ra, rb in zip(a, b):
        for (va, ma, _), (vb, mb, _) in zip(ra[0], rb[0]):
            np.testing.assert_array_equal(va.view(np.uint8), vb.view(np.uint8))
            np.testing.assert_array_equal(ma, mb)


def test_one_rank_is_the_local_full_sort(gpu_lib, lockstep):
    rng = np.random.default_rng(3)
    parts = split(rng, 1, 10_000, [CTypes.INT32], payload=WIDTHS)
    pg = lockstep(1)
    check(pg, parts, ["k0"], [True], ["first"], sizes=(3000,), output_batch_size=4096)
    assert pg.calls == []  # no collective


def test_receive_cap_is_refused_on_every_rank(gpu_lib, lockstep, monkeypatch):
    monkeypatch.setattr(S, "MAX_SHARDED_RECEIVE_ROWS", 1000)
    parts = _i64_parts([np.full(900, 1), np.full(900, 2)])  # each rank receives 900 rows: under the cap
    assert check(lockstep(2), parts, ["k"], [True], ["last"])[0] == [900, 900]
    parts = _i64_parts([np.full(1200, 1), np.concatenate([np.full(200, 1), np.full(1000, 2)])])  # 1200 rows each: refused
    pg = lockstep(2)

    def rank_fn(r):
        st = S.init_sharded_sort_state(-1, ["k"], True, "last", ["k", "p"])
        try:
            S.sort_build_consume_batch(st, table_to_device(parts[r]), True)
            return "no error"
        except B200Error as e:
            return str(e)
        finally:
            S.delete_stream_sort_state(st)
    msgs = pg.run(rank_fn)
    assert msgs[0] == msgs[1] and "would receive" in msgs[0] and "cap of 1000 rows" in msgs[0]
    assert "all_to_all_single" not in pg.calls  # refused before any row moved


def test_physical_sort_full_parallel(gpu_lib, lockstep):
    from bodo_b200.physical import OperatorResult, PhysicalSort

    rng = np.random.default_rng(11)
    R = 4
    parts = split(rng, R, 8000, [CTypes.FLOAT32], payload=[CTypes.INT64])
    glob = concat_host(parts)
    perm = oracle_perm(glob, ["k0"], [False], ["first"])

    def rank_fn(r):
        op = PhysicalSort(["k0"], False, "first", full=True, parallel=True)
        op.ConsumeBatch(table_to_device(parts[r]), OperatorResult.FINISHED)
        outs = []
        while True:
            out, res = op.ProduceBatch()
            outs.append(out.columns[1].values_numpy())
            if res == OperatorResult.FINISHED:
                break
        op.Finalize()
        return np.concatenate(outs)
    got = np.concatenate(lockstep(R).run(rank_fn))
    np.testing.assert_array_equal(got, glob.columns[1].values_numpy()[perm])


# ---- the merge form on one state: sorted runs back to back ----
def run_merge(table, runs, by, asc, nap, sizes=(1 << 30,)):
    st = S.SortState(-1, None, 0, by, asc, nap, table.names, False, 32768, None, 0, None, full=True)
    st.runs = list(runs)
    bs = batches_of(table, list(sizes))
    st._ensure(table_to_device(bs[0]))
    for i, b in enumerate(bs):
        st._consume(table_to_device(b), i == len(bs) - 1)
    st.done = True
    outs = []
    while True:
        out, last = S.produce_output_batch(st)
        outs.append(out)
        if last:
            break
    res = [(np.concatenate([o.columns[c].values_numpy() for o in outs]), np.concatenate([col_mask(o.columns[c]) for o in outs]))
           for c in range(table.n_cols)]
    S.delete_stream_sort_state(st)
    return res


@pytest.mark.parametrize("runs", [
    [1000], [0, 500], [16, 17], [1, 1, 1], [15, 16, 17, 4096, 4095], [0, 3000, 0, 1, 0],
    [256 * 16, 256 * 16 + 1, 255 * 16, 7, 0, 1, 2, 4097], [100, 0, 0, 0, 0, 0, 0, 200],
])
def test_merge_of_sorted_runs(gpu_lib, runs):
    """P sorted runs (some empty, some of one row, lengths on the merge's 16-row thread and 4096-row block edges) merge into
    the stable sort of their concatenation."""
    rng = np.random.default_rng(len(runs) * 1000 + sum(runs))
    by, asc, nap = ["k0", "k1"], [False, True], ["first", "last"]
    parts = []
    for m in runs:
        t = table(rng, m, [CTypes.INT16, CTypes.FLOAT64], payload=WIDTHS)
        parts.append(Table([Column(c.values_numpy()[oracle_perm(t, by, asc, nap)], None if c.validity is None else
                                   np.packbits(col_mask(c)[oracle_perm(t, by, asc, nap)], bitorder="little"), c.c_type, c.arr_type, m)
                            for c in t.columns], t.names))
    glob = concat_host(parts)
    perm = oracle_perm(glob, by, asc, nap)
    for sizes in ((1 << 30,), (777,)):
        got = run_merge(glob, runs, by, asc, nap, sizes)
        for c, (vals, mask) in zip(glob.columns, got):
            np.testing.assert_array_equal(vals.view(np.uint8), c.values_numpy()[perm].view(np.uint8))
            np.testing.assert_array_equal(mask, col_mask(c)[perm])


def test_merge_form_checks_the_run_lengths(gpu_lib):
    t = _i64_parts([np.arange(10)])[0]
    with pytest.raises(B200Error, match="sum of the run lengths"):
        run_merge(t, [4, 5], ["k"], [True], ["last"])
    st = S.SortState(-1, None, 0, ["k"], [True], ["last"], t.names, False, 32768, None, 0, None, full=True)
    st.runs = [3, -1]
    with pytest.raises(B200Error, match="non-negative"):
        st._ensure(table_to_device(t))


# ---- NCCL: one process per GPU ----
def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _nccl_worker(rank, world, port, q):
    import torch.distributed as dist

    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", rank))
    try:
        rng = np.random.default_rng(5)
        parts = [table(rng, 40_000 + 1000 * r, [CTypes.FLOAT64, CTypes.INT32], payload=WIDTHS) for r in range(world)]
        st = S.init_sharded_sort_state(-1, ["k0", "k1"], [True, False], ["last", "first"], parts[rank].names, output_batch_size=5000)
        S.sort_build_consume_batch(st, table_to_device(parts[rank].slice(0, 10_000), rank), False)
        S.sort_build_consume_batch(st, table_to_device(parts[rank].slice(10_000, 1 << 30), rank), True)
        outs = []
        while True:
            out, last = S.produce_output_batch(st)
            outs.append([(c.values_numpy(), col_mask(c)) for c in out.columns])
            if last:
                break
        S.delete_stream_sort_state(st)
        q.put((rank, [(np.concatenate([o[c][0] for o in outs]), np.concatenate([o[c][1] for o in outs])) for c in range(len(outs[0]))]))
    except BaseException as e:  # noqa: BLE001 (reported to the parent)
        q.put((rank, repr(e)))
    finally:
        dist.destroy_process_group()


@pytest.mark.timeout(600)
def test_nccl_ranks():
    import torch.multiprocessing as mp

    world = min(torch.cuda.device_count(), 4)
    if world < 2:
        pytest.skip("needs 2 or more GPUs")
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_nccl_worker, args=(r, world, port, q)) for r in range(world)]
    for p in procs:
        p.start()
    res = dict(q.get(timeout=500) for _ in range(world))
    for p in procs:
        p.join(timeout=60)
    for r in range(world):
        assert not isinstance(res[r], str), res[r]
    rng = np.random.default_rng(5)
    parts = [table(rng, 40_000 + 1000 * r, [CTypes.FLOAT64, CTypes.INT32], payload=WIDTHS) for r in range(world)]
    glob = concat_host(parts)
    perm = oracle_perm(glob, ["k0", "k1"], [True, False], ["last", "first"])
    for ci, c in enumerate(glob.columns):
        vals = np.concatenate([res[r][ci][0] for r in range(world)])
        mask = np.concatenate([res[r][ci][1] for r in range(world)])
        np.testing.assert_array_equal(vals.view(np.uint8), c.values_numpy()[perm].view(np.uint8))
        np.testing.assert_array_equal(mask, col_mask(c)[perm])
