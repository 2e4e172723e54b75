"""The sharded streaming groupby (init_groupby_state(..., parallel=True) through groupby_build_consume_batch /
groupby_produce_output_batch, streaming/groupby.py) against the exact groupby reference, on one GPU, with the ranks simulated as
lock-step threads of this process (tests/test_gpu_join_sharded.py's LockstepGroup).

Every rank runs the API exactly as a process per GPU would, so everything the sharded branch does runs: the all-reduced
reduce-or-shuffle decision, the raw-row shuffle through shuffle_table, the nested nunique exchanges before the outer one, and
each state's exchange in its three transports:
  * fused: exchange.get_slabs is replaced by a per-rank stand-in of exchange.Slabs (keyed by the lock-step rank: every rank is
    on device 0, so the real cache would hand one rank's slabs to all): two zeroed device slabs per rank used alternately, a
    device array of every rank's slab address for the current parity, and a handle whose barrier(channel=0) is the lock-step
    barrier.  All ranks share stream 0, so every pack is enqueued before any combine;
  * overflow: 8 KiB slabs, so finalize returns -2 and the NCCL form follows;
  * nccl: get_slabs returns None.
exchange.Slabs itself is replaced by a function that fails, so no case reaches torch's symmetric memory.

The reference (tests/test_gpu_groupby_column_types.py's exact reference and tests/test_gpu_groupby_reductions.py's for prod,
kurtosis, the boolean, bitwise and count_if aggregates) groups the global table: the rank slices concatenated in rank order, so
first / last are the first / last valid row in rank-major order.  Each rank's output groups must be owned by it (hash_keys_table
of the key columns, which tests/test_gpu_shuffle.py pins against the oracle, % R), every rank must agree on each output column's
c-type, array kind and bitmap, and the union must hold every reference group exactly once with the reference's values and NA
mask: bit for bit for the exact functions, within the bounds those files derive for the floating-point ones.

The raw-row form is forced with B200_SHUFFLE_DECISION_ROWS at 2 000 rows (and B200_COALESCE=0); its tests also pin where the rows
were aggregated: each rank's rows consumed are its own rows up to the decision plus, after it, every rank's rows that it owns.

The GPU part (161 tests) took 152 s on one H100 80GB HBM3 (700 W power limit); its budget is 5 minutes."""

import functools

import numpy as np
import pandas as pd
import pytest
import torch

from bodo_b200.table import ArrTypes, Column, CTypes, Table
from tests.helpers import table_to_device
from tests.test_gpu_groupby_column_types import (ALL_TYPES, FLOATS, MK_KEYS, MOMENTS, TNAME, _collect, _column, _match_groups,
                                                 check_column, expect, group_rows, key_column, mk_key_column)
from tests.test_gpu_groupby_float_values import _groups
from tests.test_gpu_groupby_reductions import _check_kurt
from tests.test_gpu_groupby_reductions import check as red_check
from tests.test_gpu_join_sharded import LockstepGroup, owners
from tests.test_gpu_sort import NP, gen_values
from tests.test_groupby_reductions_host import exact_kurt

gpu = pytest.mark.gpu
TRANSPORTS = {"fused": 64 << 20, "overflow": 8 << 10, "nccl": None}  # slab bytes, or None: no slabs
RS = (2, 3, 5)
EXACT = ("size", "count", "sum", "mean", "min", "max", "first", "last", "nunique") + MOMENTS
DECISION_ROWS = 2_000
NARROW = (CTypes.INT8, CTypes.UINT8, CTypes.INT16, CTypes.UINT16, CTypes.BOOL)  # 1- and 2-byte keys: shuffle_table refuses them


@pytest.fixture
def lockstep(monkeypatch):
    """lockstep(R) -> a LockstepGroup of R ranks, installed as torch.distributed for this test."""
    return lambda n: LockstepGroup(n).install(monkeypatch)


# ================================================================================================ the fused exchange's slabs
class LockstepSlabs:
    """exchange.Slabs for R lock-step ranks on device 0: rank r's view is `for_rank(r)`."""

    def __init__(self, pg, slab_bytes):
        self.pg, self.slab_bytes = pg, slab_bytes
        self.bufs = [[torch.zeros(slab_bytes, dtype=torch.uint8, device="cuda:0") for _ in range(2)] for _ in range(pg.n)]
        self.peers = [torch.tensor([self.bufs[q][p].data_ptr() for q in range(pg.n)], dtype=torch.int64, device="cuda:0")
                      for p in range(2)]
        self.parity = [0] * pg.n
        self.barriers = 0
        torch.cuda.synchronize()

    def for_rank(self, r):
        return _RankSlabs(self, r)


class _RankSlabs:
    def __init__(self, shared, rank):
        self.shared, self.rank, self.slab_bytes = shared, rank, shared.slab_bytes

    def next(self):
        """(peer pointer array on the device, my slab address, handle), as Slabs.next()"""
        s = self.shared
        p = s.parity[self.rank]
        s.parity[self.rank] ^= 1
        return int(s.peers[p].data_ptr()), int(s.bufs[self.rank][p].data_ptr()), self

    def barrier(self, channel=0):
        assert channel == 0
        self.shared.barriers += 1
        self.shared.pg.barrier_collective()


def install_transport(monkeypatch, pg, transport):
    from bodo_b200.streaming import exchange as X

    def no_symmetric_memory(*a, **k):
        raise AssertionError("the lock-step ranks must not reach torch's symmetric memory")

    monkeypatch.setattr(X, "Slabs", no_symmetric_memory)
    slab_bytes = TRANSPORTS[transport]
    if slab_bytes is None:
        monkeypatch.setattr(X, "get_slabs", lambda group, device: None)
        return None
    shared = LockstepSlabs(pg, slab_bytes)
    views = [shared.for_rank(r) for r in range(pg.n)]
    monkeypatch.setattr(X, "get_slabs", lambda group, device: views[pg.rank])
    return shared


# ================================================================================================ running the ranks
def empty_like(t):
    return Table([Column(c.data[:0], None, c.c_type, c.arr_type, 0) for c in t.columns], list(t.names))


def split_ranks(t, sizes, batches, rng):
    """rank r gets rows [sum(sizes[:r]), +sizes[r]) of host table t, cut into batches[r] batches of random sizes (zero-row ones
    included); every other non-empty batch is staged on the device.  Returns (per rank: list of batches, per rank: list of batch
    row counts)."""
    assert sum(sizes) == t.n_rows
    out, counts, lo = [], [], 0
    for r, (n, nb) in enumerate(zip(sizes, batches)):
        cuts = np.sort(rng.integers(0, n + 1, nb - 1))
        b_sizes = np.diff(np.concatenate([[0], cuts, [n]])).astype(int).tolist()
        bs = []
        for q, s in enumerate(b_sizes):
            b = t.slice(lo, lo + s) if s else empty_like(t)
            bs.append(table_to_device(b) if s and (q + r) % 2 else b)
            lo += s
        out.append(bs)
        counts.append(b_sizes)
    return out, counts


def run_ranks(lockstep, monkeypatch, R, t, batches, key_inds, funcs, transport, dropna=True, expected_groups=0,
              output_batch_size=1 << 30):
    """Every rank consumes its batches (ranks that run out pass empty batches until is_last, which all pass in the same call) and
    produces its output.  t: the global host table (for the empty batches' schema); funcs: (function, logical input column).
    Returns per rank (output batches as host tuples, info)."""
    from bodo_b200.streaming.groupby import (delete_groupby_state, get_metric, groupby_build_consume_batch,
                                             groupby_produce_output_batch, init_groupby_state)

    pg = lockstep(R)
    slabs = install_transport(monkeypatch, pg, transport)
    n_calls = max(len(b) for b in batches)
    empty = empty_like(t)

    def body(r):
        st = init_groupby_state(-1, tuple(key_inds), tuple(f for f, _ in funcs), tuple(range(len(funcs) + 1)),
                                tuple(c for _, c in funcs), parallel=True, dropna=dropna, expected_groups=expected_groups,
                                output_batch_size=output_batch_size, device=0)
        try:
            rebuilds = None
            for i in range(n_calls):
                b = batches[r][i] if i < len(batches[r]) else empty
                if i == n_calls - 1:
                    rebuilds = get_metric(st, 3)
                groupby_build_consume_batch(st, b, i == n_calls - 1, True)
            info = dict(raw=st.raw_row_mode, decided=st.shuffle_decided, shuffled=st.raw_rows_shuffled, path=st.exchange_path,
                        rows=get_metric(st, 2), rebuilds=(rebuilds, get_metric(st, 3)))
            parts = []
            while True:
                out, last = groupby_produce_output_batch(st, True)
                parts.append([(c.values_numpy().copy(), c.valid_mask_numpy(), c.c_type, c.arr_type) for c in out.columns])
                if last:
                    break
            info["n_batches"] = len(parts)
            return parts, info
        finally:
            delete_groupby_state(st)

    res = pg.run(body)
    want = {"fused": {"fused"}, "overflow": {"nccl", "fused"}, "nccl": {"nccl"}}[transport]  # (few groups fit even 8 KiB)
    assert len({i["path"] for _, i in res}) == 1 and res[0][1]["path"] in want, [i["path"] for _, i in res]
    if slabs is not None:
        assert slabs.barriers > 0
    return res


# ================================================================================================ the reference
def widen(c):
    """A 1- or 2-byte key column as the int32 column of its values: such a key is owned by the hash of the 4 low bytes of its
    widened value (shuffle_table does not take the narrow column itself)."""
    if c.c_type not in NARROW:
        return c
    return Column(c.values_numpy().astype(np.int32), c.validity, CTypes.INT32, c.arr_type, c.length)


def check_sharded(res, t, key_inds, funcs, dropna, R, df=None, what=""):
    """Compare the ranks' outputs with the reference over global table t (see the module docstring).  df: the value columns as
    pandas Series (by name) for the functions tests/test_gpu_groupby_reductions.py checks."""
    nk = len(key_inds)
    non_empty = [p for r in range(R) for p in res[r][0] if len(p[0][0])]
    out = _collect(non_empty or res[0][0])  # (asserts that the ranks agree on every column's c-type, array kind and bitmap)
    for r in range(R):
        mine = [p for p in res[r][0] if len(p[0][0])]
        if mine:
            keys = Table([widen(c) for c in _collect(mine)[:nk]])
            dest = owners(keys, range(nk), R)
            assert (dest == r).all(), (what, f"rank {r} outputs {int((dest != r).sum())} groups owned by other ranks")
    keys = [t.columns[i] for i in key_inds]
    rows, gid, groups = group_rows(keys, dropna)
    order = _match_groups(out[:nk], groups)  # every reference group exactly once in the union
    G = len(groups)
    for j, (f, c) in enumerate(funcs):
        got = out[nk + j]
        ctx = (what, f, t.names[c])
        if f in EXACT:
            check_column(got, expect(f, t.columns[c], rows, gid, G), order, ctx)
            continue
        vals = got.values_numpy()[order]
        mask = got.valid_mask_numpy()
        na = np.zeros(G, bool) if mask is None else ~mask[order]
        s = df[t.names[c]].iloc[rows].reset_index(drop=True)
        if f == "kurtosis":
            assert (got.c_type, got.arr_type) == (CTypes.FLOAT64, ArrTypes.NULLABLE_INT_BOOL), ctx
            x = s.to_numpy(dtype=np.float64, na_value=np.nan)
            _check_kurt(vals, na, [exact_kurt(x[ix]) for ix in _groups(gid, G)], ctx)
            continue
        if f.startswith("bool"):
            assert (got.c_type, got.arr_type) == (CTypes.BOOL, ArrTypes.NULLABLE_INT_BOOL), ctx
            vals = vals.astype(bool)
        elif f == "count_if":
            assert (got.c_type, got.arr_type, mask) == (CTypes.INT64, ArrTypes.NUMPY, None), ctx
        red_check(f, (vals, na), s, gid, G, str(ctx))


# ================================================================================================ data
def values_frame(n, rng):
    """the value columns: i (Int64, small), x (Float64), b (boolean), u (Int32 bit patterns), all with NA"""
    def na(p=0.1):
        return rng.random(n) < p

    return pd.DataFrame({"i": pd.arrays.IntegerArray(rng.integers(-1000, 1000, n), na()),
                         "x": pd.arrays.FloatingArray(rng.standard_normal(n) * 3 + 1, na()),
                         "b": pd.arrays.BooleanArray(rng.random(n) < 0.3, na()),
                         "u": pd.arrays.IntegerArray(rng.integers(-(2 ** 31), 2 ** 31, n).astype(np.int32), na())})


def with_keys(keys, vals, names):
    v = Table.from_pandas(vals)
    return Table(list(keys) + v.columns, list(names) + list(vals.columns))


FN_KEY = (("size", 1), ("count", 1), ("sum", 1), ("mean", 1), ("min", 1), ("max", 1), ("first", 1), ("last", 1), ("nunique", 1),
          ("var", 1), ("skew", 1))
FN_RED = (("prod", 1), ("kurtosis", 2), ("boolor_agg", 3), ("booland_agg", 3), ("boolxor_agg", 3), ("bitor_agg", 4),
          ("bitand_agg", 4), ("bitxor_agg", 4), ("count_if", 3), ("std", 2), ("var_pop", 2), ("std_pop", 2), ("sum", 2))


def rank_layout(R, n, rng):
    """unequal rank sizes, the last rank of three or more without rows, and different batch counts (ranks that run out early)"""
    w = rng.random(R) + 0.2
    if R >= 3:
        w[-1] = 0
    sizes = np.floor(w / w.sum() * n).astype(int)
    sizes[0] += n - sizes.sum()
    return sizes.tolist(), [1 + (r * 2 + 1) % 4 for r in range(R)]


# ================================================================================================ A. partial-aggregate form
@functools.lru_cache(maxsize=None)
def _data_key(ct, nullable):
    rng = np.random.default_rng(7000 + 2 * ct + nullable)
    n = 24_000
    return with_keys([key_column(ct, n, rng, nullable, 300)], values_frame(n, rng), ["k"])


@gpu
@pytest.mark.parametrize("transport", list(TRANSPORTS))
@pytest.mark.parametrize("nullable", [False, True], ids=["numpy", "nullable"])
@pytest.mark.parametrize("ct", ALL_TYPES, ids=[TNAME[c] for c in ALL_TYPES])
def test_partial_form_every_key_type(gpu_lib, lockstep, monkeypatch, ct, nullable, transport):
    """Every key type under every function: nunique through its nested exchange, first / last in rank-major order, the
    moments, prod, kurtosis, the boolean, bitwise and count_if aggregates and size, both dropna."""
    t = _data_key(ct, nullable)
    df = t.to_pandas()
    R = RS[(ct + nullable + list(TRANSPORTS).index(transport)) % 3]
    rng = np.random.default_rng(ct)
    sizes, nb = rank_layout(R, t.n_rows, rng)
    for dropna in (True, False):
        for funcs in (FN_KEY, FN_RED):
            batches, _ = split_ranks(t, sizes, nb, rng)
            res = run_ranks(lockstep, monkeypatch, R, t, batches, (0,), funcs, transport, dropna=dropna, expected_groups=8)
            assert not any(i["raw"] for _, i in res)  # (far below the decision's row count)
            check_sharded(res, t, (0,), funcs, dropna, R, df, (TNAME[ct], nullable, transport, R, dropna))


FN_MK = (("size", 1), ("count", 1), ("sum", 1), ("mean", 2), ("min", 1), ("max", 2), ("var", 2), ("skew", 2), ("prod", 1),
         ("boolor_agg", 3), ("bitxor_agg", 4), ("count_if", 3))


@functools.lru_cache(maxsize=None)
def _data_mk(case):
    types = MK_KEYS[case]
    rng = np.random.default_rng(7500 + len(types))
    n = 30_000
    keys = [mk_key_column(ct, n, rng, {2: 9, 3: 7, 4: 5}[len(types)]) for ct in types]
    vals = values_frame(n, rng)
    # key columns after the values and out of order: key_inds lists them last-first
    t = with_keys([], vals, [])
    return Table(t.columns + keys[::-1], list(t.names) + [f"k{j}" for j in reversed(range(len(types)))]), len(types)


@gpu
@pytest.mark.parametrize("transport", list(TRANSPORTS))
@pytest.mark.parametrize("case", list(MK_KEYS))
def test_partial_form_multi_column_keys(gpu_lib, lockstep, monkeypatch, case, transport):
    """2 to 4 mixed-type nullable key columns that are not the leading columns, both dropna, output_batch_size=8: produce slices
    at word granularity of the validity bitmaps (32 groups), so each rank returns ceil(its groups / 32) batches, at least one"""
    t0, nk = _data_mk(case)
    # the values first (logical 0..3), then the keys: shift the value indices of FN_MK (1..4 -> 0..3)
    t = t0
    key_inds = tuple(range(t.n_cols - 1, t.n_cols - 1 - nk, -1))
    funcs = tuple((f, c - 1) for f, c in FN_MK)
    df = t.to_pandas()
    R = RS[(nk + list(TRANSPORTS).index(transport)) % 3]
    rng = np.random.default_rng(nk)
    sizes, nb = rank_layout(R, t.n_rows, rng)
    for dropna in (True, False):
        batches, _ = split_ranks(t, sizes, nb, rng)
        res = run_ranks(lockstep, monkeypatch, R, t, batches, key_inds, funcs, transport, dropna=dropna, expected_groups=8,
                        output_batch_size=8)
        sizes_out = [sum(len(p[0][0]) for p in parts) for parts, _ in res]
        assert [i["n_batches"] for _, i in res] == [max(1, -(-g // 32)) for g in sizes_out], sizes_out
        if nk == 4:  # (600 / 160 groups: the ranks' outputs span several batches)
            assert sum(i["n_batches"] for _, i in res) > R
        check_sharded(res, t, key_inds, funcs, dropna, R, df, (case, transport, R, dropna))


@gpu
@pytest.mark.parametrize("transport", list(TRANSPORTS))
@pytest.mark.parametrize("R", RS)
def test_partial_form_tables_grow_while_combining(gpu_lib, lockstep, monkeypatch, R, transport):
    """Rank 0 holds 45 000 R distinct int64 keys, the other ranks a few rows each: every rank owns more groups (~45 000) than the
    smallest table takes (2^15), so the tables of ranks 1.. grow while the received rows are combined (their last consume call is
    empty)."""
    rng = np.random.default_rng(50 + R)
    n0, n1 = 45_000 * R, 300
    n = n0 + n1 * (R - 1)
    k = np.concatenate([rng.integers(0, 1 << 40, n0), rng.integers(0, 1 << 40, n1 * (R - 1))])
    t = with_keys([Column(k, None, CTypes.INT64, ArrTypes.NUMPY, n)], values_frame(n, rng), ["k"])
    sizes = [n0] + [n1] * (R - 1)
    batches, _ = split_ranks(t, sizes, [2] + [1] * (R - 1), rng)
    funcs = (("sum", 1), ("count", 1), ("first", 2), ("last", 1), ("nunique", 1), ("bitor_agg", 4))
    res = run_ranks(lockstep, monkeypatch, R, t, batches, (0,), funcs, transport, expected_groups=8)
    assert res[0][1]["path"] == {"overflow": "nccl"}.get(transport, transport)
    assert any(b > a for _, i in res[1:] for a, b in [i["rebuilds"]]), [i["rebuilds"] for _, i in res]
    check_sharded(res, t, (0,), funcs, True, R, t.to_pandas(), (transport, R))


# ================================================================================================ B. raw-row form
def unique_keys(ct, n, rng):
    """n keys of type ct, (nearly) all distinct where the type has room for them"""
    if ct == CTypes.BOOL:
        return rng.integers(0, 2, n).astype(np.uint8)
    if ct in FLOATS:
        return (rng.standard_normal(n) * 1e3).astype(np.float32 if ct == CTypes.FLOAT32 else np.float64)
    if ct == CTypes.UINT64:
        return rng.integers(0, 1 << 62, n, dtype=np.uint64) * np.uint64(3)  # (a third of them at or above 2^63)
    info = np.iinfo(np.dtype(NP[ct]))
    if info.bits <= 16:
        return rng.permutation(np.arange(info.min, info.max + 1))[:n].astype(info.dtype) if n <= 1 << info.bits else \
            rng.integers(info.min, info.max + 1, n).astype(info.dtype)
    return rng.integers(info.min // 2, info.max // 2, n).astype(info.dtype)


def raw_row_keys(ct, n, rng, shared=40, share=0.05, nullable=False):
    """mostly distinct keys, with `share` of the rows drawn from `shared` keys (the type's edges among them), spread over every
    rank and batch: these groups have rows on several ranks before and after the switch"""
    k = unique_keys(ct, n, rng)
    pool = gen_values(ct, shared, rng, small=False)
    if ct == CTypes.BOOL:
        pool = pool.astype(np.uint8)
    at = rng.random(n) < share
    k[at] = pool[rng.integers(0, len(pool), int(at.sum()))]
    return _column(k, ct, rng, nullable, na_frac=0.02)


def check_raw_rows(res, t, key_inds, R, counts, batches):
    """every rank switched after its first consume call; its rows consumed = its own first batch + every rank's later rows that
    it owns (where shuffle_table sends them); its raw_rows_shuffled = its own later rows"""
    later = [sum(c[1:]) for c in counts]
    first = [c[0] for c in counts]
    assert sum(first) >= DECISION_ROWS
    dest = owners(t, key_inds, R)
    src = np.repeat(np.arange(R), [sum(c) for c in counts])
    pos = np.concatenate([np.arange(sum(c)) for c in counts])
    after = pos >= np.repeat(first, [sum(c) for c in counts])
    for r, (_, i) in enumerate(res):
        assert i["decided"] and i["raw"], (r, i)
        assert i["shuffled"] == later[r], (r, i, later)
        assert i["rows"] == first[r] + int((after & (dest == r)).sum()), (r, i["rows"], first[r])
    assert sum(later) > 0


def raw_layout(R, n):
    """rank sizes (uneven, none empty) and batch counts; the first batch of every rank is cut at n / (3 R) rows"""
    sizes = [n // R + (37 * r) % 500 - 250 for r in range(R)]
    sizes[0] += n - sum(sizes)
    return sizes


def split_raw(t, sizes, rng, n_batches=4):
    """rank r's rows in n_batches batches, the first one of a third of its share (so the decision falls after it)"""
    out, counts, lo = [], [], 0
    for r, n in enumerate(sizes):
        b0 = n // 3
        cuts = np.sort(rng.integers(b0, n + 1, n_batches - 2))
        b_sizes = np.diff(np.concatenate([[0, b0], cuts, [n]])).astype(int).tolist()
        bs = []
        for q, s in enumerate(b_sizes):
            b = t.slice(lo, lo + s) if s else empty_like(t)
            bs.append(table_to_device(b) if s and (q + r) % 2 else b)
            lo += s
        out.append(bs)
        counts.append(b_sizes)
    return out, counts


FN_RAW = (("size", 1), ("count", 1), ("sum", 1), ("min", 2), ("max", 1), ("nunique", 1), ("mean", 2), ("bitxor_agg", 4))


@gpu
@pytest.mark.parametrize("nullable", [False, True], ids=["numpy", "nullable"])
@pytest.mark.parametrize("ct", ALL_TYPES, ids=[TNAME[c] for c in ALL_TYPES])
def test_raw_rows_every_key_type(gpu_lib, lockstep, monkeypatch, ct, nullable):
    """After the switch a group's raw rows go where shuffle_table hashes them and its partials go where the exchange pack hashes
    them: the two must agree for every key type shuffle_table partitions, or the owner check fails.  nunique through the raw
    rows too.  A 1- or 2-byte key (which shuffle_table refuses) keeps the partial-aggregate form."""
    monkeypatch.setenv("B200_SHUFFLE_DECISION_ROWS", str(DECISION_ROWS))
    monkeypatch.setenv("B200_COALESCE", "0")
    transport = list(TRANSPORTS)[(ct + nullable) % 3]
    R = RS[(ct + 2 * nullable) % 3]
    rng = np.random.default_rng(8000 + 2 * ct + nullable)
    n = 4_000 * R
    t = with_keys([raw_row_keys(ct, n, rng, nullable=nullable)], values_frame(n, rng), ["k"])
    sizes = raw_layout(R, n)
    dropna = bool(ct % 2)
    batches, counts = split_raw(t, sizes, rng)
    res = run_ranks(lockstep, monkeypatch, R, t, batches, (0,), FN_RAW, transport, dropna=dropna)
    if ct in NARROW:
        assert all(i["decided"] and not i["raw"] and i["shuffled"] == 0 for _, i in res), [i for _, i in res]
    else:
        check_raw_rows(res, t, (0,), R, counts, batches)
    check_sharded(res, t, (0,), FN_RAW, dropna, R, t.to_pandas(), (TNAME[ct], nullable, transport, R))


@gpu
@pytest.mark.parametrize("transport", list(TRANSPORTS))
def test_raw_rows_float_key_signed_zero_nan_and_na(gpu_lib, lockstep, monkeypatch, transport):
    """One nullable float64 key with -0.0 and 0.0 (one group), NaN and NA (two groups) under dropna=False, on both routes."""
    monkeypatch.setenv("B200_SHUFFLE_DECISION_ROWS", str(DECISION_ROWS))
    monkeypatch.setenv("B200_COALESCE", "0")
    R = 3
    rng = np.random.default_rng(8500 + list(TRANSPORTS).index(transport))
    n = 15_000
    k = rng.standard_normal(n) * 1e3
    special = rng.random(n) < 0.06
    k[special] = np.array([-0.0, 0.0, np.nan, np.nan, 1.5])[rng.integers(0, 5, int(special.sum()))]
    valid = ~(rng.random(n) < 0.02)
    key = Column(k, np.packbits(valid, bitorder="little"), CTypes.FLOAT64, ArrTypes.NULLABLE_INT_BOOL, n)
    t = with_keys([key], values_frame(n, rng), ["k"])
    batches, counts = split_raw(t, raw_layout(R, n), rng)
    res = run_ranks(lockstep, monkeypatch, R, t, batches, (0,), FN_RAW, transport, dropna=False)
    check_raw_rows(res, t, (0,), R, counts, batches)
    check_sharded(res, t, (0,), FN_RAW, False, R, t.to_pandas(), transport)
    groups = group_rows([key], False)[2]
    assert {(1, 0), (2, 0), (0, 0)} <= {tuple(g) for g in groups.tolist()}  # NA, NaN and the one zero group


@gpu
@pytest.mark.parametrize("transport", list(TRANSPORTS))
@pytest.mark.parametrize("R", RS)
def test_raw_rows_multi_column_keys(gpu_lib, lockstep, monkeypatch, R, transport):
    """(int32, uint64, float32) nullable keys, mostly distinct tuples, a shared set of tuples on every rank"""
    monkeypatch.setenv("B200_SHUFFLE_DECISION_ROWS", str(DECISION_ROWS))
    monkeypatch.setenv("B200_COALESCE", "0")
    rng = np.random.default_rng(8700 + R)
    n = 4_000 * R
    keys = [raw_row_keys(ct, n, rng, shared=6, share=0.1, nullable=True) for ct in (CTypes.INT32, CTypes.UINT64, CTypes.FLOAT32)]
    t = with_keys(keys, values_frame(n, rng), ["a", "b", "c"])
    funcs = tuple((f, c + 2) for f, c in FN_MK)
    batches, counts = split_raw(t, raw_layout(R, n), rng)
    dropna = R != 3
    res = run_ranks(lockstep, monkeypatch, R, t, batches, (0, 1, 2), funcs, transport, dropna=dropna)
    check_raw_rows(res, t, (0, 1, 2), R, counts, batches)
    check_sharded(res, t, (0, 1, 2), funcs, dropna, R, t.to_pandas(), (transport, R))


def first_last_data(R, rng):
    """Mostly distinct int64 keys, plus 64 keys with rows on every rank in every batch, so that a group's first valid row in
    rank-major order (a lower rank's later batch) reaches its owner after the owner's own earlier rows."""
    n = 4_000 * R
    k = raw_row_keys(CTypes.INT64, n, rng, shared=64, share=0.08)
    return with_keys([k], values_frame(n, rng), ["k"])


@gpu
@pytest.mark.parametrize("transport", list(TRANSPORTS))
@pytest.mark.parametrize("R", RS)
def test_first_last_keep_rank_major_order_where_keys_are_unique(gpu_lib, lockstep, monkeypatch, R, transport):
    """With unique keys the state would switch to raw rows; a raw row is numbered by the rank that consumes it, so first / last
    would follow owner arrival instead of rank-major order.  A state with first or last stays in the partial-aggregate form."""
    monkeypatch.setenv("B200_SHUFFLE_DECISION_ROWS", str(DECISION_ROWS))
    monkeypatch.setenv("B200_COALESCE", "0")
    rng = np.random.default_rng(8900 + R)
    t = first_last_data(R, rng)
    funcs = (("first", 1), ("last", 1), ("first", 2), ("last", 3), ("count", 1), ("nunique", 4))
    batches, counts = split_raw(t, raw_layout(R, t.n_rows), rng)
    res = run_ranks(lockstep, monkeypatch, R, t, batches, (0,), funcs, transport)
    check_sharded(res, t, (0,), funcs, True, R, t.to_pandas(), (transport, R))
    assert all(i["decided"] and not i["raw"] and i["shuffled"] == 0 for _, i in res), [i for _, i in res]
    # the same data without first / last does switch
    res = run_ranks(lockstep, monkeypatch, R, t, batches, (0,), funcs[4:], transport)
    check_raw_rows(res, t, (0,), R, counts, batches)
    check_sharded(res, t, (0,), funcs[4:], True, R, t.to_pandas(), (transport, R))


# ================================================================================================ C. the decision
def decision_table(uniq_per_rank, n_per_rank, rng):
    """rank r's keys: a uniq_per_rank[r] share of distinct keys, the rest from 20 keys"""
    ks = []
    for r, (u, n) in enumerate(zip(uniq_per_rank, n_per_rank)):
        k = (rng.integers(0, 1 << 40, n) << 3) + r  # (distinct across ranks)
        dup = rng.random(n) >= u
        k[dup] = rng.integers(0, 20, int(dup.sum()))
        ks.append(k)
    k = np.concatenate(ks)
    return with_keys([Column(k, None, CTypes.INT64, ArrTypes.NUMPY, len(k))], values_frame(len(k), rng), ["k"])


FN_DEC = (("sum", 1), ("count", 2), ("max", 1), ("nunique", 4))


@gpu
@pytest.mark.parametrize("transport", list(TRANSPORTS))
def test_decision_below_threshold_keeps_the_partial_form(gpu_lib, lockstep, monkeypatch, transport):
    monkeypatch.setenv("B200_SHUFFLE_DECISION_ROWS", str(DECISION_ROWS))
    monkeypatch.setenv("B200_COALESCE", "0")
    R = 3
    rng = np.random.default_rng(9100)
    t = decision_table([0.5, 0.6, 0.4], [5_000] * R, rng)
    batches, counts = split_raw(t, [5_000] * R, rng)
    res = run_ranks(lockstep, monkeypatch, R, t, batches, (0,), FN_DEC, transport)
    assert all(i["decided"] and not i["raw"] and i["shuffled"] == 0 for _, i in res), [i for _, i in res]
    assert [i["rows"] for _, i in res] == [5_000] * R  # (every rank aggregated its own rows)
    check_sharded(res, t, (0,), FN_DEC, True, R, t.to_pandas(), transport)


@gpu
@pytest.mark.parametrize("summed", ["above", "below"])
@pytest.mark.parametrize("R", [2, 5])
def test_ranks_with_different_uniqueness_decide_alike(gpu_lib, lockstep, monkeypatch, R, summed):
    """Rank 0's keys are all distinct, the others' almost all duplicates (or the reverse); the decision is made from the counts
    summed over the ranks, so every rank takes the same form: the raw-row form when the summed uniqueness reaches the
    threshold (0.85), even on ranks whose own uniqueness is far below it, the partial form otherwise."""
    monkeypatch.setenv("B200_SHUFFLE_DECISION_ROWS", str(DECISION_ROWS))
    monkeypatch.setenv("B200_COALESCE", "0")
    rng = np.random.default_rng(9200 + R)
    if summed == "above":  # rank 0: 97 % of the rows, all distinct; the others: 3 % of duplicates
        n = [12_000] + [max(1, 360 // (R - 1))] * (R - 1)
        u = [1.0] + [0.0] * (R - 1)
    else:  # rank 0 distinct but small; the others large and duplicated
        n = [3_000] + [6_000] * (R - 1)
        u = [1.0] + [0.05] * (R - 1)
    t = decision_table(u, n, rng)
    batches, counts = split_raw(t, n, rng)
    first = [c[0] for c in counts]
    res = run_ranks(lockstep, monkeypatch, R, t, batches, (0,), FN_DEC, "overflow")
    modes = {i["raw"] for _, i in res}
    assert len(modes) == 1 and all(i["decided"] for _, i in res), [i for _, i in res]
    assert modes == {summed == "above"}
    if summed == "above":
        check_raw_rows(res, t, (0,), R, counts, batches)
    check_sharded(res, t, (0,), FN_DEC, True, R, t.to_pandas(), (R, summed))
    assert sum(first) >= DECISION_ROWS


@gpu
@pytest.mark.parametrize("transport", list(TRANSPORTS))
def test_coalesced_small_batches_defer_the_decision(gpu_lib, lockstep, monkeypatch, transport):
    """int64 key with sum / count (the coalescing signature), coalescing on: small batches wait in the device buffer, the rows
    consumed stay below the decision's count, the decision is deferred, and the result is still exact."""
    monkeypatch.setenv("B200_SHUFFLE_DECISION_ROWS", str(DECISION_ROWS))
    monkeypatch.delenv("B200_COALESCE", raising=False)
    R = 3
    rng = np.random.default_rng(9300)
    n = 6_000
    k = rng.integers(0, 1 << 40, n * R)  # all distinct: the raw-row form, were it decided
    v = rng.integers(-(1 << 40), 1 << 40, n * R)
    t = Table([Column(k, None, CTypes.INT64, ArrTypes.NUMPY, n * R), Column(v, None, CTypes.INT64, ArrTypes.NUMPY, n * R)], ["k", "v"])
    batches = [[t.slice(r * n + q * 1000, r * n + (q + 1) * 1000) for q in range(6)] for r in range(R)]
    funcs = (("sum", 1), ("count", 1), ("size", 1))
    res = run_ranks(lockstep, monkeypatch, R, t, batches, (0,), funcs, transport)
    assert all(not i["decided"] and not i["raw"] for _, i in res), [i for _, i in res]
    check_sharded(res, t, (0,), funcs, True, R, None, transport)
