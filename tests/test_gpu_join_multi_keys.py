"""Multi-column equi-join keys (2..4 key columns per side).  Keys compare column by column on their canonical values (integers
widened to int64, floats with -0.0 as 0.0 and NaN as NA); NA is part of the key tuple: under is_na_equal=True NA equals NA within a
column, under False a row with any NA key column matches nothing.

Expected rows come from the CPU oracle's single-key hash join over dense int64 ids of the key tuples (factorized here over
build and probe together, the NA pattern part of the tuple; under is_na_equal=False a tuple with an NA column is an invalid key),
and from pandas where pandas defines the result (is_na_equal=True)."""

import numpy as np
import pandas as pd
import pytest

from bodo_b200 import _lib
from bodo_b200._lib import ffi
from bodo_b200.streaming.join import (build_runtime_filter, delete_join_state, get_metric, init_join_state, join_build_consume_batch,
                                      join_probe_consume_batch, runtime_join_filter)
from bodo_b200.table import ArrTypes, Column, CTable, CTypes, Table
from tests.helpers import table_to_device
from tests.test_gpu_join import assert_rowset_equal

pytestmark = pytest.mark.gpu

NAN = np.nan


def col(values, valid=None, c_type=-1):
    """A host column; `valid` (bool array) gives it an Arrow bitmap."""
    values = np.ascontiguousarray(values)
    bm = None
    if valid is not None:
        bits = np.packbits(np.asarray(valid, dtype=np.uint8), bitorder="little")
        bm = np.zeros(len(bits) + 8, dtype=np.uint8)
        bm[: len(bits)] = bits
    return Column(values, bm, c_type, ArrTypes.NULLABLE_INT_BOOL if valid is not None else ArrTypes.NUMPY, len(values))


def canon(c: Column):
    """(canonical int64 value, valid) of a key column: integers widened, floats as their bits with -0.0 as 0.0; NaN is NA."""
    v = c.values_numpy()
    m = c.valid_mask_numpy()
    valid = np.ones(len(v), dtype=bool) if m is None else m.copy()
    if v.dtype.kind == "f":
        d = v.astype(np.float64)
        valid &= ~np.isnan(d)
        k = np.where(d == 0, 0.0, d).view(np.int64).copy()
    else:
        k = v.view(np.int64).copy() if v.dtype == np.uint64 else v.astype(np.int64)
    k[~valid] = 0
    return k, valid


def tuple_ids(bt, bkeys, pt, pkeys, is_na_equal):
    """Dense int64 ids of the key tuples of both sides and their validity (the oracle's single-key input)."""
    parts = []
    for t, keys in ((bt, bkeys), (pt, pkeys)):
        cs = [canon(t.columns[j]) for j in keys]
        parts.append(pd.DataFrame({**{f"k{j}": k for j, (k, _) in enumerate(cs)}, **{f"v{j}": v for j, (_, v) in enumerate(cs)}}))
    both = pd.concat(parts, ignore_index=True)
    ids = both.groupby(list(both.columns), sort=False).ngroup().to_numpy().astype(np.int64)
    allv = both[[c for c in both.columns if c.startswith("v")]].all(axis=1).to_numpy()
    valid = np.ones(len(ids), dtype=bool) if is_na_equal else allv
    nb = bt.n_rows
    return ids[:nb], valid[:nb], ids[nb:], valid[nb:]


def col_bits(c: Column, idx=None):
    """(int64 bits, valid) of an output / input column, gathered at idx (-1: NULL)."""
    v = c.values_numpy()
    if v.dtype.kind == "f":
        v = v.view(np.int64 if v.dtype.itemsize == 8 else np.int32)
    v = v.view(np.int64) if v.dtype == np.uint64 else v.astype(np.int64)
    m = c.valid_mask_numpy()
    m = np.ones(len(v), dtype=bool) if m is None else m
    if idx is not None:  # index -1 picks the appended NULL
        v, m = np.append(v, 0)[idx], np.append(m, False)[idx]
    return np.where(m, v, 0), m


def rows_sorted(arrays):
    a = np.stack([x.astype(np.int64) for x in arrays], axis=1) if arrays else np.zeros((0, 0), np.int64)
    if len(a) == 0:
        return a
    return a[np.lexsort(a.T[::-1])]


def expected(oracle, bt, bkeys, pt, pkeys, bo, po, is_na_equal):
    bid, bv, pid, pv = tuple_ids(bt, bkeys, pt, pkeys, is_na_equal)
    bi, pi = oracle.hash_join(bid, bv, pid, pv, bo, po, is_na_equal)
    arrays = []
    for t, idx in ((bt, bi), (pt, pi)):
        for c in t.columns:
            arrays += list(col_bits(c, idx))
    return rows_sorted(arrays)


def got_rows(outs):
    per = [[] for _ in range(outs[0].n_cols)]
    for o in outs:
        for j, c in enumerate(o.columns):
            per[j].append(col_bits(c))
    arrays = []
    for parts in per:
        arrays += [np.concatenate([p[0] for p in parts]), np.concatenate([p[1] for p in parts])]
    return rows_sorted(arrays)


def run(bt, bkeys, pt, pkeys, bo=False, po=False, is_na_equal=True, to_device=True, batch=None, used_cols=None, **kind):
    """One join state fed `batch`-row build then probe batches: (output tables copied to the host, metrics 5..7)."""
    st = init_join_state(-1, bkeys, pkeys, tuple(bt.names), tuple(pt.names), bo, po, is_na_equal=is_na_equal, **kind)
    bs = batch or max(bt.n_rows, pt.n_rows, 1)
    for i0 in range(0, max(bt.n_rows, 1), bs):
        b = bt.slice(i0, i0 + bs)
        join_build_consume_batch(st, table_to_device(b) if to_device else b, i0 + bs >= bt.n_rows)
    outs = []
    for i0 in range(0, max(pt.n_rows, 1), bs):
        p = pt.slice(i0, i0 + bs)
        out, _, _ = join_probe_consume_batch(st, table_to_device(p) if to_device else p, i0 + bs >= pt.n_rows, True, used_cols)
        outs.append(Table([Column(c.values_numpy().copy(), None if c.validity is None else np.packbits(c.valid_mask_numpy(), bitorder="little"),
                                  c.c_type, c.arr_type, c.length) for c in out.columns], list(out.names)))
    m = [get_metric(st, j) for j in (5, 6, 7)]
    delete_join_state(st)
    return outs, m


# ---- key columns of mixed types ----
def key_values(rng, kind, n, side):
    """Values from a small pool, so that tuples share most columns; float pools hold NaN, -0.0 (build) / 0.0 (probe) and ±inf."""
    if kind == "float64" or kind == "float32":
        pool = [NAN, np.inf, -np.inf, 1.5, -2.25, 7.0, -0.0 if side == "build" else 0.0]
        return rng.choice(np.array(pool, dtype=kind), n), -1
    if kind == "date":
        return rng.integers(18_000, 18_006, n).astype(np.int32), CTypes.DATE
    lo, hi = {"uint8": (250, 256), "int16": (-3, 3)}.get(kind, (-2, 4))
    return rng.integers(lo, hi, n).astype(kind), -1


SCHEMAS = {
    "int64+int32": ["int64", "int32"],
    "date+int64": ["date", "int64"],
    "float64+int64+int32": ["float64", "int64", "int32"],
    "uint8+int16": ["uint8", "int16"],
    "float32+int32": ["float32", "int32"],
    "int64+float64+int32+uint8": ["int64", "float64", "int32", "uint8"],
}


def key_tables(rng, kinds, nb, npr, nullable=True):
    """Build and probe tables with the key columns NOT in the leading positions and in a different order on each side.  Build:
    payload, k0, payload, k1, ...; probe: the keys reversed, a payload in the middle.  Returns (bt, bkeys, pt, pkeys)."""
    tabs = {}
    for side, n in (("build", nb), ("probe", npr)):
        cols = []
        for j, kind in enumerate(kinds):
            v, ct = key_values(rng, kind, n, side)
            valid = (rng.random(n) > 0.1) if nullable and j % 2 == 0 else None
            cols.append(col(v, valid, ct))
        tabs[side] = cols
    nk = len(kinds)
    b = [col(rng.integers(-(1 << 40), 1 << 40, nb))]
    bkeys = []
    for j in range(nk):
        bkeys.append(len(b))
        b.append(tabs["build"][j])
        if j == 0:
            b.append(col(rng.random(nb).astype(np.float32), rng.random(nb) > 0.2))
    p, pkeys = [], [None] * nk
    for j in reversed(range(nk)):
        pkeys[j] = len(p)
        p.append(tabs["probe"][j])
        if j == nk - 1:
            p.append(col(rng.integers(0, 1000, npr).astype(np.int32)))
    bt = Table(b, [f"b{i}" for i in range(len(b))])
    pt = Table(p, [f"p{i}" for i in range(len(p))])
    return bt, tuple(bkeys), pt, tuple(pkeys)


HOW = {"inner": (False, False), "left": (False, True), "right": (True, False), "outer": (True, True)}  # probe = left table


@pytest.mark.parametrize("schema", list(SCHEMAS))
@pytest.mark.parametrize("how", list(HOW))
@pytest.mark.parametrize("is_na_equal", [True, False])
def test_mixed_type_keys_every_outer_kind(gpu_lib, oracle, schema, how, is_na_equal):
    rng = np.random.default_rng([70, list(SCHEMAS).index(schema), list(HOW).index(how), int(is_na_equal)])
    bt, bkeys, pt, pkeys = key_tables(rng, SCHEMAS[schema], 2_500, 4_000)
    bo, po = HOW[how]
    to_device = how in ("inner", "outer")
    outs, m = run(bt, bkeys, pt, pkeys, bo, po, is_na_equal, to_device, batch=1_700)
    assert m == [0, 0, 0]  # multi-column keys always take the general (CSR) path
    np.testing.assert_array_equal(got_rows(outs), expected(oracle, bt, bkeys, pt, pkeys, bo, po, is_na_equal))


@pytest.mark.parametrize("is_na_equal", [True, False])
@pytest.mark.parametrize("to_device", [False, True])
def test_anti_and_mark_joins(gpu_lib, oracle, is_na_equal, to_device):
    rng = np.random.default_rng(71)
    bt, bkeys, pt, pkeys = key_tables(rng, ["float64", "int64", "int32"], 3_000, 20_000)
    bid, bv, pid, pv = tuple_ids(bt, bkeys, pt, pkeys, is_na_equal)
    has = pv & np.isin(pid, bid[bv])
    kept_p = list(range(pt.n_cols))
    anti, m = run(bt, bkeys, pt, pkeys, is_na_equal=is_na_equal, to_device=to_device, batch=7_000, used_cols=([], kept_p), is_anti_join=True)
    assert m == [0, 0, 0]
    rows = np.flatnonzero(~has)
    exp = rows_sorted([a for c in pt.columns for a in col_bits(c, rows)])
    np.testing.assert_array_equal(got_rows(anti), exp)
    mark, _ = run(bt, bkeys, pt, pkeys, is_na_equal=is_na_equal, to_device=to_device, batch=7_000, used_cols=([], kept_p), is_mark_join=True)
    flags = np.concatenate([o.columns[-1].values_numpy().astype(bool) for o in mark])
    np.testing.assert_array_equal(flags, has)  # a mark join emits the probe rows in order
    k0 = np.concatenate([col_bits(o.columns[0])[0] for o in mark])
    np.testing.assert_array_equal(k0, col_bits(pt.columns[0])[0])


def test_negative_zero_inside_a_tuple(gpu_lib, oracle):
    """-0.0 and 0.0 are one key inside a tuple; NaN joins NaN only under is_na_equal.  The build key columns carry the build rows'
    bits (-0.0 stays -0.0)."""
    bt = Table([col(np.array([-0.0, 1.0, NAN, -0.0], dtype=np.float64)), col(np.array([5, 5, 5, 6], dtype=np.int32)),
                col(np.arange(4, dtype=np.int64))], ["k0", "k1", "b"])
    pt = Table([col(np.array([0.0, 0.0, NAN, 1.0, -0.0], dtype=np.float64)), col(np.array([5, 6, 5, 6, 7], dtype=np.int32))], ["k0", "k1"])
    for na_eq, n_exp in ((True, 3), (False, 2)):
        outs, _ = run(bt, (0, 1), pt, (0, 1), is_na_equal=na_eq)
        np.testing.assert_array_equal(got_rows(outs), expected(oracle, bt, (0, 1), pt, (0, 1), False, False, na_eq))
        assert outs[0].n_rows == n_exp
        k0 = outs[0].columns[0].values_numpy()
        assert np.signbit(k0[k0 == 0]).all()  # both (0.0, 5) and (0.0, 6) matched a -0.0 build row


def test_duplicates_unique_and_empty_build(gpu_lib, oracle, monkeypatch):
    rng = np.random.default_rng(72)
    n = 20_000
    # many-to-many: every tuple 1..40 times on each side
    a, b = rng.integers(0, 30, n), rng.integers(0, 20, n).astype(np.int32)
    bt = Table([col(a), col(b), col(rng.integers(0, 1 << 40, n))], ["a", "b", "x"])
    pa, pb = rng.integers(0, 35, n), rng.integers(0, 20, n).astype(np.int32)
    pt = Table([col(pa), col(pb), col(rng.random(n))], ["a", "b", "y"])
    outs, m = run(bt, (0, 1), pt, (0, 1), batch=6_000)
    assert m == [0, 0, 0]
    np.testing.assert_array_equal(got_rows(outs), expected(oracle, bt, (0, 1), pt, (0, 1), False, False, True))
    # unique build tuples on an all-8-byte, bitmap-free schema (what a single int64 key would run inline): the CSR form, and
    # B200_JOIN_INLINE=0 changes nothing
    perm = rng.permutation(n)
    ub = Table([col(perm // 8), col(perm % 8), col(rng.integers(0, 1 << 40, n))], ["a", "b", "x"])
    up = Table([col(rng.integers(0, n // 8 + 10, 3 * n)), col(rng.integers(0, 10, 3 * n)), col(rng.integers(0, 1 << 40, 3 * n))], ["a", "b", "y"])
    exp = expected(oracle, ub, (0, 1), up, (0, 1), False, False, True)
    for env in ("1", "0"):
        monkeypatch.setenv("B200_JOIN_INLINE", env)
        outs, m = run(ub, (0, 1), up, (0, 1), batch=25_000)
        assert m == [0, 0, 0]
        np.testing.assert_array_equal(got_rows(outs), exp)
    # empty build side
    eb = Table([col(np.zeros(0, np.int64)), col(np.zeros(0, np.int32)), col(np.zeros(0, np.int64))], ["a", "b", "x"])
    for bo, po in HOW.values():
        outs, _ = run(eb, (0, 1), pt, (0, 1), bo, po)
        assert sum(o.n_rows for o in outs) == (n if po else 0)
        np.testing.assert_array_equal(got_rows(outs), expected(oracle, eb, (0, 1), pt, (0, 1), bo, po, True))


@pytest.mark.parametrize("how", ["inner", "left"])
def test_large_tuples_that_differ_in_one_column(gpu_lib, how):
    """4 M distinct build tuples (a, b) = (x >> 2, x & 3); probe tuples (a', b') with b' in [0, 8): half of them agree with a build
    tuple in a but not in b.  Slot walks, tag hits and column compares at a real table size; checked by arithmetic."""
    import torch

    dev = torch.device("cuda", 0)
    g = torch.Generator(device=dev).manual_seed(73)
    nb, npr = 1 << 22, 12_000_000
    x = torch.randperm(nb, device=dev, generator=g)
    bt = Table([Column(x >> 2), Column((x & 3).to(torch.int32)), Column(x * 7 + 1)], ["a", "b", "x"])
    pa = torch.randint(0, nb // 4 + 1000, (npr,), device=dev, generator=g)
    pb = torch.randint(0, 8, (npr,), device=dev, generator=g, dtype=torch.int32)
    pt = Table([Column(pb), Column(torch.arange(npr, device=dev)), Column(pa)], ["b", "i", "a"])
    st = init_join_state(-1, (0, 1), (2, 0), ("a", "b", "x"), ("b", "i", "a"), False, how == "left")
    join_build_consume_batch(st, bt, True)
    out, _, _ = join_probe_consume_batch(st, pt, True, True)
    c = [torch.as_tensor(cc.data, device=dev)[: out.n_rows] for cc in out.columns]  # a, b, x, b', i, a'
    match = (pa < nb // 4) & (pb < 4)
    if how == "inner":
        assert out.n_rows == int(match.sum())
        assert torch.equal(c[0], c[5]) and torch.equal(c[1], c[3])
        assert torch.equal(c[2], ((c[0] << 2) | c[1].to(torch.int64)) * 7 + 1)
        assert torch.equal(torch.sort(c[4]).values, torch.nonzero(match).flatten())
    else:
        assert out.n_rows == npr and out.columns[2].validity is not None
        valid = torch.as_tensor(out.columns[2].valid_mask_numpy(), device=dev)
        order = torch.argsort(c[4])
        assert torch.equal(c[4][order], torch.arange(npr, device=dev))
        assert torch.equal(valid[order], match)
        mx = c[2][order][match]
        assert torch.equal(mx, ((pa[match] << 2) | pb[match].to(torch.int64)) * 7 + 1)
    delete_join_state(st)


@pytest.mark.parametrize("bad", ["count", "five", "int_width", "float_int", "float_width"])
def test_key_type_and_count_errors(gpu_lib, bad):
    n = 10
    ints = lambda dt: col(np.arange(n).astype(dt))
    if bad == "count":
        with pytest.raises(_lib.B200Error, match="same number"):
            init_join_state(-1, (0, 1), (0,), ("a", "b"), ("a", "b"), False, False)
        return
    if bad == "five":
        with pytest.raises(_lib.B200Error, match="1 to 4"):
            init_join_state(-1, tuple(range(5)), tuple(range(5)), tuple("abcde"), tuple("abcde"), False, False)
        return
    b_dt, p_dt = {"int_width": ("int64", "int32"), "float_int": ("float64", "int64"), "float_width": ("float64", "float32")}[bad]
    bt = Table([ints("int32"), ints(b_dt), ints("int64")], ["a", "b", "c"])
    pt = Table([ints("int32"), ints(p_dt)], ["a", "b"])
    st = init_join_state(-1, (0, 1), (0, 1), ("a", "b", "c"), ("a", "b"), False, False)
    join_build_consume_batch(st, table_to_device(bt), True)
    try:
        for call in (lambda: join_probe_consume_batch(st, table_to_device(pt), True),
                     lambda: runtime_join_filter((st,), table_to_device(pt), ((0, 1),))):
            with pytest.raises(_lib.B200Error) as e:
                call()
            msg = str(e.value)
            assert "key position 1" in msg and np.dtype(b_dt).name in msg and np.dtype(p_dt).name in msg, msg
    finally:
        delete_join_state(st)


# ---- runtime filter ----
def filter_keep(st, pt, key_cols, use_mm):
    import torch

    L = _lib.lib()
    keep = torch.zeros(pt.n_rows + 8, dtype=torch.uint8, device="cuda:0")
    ct = CTable(pt)  # owns the column descriptors ct.ptr points to, so it must outlive the call
    rc = L.b200_join_runtime_filter_n(st.handle, ct.ptr, ffi.new("int32_t[]", list(key_cols)), len(key_cols),
                                      ffi.new("int32_t[]", list(use_mm)), 1, ffi.cast("uint8_t*", keep.data_ptr()))
    _lib.check(rc, "runtime filter")
    return keep[: pt.n_rows].cpu().numpy().astype(bool)


@pytest.mark.parametrize("kinds", [["int64"], ["float64"], ["float64", "int64", "int32"]], ids="+".join)
@pytest.mark.parametrize("is_na_equal", [True, False])
def test_runtime_filter_has_no_false_negatives(gpu_lib, kinds, is_na_equal):
    """Key columns 0 and 2 are nullable and float columns hold NaN: under is_na_equal a probe row with NA key columns that has a
    partner on the build side must pass the filter, for one key column as for several."""
    rng = np.random.default_rng(74)
    bt, bkeys, pt, pkeys = key_tables(rng, kinds, 5_000, 200_000)
    st = init_join_state(-1, bkeys, pkeys, tuple(bt.names), tuple(pt.names), False, False, is_na_equal=is_na_equal)
    join_build_consume_batch(st, table_to_device(bt), True)
    _, bounds = build_runtime_filter(st)
    assert len(bounds) == len(kinds)
    bid, bv, pid, pv = tuple_ids(bt, bkeys, pt, pkeys, is_na_equal)
    # integer columns: plain min / max over the non-NA values of the build rows that can match
    for j in [j for j, kind in enumerate(kinds) if kind.startswith("int")]:
        k, v = canon(bt.columns[bkeys[j]])
        assert bounds[j] == (int(k[v & bv].min()), int(k[v & bv].max()))
    dpt = table_to_device(pt)
    keep = filter_keep(st, dpt, pkeys, [1] * len(kinds))
    partner = pv & np.isin(pid, bid[bv])
    assert keep[partner].all()  # no false negatives
    if not is_na_equal:
        assert not keep[~pv].any()  # a row with an NA key column can never match
    kept = runtime_join_filter((st,), dpt, (pkeys,))
    assert kept.n_rows == keep.sum()
    out, _, _ = join_probe_consume_batch(st, kept, True, True)
    u, cnt = np.unique(bid[bv], return_counts=True)
    pos = np.searchsorted(u, pid[partner])
    assert out.n_rows == cnt[pos].sum()
    delete_join_state(st)


def test_runtime_filter_bounds_absent_columns_and_entry_points(gpu_lib):
    rng = np.random.default_rng(75)
    nb, npr = 10_000, 100_000
    bt = Table([col(rng.integers(0, 1000, nb)), col(rng.integers(100, 201, nb).astype(np.int32)), col(rng.random(nb))], ["a", "b", "x"])
    pb = rng.integers(0, 400, npr).astype(np.int32)
    pt = table_to_device(Table([col(rng.random(npr)), col(pb), col(rng.integers(0, 1000, npr))], ["y", "b", "a"]))
    st = init_join_state(-1, (0, 1), (2, 1), ("a", "b", "x"), ("y", "b", "a"), False, False)
    join_build_consume_batch(st, table_to_device(bt), True)
    _, bounds = build_runtime_filter(st)
    assert bounds[1] == (int(bt.columns[1].data.min()), int(bt.columns[1].data.max()))
    inb = (pb >= bounds[1][0]) & (pb <= bounds[1][1])
    # column a absent: no bloom filter, only b's bounds apply
    np.testing.assert_array_equal(filter_keep(st, pt, (-1, 1), (1, 1)), inb)
    assert filter_keep(st, pt, (-1, 1), (1, 0)).all()  # b's bounds switched off: nothing drops a row
    both = filter_keep(st, pt, (2, 1), (1, 1))
    assert not both[~inb].any() and both.sum() < inb.sum()  # the bloom filter drops more
    # every key column absent: the table passes through
    assert runtime_join_filter((st,), pt, ((-1, -1),)).n_rows == npr
    assert runtime_join_filter((st,), pt, ((2, 1),), ((0, 1),)).n_rows <= inb.sum()
    L = _lib.lib()
    # the _n bounds entry point installs per-column bounds: an empty range on b drops every row
    _lib.check(L.b200_join_set_key_bounds_n(st.handle, ffi.new("int64_t[]", [0, 10_000, 1, 0]), 2))
    assert not filter_keep(st, pt, (2, 1), (1, 1)).any()
    assert L.b200_join_set_key_bounds_n(st.handle, ffi.new("int64_t[]", [0, 1]), 1) < 0
    delete_join_state(st)


@pytest.mark.parametrize("how", ["inner", "left", "right", "outer"])
def test_physical_merge_list_keys_equals_pandas(gpu_lib, how):
    from bodo_b200.physical import merge

    rng = np.random.default_rng(76)
    left = pd.DataFrame({"x": rng.integers(0, 1000, 3_000), "suppkey": rng.integers(0, 6, 3_000).astype(np.int32),
                         "partkey": rng.integers(0, 50, 3_000), "price": rng.choice([0.5, 1.5, NAN, -0.0], 3_000)})
    right = pd.DataFrame({"pk": rng.integers(0, 60, 900), "qty": rng.random(900), "px": rng.choice([0.5, 1.5, NAN, 0.0], 900),
                          "sk": rng.integers(0, 6, 900).astype(np.int32)})
    got = merge(left, right, left_on=["partkey", "suppkey", "price"], right_on=["pk", "sk", "px"], how=how, batch_size=1_000)
    exp = right.merge(left, left_on=["pk", "sk", "px"], right_on=["partkey", "suppkey", "price"], how={"left": "right", "right": "left"}.get(how, how))
    assert_rowset_equal(got, exp)
    with pytest.raises(ValueError):
        merge(left, right, left_on=["partkey", "suppkey"], right_on=["pk"])


def _sharded_worker(rank, world, port, q):
    import os

    import torch
    import torch.distributed as dist
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", rank))
    try:
        from oracle import oracle as O
        rng = np.random.default_rng(77)  # the same global tables on every rank; each rank feeds its own row slice
        bt, bkeys, pt, pkeys = key_tables(rng, ["int64", "float64", "int32"], 20_000, 60_000, nullable=False)
        results = {}
        for name, kw, bo, po, na_eq in (("shuffle", {}, False, False, False), ("shuffle-outer", {}, True, True, True),
                                        ("broadcast", {"force_broadcast": True}, False, True, True)):
            os.environ["BODO_BCAST_JOIN_THRESHOLD"] = "0" if name != "broadcast" else str(10 << 20)
            st = init_join_state(-1, bkeys, pkeys, tuple(bt.names), tuple(pt.names), bo, po, build_parallel=True, probe_parallel=True,
                                 device=rank, is_na_equal=na_eq, **kw)
            bchunk, pchunk = (bt.n_rows + world - 1) // world, (pt.n_rows + world - 1) // world
            join_build_consume_batch(st, bt.slice(rank * bchunk, (rank + 1) * bchunk), True)
            out, _, _ = join_probe_consume_batch(st, pt.slice(rank * pchunk, (rank + 1) * pchunk), True, True)
            host = Table([Column(c.values_numpy().copy(), None if c.validity is None else np.packbits(c.valid_mask_numpy(), bitorder="little"),
                                 c.c_type, c.arr_type, c.length) for c in out.columns], list(out.names))
            delete_join_state(st)
            allg = [None] * world
            dist.all_gather_object(allg, got_rows([host]))
            if rank == 0:
                g = rows_sorted(list(np.concatenate(allg).T))
                e = expected(O, bt, bkeys, pt, pkeys, bo, po, na_eq)
                results[name] = bool(g.shape == e.shape and np.array_equal(g, e))
        q.put((rank, results))
    except Exception:
        import traceback
        q.put((rank, traceback.format_exc()))
    finally:
        dist.destroy_process_group()


@pytest.mark.timeout(600)
def test_sharded_join_two_gpus(gpu_lib):
    """Partitioned (hash_keys over the three key columns) and broadcast multi-key joins over the ranks; the union of the ranks'
    outputs equals the oracle's join of the global tables.  NaN keys are numpy NaN on both sides, so they hash alike."""
    import socket

    import torch
    import torch.multiprocessing as mp
    world = min(torch.cuda.device_count(), 4)
    if world < 2:
        pytest.skip("needs at least 2 GPUs")
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=_sharded_worker, args=(r, world, port, q)) for r in range(world)]
    for p in procs:
        p.start()
    res = [q.get(timeout=500) for _ in range(world)]
    for p in procs:
        p.join(timeout=60)
    for r in res:
        assert isinstance(r[1], dict), r
    r0 = [r for r in res if r[0] == 0][0][1]
    assert r0 == {"shuffle": True, "shuffle-outer": True, "broadcast": True}, r0
