"""The groupby against an exact reference for every key and value column type, single- and multi-column keys.

Reference (CPU, below: plain numpy over the input Table, no pandas groupby, no device):
  * group identity: a key cell is NA when its validity bit is clear; an integer, bool or temporal cell is its exact value in its
    own type (uint64 by its bit pattern, i.e. as unsigned); a float cell is its float64 value with -0.0 folded onto 0.0, and
    every NaN is one value, distinct from NA.  A group is the tuple of its key cells, NA-ness included, so (NA, 0) and (0, 0) are
    two groups.  dropna=True drops every row with an NA or NaN key component.
  * size / count: rows / non-NA values (NaN is NA); int64, numpy.
  * sum of an integer or bool column: the exact sum mod 2^64, bit for bit; int64 for signed and bool inputs, uint64 for unsigned
    ones; the input's array kind, except that a bool input gives a nullable output.  Of a float column: the input's type,
    |got - exact| <= gamma_{n-1} sum|x| (+ one float32 rounding).
  * mean: the exact rational sum of float64(value) over the count, rounded once; float64, nullable (NA without values).  Bit for
    bit when the group's values are integers with sum|x| < 2^52 (every partial sum is then exact in any order), otherwise
    |got - exact| <= gamma_{n-1} sum|x| / n + u |exact|.
  * min / max: the least / greatest valid value in the input's type, bit for bit (floats in IEEE total order, -0.0 < 0.0, NaN
    skipped); uint64 is refused by the constructor.  first / last: the cell of the first / last valid row in arrival order.
    nunique: distinct valid values (floats: -0.0 equals 0.0, NaN is NA).  These three take single-column keys only.
  * var / std / var_pop / std_pop / skew: exact_moments of float64(value), within var_tol / skew_tol
    (tests/test_gpu_groupby_float_values.py derives both bounds).
Every output column's c_type and array kind is pinned as well; a nullable output's NA mask must match the reference's.

What runs through it: every key type (numpy and nullable, both dropna) through host batches and one device batch, and every key
type wide enough for it through a table that grows; the SM-partitioned generic kernels (SPG-G) for the key types they accept; every value type under an int64 key;
multi-column keys of 2, 3 and 4 mixed-type nullable columns (every NA mask, tuples that differ only in NA-ness, -0.0 / 0.0 and
NaN components), including one of more than a million groups sliced by a small output batch; and mean / var / std / skew of
uint64 values at and above 2^63 through every path of the float-values file (host, device, growth, multi-column key, special
slots, fused and NCCL exchanges), which read those values as negative before load_as_f64 widened uint64 as unsigned."""

import functools
import math
from fractions import Fraction

import numpy as np
import pytest

from bodo_b200.table import ArrTypes, Column, CTypes, Table, np_dtype_of
from tests.test_gpu_groupby_float_values import (PATHS, U, _groups, _total_order, exact_moments, gamma, run_path, skew_tol,
                                                 var_tol)
from tests.test_gpu_sort import KEY_TYPES, gen_values, make_column

ALL_TYPES = KEY_TYPES  # the 14 fixed-width column types
FLOATS = (CTypes.FLOAT32, CTypes.FLOAT64)
TEMPORAL = (CTypes.DATE, CTypes.DATETIME, CTypes.TIMEDELTA)
SIGNED = (CTypes.INT8, CTypes.INT16, CTypes.INT32, CTypes.INT64) + TEMPORAL
MOMENTS = ("var", "std", "var_pop", "std_pop", "skew")
TNAME = {v: k.lower() for k, v in vars(CTypes).items() if isinstance(v, int)}
INT64_MIN, INT64_MAX = np.iinfo(np.int64).min, np.iinfo(np.int64).max
HOST_BATCH = 4_097


# ---- exact reference ---------------------------------------------------------------------------------------------------

def encode(col: Column):
    """(state, code) per cell: state 0 = a value, 1 = NA, 2 = NaN; code = the value's identity (an integer / temporal cell's
    exact bits, a float's float64 bits with -0.0 folded onto 0.0), 0 unless state is 0."""
    v = col.values_numpy()
    state = np.zeros(len(v), np.int64)
    if col.validity is not None:
        state[~col.valid_mask_numpy()] = 1
    if v.dtype.kind == "f":
        d = v.astype(np.float64)
        state[(state == 0) & np.isnan(d)] = 2
        code = np.where(d == 0, 0.0, d).view(np.int64)
    elif v.dtype.itemsize == 8:
        code = v.view(np.int64)
    else:
        code = v.astype(np.int64)  # (bool storage and the narrow types: their exact value)
    return state, np.where(state == 0, code, 0)


def key_matrix(keys):
    return np.stack([a for c in keys for a in encode(c)], axis=1)


def group_rows(keys, dropna):
    """-> (kept rows in arrival order, group id of each kept row, the groups' key matrix (state, code per column) in
    lexicographic order)"""
    M = key_matrix(keys)
    keep = (M[:, 0::2] == 0).all(axis=1) if dropna else np.ones(len(M), bool)
    rows = np.flatnonzero(keep)
    groups, gid = np.unique(M[rows], axis=0, return_inverse=True)
    return rows, gid.reshape(-1), groups


def _valid_values(col, rows):
    v = col.values_numpy()[rows]
    ok = col.valid_mask_numpy()[rows] if col.validity is not None else np.ones(len(rows), bool)
    if col.c_type in FLOATS:
        ok &= ~np.isnan(v)
    return v, ok


def _exact_means(x, g, G, cnt):
    """exact mean, sum|x| and "bit-exact" (integers, sum|x| < 2^52) per group of the float64 values x with group ids g"""
    abs_sum = np.zeros(G)
    np.add.at(abs_sum, g, np.abs(x))
    if not (np.isfinite(x).all() and (x == np.round(x)).all()):
        refs = [exact_moments(x[ix]) for ix in _groups(g, G)]
        return np.array([np.nan if r["mean"] is None else r["mean"] for r in refs]), np.array([r["abs_sum"] for r in refs]), np.zeros(G, bool)
    with np.errstate(invalid="ignore", divide="ignore"):
        if np.abs(x).sum() < 2.0 ** 53:  # int64 sums are exact and so are their float64 images: one rounded division
            s = np.zeros(G, np.int64)
            np.add.at(s, g, x.astype(np.int64))
            mean = s / cnt
        else:
            order = np.argsort(g, kind="stable")
            b = np.searchsorted(g[order], np.arange(G + 1))
            xs = x[order].tolist()
            mean = np.array([float(Fraction(sum(int(t) for t in xs[b[j]:b[j + 1]]), int(cnt[j]))) if cnt[j] else np.nan
                             for j in range(G)])
    return mean, abs_sum, abs_sum < 2.0 ** 52


def expect(f, col, rows, gid, G, sample=None):
    """The reference's output column of function f over `col`: a dict of c_type, arr_type, `valid` (the reference defines a
    value), `bitmap` (the output carries validity) and either `bits` (compared bit for bit), `mean`, `fsum` or `moments`."""
    ct, at = col.c_type, col.arr_type
    v, ok = _valid_values(col, rows)
    cnt = np.bincount(gid[ok], minlength=G)
    seen = cnt > 0
    e = dict(fn=f, ct=ct, at=at, valid=np.ones(G, bool), bitmap=at == ArrTypes.NULLABLE_INT_BOOL)
    if f in ("size", "count", "nunique"):
        if f == "size":
            n = np.bincount(gid, minlength=G)
        elif f == "count":
            n = cnt
        else:
            code = encode(col)[1][rows][ok]
            n = np.bincount(np.unique(np.stack([gid[ok], code], axis=1), axis=0)[:, 0], minlength=G)
        e.update(ct=CTypes.INT64, at=ArrTypes.NUMPY, bitmap=False, bits=n.astype(np.int64))
    elif f == "sum" and ct not in FLOATS:
        w = v.astype(np.int64).view(np.uint64) if ct in SIGNED else v.astype(np.uint64)
        s = np.zeros(G, np.uint64)
        np.add.at(s, gid[ok], w[ok])
        signed = ct in SIGNED or ct == CTypes.BOOL
        e.update(ct=CTypes.INT64 if signed else CTypes.UINT64, bits=s.view(np.int64) if signed else s)
        if ct == CTypes.BOOL:
            e.update(at=ArrTypes.NULLABLE_INT_BOOL, bitmap=True)
    elif f == "sum":
        x = v[ok].astype(np.float64)
        e["fsum"] = [exact_moments(x[ix]) for ix in _groups(gid[ok], G)]
    elif f == "mean":
        x = v[ok].astype(np.float64)
        e.update(ct=CTypes.FLOAT64, at=ArrTypes.NULLABLE_INT_BOOL, bitmap=True, valid=seen, n=cnt)
        e["mean"], e["abs_sum"], e["bit_exact"] = _exact_means(x, gid[ok], G, cnt)
    elif f in ("min", "max"):
        mn = f == "min"
        if ct in FLOATS:
            key = _total_order(v.astype(np.float64))
            m = np.full(G, INT64_MAX if mn else INT64_MIN, np.int64)
            (np.minimum if mn else np.maximum).at(m, gid[ok], key[ok])
            dec = np.where(m < 0, m ^ np.int64(INT64_MAX), m).view(np.float64)
            bits = np.where(seen, dec, np.nan).astype(v.dtype)
        else:
            m = np.full(G, INT64_MAX if mn else INT64_MIN, np.int64)
            (np.minimum if mn else np.maximum).at(m, gid[ok], v[ok].astype(np.int64))
            bits = np.where(seen, m, 0).astype(v.dtype)
        e.update(valid=seen, bits=bits)
    elif f in ("first", "last"):
        pos = np.flatnonzero(ok)
        idx = np.full(G, len(v) if f == "first" else -1, np.int64)
        (np.minimum if f == "first" else np.maximum).at(idx, gid[pos], pos)
        bits = v[np.where(seen, idx, 0)] if len(v) else np.zeros(G, v.dtype)
        bits = np.where(seen, bits, np.nan if ct in FLOATS else 0).astype(v.dtype)
        e.update(valid=seen, bits=bits)
    else:
        assert f in MOMENTS, f
        x = v[ok].astype(np.float64)
        order = np.argsort(gid[ok], kind="stable")
        b = np.searchsorted(gid[ok][order], np.arange(G + 1))
        pick = range(G) if sample is None or G <= sample else np.linspace(0, G - 1, sample).astype(np.int64)
        e.update(ct=CTypes.FLOAT64, at=ArrTypes.NULLABLE_INT_BOOL, bitmap=True)
        e["moments"] = {int(g): exact_moments(x[order[b[g]:b[g + 1]]]) for g in pick}
    return e


def reference(keys, vals, fn, cols, dropna, sample=None):
    """-> (the groups' key matrix, one expect() dict per function); cols index `vals`"""
    rows, gid, groups = group_rows(keys, dropna)
    return groups, [expect(f, vals[c], rows, gid, len(groups), sample) for f, c in zip(fn, cols)]


# ---- comparing a device result with the reference ---------------------------------------------------------------------

def _uint_view(a):
    return np.ascontiguousarray(a).view(f"u{a.dtype.itemsize}")


def _match_groups(out_keys, groups):
    """row order of the device output that lines it up with the reference's groups (each group exactly once)"""
    M = key_matrix(out_keys)
    assert M.shape == groups.shape, (M.shape, groups.shape)
    order = np.lexsort(M.T[::-1])
    bad = np.flatnonzero((M[order] != groups).any(axis=1))
    assert len(bad) == 0, ("group keys differ", bad[:5], M[order][bad[:5]], groups[bad[:5]])
    return order


def check_column(got: Column, e, order, what):
    ctx = (what, e["fn"])
    assert (got.c_type, got.arr_type) == (e["ct"], e["at"]), ctx + ((got.c_type, got.arr_type), (e["ct"], e["at"]))
    vals = got.values_numpy()[order]
    assert vals.dtype == np_dtype_of(e["ct"]), ctx + (vals.dtype,)
    mask = got.valid_mask_numpy()
    assert (mask is not None) == e["bitmap"], ctx + ("validity bitmap",)
    if mask is not None:
        mask = mask[order]
    if "moments" in e:
        for g, r in e["moments"].items():
            x, ex = vals[g], r[e["fn"]]
            c = ctx + (g, r["n"], x, ex)
            if ex is None:
                assert not mask[g], c
                continue
            assert mask[g], c
            if not math.isfinite(ex):
                assert x == ex or (math.isnan(ex) and math.isnan(x)), c
            elif e["fn"] == "skew":
                assert abs(x - ex) <= skew_tol(r), c + (skew_tol(r),)
            else:
                assert abs(x - ex) <= var_tol(r) * abs(ex), c + (var_tol(r),)
        return
    if mask is not None:
        bad = np.flatnonzero(mask != e["valid"])
        assert len(bad) == 0, ctx + ("NA mask", bad[:5])
    if "fsum" in e:
        ex = np.array([r["sum"] for r in e["fsum"]])
        n, abs_sum = np.array([r["n"] for r in e["fsum"]]), np.array([r["abs_sum"] for r in e["fsum"]])
        fin = np.isfinite(ex)
        got = vals.astype(np.float64)
        assert ((got[~fin] == ex[~fin]) | (np.isnan(got[~fin]) & np.isnan(ex[~fin]))).all(), ctx
        r32 = 2.0 ** -24 if e["ct"] == CTypes.FLOAT32 else 0.0  # the float32 output is the float64 sum rounded once more
        with np.errstate(invalid="ignore"):  # (groups with ±inf: compared exactly above)
            bound = gamma(n - 1) * abs_sum * (1 + r32) + r32 * np.abs(ex)
            bad = np.flatnonzero(fin & ~(np.abs(got - ex) <= bound))
        assert len(bad) == 0, ctx + (bad[:5], got[bad[:5]], ex[bad[:5]])
        return
    if "mean" in e:
        ex, valid = e["mean"], e["valid"]
        exact = valid & e["bit_exact"]
        bad = np.flatnonzero(exact & (_uint_view(vals) != _uint_view(ex)))
        assert len(bad) == 0, ctx + ("bit-exact mean", bad[:5], vals[bad[:5]], ex[bad[:5]])
        fin = valid & ~exact & np.isfinite(ex)
        n = np.maximum(e["n"], 1)
        with np.errstate(invalid="ignore"):  # (groups with ±inf or without values: compared below / by the NA mask)
            bound = gamma(n - 1) * e["abs_sum"] / n * (1 + U) + U * np.abs(ex)
            bad = np.flatnonzero(fin & ~(np.abs(vals - ex) <= bound))
        assert len(bad) == 0, ctx + ("mean", bad[:5], vals[bad[:5]], ex[bad[:5]])
        inf = valid & ~np.isfinite(ex)
        assert ((vals[inf] == ex[inf]) | (np.isnan(vals[inf]) & np.isnan(ex[inf]))).all(), ctx
        return
    exp, valid = e["bits"], e["valid"]
    assert exp.dtype.itemsize == vals.dtype.itemsize, ctx
    bad = np.flatnonzero(valid & (_uint_view(vals) != _uint_view(exp)))
    assert len(bad) == 0, ctx + (bad[:5], vals[bad[:5]], exp[bad[:5]])
    if mask is None and vals.dtype.kind == "f":  # a numpy float output marks a group without values by NaN
        assert np.isnan(vals[~valid]).all(), ctx


def check_result(out, nk, groups, exp, what):
    order = _match_groups(out[:nk], groups)
    for j, e in enumerate(exp):
        check_column(out[nk + j], e, order, what)


# ---- running the device groupby ---------------------------------------------------------------------------------------

def _collect(parts):
    """output batches (lists of host (values, mask, c_type, arr_type)) -> one host Column per output column"""
    cols = []
    for j in range(len(parts[0])):
        ps = [p[j] for p in parts]
        assert len({(p[2], p[3], p[1] is None) for p in ps}) == 1, "output batches disagree on a column's type"
        data = np.concatenate([p[0] for p in ps])
        mask = None if ps[0][1] is None else np.concatenate([p[1] for p in ps])
        cols.append(Column(data, None if mask is None else np.packbits(mask, bitorder="little"), ps[0][2], ps[0][3], len(data)))
    return cols


def run(table, nk, fn, cols, dropna=True, feed="host", expected_groups=0, output_batch_size=1 << 30, device_batch=None):
    """Groups `table` by its first nk columns; fn[j] reads column cols[j] (a logical index).  feed: "host" (HOST_BATCH-row host
    batches) or "device" (device batches of device_batch rows, default one batch).  Returns (output columns on the host,
    metrics, number of output batches)."""
    from bodo_b200.streaming.groupby import (delete_groupby_state, get_metric, groupby_build_consume_batch,
                                             groupby_produce_output_batch, init_groupby_state)
    from tests.helpers import table_to_device

    st = init_groupby_state(-1, tuple(range(nk)), fn, tuple(range(len(fn) + 1)), cols, dropna=dropna,
                            expected_groups=expected_groups, output_batch_size=output_batch_size)
    n = table.n_rows
    step = HOST_BATCH if feed == "host" else (device_batch or max(n, 1))
    starts = list(range(0, n, step)) or [0]
    try:
        for i, r0 in enumerate(starts):
            b = table.slice(r0, r0 + step)
            groupby_build_consume_batch(st, b if feed == "host" else table_to_device(b), i == len(starts) - 1, True)
        parts = []
        while True:
            out, last = groupby_produce_output_batch(st, True)
            parts.append([(c.values_numpy().copy(), c.valid_mask_numpy(), c.c_type, c.arr_type) for c in out.columns])
            if last:
                break
        metrics = {w: get_metric(st, w) for w in (3, 8, 10, 12, 14)}
    finally:
        delete_groupby_state(st)
    return _collect(parts), metrics, len(parts)


# ---- data ---------------------------------------------------------------------------------------------------------------

def _column(data, ct, rng, nullable, na_frac=0.15):
    data = np.ascontiguousarray(data.astype(np.uint8) if ct == CTypes.BOOL else data)
    if not nullable:
        return Column(data, None, ct, ArrTypes.NUMPY, len(data))
    valid = rng.random(len(data)) >= na_frac
    return Column(data, np.packbits(valid, bitorder="little"), ct, ArrTypes.NULLABLE_INT_BOOL, len(data))


def key_column(ct, n, rng, nullable, n_distinct):
    """keys drawn from n_distinct values of the type, its edge values among them (gen_values: min, max, 0, 1; floats: ±0.0,
    ±inf, NaN, subnormals, max; INT64_MIN, the table's marker key, for int64 / datetime / timedelta)"""
    pool = gen_values(ct, n_distinct, rng, small=False)
    if ct == CTypes.UINT64:
        pool[-1] = 2 ** 63
    return _column(pool[rng.integers(0, len(pool), n)], ct, rng, nullable)


def value_column(ct, n, rng, nullable):
    """gen_values' small values with the type's edges mixed in; a float max becomes 2.5 (a sum past it overflows in an order-
    dependent way: the float-values file pins floats at the overflow edge)"""
    c = make_column(ct, n, rng, nullable)
    if ct in FLOATS:
        big = np.isfinite(c.data) & (np.abs(c.data) > 1e30)
        c.data[big] = np.copysign(2.5, c.data[big])
    return c


# ---- the reference pinned on the CPU ----------------------------------------------------------------------------------

def test_reference_against_pandas():
    """Integer values with sums far below 2^53 and no NaN keys, where pandas' groupby is exact: sizes, counts, sums, means,
    min / max / first / last / nunique bit for bit, the moments to 1e-9, over a 3-column key with NA and uint64 2^63 / 2^64 - 1
    components and -0.0 / 0.0 float components, both dropna values."""
    import pandas as pd

    rng = np.random.default_rng(11)
    n = 4_000
    k0 = rng.integers(-3, 3, n).astype(np.int16)
    k0_valid = rng.random(n) >= 0.2
    k1 = np.array([0, 5, 2 ** 63, 2 ** 64 - 1], dtype=np.uint64)[rng.integers(0, 4, n)]
    k2 = np.array([-0.0, 0.0, 1.5, -2.0])[rng.integers(0, 4, n)]
    v = rng.integers(-1000, 1000, n)
    v_valid = rng.random(n) >= 0.2
    cols = [Column(k0, np.packbits(k0_valid, bitorder="little"), CTypes.INT16, ArrTypes.NULLABLE_INT_BOOL, n),
            Column(k1, None, CTypes.UINT64, ArrTypes.NUMPY, n), Column(k2, None, CTypes.FLOAT64, ArrTypes.NUMPY, n),
            Column(v, np.packbits(v_valid, bitorder="little"), CTypes.INT64, ArrTypes.NULLABLE_INT_BOOL, n)]
    df = pd.DataFrame({"k0": pd.arrays.IntegerArray(k0, ~k0_valid), "k1": k1, "k2": k2, "v": pd.arrays.IntegerArray(v, ~v_valid)})
    pd_fn = {"size": lambda g: g.size(), "count": lambda g: g.count(), "sum": lambda g: g.sum(), "mean": lambda g: g.mean(),
             "min": lambda g: g.min(), "max": lambda g: g.max(), "first": lambda g: g.first(), "last": lambda g: g.last(),
             "nunique": lambda g: g.nunique(), "var": lambda g: g.var(), "std": lambda g: g.std(),
             "var_pop": lambda g: g.var(ddof=0), "std_pop": lambda g: g.std(ddof=0), "skew": lambda g: g.skew()}
    for nk, fns in ((3, ("size", "count", "sum", "mean", "min", "max") + MOMENTS), (1, ("first", "last", "nunique", "sum", "mean"))):
        for dropna in (True, False):
            rows, gid, groups = group_rows(cols[:nk], dropna)
            G = len(groups)
            g = df.groupby([f"k{j}" for j in range(nk)], dropna=dropna, sort=False)
            pid = g.ngroup().to_numpy(dtype=np.float64, na_value=np.nan)
            np.testing.assert_array_equal(np.flatnonzero(~np.isnan(pid)), rows)
            pairs = np.unique(np.stack([gid, pid[rows].astype(np.int64)], axis=1), axis=0)
            assert len(pairs) == G == g.ngroups  # the same partition of the kept rows
            to_pd = pairs[:, 1]  # reference group -> pandas group
            for f in fns:
                e = expect(f, cols[3], rows, gid, G)
                s = pd_fn[f](g["v"]).iloc[to_pd]
                na = s.isna().to_numpy()
                if "moments" in e:
                    got = np.array([np.nan if e["moments"][j][f] is None else e["moments"][j][f] for j in range(G)])
                    np.testing.assert_array_equal(np.isnan(got), na, err_msg=f)
                    np.testing.assert_allclose(got[~na], s.to_numpy(dtype=np.float64)[~na], rtol=1e-9, atol=1e-12, err_msg=f)
                    continue
                ref = e["mean"] if f == "mean" else e["bits"]
                np.testing.assert_array_equal(~e["valid"], na, err_msg=f)
                np.testing.assert_array_equal(ref[~na], s.to_numpy(dtype=ref.dtype, na_value=0)[~na], err_msg=f)
                if f == "mean":
                    assert e["bit_exact"].all()
    # the value identity of the reference: uint64 compares unsigned, NaN is one key distinct from NA, -0.0 is 0.0
    u = Column(np.array([2 ** 63, 2 ** 63, 2 ** 64 - 1, 0], dtype=np.uint64), None, CTypes.UINT64, ArrTypes.NUMPY, 4)
    assert len(group_rows([u], True)[2]) == 3
    fl = Column(np.array([np.nan, -np.nan, -0.0, 0.0, 1.0]), np.packbits([1, 1, 1, 1, 0], bitorder="little"), CTypes.FLOAT64,
                ArrTypes.NULLABLE_INT_BOOL, 5)
    assert len(group_rows([fl], False)[2]) == 3 and len(group_rows([fl], True)[2]) == 1
    mean = expect("mean", u, np.arange(4), np.array([0, 0, 1, 1]), 2)
    assert list(mean["mean"]) == [2.0 ** 63, 2.0 ** 63] and not mean["bit_exact"].any()


# ---- a. every key type, single column ---------------------------------------------------------------------------------

FN_A = ("size", "count", "sum", "mean", "min", "max", "first", "last", "nunique", "var", "skew")


@functools.lru_cache(maxsize=None)
def _data_a(ct, nullable):
    rng = np.random.default_rng(1000 + 2 * ct + nullable)
    n = 12_000
    return Table([key_column(ct, n, rng, nullable, 200), value_column(CTypes.INT64, n, rng, True),
                  value_column(CTypes.FLOAT64, n, rng, True)], ["k", "i", "x"])


@pytest.mark.gpu
@pytest.mark.parametrize("dropna", [True, False], ids=["dropna", "keepna"])
@pytest.mark.parametrize("nullable", [False, True], ids=["numpy", "nullable"])
@pytest.mark.parametrize("ct", ALL_TYPES, ids=[TNAME[c] for c in ALL_TYPES])
def test_every_key_type(gpu_lib, ct, nullable, dropna):
    t = _data_a(ct, nullable)
    for vcol in (1, 2):  # (one value column per state: both at once would need more than 16 accumulator columns)
        cols = (vcol,) * len(FN_A)
        groups, exp = reference(t.columns[:1], t.columns, FN_A, cols, dropna)
        for feed in ("host", "device"):
            out, m, _ = run(t, 1, FN_A, cols, dropna=dropna, feed=feed, expected_groups=8)
            check_result(out, 1, groups, exp, (TNAME[ct], nullable, dropna, t.names[vcol], feed))
            assert m[8] == m[10] == m[12] == m[14] == 0, m  # the direct kernel


# The smallest table has 2^16 slots whatever expected_groups says (it takes 2^15 groups), and the 12 000-row inputs above fit
# it.  Here every key type wide enough for it brings ~40 000 groups, so the table grows (fail list, settle, rehash_kernel).
WIDE_KEYS = tuple(c for c in ALL_TYPES if c not in (CTypes.INT8, CTypes.UINT8, CTypes.BOOL))
FN_GROW = ("size", "count", "sum", "mean", "min", "max", "first", "last", "nunique")


@pytest.mark.gpu
@pytest.mark.parametrize("nullable", [False, True], ids=["numpy", "nullable"])
@pytest.mark.parametrize("ct", WIDE_KEYS, ids=[TNAME[c] for c in WIDE_KEYS])
def test_every_key_type_through_table_growth(gpu_lib, ct, nullable):
    rng = np.random.default_rng(1500 + 2 * ct + nullable)
    n = 200_000
    t = Table([key_column(ct, n, rng, nullable, 70_000), value_column(CTypes.INT64, n, rng, True)], ["k", "v"])
    cols = (1,) * len(FN_GROW)
    for dropna in (True, False):
        groups, exp = reference(t.columns[:1], t.columns, FN_GROW, cols, dropna)
        assert len(groups) > 1 << 15
        for feed in ("host", "device"):
            out, m, _ = run(t, 1, FN_GROW, cols, dropna=dropna, feed=feed, expected_groups=8)
            check_result(out, 1, groups, exp, (TNAME[ct], nullable, dropna, feed))
            assert m[3] > 0 and m[8] == m[10] == m[12] == m[14] == 0, m  # grew, on the direct kernel


# ---- b. key types on the SM-partitioned generic path (SPG-G) ----------------------------------------------------------

SPGG_KEYS = (CTypes.INT32, CTypes.UINT32, CTypes.DATE, CTypes.INT64, CTypes.DATETIME, CTypes.TIMEDELTA)
FN_B = ("sum", "count", "mean", "min", "max")


@pytest.mark.gpu
@pytest.mark.timeout(300)
@pytest.mark.parametrize("nullable", [False, True], ids=["numpy", "nullable"])
@pytest.mark.parametrize("ct", SPGG_KEYS, ids=[TNAME[c] for c in SPGG_KEYS])
def test_key_types_on_the_generic_sm_partitioned_path(gpu_lib, ct, nullable):
    """2^21 + 4097 device rows (the first 2^20 learn the cardinality through the direct kernel, the rest go through SPG-G),
    3000 key values with the type's edges; a full-range nullable value column, int64 under a nullable key and int32 under a
    numpy one, so both value widths meet both key widths."""
    rng = np.random.default_rng(2000 + 2 * ct + nullable)
    n = (1 << 21) + 4_097
    vt = CTypes.INT64 if nullable else CTypes.INT32
    t = Table([key_column(ct, n, rng, nullable, 3000), make_column(vt, n, rng, True, small=False)], ["k", "v"])
    for dropna in (True, False):
        groups, exp = reference(t.columns[:1], t.columns, FN_B, (1,) * 5, dropna)
        out, m, _ = run(t, 1, FN_B, (1,) * 5, dropna=dropna, feed="device")
        check_result(out, 1, groups, exp, (TNAME[ct], nullable, dropna))
        assert m[12] > 0, m  # the SPG-G kernels ran


# ---- c. every value type ----------------------------------------------------------------------------------------------

def fn_for_value(ct):
    """every function the constructor accepts for a value column of type ct (temporal: the SQL-meaningful ones)"""
    if ct in TEMPORAL:
        return ("size", "count", "min", "max", "first", "last", "nunique")
    mm = () if ct == CTypes.UINT64 else ("min", "max")
    return ("size", "count", "sum", "mean") + mm + ("first", "last", "nunique") + MOMENTS


@functools.lru_cache(maxsize=None)
def _data_c(vt, key_nullable, value_nullable):
    rng = np.random.default_rng(3000 + 4 * vt + 2 * key_nullable + value_nullable)
    n = 10_000
    k, v = key_column(CTypes.INT64, n, rng, key_nullable, 150), value_column(vt, n, rng, value_nullable)
    if vt == CTypes.UINT64:  # a third of the groups hold only values at or above 2^63
        big = (k.data % 3 == 0)
        v.data[big] = np.uint64(2 ** 63) + rng.integers(0, 2 ** 62, int(big.sum()), dtype=np.uint64) * np.uint64(2)
        v.data[big & (rng.random(n) < 0.1)] = np.uint64(2 ** 64 - 1)
    return Table([k, v], ["k", "v"])


@pytest.mark.gpu
@pytest.mark.parametrize("value_nullable", [False, True], ids=["vnumpy", "vnullable"])
@pytest.mark.parametrize("key_nullable", [False, True], ids=["knumpy", "knullable"])
@pytest.mark.parametrize("vt", ALL_TYPES, ids=[TNAME[c] for c in ALL_TYPES])
def test_every_value_type(gpu_lib, vt, key_nullable, value_nullable):
    t = _data_c(vt, key_nullable, value_nullable)
    fn = fn_for_value(vt)
    for dropna in (True, False):
        groups, exp = reference(t.columns[:1], t.columns, fn, (1,) * len(fn), dropna)
        for feed in ("host", "device"):
            out, _, _ = run(t, 1, fn, (1,) * len(fn), dropna=dropna, feed=feed, expected_groups=8)
            check_result(out, 1, groups, exp, (TNAME[vt], key_nullable, value_nullable, dropna, feed))
    if vt == CTypes.UINT64:
        from bodo_b200._lib import B200Error

        for f in ("min", "max"):
            with pytest.raises(B200Error, match="min/max of uint64 is not supported"):
                run(t, 1, ("count", f), (1, 1))


# ---- d. multi-column keys ---------------------------------------------------------------------------------------------

MK_KEYS = {"int8-uint64": (CTypes.INT8, CTypes.UINT64), "bool-date-float32": (CTypes.BOOL, CTypes.DATE, CTypes.FLOAT32),
           "uint16-int64-float64-timedelta": (CTypes.UINT16, CTypes.INT64, CTypes.FLOAT64, CTypes.TIMEDELTA)}
FN_D = ("size", "count", "sum", "mean", "min", "max") + MOMENTS


def mk_key_column(ct, n, rng, pool_size):
    """a nullable key component over pool_size values: 0 and the type's edges (uint64: 2^63; floats: -0.0, 0.0 and NaN); an
    NA cell holds 0, so a tuple with an NA component has a twin that differs from it only in NA-ness"""
    pool = gen_values(ct, pool_size, rng, small=False)
    pool[0] = 0
    if ct in FLOATS:
        pool[1:3] = [-0.0, np.nan]
    if ct == CTypes.UINT64:
        pool[1] = 2 ** 63
    c = _column(pool[rng.integers(0, len(pool), n)], ct, rng, True, na_frac=0.25)
    c.data[~c.valid_mask_numpy()] = 0
    return c


@functools.lru_cache(maxsize=None)
def _data_d(case):
    types = MK_KEYS[case]
    rng = np.random.default_rng(4000 + len(types))
    n = 40_000
    pool = {2: 9, 3: 7, 4: 5}[len(types)]
    keys = [mk_key_column(ct, n, rng, pool) for ct in types]
    return Table(keys + [value_column(CTypes.INT64, n, rng, True)], [f"k{j}" for j in range(len(types))] + ["v"])


@pytest.mark.gpu
@pytest.mark.parametrize("feed", ["host", "device"])
@pytest.mark.parametrize("dropna", [True, False], ids=["dropna", "keepna"])
@pytest.mark.parametrize("case", list(MK_KEYS))
def test_multi_column_keys(gpu_lib, case, dropna, feed):
    t = _data_d(case)
    nk = len(MK_KEYS[case])
    masks = np.stack([c.valid_mask_numpy() for c in t.columns[:nk]], axis=1) @ (1 << np.arange(nk))
    assert len(np.unique(masks)) == 1 << nk  # every NA mask of the tuple occurs
    groups, exp = reference(t.columns[:nk], t.columns, FN_D, (nk,) * len(FN_D), dropna)
    out, m, n_batches = run(t, nk, FN_D, (nk,) * len(FN_D), dropna=dropna, feed=feed, expected_groups=8, output_batch_size=32)
    check_result(out, nk, groups, exp, (case, dropna, feed))
    assert n_batches == -(-len(groups) // 32) > 1  # produce sliced the output
    if not dropna:  # groups that differ from another group only in one component's NA-ness, e.g. (NA, 0) beside (0, 0)
        seen = {tuple(r) for r in groups.tolist()}
        twins = sum(tuple(r[:2 * j] + [0] + r[2 * j + 1:]) in seen for r in groups.tolist() for j in range(nk) if r[2 * j] == 1)
        assert twins > 0


@pytest.mark.gpu
@pytest.mark.parametrize("f", ["first", "last", "nunique"])
def test_multi_column_keys_refuse_single_key_functions(gpu_lib, f):
    from bodo_b200._lib import B200Error

    t = _data_d("int8-uint64")
    msg = "nunique is supported for single-column keys" if f == "nunique" else "first / last are supported for single-column keys"
    with pytest.raises(B200Error, match=msg):
        run(t, 2, ("count", f), (2, 2))


@pytest.mark.gpu
@pytest.mark.timeout(600)
def test_multi_column_keys_over_a_million_groups(gpu_lib):
    """(int16, uint32, bool) nullable keys, ~1.5 M groups with no size hint (the default table takes 2^20 groups, so it grows
    mid-batch: fail list, settle, rehash_mk_kernel),
    device batches of 700 001 rows and an output batch of 300 000 groups; the moments are checked on 4000 groups spread over the
    output."""
    rng = np.random.default_rng(5)
    n = 1 << 21
    keys = [_column(rng.integers(-1000, 1001, n).astype(np.int16), CTypes.INT16, rng, True, 0.05),
            _column(rng.integers(0, 600, n).astype(np.uint32), CTypes.UINT32, rng, True, 0.05),
            _column(rng.integers(0, 2, n).astype(bool), CTypes.BOOL, rng, True, 0.05)]
    t = Table(keys + [_column(rng.integers(-1000, 1001, n).astype(np.int32), CTypes.INT32, rng, True)], ["a", "b", "c", "v"])
    groups, exp = reference(t.columns[:3], t.columns, FN_D, (3,) * len(FN_D), False, sample=4000)
    assert len(groups) > 1_000_000
    out, m, n_batches = run(t, 3, FN_D, (3,) * len(FN_D), dropna=False, feed="device", output_batch_size=300_000,
                            device_batch=700_001)
    check_result(out, 3, groups, exp, "1M groups")
    assert m[3] > 0 and n_batches == -(-len(groups) // 300_000), (m, n_batches)


# ---- e. mean / var / std / skew of uint64 values at and above 2^63 ----------------------------------------------------

@functools.lru_cache(maxsize=None)
def _u64_data():
    rng = np.random.default_rng(6)
    G, n = 64, 40_000
    gid = rng.integers(0, G, n)
    base = np.uint64(2 ** 63)
    u = base + rng.integers(0, 2 ** 40, n, dtype=np.uint64) * (gid.astype(np.uint64) % np.uint64(7) + np.uint64(1))
    top = gid % 4 == 1  # groups next to 2^64 - 1
    u[top] = np.uint64(2 ** 64 - 1) - rng.integers(0, 2 ** 52, int(top.sum()), dtype=np.uint64)
    ends = gid % 4 == 2  # groups of {2^63, 2^64 - 1} only
    u[ends] = np.where(rng.random(int(ends.sum())) < 0.5, base, np.uint64(2 ** 64 - 1))
    return gid, G, u


@pytest.mark.gpu
@pytest.mark.parametrize("path", PATHS)
def test_uint64_moments_at_and_above_2_63(gpu_lib, path):
    gid, G, u = _u64_data()
    fn = ("mean", "var", "std", "var_pop", "std_pop", "skew", "count")
    got = run_path(path, gid, G, {"u": u}, fn, ("u",) * len(fn))
    refs = [exact_moments(u[ix].astype(np.float64)) for ix in _groups(gid, G)]
    (mean, na), n = got[0], np.array([r["n"] for r in refs])
    assert not na.any() and (mean >= 2.0 ** 63).all(), (path, mean.min())  # (read as int64, every mean would be negative)
    np.testing.assert_array_equal(got[-1][0], n)
    for (vals, na), f in zip(got[:-1], fn):
        for g, r in enumerate(refs):
            e, x = r[f], vals[g]
            ctx = (path, f, g, r["n"], x, e)
            assert e is not None and not na[g], ctx
            if f == "mean":
                assert abs(x - e) <= gamma(r["n"] - 1) * r["abs_sum"] / r["n"] * (1 + U) + U * abs(e), ctx
            elif f == "skew":
                assert abs(x - e) <= skew_tol(r), ctx + (skew_tol(r),)
            else:
                assert abs(x - e) <= var_tol(r) * abs(e), ctx + (var_tol(r),)
