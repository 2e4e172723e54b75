"""Value window functions (SUM, COUNT, MEAN, MIN, MAX, FIRST_VALUE, LAST_VALUE over the "range", "rows" and "partition" frames;
LAG, LEAD) on the GPU.

The oracle is numpy over tests/test_gpu_sort.py's stable permutation (partition keys ascending NA last, order keys, arrival).
Partition and peer boundaries come from adjacent equality of (isna, key) in that order, and each row's frame end from them,
independently of the device.  Integer sums (wrapping in 64 bits), counts, means of integers, min / max / first / last / lag / lead
are compared bit for bit.  Float sums and means are compared with an exact reference (each finite double is an integer multiple
of 2^-1074, so prefix sums of Python ints are exact): |got - exact| <= gamma_(m-1) * sum|v| for a frame of m valid cells, with
gamma_k = k u / (1 - k u) and u = 2^-53, the bound of any summation order; +-inf are counted apart."""

import math

import numpy as np
import pandas as pd
import pytest
import torch

from bodo_b200 import _lib
from bodo_b200._lib import B200Error, ffi
from bodo_b200.streaming import window as W
from bodo_b200.table import ArrTypes, Column, CTypes, Table, np_dtype_of
from tests.helpers import table_to_device
from tests.test_gpu_sort import KEY_TYPES, batches_of, col_mask, make_column, oracle_perm

pytestmark = pytest.mark.gpu

TILE = 2048
CHUNK = 1 << 24
FRAMES = ("range", "rows", "partition")
TEMPORAL = (CTypes.DATE, CTypes.DATETIME, CTypes.TIMEDELTA)
UNSIGNED = (CTypes.UINT8, CTypes.UINT16, CTypes.UINT32, CTypes.UINT64)
U = 2.0 ** -53


@pytest.fixture(autouse=True)
def _return_device_memory():
    yield
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    _lib.lib().b200_pool_trim(torch.cuda.current_device(), 0)


def _sorted_col(table, name, perm):
    c = table.columns[table.names.index(name)]
    return c.values_numpy()[perm], col_mask(c)[perm], c.c_type


def bounds(table, part, order, asc, nap):
    """(perm, P, partition end (exclusive), {frame: e}) from adjacent equality of (isna, key) in the stable order."""
    perm = oracle_perm(table, part + order, [True] * len(part) + list(asc), ["last"] * len(part) + list(nap))
    n = len(perm)
    idx = np.arange(n, dtype=np.int64)

    def adjacent_equal(name):
        v, m, _ = _sorted_col(table, name, perm)
        na = ~m
        if v.dtype.kind == "f":
            na |= np.isnan(v)
        v = np.where(na, 0, v)
        return (na[1:] == na[:-1]) & (v[1:] == v[:-1])

    pstart, qstart = np.ones(n, bool), np.ones(n, bool)
    if n:
        peq = np.ones(n - 1, bool)
        for k in part:
            peq &= adjacent_equal(k)
        oeq = peq.copy()
        for k in order:
            oeq &= adjacent_equal(k)
        pstart[1:], qstart[1:] = ~peq, ~oeq

    def ends(starts):
        s = np.flatnonzero(starts)
        return np.append(s[1:], n)[np.cumsum(starts) - 1] if n else idx

    P = np.maximum.accumulate(np.where(pstart, idx, 0)) if n else idx
    pe = ends(pstart)
    return perm, P, pe, {"rows": idx, "range": ends(qstart) - 1, "partition": pe - 1}


def _exact_ints(v):
    """Each finite double as the exact integer x * 2^1074 (non-finite cells: 0)."""
    out = []
    for x in v.tolist():
        num, den = x.as_integer_ratio() if math.isfinite(x) else (0, 1)
        out.append(num * ((1 << 1074) // den))
    return out


def _prefix(a):
    p = [0]
    for x in a:
        p.append(p[-1] + x)
    return p


def expected(table, fn, perm, P, pe, ends):
    """(values, validity) of one value function, from its definition; float sum / mean: (exact, validity, tolerance) instead."""
    name, fname = fn[0], fn[1]
    n = len(perm)
    idx = np.arange(n, dtype=np.int64)
    if fname in ("lag", "lead"):
        v, m, ct = _sorted_col(table, fn[2], perm)
        k = fn[3] if len(fn) > 3 else 1
        default = fn[4] if len(fn) > 4 else None
        src = idx - k if fname == "lag" else idx + k
        ok = (src >= P) & (src < pe)
        s = np.where(ok, src, 0)
        vals = v[s].copy() if n else v.copy()
        valid = np.where(ok, m[s], default is not None) if n else m.copy()
        if default is not None:
            vals[~ok] = np.array(default).astype(v.dtype)
        vals[~valid] = 0
        return vals, valid
    e = ends[fn[3] if len(fn) > 3 else "range"]
    if fn[2] is None:  # count(*)
        return e - P + 1, np.ones(n, bool)
    v, m, ct = _sorted_col(table, fn[2], perm)
    if fname in ("first_value", "last_value"):
        s = P if fname == "first_value" else e
        vals, valid = v[s].copy(), m[s].copy()
        vals[~valid] = 0
        return vals, valid
    flt = v.dtype.kind == "f"
    good = m & ~np.isnan(v) if flt else m.copy()
    cnt = np.concatenate([[0], np.cumsum(good)])
    c = cnt[e + 1] - cnt[P]
    if fname == "count":
        return c.astype(np.int64), np.ones(n, bool)
    if fname in ("min", "max"):
        # the earliest row holding the least / greatest valid value, -0.0 == 0.0, in the frame [P, e]
        vals, valid = np.zeros_like(v), c > 0
        key = [0.0 if x == 0 else x for x in v.tolist()]  # Python numbers: exact for every integer type; -0.0 ties 0.0
        best = np.full(n, -1, np.int64)  # the earliest row holding the frame's least / greatest value, for the frame [P, i]
        for i in range(n):
            b = best[i - 1] if i > P[i] else -1
            if good[i] and (b < 0 or (key[i] < key[b] if fname == "min" else key[i] > key[b])):
                b = i
            best[i] = b
        b = best[e]
        vals[b >= 0] = v[b[b >= 0]]
        return vals, valid
    if not flt:
        x = np.where(good, v, 0)
        x = x.astype(np.int64).view(np.uint64) if v.dtype.kind in "ib" else x.astype(np.uint64)
        S = np.concatenate([[np.uint64(0)], np.cumsum(x, dtype=np.uint64)])
        s = S[e + 1] - S[P]
        if fname == "sum":
            out = s.view(np.int64) if ct not in UNSIGNED else s
            return np.where(c > 0, out, 0), c > 0
        sd = s.view(np.int64).astype(np.float64) if ct not in UNSIGNED else s.astype(np.float64)
        return np.where(c > 0, sd / np.maximum(c, 1), 0.0), c > 0
    # floats: exact reference, with infinities counted apart
    vv = np.where(good, v, 0).astype(np.float64)
    fin = np.isfinite(vv)
    ex = _prefix(_exact_ints(np.where(fin, vv, 0)))
    ab = np.concatenate([[0.0], np.cumsum(np.abs(np.where(fin, vv, 0)))])
    pinf = np.concatenate([[0], np.cumsum(vv == np.inf)])
    ninf = np.concatenate([[0], np.cumsum(vv == -np.inf)])
    exact = np.empty(n)
    tol = np.empty(n)
    for i in range(n):
        a, b = int(P[i]), int(e[i]) + 1
        ip, ineg = pinf[b] - pinf[a], ninf[b] - ninf[a]
        mm = int(c[i])
        g = (mm - 1) * U / (1 - (mm - 1) * U) if mm > 1 else 0.0
        if ip or ineg:
            exact[i], tol[i] = (np.nan if ip and ineg else np.inf if ip else -np.inf), 0.0
            continue
        exact[i] = (ex[b] - ex[a]) / (1 << 1074)
        tol[i] = g * (ab[b] - ab[a])
    if fname == "mean":
        exact = np.where(c > 0, exact / np.maximum(c, 1), 0.0)
        tol = tol / np.maximum(c, 1) + 2 * U * np.abs(exact)
    if ct == CTypes.FLOAT32 and fname == "sum":
        tol = tol * (1 + 2.0 ** -23) + 2.0 ** -24 * (np.abs(exact) + tol)
    return exact, c > 0, tol


def out_type(table, fn):
    if fn[1] == "count":
        return CTypes.INT64, ArrTypes.NUMPY
    ct = table.columns[table.names.index(fn[2])].c_type
    if fn[1] == "mean":
        return CTypes.FLOAT64, ArrTypes.NULLABLE_INT_BOOL
    if fn[1] == "sum":
        return (ct if ct in (CTypes.FLOAT32, CTypes.FLOAT64) else CTypes.UINT64 if ct in UNSIGNED else CTypes.INT64), ArrTypes.NULLABLE_INT_BOOL
    return ct, ArrTypes.NULLABLE_INT_BOOL


def run(table, part, order, asc, nap, funcs, sizes=(1 << 30,), device=True, output_batch_size=32768):
    st = W.init_window_state(-1, part, order, asc, nap, funcs, table.names, output_batch_size=output_batch_size)
    bs = batches_of(table, list(sizes))
    for i, b in enumerate(bs):
        W.window_build_consume_batch(st, table_to_device(b) if device else b, i == len(bs) - 1)
    outs = []
    while True:
        out, last = W.window_produce_output_batch(st)
        outs.append(out)
        if last:
            break
    W_cols = table.n_cols + len(funcs)
    res = [(np.concatenate([o.columns[c].values_numpy() for o in outs]), np.concatenate([col_mask(o.columns[c]) for o in outs]),
            outs[0].columns[c]) for c in range(W_cols)]
    W.delete_window_state(st)
    return res, [o.n_rows for o in outs]


def check(table, part, order, asc, nap, funcs, **kw):
    part, order = list(part), list(order)
    perm, P, pe, ends = bounds(table, part, order, asc, nap)
    got, sizes = run(table, part, order, asc, nap, funcs, **kw)
    for c, (vals, mask, _) in zip(table.columns, got):
        np.testing.assert_array_equal(vals.view(np.uint8), c.values_numpy()[perm].view(np.uint8))
        np.testing.assert_array_equal(mask, col_mask(c)[perm])
    for fn, (vals, mask, oc) in zip(funcs, got[table.n_cols:]):
        ct, at = out_type(table, fn)
        assert (oc.c_type, oc.arr_type) == (ct, at), fn
        assert vals.dtype == np_dtype_of(ct), fn
        exp = expected(table, fn, perm, P, pe, ends)
        np.testing.assert_array_equal(mask, exp[1], err_msg=str(fn))
        if len(exp) == 2:
            e = exp[0].astype(vals.dtype) if exp[0].dtype != vals.dtype else exp[0]
            got_bits = np.where(mask, vals.view(f"u{vals.itemsize}"), 0)
            np.testing.assert_array_equal(got_bits, np.where(mask, e.view(f"u{vals.itemsize}"), 0), err_msg=str(fn))
        else:
            exact, valid, tol = exp
            g = vals.astype(np.float64)[valid]
            x, t = exact[valid], tol[valid]
            nonfinite = ~np.isfinite(x)
            np.testing.assert_array_equal(g[nonfinite], x[nonfinite], err_msg=str(fn))
            assert np.all(np.abs(g[~nonfinite] - x[~nonfinite]) <= t[~nonfinite]), fn
    return got, sizes


def float_values(ct, n, rng, nullable):
    """Normal values over a few magnitudes, with +-inf, NaN, -0.0 and subnormals mixed in (no value near the type's max, whose
    sums would overflow)."""
    dt = np.dtype("float32" if ct == CTypes.FLOAT32 else "float64")
    v = (rng.standard_normal(n) * 10.0 ** rng.integers(-3, 4, n)).astype(dt)
    edge = np.array([np.inf, -np.inf, np.nan, -0.0, 0.0, np.finfo(dt).smallest_subnormal], dtype=dt)
    pos = rng.integers(0, n, min(n, 3 * len(edge)))
    v[pos] = np.resize(edge, len(pos))
    if not nullable:
        return Column(v, None, ct, ArrTypes.NUMPY, n)
    return Column(v, np.packbits(rng.random(n) >= 0.15, bitorder="little"), ct, ArrTypes.NULLABLE_INT_BOOL, n)


def all_funcs(col, ct, lag_default=None):
    fs = []
    for fr in FRAMES:
        names = ["count", "min", "max", "first_value", "last_value"] + ([] if ct in TEMPORAL else ["sum", "mean"])
        fs += [(f"{f}_{fr}", f, col, fr) for f in names]
        fs.append((f"cnt_{fr}", "count", None, fr))
    fs += [("lag1", "lag", col), ("lead0", "lead", col, 0), ("lag3", "lag", col, 3, lag_default), ("lead2", "lead", col, 2, lag_default)]
    return fs


def _default_for(ct):
    return {CTypes.BOOL: True, CTypes.FLOAT32: 0.5, CTypes.FLOAT64: -2.25}.get(ct, 7)


# ---- every function x every frame x every value type ----
@pytest.mark.parametrize("ct", KEY_TYPES)
@pytest.mark.parametrize("nullable", [False, True])
def test_value_types(gpu_lib, ct, nullable):
    rng = np.random.default_rng(300 + ct * 2 + nullable)
    n = 3000
    if ct in (CTypes.FLOAT32, CTypes.FLOAT64):
        x = float_values(ct, n, rng, nullable)
    else:
        x = make_column(ct, n, rng, nullable, small=False)  # full-range integers: int64 sums wrap, uint64 sums exceed 2^63
    g = make_column(CTypes.INT8, n, rng, False)
    o = make_column(CTypes.INT16, n, rng, True, na_frac=0.1)  # many peers: "range" and "rows" differ
    t = Table([g, o, x], ["g", "o", "x"])
    check(t, ["g"], ["o"], [True], ["last"], all_funcs("x", ct, _default_for(ct)), sizes=(777,))


def test_sum_wraps_in_64_bits(gpu_lib):
    n = 1000
    big = np.full(n, np.iinfo(np.int64).max - 5, np.int64)
    ubig = np.full(n, np.uint64(1) << np.uint64(63), np.uint64)
    t = Table([Column(np.zeros(n, np.int64)), Column(np.arange(n, dtype=np.int64)), Column(big), Column(ubig)], ["g", "o", "b", "u"])
    check(t, ["g"], ["o"], [True], ["last"], [("sb", "sum", "b", "rows"), ("mb", "mean", "b", "partition"), ("su", "sum", "u", "rows"),
                                              ("mu", "mean", "u", "range")])


@pytest.mark.parametrize("part,order", [([], ["o"]), (["g"], []), ([], ["g"]), (["g", "o"], ["h", "x"])])
def test_key_shapes(gpu_lib, part, order):
    """No PARTITION BY; no ORDER BY ("range" is then "partition"); 4 keys; the value column may be a key."""
    rng = np.random.default_rng(31)
    n = 5000
    t = Table([make_column(CTypes.INT32, n, rng, True, na_frac=0.1), make_column(CTypes.INT8, n, rng, False),
               make_column(CTypes.UINT16, n, rng, True), float_values(CTypes.FLOAT64, n, rng, True)], ["g", "o", "h", "x"])
    fs = [(f"{f}_{fr}", f, "x", fr) for f in ("sum", "mean", "min", "last_value") for fr in FRAMES]
    fs += [("c", "count", None), ("lg", "lag", "x", 2, 1.5), ("kmin", "min", (part + order)[0], "rows"),
           ("ksum", "sum", (part + order)[0], "range")]
    check(t, part, order, [False] * len(order), ["first"] * len(order), fs, sizes=(1500,))


def test_no_order_by_range_is_partition(gpu_lib):
    rng = np.random.default_rng(32)
    n = 4000
    t = Table([make_column(CTypes.INT16, n, rng, False), float_values(CTypes.FLOAT64, n, rng, True)], ["g", "x"])
    got, _ = run(t, ["g"], [], [], [], [("a", "sum", "x", "range"), ("b", "sum", "x", "partition"), ("c", "max", "x"),
                                        ("d", "max", "x", "partition")])
    for a, b in ((2, 3), (4, 5)):
        np.testing.assert_array_equal(got[a][0].view(np.uint64), got[b][0].view(np.uint64))
        np.testing.assert_array_equal(got[a][1], got[b][1])


def test_lag_lead_edges(gpu_lib):
    sizes = [1, 2, 3, 5, 8, 100]
    g = np.repeat(np.arange(len(sizes)), sizes)
    n = len(g)
    rng = np.random.default_rng(33)
    perm = rng.permutation(n)
    cols = [Column(g[perm].astype(np.int64)), Column(rng.integers(0, 4, n).astype(np.int64))]
    names = ["g", "o"]
    fs = []
    for ct in (CTypes.INT8, CTypes.UINT64, CTypes.FLOAT32, CTypes.BOOL, CTypes.DATE, CTypes.DATETIME):
        names.append(f"x{ct}")
        cols.append(make_column(ct, n, rng, True, small=False))
        d = _default_for(ct)
        for k in (0, 1, 4, 99, 100, 1000, (1 << 31) - 1):
            fs += [(f"lag{k}_{ct}", "lag", f"x{ct}", k), (f"lead{k}_{ct}", "lead", f"x{ct}", k, d)]
    for i in range(0, len(fs), 30 - len(cols)):  # at most 32 output columns per state
        check(Table(cols, names), ["g"], ["o"], [True], ["last"], fs[i:i + 30 - len(cols)])


@pytest.mark.parametrize("n", [1, 2, TILE - 1, TILE, TILE + 1, 3 * TILE + 17, 40_000])
def test_tile_edges(gpu_lib, n):
    """One partition spans many tiles (cross-tile carries); partitions and peer groups straddle tile edges."""
    rng = np.random.default_rng(n)
    i = np.arange(n)
    t = Table([Column((i // 15000).astype(np.int64)), Column((i // 7 % 5).astype(np.int64)),
               make_column(CTypes.INT32, n, rng, True, small=False), float_values(CTypes.FLOAT64, n, rng, True)], ["g", "o", "x", "f"])
    fs = [("sx", "sum", "x", "rows"), ("mx", "max", "x", "range"), ("nx", "min", "x", "partition"), ("cf", "count", "f", "rows"),
          ("sf", "sum", "f", "rows"), ("af", "mean", "f", "partition"), ("lf", "last_value", "f", "range"), ("c", "count", None, "rows"),
          ("lg", "lead", "x", 2047)]
    check(t, ["g"], ["o"], [True], ["last"], fs, sizes=(TILE - 1, TILE, TILE + 1))


def test_determinism_across_batches_and_frame_ends(gpu_lib):
    """Float sums are bit-identical for any batch split, host or device; rows that share a frame end share their bits."""
    rng = np.random.default_rng(34)
    n = 30_000
    t = Table([Column(rng.integers(0, 5, n).astype(np.int64)), Column(rng.integers(0, 50, n).astype(np.int64)),
               float_values(CTypes.FLOAT64, n, rng, True), float_values(CTypes.FLOAT32, n, rng, False)], ["g", "o", "x", "y"])
    fs = [(f"{f}{c}_{fr}", f, c, fr) for c in ("x", "y") for f in ("sum", "mean") for fr in FRAMES]
    ref, _ = run(t, ["g"], ["o"], [True], ["last"], fs)
    for sizes, dev in (((1000,), True), ((4096, 17), False), ((TILE,), True), ((7777,), False)):
        got, _ = run(t, ["g"], ["o"], [True], ["last"], fs, sizes=sizes, device=dev)
        for a, b in zip(ref[4:], got[4:]):
            np.testing.assert_array_equal(a[0].view(f"u{a[0].itemsize}"), b[0].view(f"u{b[0].itemsize}"))
            np.testing.assert_array_equal(a[1], b[1])
    perm, P, pe, ends = bounds(t, ["g"], ["o"], [True], ["last"])
    for j, fn in enumerate(fs):
        e = ends[fn[3]]
        v = ref[4 + j][0]
        np.testing.assert_array_equal(v.view(f"u{v.itemsize}"), v[e].view(f"u{v.itemsize}"), err_msg=str(fn))


def test_mixed_with_ranking(gpu_lib):
    from tests.test_gpu_window import ALL, oracle

    rng = np.random.default_rng(35)
    n = 10_000
    t = Table([make_column(CTypes.INT16, n, rng, True), make_column(CTypes.INT32, n, rng, True), float_values(CTypes.FLOAT64, n, rng, True)],
              ["g", "o", "x"])
    vals = [("s", "sum", "x", "rows"), ("lg", "lag", "x", 1, 0.0), ("mx", "max", "o", "partition")]
    funcs = [ALL[0], vals[0], ALL[1], ALL[5], vals[1], ALL[3], vals[2]]
    alone, _ = check(t, ["g"], ["o"], [True], ["last"], vals)
    got, _ = run(t, ["g"], ["o"], [True], ["last"], funcs)
    perm, exp, _ = oracle(t, ["g"], ["o"], [True], ["last"], [f for f in funcs if f[1] in W.FUNCS])
    vi = 0
    for j, f in enumerate(funcs):
        vals_, mask, oc = got[3 + j]
        if f[1] in W.FUNCS:
            np.testing.assert_array_equal(vals_.view(np.uint64), exp[f[0]].view(np.uint64), err_msg=f[0])
            assert oc.arr_type == ArrTypes.NUMPY
        else:
            a = alone[3 + vi]
            np.testing.assert_array_equal(vals_.view(f"u{vals_.itemsize}"), a[0].view(f"u{a[0].itemsize}"))
            np.testing.assert_array_equal(mask, a[1])
            vi += 1


def test_output_slicing_and_zero_rows(gpu_lib):
    rng = np.random.default_rng(36)
    n = 10_000
    t = Table([make_column(CTypes.INT8, n, rng, False), make_column(CTypes.INT32, n, rng, True), float_values(CTypes.FLOAT32, n, rng, True)],
              ["g", "o", "x"])
    fs = [("s", "sum", "x", "rows"), ("m", "mean", "o", "partition"), ("l", "lag", "x", 2), ("c", "count", "x")]
    _, sizes = check(t, ["g"], ["o"], [True], ["last"], fs, output_batch_size=1000)
    assert sizes == [1024] * 9 + [n - 9 * 1024]
    z = Table([Column(np.empty(0, np.int64)), Column(np.empty(0, np.float32), np.empty(0, np.uint8), CTypes.FLOAT32,
                                                      ArrTypes.NULLABLE_INT_BOOL, 0)], ["g", "x"])
    fs = [("s", "sum", "x"), ("c", "count", None), ("m", "mean", "g"), ("mn", "min", "x"), ("lg", "lead", "g", 1, 3), ("r", "rank")]
    got, sizes = run(z, ["g"], [], [], [], fs)
    assert sizes == [0] and all(len(v) == 0 for v, _, _ in got)
    assert [(c.c_type, c.arr_type) for _, _, c in got[2:]] == [
        (CTypes.FLOAT32, ArrTypes.NULLABLE_INT_BOOL), (CTypes.INT64, ArrTypes.NUMPY), (CTypes.FLOAT64, ArrTypes.NULLABLE_INT_BOOL),
        (CTypes.FLOAT32, ArrTypes.NULLABLE_INT_BOOL), (CTypes.INT64, ArrTypes.NULLABLE_INT_BOOL), (CTypes.INT64, ArrTypes.NUMPY)]


def test_large_input_against_torch(gpu_lib):
    """2^24 + a few tiles of device rows against a torch recomputation: a segmented cumsum through offsets at P, and a cummax
    over (partition id << 32) | value."""
    n = CHUNK + 3 * TILE + 5
    dev = torch.device("cuda", 0)
    g = torch.Generator(device=dev).manual_seed(37)
    pk = torch.randint(0, 50, (n,), generator=g, device=dev, dtype=torch.int64)  # partitions of ~340k rows: many tiles each
    x = torch.randint(0, 1 << 31, (n,), generator=g, device=dev, dtype=torch.int64)
    rid = torch.arange(n, device=dev, dtype=torch.int64)
    funcs = [("s", "sum", "x", "rows"), ("m", "max", "x", "rows"), ("c", "count", None, "partition"), ("lg", "lag", "x", 1, -1)]
    st = W.init_window_state(-1, ["p"], ["r"], [True], ["last"], funcs, ["p", "r", "x"], output_batch_size=1 << 30)
    b = 3_000_000
    for r0 in range(0, n, b):
        t = Table([Column(pk[r0:r0 + b]), Column(rid[r0:r0 + b]), Column(x[r0:r0 + b])], ["p", "r", "x"])
        W.window_build_consume_batch(st, t, r0 + b >= n)
    out, last = W.window_produce_output_batch(st)
    assert last and out.n_rows == n
    got = [torch.as_tensor(c.data, device=dev) for c in out.columns]
    idx = torch.sort(pk, stable=True).indices
    assert torch.equal(got[1], idx)
    sp, sx = pk[idx], x[idx]
    i = torch.arange(n, device=dev, dtype=torch.int64)
    ps = torch.ones(n, dtype=torch.bool, device=dev)
    ps[1:] = torch.diff(sp) != 0
    P = torch.cummax(torch.where(ps, i, 0), 0).values
    cs = torch.cumsum(sx, 0)
    before = torch.where(P > 0, cs[(P - 1).clamp(min=0)], 0)
    assert torch.equal(got[3], cs - before)
    pid = torch.cumsum(ps.to(torch.int64), 0) - 1
    assert torch.equal(got[4], torch.cummax((pid << 32) | sx, 0).values & 0xFFFFFFFF)
    assert torch.equal(got[5], torch.bincount(pid)[pid])
    exp_lag = torch.where(ps, -1, torch.roll(sx, 1))
    assert torch.equal(got[6], exp_lag)
    for c in (3, 4, 6):
        assert out.columns[c].valid_mask_numpy().all()
    W.delete_window_state(st)


# ---- pandas ----
def test_pandas_cross_checks_without_na(gpu_lib):
    from bodo_b200.physical import window

    rng = np.random.default_rng(38)
    n = 40_000
    df = pd.DataFrame({"p": rng.integers(0, 300, n), "o": rng.integers(0, 50, n), "i": rng.integers(-1000, 1000, n),
                       "f": rng.integers(-2000, 2000, n) / 8.0})  # eighths: float sums are exact, in any order
    funcs = [("cs", "sum", "i", "rows"), ("cmin", "min", "f", "rows"), ("cmax", "max", "i", "rows"), ("fs", "sum", "f", "rows"),
             ("ts", "sum", "i", "partition"), ("tm", "mean", "f", "partition"), ("tmin", "min", "i", "partition"),
             ("tmax", "max", "f", "partition"), ("tc", "count", "f", "partition"), ("tz", "count", None, "partition"),
             ("tf", "first_value", "i", "partition"), ("tl", "last_value", "f", "partition"), ("sh", "lag", "i", 3, -7),
             ("sl", "lead", "f", 2, 0.5)]
    got = window(df, "p", "o", funcs, batch_size=7000)
    srt = df.sort_values(["p", "o"], kind="stable").reset_index(drop=True)
    gb = srt.groupby("p", sort=False)
    exp = {"cs": gb["i"].cumsum(), "cmin": gb["f"].cummin(), "cmax": gb["i"].cummax(), "fs": gb["f"].cumsum(),
           "ts": gb["i"].transform("sum"), "tm": gb["f"].transform("mean"), "tmin": gb["i"].transform("min"),
           "tmax": gb["f"].transform("max"), "tc": gb["f"].transform("count"), "tz": gb["f"].transform("size"),
           "tf": gb["i"].transform("first"), "tl": gb["f"].transform("last"), "sh": gb["i"].shift(3, fill_value=-7),
           "sl": gb["f"].shift(-2, fill_value=0.5)}
    for k, e in exp.items():
        np.testing.assert_array_equal(got[k].to_numpy(dtype=np.float64), e.to_numpy(dtype=np.float64), err_msg=k)


def test_pandas_differences_with_na(gpu_lib):
    """With NA cells: cumsum / cummin / cummax give NA at NA rows, the "rows" frame the aggregate so far; transform("sum") of an
    all-NA partition gives 0, SUM gives NA."""
    from bodo_b200.physical import window

    df = pd.DataFrame({"p": [0, 0, 0, 1, 1, 2], "x": pd.array([1.0, None, 2.0, None, None, 4.0], dtype="Float64")})
    got = window(df, "p", [], [("cs", "sum", "x", "rows"), ("cm", "max", "x", "rows"), ("ts", "sum", "x", "partition")])
    gb = df.groupby("p")["x"]
    assert gb.cumsum().isna().tolist() == [False, True, False, True, True, False]
    assert got["cs"].tolist()[:3] == [1.0, 1.0, 3.0] and got["cm"].tolist()[:3] == [1.0, 1.0, 2.0]
    assert gb.transform("sum").tolist()[3:5] == [0.0, 0.0]
    assert got["ts"].isna().tolist() == [False, False, False, True, True, False]


def test_share_of_partition_and_qualify_on_running_total(gpu_lib):
    """x / SUM(x) OVER (PARTITION BY p), and QUALIFY SUM(x) OVER (PARTITION BY p ORDER BY t ROWS ...) <= 100."""
    from bodo_b200.expr import col, lit
    from bodo_b200.physical import PhysicalFilterProject, PhysicalReadPandas, PhysicalWindow, ResultCollector, run_pipeline

    rng = np.random.default_rng(39)
    n = 20_000
    df = pd.DataFrame({"p": rng.integers(0, 500, n), "t": rng.integers(0, 1000, n), "x": rng.integers(1, 30, n).astype(np.float64)})
    op = PhysicalWindow("p", "t", [("tot", "sum", "x", "partition"), ("run", "sum", "x", "rows")])
    run_pipeline(PhysicalReadPandas(df, 4096), [], op)
    coll = ResultCollector()
    run_pipeline(op, [PhysicalFilterProject(col("run") <= lit(100.0), [("p", col("p")), ("t", col("t")), ("share", col("x") / col("tot"))])],
                 coll)
    op.Finalize()
    key = ["p", "t", "share"]  # the filter does not keep the window's row order
    got = coll.result().astype({"p": np.int64, "t": np.int64, "share": np.float64}).sort_values(key).reset_index(drop=True)
    srt = df.sort_values(["p", "t"], kind="stable").reset_index(drop=True)
    gb = srt.groupby("p", sort=False)["x"]
    srt["share"] = srt["x"] / gb.transform("sum")
    exp = srt[gb.cumsum() <= 100.0].sort_values(key).reset_index(drop=True)
    np.testing.assert_array_equal(got["p"].to_numpy(dtype=np.int64), exp["p"].to_numpy())
    np.testing.assert_array_equal(got["t"].to_numpy(dtype=np.int64), exp["t"].to_numpy())
    np.testing.assert_array_equal(got["share"].to_numpy(dtype=np.float64), exp["share"].to_numpy())


# ---- errors ----
def test_device_side_validation(gpu_lib):
    """The C entry rejects what the Python layer would have refused, for callers that use the ABI directly."""
    L = _lib.lib()
    c_types = ffi.new("int8_t[]", [CTypes.INT64, CTypes.DATETIME])
    a_types = ffi.new("int8_t[]", [ArrTypes.NUMPY, ArrTypes.NUMPY])
    one = ffi.new("int32_t[]", [1])

    def init(code, col, frame, arg=0, valid=0, n_funcs=1):
        fs = ffi.new("b200_window_func[]", max(1, n_funcs))
        for d in fs:
            d.code, d.col, d.frame, d.arg, d.default_valid = code, col, frame, arg, valid
        h = L.b200_window_state_init(-1, c_types, a_types, 2, 1, 0, one, one, fs, n_funcs, 1024, 0, ffi.NULL)
        if h != ffi.NULL:
            L.b200_delete_sort_state(h)
            return None
        return ffi.string(L.b200_last_error()).decode()

    assert init(6, 0, 2) is None and init(13, 1, 0, 5, 1) is None and init(7, -1, 3) is None
    assert "column index out of range" in init(6, 2, 1)
    assert "column index out of range" in init(9, -1, 1)
    assert "lag and lead take no frame" in init(14, 0, 1)
    assert "no column and no frame" in init(1, -1, 2)
    assert "unknown frame" in init(6, 0, 0)
    assert "unknown frame" in init(11, 0, 6)
    assert "sum and mean need" in init(8, 1, 1)
    assert "offset k" in init(13, 0, 0, 1 << 31)
    assert "offset k" in init(14, 0, 0, -1)
    assert "unknown function code" in init(25, 0, 1)
    assert "at most 32" in init(7, 0, 1, n_funcs=31)


def test_type_errors_at_first_consume(gpu_lib):
    n = 4
    t = Table([Column(np.arange(n, dtype=np.int64)), Column(np.arange(n, dtype=np.int64), None, CTypes.DATETIME),
               Column(np.zeros(n, np.int8))], ["k", "ts", "b"])
    for funcs, msg in (([("s", "sum", "ts")], "sum and mean need"), ([("m", "mean", "ts", "rows")], "sum and mean need"),
                       ([("l", "lag", "b", 1, 300)], "not exactly representable"), ([("l", "lead", "b", 1, 0.5)], "not exactly representable")):
        st = W.init_window_state(-1, ["k"], [], True, "last", funcs, t.names)
        with pytest.raises(B200Error, match=msg):
            W.window_build_consume_batch(st, t, True)
        W.delete_window_state(st)
