"""Bounded ROWS frames (("rows", start, end): k PRECEDING / k FOLLOWING) and NTH_VALUE on the GPU.

The oracle is numpy over [lo, hi] per row, from tests/test_gpu_window_values.py's partition boundaries (adjacent equality of
(isna, key) in the stable order) and the frame's definition, independently of the device.  Integer sums (wrapping in 64 bits),
counts, means of integers, min / max (through a sparse table over (rank of the value, position)), first / last / nth are compared
bit for bit.  Float sums and means are compared with the exact reference (each finite double is an integer multiple of 2^-1074):
|got - exact| <= gamma_min(m-1, h) * sum|v| for m valid cells, with h = 10 + 3 floor(log2 W) the combination tree's height for a
frame of W rows (DESIGN §3c)."""

import numpy as np
import pandas as pd
import pytest
import torch

from bodo_b200 import _lib
from bodo_b200._lib import ffi
from bodo_b200.streaming import window as W
from bodo_b200.table import ArrTypes, Column, CTypes, Table, np_dtype_of
from tests.test_gpu_sort import KEY_TYPES, col_mask, make_column
from tests.test_gpu_window_values import (CHUNK, TEMPORAL, TILE, U, UNSIGNED, _exact_ints, _prefix, _sorted_col, bounds,
                                          float_values, out_type, run)

pytestmark = pytest.mark.gpu

BIG = (1 << 31) - 1
FRAMES = [(-3, 0), (0, 3), (-2, 2), (0, 0), (-5, -2), (2, 5), (None, 3), (-3, None), (0, None), (None, -1), (-BIG, BIG),
          (-BIG, -4000), (4000, BIG)]


@pytest.fixture(autouse=True)
def _return_device_memory():
    yield
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    _lib.lib().b200_pool_trim(torch.cuda.current_device(), 0)


def frame_of(fn):
    if fn[1] == "nth_value":
        return fn[4] if len(fn) > 4 else "range"
    return fn[3] if len(fn) > 3 else "range"


def lo_hi(fr, P, pe, ends):
    n = len(P)
    i = np.arange(n, dtype=np.int64)
    if isinstance(fr, str):
        return P.copy(), ends[fr].copy()
    _, s, e = fr
    lo = P.copy() if s is None else np.maximum(P, i + s)
    hi = pe - 1 if e is None else np.minimum(pe - 1, i + e)
    return lo, hi


def _range_min(key, lo, hi):
    """min(key[lo..hi]) per row (lo <= hi) through a sparse table."""
    st = [key]
    while (1 << len(st)) <= len(key):
        p, h = st[-1], 1 << (len(st) - 1)
        st.append(np.minimum(p[:-h], p[h:]))
    k = ilog2(hi - lo + 1)
    out = np.empty(len(lo), np.int64)
    for kk in np.unique(k):
        s = k == kk
        t = st[kk]
        out[s] = np.minimum(t[lo[s]], t[hi[s] - (1 << kk) + 1])
    return out


def ilog2(w):
    """floor(log2(w)) of positive integers (1 for w < 1), exactly."""
    return np.frexp(np.maximum(w, 1).astype(np.float64))[1].astype(np.int64) - 1


def height(w):
    return 10 + 3 * ilog2(w)


def expected(table, fn, perm, P, pe, ends):
    """(values, validity) of one function over [lo, hi]; float sum / mean: (exact, validity, tolerance) instead."""
    n = len(perm)
    lo, hi = lo_hi(frame_of(fn), P, pe, ends)
    nonempty = lo <= hi
    if fn[2] is None:  # count(*)
        return np.maximum(hi - lo + 1, 0), np.ones(n, bool)
    v, m, ct = _sorted_col(table, fn[2], perm)
    fname = fn[1]
    if fname in ("first_value", "last_value", "nth_value"):
        src = lo if fname == "first_value" else hi if fname == "last_value" else lo + fn[3] - 1
        ok = nonempty & (src <= hi)
        s = np.where(ok, src, 0)
        vals, valid = v[s].copy(), ok & m[s]
        vals[~valid] = 0
        return vals, valid
    flt = v.dtype.kind == "f"
    good = m & ~np.isnan(v) if flt else m.copy()
    cnt = np.concatenate([[0], np.cumsum(good)])
    a, b = np.where(nonempty, lo, 0), np.where(nonempty, hi + 1, 0)
    c = cnt[b] - cnt[a]
    if fname == "count":
        return c.astype(np.int64), np.ones(n, bool)
    if fname in ("min", "max"):
        # -0.0 ties 0.0; Python numbers are exact for every integer type; NA and NaN cells are excluded below
        pykey = [0 if not ok or x == 0 else x for ok, x in zip(good.tolist(), v.tolist())]
        order = sorted(range(n), key=lambda j: pykey[j])
        rank = np.empty(n, np.int64)
        r = -1
        for t, j in enumerate(order):
            if t == 0 or pykey[j] != pykey[order[t - 1]]:
                r += 1
            rank[j] = r
        if fname == "max":
            rank = r - rank
        key = np.where(good, rank * n + np.arange(n), np.iinfo(np.int64).max)
        best = _range_min(key, a, np.maximum(b - 1, a))
        valid = c > 0
        vals = np.zeros_like(v)
        vals[valid] = v[best[valid] % n]
        return vals, valid
    if not flt:
        x = np.where(good, v, 0)
        x = x.astype(np.int64).view(np.uint64) if v.dtype.kind in "ib" else x.astype(np.uint64)
        S = np.concatenate([[np.uint64(0)], np.cumsum(x, dtype=np.uint64)])
        s = S[b] - S[a]
        if fname == "sum":
            out = s.view(np.int64) if ct not in UNSIGNED else s
            return np.where(c > 0, out, 0), c > 0
        sd = s.view(np.int64).astype(np.float64) if ct not in UNSIGNED else s.astype(np.float64)
        return np.where(c > 0, sd / np.maximum(c, 1), 0.0), c > 0
    vv = np.where(good, v, 0).astype(np.float64)
    fin = np.isfinite(vv)
    ex = _prefix(_exact_ints(np.where(fin, vv, 0)))
    ab = np.concatenate([[0.0], np.cumsum(np.abs(np.where(fin, vv, 0)))])
    pinf = np.concatenate([[0], np.cumsum(vv == np.inf)])
    ninf = np.concatenate([[0], np.cumsum(vv == -np.inf)])
    h = height(hi - lo + 1)
    exact, tol = np.zeros(n), np.zeros(n)
    for i in range(n):
        ai, bi = int(a[i]), int(b[i])
        ip, ineg = pinf[bi] - pinf[ai], ninf[bi] - ninf[ai]
        if ip or ineg:
            exact[i] = np.nan if ip and ineg else np.inf if ip else -np.inf
            continue
        k = min(int(c[i]) - 1, int(h[i]))
        g = k * U / (1 - k * U) if k > 0 else 0.0
        exact[i] = (ex[bi] - ex[ai]) / (1 << 1074)
        tol[i] = g * (ab[bi] - ab[ai])
    if fname == "mean":
        exact = np.where(c > 0, exact / np.maximum(c, 1), 0.0)
        tol = tol / np.maximum(c, 1) + 2 * U * np.abs(exact)
    if ct == CTypes.FLOAT32 and fname == "sum":
        tol = tol * (1 + 2.0 ** -23) + 2.0 ** -24 * (np.abs(exact) + tol)
    return exact, c > 0, tol


def check(table, part, order, funcs, asc=None, nap=None, **kw):
    part, order = list(part), list(order)
    asc = [True] * len(order) if asc is None else asc
    nap = ["last"] * len(order) if nap is None else nap
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


def frame_funcs(col, ct, frames):
    fs = []
    for j, (s, e) in enumerate(frames):
        fr = ("rows", s, e)
        names = ["count", "min", "max", "first_value", "last_value"] + ([] if ct in TEMPORAL else ["sum", "mean"])
        fs += [(f"{f}{j}", f, col, fr) for f in names]
        fs += [(f"cz{j}", "count", None, fr), (f"nth{j}", "nth_value", col, 1 + j % 4, fr)]
    return fs


def in_states(fs, n_cols):
    per = 32 - n_cols
    return [fs[i:i + per] for i in range(0, len(fs), per)]


# ---- every function x every value type x every frame ----
@pytest.mark.parametrize("ct", KEY_TYPES)
@pytest.mark.parametrize("nullable", [False, True])
def test_value_types(gpu_lib, ct, nullable):
    rng = np.random.default_rng(700 + ct * 2 + nullable)
    n = 1500
    x = float_values(ct, n, rng, nullable) if ct in (CTypes.FLOAT32, CTypes.FLOAT64) else make_column(ct, n, rng, nullable, small=False)
    t = Table([make_column(CTypes.INT8, n, rng, False), make_column(CTypes.INT16, n, rng, True, na_frac=0.1), x], ["g", "o", "x"])
    fs = frame_funcs("x", ct, FRAMES) + [("nth_r", "nth_value", "x", 2), ("nth_w", "nth_value", "x", 3, "rows"),
                                         ("nth_p", "nth_value", "x", 5, "partition"), ("nth_big", "nth_value", "x", BIG, "partition")]
    for chunk in in_states(fs, 3):
        check(t, ["g"], ["o"], chunk, sizes=(777,))


def test_cancellation_is_exact(gpu_lib):
    """SUM over 1 PRECEDING of [2^60, 1, 1, ...]: a prefix difference gives 0 or 4, the tree exactly 2."""
    n = 50
    x = np.ones(n)
    x[0] = 2.0 ** 60
    t = Table([Column(np.zeros(n, np.int64)), Column(np.arange(n, dtype=np.int64)), Column(x)], ["g", "o", "x"])
    got, _ = run(t, ["g"], ["o"], [True], ["last"], [("s", "sum", "x", ("rows", -1, 0)), ("m", "mean", "x", ("rows", -1, 0))])
    assert got[3][0][0] == 2.0 ** 60 and np.all(got[3][0][2:] == 2.0)
    assert np.all(got[4][0][2:] == 1.0)


@pytest.mark.parametrize("k", [3, 4, 6, 11])
def test_widths_around_the_stored_levels(gpu_lib, k):
    """Frames of 2^k - 1, 2^k and 2^k + 1 rows, trailing, leading and centred, in one partition of many tiles."""
    rng = np.random.default_rng(k)
    n = 3 * TILE + 101
    t = Table([Column(np.zeros(n, np.int64)), Column(rng.permutation(n).astype(np.int64)),
               make_column(CTypes.INT64, n, rng, True, small=False), float_values(CTypes.FLOAT64, n, rng, True)], ["g", "o", "x", "f"])
    fs = []
    for w in ((1 << k) - 1, 1 << k, (1 << k) + 1):
        for j, fr in enumerate([("rows", -(w - 1), 0), ("rows", 0, w - 1), ("rows", -(w // 2), w - 1 - w // 2)]):
            fs += [(f"sx{w}_{j}", "sum", "x", fr), (f"mx{w}_{j}", "max", "x", fr), (f"sf{w}_{j}", "sum", "f", fr),
                   (f"nf{w}_{j}", "min", "f", fr)]
    for chunk in in_states(fs, 4):
        check(t, ["g"], ["o"], chunk)


@pytest.mark.parametrize("n", [1, 7, 8, 9, TILE - 1, TILE, TILE + 1, 3 * TILE + 17, 40_000])
def test_tile_edges(gpu_lib, n):
    rng = np.random.default_rng(n + 1)
    i = np.arange(n)
    t = Table([Column((i // 15000).astype(np.int64)), Column((i // 7 % 5).astype(np.int64)),
               make_column(CTypes.INT32, n, rng, True, small=False), float_values(CTypes.FLOAT64, n, rng, True)], ["g", "o", "x", "f"])
    fs = [("sx", "sum", "x", ("rows", -100, 3)), ("mx", "max", "x", ("rows", -2047, 0)), ("nx", "min", "x", ("rows", 0, 5000)),
          ("cf", "count", "f", ("rows", -9, 9)), ("sf", "sum", "f", ("rows", -1000, None)), ("af", "mean", "f", ("rows", None, 2048)),
          ("lf", "last_value", "f", ("rows", -3, 2049)), ("c", "count", None, ("rows", -8, -1)), ("nt", "nth_value", "x", 2049, "range")]
    check(t, ["g"], ["o"], fs, sizes=(TILE - 1, TILE, TILE + 1))


def test_large_input_against_torch(gpu_lib):
    """2^24 + a few tiles of device rows: integer sums against cumsum differences, max against a torch sparse table."""
    n = CHUNK + 3 * TILE + 5
    dev = torch.device("cuda", 0)
    g = torch.Generator(device=dev).manual_seed(71)
    pk = torch.randint(0, 50, (n,), generator=g, device=dev, dtype=torch.int64)
    x = torch.randint(-(1 << 40), 1 << 40, (n,), generator=g, device=dev, dtype=torch.int64)
    rid = torch.arange(n, device=dev, dtype=torch.int64)
    funcs = [("s", "sum", "x", ("rows", -1000, 500)), ("m", "max", "x", ("rows", -70000, 0)), ("c", "count", None, ("rows", -5, 5))]
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
    pid = torch.cumsum(ps.to(torch.int64), 0) - 1
    pe = P + torch.bincount(pid)[pid]
    cs = torch.cat([torch.zeros(1, dtype=torch.int64, device=dev), torch.cumsum(sx, 0)])
    lo, hi = torch.maximum(P, i - 1000), torch.minimum(pe - 1, i + 500)
    assert torch.equal(got[3], cs[hi + 1] - cs[lo])
    lo = torch.maximum(P, i - 70000)
    levels = [sx]
    while (1 << len(levels)) <= 70001:
        p, h = levels[-1], 1 << (len(levels) - 1)
        levels.append(torch.maximum(p[:-h], p[h:]))
    w = i - lo + 1
    k = torch.frexp(w.to(torch.float64))[1].to(torch.int64) - 1
    exp = torch.empty_like(sx)
    for kk in range(len(levels)):
        s = k == kk
        if bool(s.any()):
            exp[s] = torch.maximum(levels[kk][lo[s]], levels[kk][i[s] - (1 << kk) + 1])
    del levels
    assert torch.equal(got[4], exp)
    assert torch.equal(got[5], torch.minimum(pe - 1, i + 5) - torch.maximum(P, i - 5) + 1)
    for c in (3, 4):
        assert out.columns[c].valid_mask_numpy().all()
    W.delete_window_state(st)


def test_determinism_across_batches(gpu_lib):
    rng = np.random.default_rng(72)
    n = 30_000
    t = Table([Column(rng.integers(0, 5, n).astype(np.int64)), Column(rng.integers(0, 50, n).astype(np.int64)),
               float_values(CTypes.FLOAT64, n, rng, True), float_values(CTypes.FLOAT32, n, rng, False)], ["g", "o", "x", "y"])
    fs = [(f"{f}{c}{j}", f, c, ("rows", s, e)) for c in ("x", "y") for f in ("sum", "mean")
          for j, (s, e) in enumerate([(-6, 0), (-300, 300), (None, 77), (5, None)])]
    ref, _ = run(t, ["g"], ["o"], [True], ["last"], fs)
    for sizes, dev in (((1000,), True), ((4096, 17), False), ((TILE,), True)):
        got, _ = run(t, ["g"], ["o"], [True], ["last"], fs, sizes=sizes, device=dev)
        for a, b in zip(ref[4:], got[4:]):
            np.testing.assert_array_equal(a[0].view(f"u{a[0].itemsize}"), b[0].view(f"u{b[0].itemsize}"))
            np.testing.assert_array_equal(a[1], b[1])


def test_spellings_of_the_unbounded_frames(gpu_lib):
    rng = np.random.default_rng(73)
    n = 20_000
    t = Table([Column(rng.integers(0, 7, n).astype(np.int64)), Column(rng.integers(0, 500, n).astype(np.int64)),
               float_values(CTypes.FLOAT64, n, rng, True)], ["g", "o", "x"])
    fs = []
    for f in ("sum", "mean", "min", "max", "count", "first_value", "last_value"):
        fs += [(f"{f}_r", f, "x", "rows"), (f"{f}_r2", f, "x", ("rows", None, 0)), (f"{f}_p", f, "x", "partition"),
               (f"{f}_p2", f, "x", ("rows", None, None))]
    got, _ = run(t, ["g"], ["o"], [True], ["last"], fs)
    for j in range(0, len(fs), 2):
        a, b = got[3 + j], got[4 + j]
        np.testing.assert_array_equal(a[0].view(np.uint64), b[0].view(np.uint64), err_msg=str(fs[j]))
        np.testing.assert_array_equal(a[1], b[1])


def test_mixed_state_keeps_old_columns(gpu_lib):
    rng = np.random.default_rng(74)
    n = 10_000
    t = Table([make_column(CTypes.INT16, n, rng, True), make_column(CTypes.INT32, n, rng, True), float_values(CTypes.FLOAT64, n, rng, True)],
              ["g", "o", "x"])
    old = [("rn", "row_number"), ("s", "sum", "x", "rows"), ("lg", "lag", "x", 1, 0.0), ("dr", "dense_rank"), ("mx", "max", "o", "range")]
    new = [("ms", "sum", "x", ("rows", -3, 3)), ("nv", "nth_value", "o", 2), ("mn", "min", "x", ("rows", -10, 0)),
           ("fv", "first_value", "x", ("rows", 1, 4))]
    alone, _ = run(t, ["g"], ["o"], [True], ["last"], old)
    mixed = [old[0], new[0], old[1], old[2], new[1], old[3], new[2], old[4], new[3]]
    got, _ = run(t, ["g"], ["o"], [True], ["last"], mixed)
    for j, f in enumerate(mixed):
        if f in old:
            a, b = alone[3 + old.index(f)], got[3 + j]
            np.testing.assert_array_equal(a[0].view(f"u{a[0].itemsize}"), b[0].view(f"u{b[0].itemsize}"), err_msg=f[0])
            np.testing.assert_array_equal(a[1], b[1])
    check(t, ["g"], ["o"], new)


# ---- pandas ----
@pytest.mark.parametrize("with_na", [False, True])
def test_pandas_rolling(gpu_lib, with_na):
    from bodo_b200.physical import window

    rng = np.random.default_rng(75 + with_na)
    n = 20_000
    f = rng.integers(-2000, 2000, n) / 8.0  # eighths: float sums are exact in any order
    if with_na:
        f = pd.array(np.where(rng.random(n) < 0.2, np.nan, f), dtype="Float64")
        f[rng.random(n) < 0.2] = pd.NA
    df = pd.DataFrame({"p": rng.integers(0, 300, n), "o": rng.permutation(n), "f": f})
    funcs = [("s7", "sum", "f", ("rows", -6, 0)), ("m7", "mean", "f", ("rows", -6, 0)), ("n7", "min", "f", ("rows", -6, 0)),
             ("x7", "max", "f", ("rows", -6, 0)), ("c7", "count", "f", ("rows", -6, 0)), ("sc", "sum", "f", ("rows", -3, 3)),
             ("xf", "max", "f", ("rows", 0, 9))]
    got = window(df, "p", "o", funcs, batch_size=7000)
    srt = df.sort_values(["p", "o"], kind="stable").reset_index(drop=True)
    srt["f"] = srt["f"].astype(np.float64)
    gb = srt.groupby("p", sort=False)["f"]

    def roll(r, how):
        return getattr(r, how)().reset_index(level=0, drop=True).sort_index()

    fwd = pd.api.indexers.FixedForwardWindowIndexer(window_size=10)
    exp = {"s7": roll(gb.rolling(7, min_periods=1), "sum"), "m7": roll(gb.rolling(7, min_periods=1), "mean"),
           "n7": roll(gb.rolling(7, min_periods=1), "min"), "x7": roll(gb.rolling(7, min_periods=1), "max"),
           "c7": roll(gb.rolling(7, min_periods=0), "count"), "sc": roll(gb.rolling(7, center=True, min_periods=1), "sum"),
           "xf": roll(gb.rolling(fwd, min_periods=1), "max")}
    for k, e in exp.items():
        np.testing.assert_array_equal(got[k].to_numpy(dtype=np.float64, na_value=np.nan), e.to_numpy(dtype=np.float64), err_msg=k)


# ---- errors ----
def test_device_side_validation(gpu_lib):
    L = _lib.lib()
    c_types = ffi.new("int8_t[]", [CTypes.INT64, CTypes.DATETIME])
    a_types = ffi.new("int8_t[]", [ArrTypes.NUMPY, ArrTypes.NUMPY])
    one = ffi.new("int32_t[]", [1])
    UP, UF = W.UNBOUNDED_PRECEDING, W.UNBOUNDED_FOLLOWING

    def init(code, col, frame, arg=0, start=UP, end=UF):
        fs = ffi.new("b200_window_func[]", 1)
        fs[0].code, fs[0].col, fs[0].frame, fs[0].arg = code, col, frame, arg
        fs[0].rows.start, fs[0].rows.end = start, end
        h = L.b200_window_state_init(-1, c_types, a_types, 2, 1, 0, one, one, fs, 1, 1024, 0, ffi.NULL)
        if h != ffi.NULL:
            L.b200_delete_sort_state(h)
            return None
        return ffi.string(L.b200_last_error()).decode()

    assert init(6, 0, 4, 0, -3, 0) is None and init(15, 1, 1, 2) is None and init(7, -1, 4, 0, 0, 0) is None
    assert init(15, 0, 4, 1, UP, 5) is None and init(11, 0, 2) is None and init(9, 0, 4, 0, -(2 ** 31 - 1), 2 ** 31 - 1) is None
    assert "nth_value needs n" in init(15, 0, 1, 0)
    assert "nth_value needs n" in init(15, 0, 1, 1 << 31)
    assert "column index out of range" in init(15, -1, 1, 1)
    assert "row offset" in init(6, 0, 4, 0, -(1 << 31), 0)
    assert "row offset" in init(6, 0, 4, 0, 0, 1 << 31)
    assert "row offset" in init(6, 0, 4, 0, UF, UF)
    assert "row offset" in init(6, 0, 4, 0, UP, UP)
    assert "start after frame end" in init(6, 0, 4, 0, 2, 1)
    assert "lag and lead take no frame" in init(13, 0, 4, 1)
    assert "no column and no frame" in init(0, -1, 4)
    assert "unknown frame" in init(6, 0, 6)
    assert "unknown function code" in init(25, 0, 1)
    assert "sum and mean need" in init(8, 1, 4, 0, -1, 1)
