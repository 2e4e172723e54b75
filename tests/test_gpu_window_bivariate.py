"""COVAR_SAMP / COVAR_POP / CORR / REGR_SLOPE / REGR_INTERCEPT window functions on the GPU, over the cumulative frames, bounded
ROWS frames and RANGE frames.

The oracle is exact: each cell as a double (what the device converts it to) is an integer multiple of 2^-1074, so with X, Y the
scaled integers of a frame's m counted pairs (both cells valid, non-NaN and finite), Sxx = (m sum X^2 - (sum X)^2) / (m 2^2148),
Syy and Sxy = (m sum XY - sum X sum Y) / (m 2^2148) are Python rationals, from prefix sums.  slope* = Sxy / Sxx and
intercept* = my - slope* mx are exact rationals, and corr* is rounded from the rational Sxy^2 / (Sxx Syy) with Sxy's sign.  The
device must match the validity exactly and lie within the bound of DESIGN §3c,
    |Sxy - Sxy*| <= sqrt(h) (gamma_{21h} sqrt(Sxx* Syy*) + gamma_{8h} (|mx*| sqrt(m Syy*) + |my*| sqrt(m Sxx*))),
(Sxx and Syy: the same with x = y), with h the combination height (tests/test_gpu_window_moments.py's), and the first-order bounds
§3c derives from it for corr, slope and intercept.  Frame bounds come from tests/test_gpu_window_frames.py's lo_hi and
tests/test_gpu_window_ranges.py's range_lo_hi, independently of the device."""

import math
from fractions import Fraction

import numpy as np
import pandas as pd
import pytest
import torch

from bodo_b200 import _lib
from bodo_b200._lib import ffi
from bodo_b200.streaming import window as W
from bodo_b200.table import ArrTypes, Column, CTypes, Table
from tests.test_gpu_sort import col_mask, make_column
from tests.test_gpu_window_frames import FRAMES as BOUNDED, ilog2, in_states, lo_hi
from tests.test_gpu_window_moments import gamma
from tests.test_gpu_window_ranges import range_lo_hi
from tests.test_gpu_window_values import CHUNK, TILE, U, _sorted_col, bounds, float_values, run

pytestmark = pytest.mark.gpu

FUNCS = ("covar_samp", "covar_pop", "corr", "regr_slope", "regr_intercept")
CUMULATIVE = ("range", "rows", "partition")
RANGES = [(-3, 0), (-2, 2), (0, 0), (2, 5), (None, 3), (-5, None)]
ALL_FRAMES = list(CUMULATIVE) + [("rows", s, e) for s, e in BOUNDED] + [("range_between", s, e) for s, e in RANGES]


@pytest.fixture(autouse=True)
def _return_device_memory():
    yield
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    _lib.lib().b200_pool_trim(torch.cuda.current_device(), 0)


def frame_of(fn):
    return fn[4] if len(fn) > 4 else "range"


def _scaled(table, col, perm):
    """The sorted column as doubles, its counted mask (valid and non-NaN), its +-inf mask and the exact scaled integers of its
    finite cells (0 elsewhere)."""
    v, mask, _ = _sorted_col(table, col, perm)
    d = v.astype(np.float64)
    good = mask & ~np.isnan(d)
    inf = good & np.isinf(d)
    S = [num * ((1 << 1074) // den) for num, den in (x.as_integer_ratio() if f else (0, 1) for x, f in zip(d.tolist(), (good & ~inf).tolist()))]
    return good, inf, S


def _prefix(a):
    p = [0]
    for x in a:
        p.append(p[-1] + x)
    return p


def frame_bounds(table, order, fr, perm, P, pe, ends):
    if isinstance(fr, tuple) and fr[0] == "range_between":
        return range_lo_hi(table, order, [True], ["last"], fr, perm, P, pe, ends)
    return lo_hi(fr, P, pe, ends)


def exact_comoments(table, perm, ycol, xcol, lo, hi, cumulative):
    """Per row over [lo, hi]: m, Sxx*, Syy*, Sxy* and the means as Fractions (None when m = 0 or the pairs hold +-inf), whether
    x / y holds +-inf among the counted pairs, and h."""
    gy, iy, Y = _scaled(table, ycol, perm)
    gx, ix, X = _scaled(table, xcol, perm)
    pair = gx & gy
    X = [x if p else 0 for x, p in zip(X, pair.tolist())]
    Y = [y if p else 0 for y, p in zip(Y, pair.tolist())]
    SX, SY = _prefix(X), _prefix(Y)
    SXX, SYY, SXY = _prefix([x * x for x in X]), _prefix([y * y for y in Y]), _prefix([x * y for x, y in zip(X, Y)])
    cnt = np.concatenate([[0], np.cumsum(pair)])
    nx, ny = np.concatenate([[0], np.cumsum(pair & ix)]), np.concatenate([[0], np.cumsum(pair & iy)])
    a, b = np.where(lo <= hi, lo, 0), np.where(lo <= hi, hi + 1, 0)
    m = cnt[b] - cnt[a]
    xinf, yinf = nx[b] - nx[a] > 0, ny[b] - ny[a] > 0
    out = []
    for i in range(len(lo)):
        mi = int(m[i])
        if mi == 0 or xinf[i] or yinf[i]:
            out.append(None)
            continue
        ai, bi = int(a[i]), int(b[i])
        sx, sy = SX[bi] - SX[ai], SY[bi] - SY[ai]
        den = mi << 2148
        out.append((Fraction(mi * (SXX[bi] - SXX[ai]) - sx * sx, den), Fraction(mi * (SYY[bi] - SYY[ai]) - sy * sy, den),
                    Fraction(mi * (SXY[bi] - SXY[ai]) - sx * sy, den), Fraction(sx, mi << 1074), Fraction(sy, mi << 1074)))
    h = np.maximum(m - 1, 0)
    if not cumulative:
        h = np.minimum(h, 10 + 3 * ilog2(hi - lo + 1))
    return m, out, xinf, yinf, h


def _corr_exact(sxx, syy, sxy):
    """sign(Sxy) sqrt(Sxy^2 / (Sxx Syy)), rounded from the exact rational (within one ulp)."""
    q = sxy * sxy / (sxx * syy)
    k = 120
    r = Fraction(math.isqrt(q.numerator * 4**k // q.denominator), 2**k)
    return math.copysign(float(r), float(sxy)) if sxy != 0 else 0.0


def expected(fname, m, ex, xinf, yinf, h):
    """(exact value, validity, tolerance, NaN expected) per row.  Tolerances: e_ab the §3c bound on S_ab; covar_samp / covar_pop
    divide it; corr takes e_xy / D + |corr*| (e_xx / Sxx* + e_yy / Syy*) / 2 with D = sqrt(Sxx* Syy*), slope
    (e_xy + |slope*| e_xx) / (Sxx* - e_xx), intercept |mx*| e_slope + the means' gamma_{4h} (|m*| + sqrt(S* / m)) each, all
    doubled for the second-order terms, plus the final operations' rounding."""
    n = len(m)
    val, valid, tol, nan = np.zeros(n), np.zeros(n, bool), np.zeros(n), xinf | yinf
    for i in range(n):
        mi, hi = int(m[i]), int(h[i])
        if ex[i] is None:  # m = 0, or +-inf among the pairs (a NaN; corr / regr's validity is checked by the caller)
            valid[i] = mi >= (2 if fname == "covar_samp" else 1) if fname in ("covar_samp", "covar_pop") else False
            continue
        sxx, syy, sxy, mx, my = ex[i]
        fx, fy = float(sxx), float(syy)
        amx, amy = abs(float(mx)), abs(float(my))
        g21, g8, sh = gamma(21 * hi), gamma(8 * hi), math.sqrt(hi)

        def e(a, b, ma, mb):
            return sh * (g21 * math.sqrt(a) * math.sqrt(b) + g8 * (ma * math.sqrt(mi * b) + mb * math.sqrt(mi * a)))

        exy, exx, eyy = e(fx, fy, amx, amy), e(fx, fx, amx, amx), e(fy, fy, amy, amy)
        if fname in ("covar_samp", "covar_pop"):
            d = mi - (1 if fname == "covar_samp" else 0)
            valid[i] = d >= 1
            if valid[i]:
                val[i] = float(sxy / d)
                tol[i] = exy / d + 2 * U * abs(val[i])
        elif fname == "corr":
            valid[i] = mi >= 2 and sxx != 0 and syy != 0
            if valid[i]:
                val[i] = _corr_exact(sxx, syy, sxy)
                tol[i] = 2 * (exy / (math.sqrt(fx) * math.sqrt(fy)) + abs(val[i]) * 0.5 * (exx / fx + eyy / fy)) + 4 * U
        else:
            valid[i] = sxx != 0
            if valid[i]:
                slope = sxy / sxx
                ts = 2 * (exy + abs(float(slope)) * exx) / max(fx - exx, 1e-300) + 2 * U * abs(float(slope))
                if fname == "regr_slope":
                    val[i], tol[i] = float(slope), ts
                else:
                    val[i] = float(my - slope * mx)
                    emx, emy = gamma(4 * hi) * (amx + math.sqrt(fx / mi)), gamma(4 * hi) * (amy + math.sqrt(fy / mi))
                    tol[i] = 2 * (emy + amx * ts + abs(float(slope)) * emx + ts * emx) + 4 * U * (amy + abs(float(slope)) * amx) + 2 * U * abs(val[i])
    return val, valid, tol, nan


def check(table, part, order, funcs, **kw):
    part, order = list(part), list(order)
    perm, P, pe, ends = bounds(table, part, order, [True] * len(order), ["last"] * len(order))
    got, sizes = run(table, part, order, [True] * len(order), ["last"] * len(order), funcs, **kw)
    for c, (vals, mask, _) in zip(table.columns, got):
        np.testing.assert_array_equal(vals.view(np.uint8), c.values_numpy()[perm].view(np.uint8))
    cache = {}
    for fn, (vals, mask, oc) in zip(funcs, got[table.n_cols:]):
        assert (oc.c_type, oc.arr_type) == (CTypes.FLOAT64, ArrTypes.NULLABLE_INT_BOOL), fn
        fr = frame_of(fn)
        key = (fn[2], fn[3], str(fr))
        if key not in cache:
            lo, hi = frame_bounds(table, order, fr, perm, P, pe, ends)
            cache[key] = exact_comoments(table, perm, fn[2], fn[3], lo, hi, isinstance(fr, str)), lo, hi
        (m, ex, xinf, yinf, h), lo, hi = cache[key]
        exact, valid, tol, nan = expected(fn[1], m, ex, xinf, yinf, h)
        inf_rows = np.array([e is None for e in ex]) & (m >= 1)
        if fn[1] in ("covar_samp", "covar_pop"):
            np.testing.assert_array_equal(mask, valid, err_msg=str(fn))
        else:  # with +-inf among the pairs the NA test reads the device's exact Sxx = 0 (equal x) / Syy = 0 (equal y)
            fin = ~inf_rows
            np.testing.assert_array_equal(mask[fin], valid[fin], err_msg=str(fn))
            assert np.all(mask[inf_rows] <= (m[inf_rows] >= (1 if fn[1] != "corr" else 2))), fn
        assert np.isnan(vals[mask & inf_rows]).all(), fn  # a frame whose pairs hold +-inf gives a valid NaN
        ok = mask & ~inf_rows
        if fn[1] == "corr":
            assert np.all(np.abs(vals[ok]) <= 1.0), fn
        err = np.abs(vals[ok] - exact[ok])
        bad = np.flatnonzero(~(err <= tol[ok]))
        assert bad.size == 0, (fn, vals[ok][bad[:5]], exact[ok][bad[:5]], tol[ok][bad[:5]])
    return got, sizes


def bivariate_funcs(y, x, frames):
    return [(f"{f}{j}", f, y, x, fr) for j, fr in enumerate(frames) for f in FUNCS]


def _no_subnormal(c):
    """float_values' column with its float64 subnormal replaced by 0.0: the square of a subnormal difference underflows to 0,
    which would make the device's Sxx exactly 0 where Sxx* is positive (1e-647)."""
    v = np.asarray(c.data)
    if v.dtype == np.float64:
        v[(v != 0) & (np.abs(v) < np.finfo(np.float64).tiny)] = 0.0
    return c


def _values(ct, n, rng, nullable):
    if ct in (CTypes.FLOAT32, CTypes.FLOAT64):
        return _no_subnormal(float_values(ct, n, rng, nullable))
    return make_column(ct, n, rng, nullable, small=False)


# ---- every function x every frame x pairs of value types ----
PAIRS = [(CTypes.FLOAT64, CTypes.FLOAT64, True, True), (CTypes.FLOAT64, CTypes.INT8, True, False), (CTypes.INT64, CTypes.UINT32, False, True),
         (CTypes.FLOAT32, CTypes.FLOAT64, True, False), (CTypes.BOOL, CTypes.INT16, True, True), (CTypes.UINT64, CTypes.FLOAT32, False, True),
         (CTypes.INT32, CTypes.UINT8, True, True), (CTypes.UINT16, CTypes.BOOL, False, False)]


@pytest.mark.parametrize("yct,xct,ynull,xnull", PAIRS)
def test_value_type_pairs(gpu_lib, yct, xct, ynull, xnull):
    rng = np.random.default_rng(1200 + 16 * yct + xct)
    n = 1200
    o = make_column(CTypes.INT16, n, rng, True, na_frac=0.1)
    o.data = np.asarray(o.data) % 300  # ties, so RANGE frames differ from ROWS frames
    t = Table([make_column(CTypes.INT8, n, rng, False), o, _values(yct, n, rng, ynull), _values(xct, n, rng, xnull)], ["g", "o", "y", "x"])
    for chunk in in_states(bivariate_funcs("y", "x", ALL_FRAMES), 4):
        check(t, ["g"], ["o"], chunk, sizes=(777,))


# ---- exact invariants ----
def test_symmetry_self_correlation_and_bounds(gpu_lib):
    """covar and corr bit-symmetric in (y, x); corr(x, x) exactly 1.0 where valid; |corr| <= 1 everywhere."""
    rng = np.random.default_rng(1300)
    n = 9000
    t = Table([Column(rng.integers(0, 7, n).astype(np.int64)), Column(rng.integers(0, 500, n).astype(np.int64)),
               _values(CTypes.FLOAT64, n, rng, True), Column(1e6 + rng.standard_normal(n) * 1e-3), make_column(CTypes.INT32, n, rng, True, small=False)],
              ["g", "o", "a", "b", "c"])
    frames = ["range", "rows", "partition", ("rows", -19, 0), ("rows", -3, 300), ("range_between", -5, 2)]
    for y, x in (("a", "b"), ("a", "c"), ("b", "c")):
        fs = [(f"{f}{j}{s}", f, *cols, fr) for j, fr in enumerate(frames) for f in ("covar_samp", "covar_pop", "corr")
              for s, cols in (("f", (y, x)), ("r", (x, y)))]
        res = {}
        for chunk in in_states(fs, 5):
            got, _ = run(t, ["g"], ["o"], [True], ["last"], chunk)
            res.update({fn[0]: got[5 + k] for k, fn in enumerate(chunk)})
        for fn in fs:
            if fn[0].endswith("f"):
                a, b = res[fn[0]], res[fn[0][:-1] + "r"]
                np.testing.assert_array_equal(a[0].view(np.uint64), b[0].view(np.uint64), err_msg=str(fn))
                np.testing.assert_array_equal(a[1], b[1])
            if fn[1] == "corr":
                v, mk, _ = res[fn[0]]
                assert np.all(np.abs(v[mk & ~np.isnan(v)]) <= 1.0)
    fs = [(f"cc{j}{c}", "corr", c, c, fr) for j, fr in enumerate(frames) for c in ("a", "b", "c")]
    for chunk in in_states(fs, 5):
        got, _ = run(t, ["g"], ["o"], [True], ["last"], chunk)
        for k, fn in enumerate(chunk):
            v, mk, _ = got[5 + k]
            fin = mk & ~np.isnan(v)  # +-inf in the frame: a valid NaN
            assert fin.sum() > 0 and (v[fin] == 1.0).all(), fn


def test_edges_equal_x_inf_nan_and_few_pairs(gpu_lib):
    """Per partition: m = 0 / 1 / 2, an equal-valued x (corr, slope, intercept NA; covariances exactly 0.0), +-inf (valid NaN),
    NaN and NA dropped pairwise, and y valid where x is NA throughout."""
    nan, inf = np.nan, np.inf
    parts = [([nan, 1.0], [2.0, nan]),            # m = 0
             ([1.0, 5.0], [nan, 2.0]),            # m = 1
             ([1.0, 4.0], [2.0, 8.0]),            # m = 2: slope 0.5 exactly, corr 1
             ([3.0, 1.0, 7.0, 2.0], [5.0] * 4),   # x constant
             ([0.1] * 6, [0.3, 0.7, 0.1, 0.9, 0.2, 0.4]),  # y constant: slope 0.0 exactly, corr NA
             ([1.0, 2.0, 3.0], [1.0, inf, 2.0]),  # inf in x
             ([1.0, -inf, 3.0], [1.0, 2.0, 3.0]),  # inf in y
             ([1.0, 2.0, 3.0, 4.0], [None] * 4),  # x NA throughout
             ([2.0, 4.0, nan, 8.0], [1.0, 2.0, 3.0, 4.0])]
    g = np.concatenate([np.full(len(p[0]), k) for k, p in enumerate(parts)]).astype(np.int64)
    y = np.concatenate([np.array(p[0], dtype=np.float64) for p in parts])
    xs = [v for p in parts for v in p[1]]
    xvalid = np.array([v is not None for v in xs])
    x = np.array([0.0 if v is None else v for v in xs])
    n = len(y)
    t = Table([Column(g), Column(np.arange(n, dtype=np.int64)), Column(y),
               Column(x, np.packbits(xvalid, bitorder="little"), CTypes.FLOAT64, ArrTypes.NULLABLE_INT_BOOL, n)], ["g", "o", "y", "x"])
    fs = bivariate_funcs("y", "x", ["partition", "rows", ("rows", -1, 0)])
    got, _ = check(t, ["g"], ["o"], fs)
    res = {fn[0]: got[4 + j] for j, fn in enumerate(fs)}
    off = np.cumsum([0] + [len(p[0]) for p in parts])
    sl = {k: slice(off[k], off[k + 1]) for k in range(len(parts))}
    for f in FUNCS:
        assert not res[f"{f}0"][1][sl[0]].any() and not res[f"{f}0"][1][sl[7]].any()  # no pairs
    assert res["covar_pop0"][1][sl[1]].all() and (res["covar_pop0"][0][sl[1]] == 0.0).all()  # m = 1
    for f in ("covar_samp", "corr", "regr_slope", "regr_intercept"):
        assert not res[f"{f}0"][1][sl[1]].any()
    assert (res["regr_slope0"][0][sl[2]] == 0.5).all() and (res["corr0"][0][sl[2]] == 1.0).all() and (res["covar_samp0"][0][sl[2]] == 9.0).all()
    assert (res["regr_intercept0"][0][sl[2]] == 0.0).all()
    for j in range(3):
        for f in ("corr", "regr_slope", "regr_intercept"):
            assert not res[f"{f}{j}"][1][sl[3]].any(), (f, j)
        for f in ("covar_samp", "covar_pop"):
            v, mk, _ = res[f"{f}{j}"]
            assert (v[sl[3]][mk[sl[3]]] == 0.0).all() and mk[sl[3]].any()
        v, mk, _ = res[f"regr_slope{j}"]
        assert (v[sl[4]][mk[sl[4]]] == 0.0).all() and mk[sl[4]].any()
        assert not res[f"corr{j}"][1][sl[4]].any()
    for k in (5, 6):
        for f in FUNCS:
            v, mk, _ = res[f"{f}0"]
            assert mk[sl[k]].all() and np.isnan(v[sl[k]]).all(), (k, f)
    assert (res["regr_slope0"][0][sl[8]] == 2.0).all() and (res["corr0"][0][sl[8]] == 1.0).all()


def test_catastrophic_cancellation(gpu_lib):
    """x = 1.7e9 + U[0, 1000), y = 3x + noise: corr and slope within 1e-6 of exact in every frame, where the one-pass formula
    sum xy - sum x sum y / m fails the same check."""
    rng = np.random.default_rng(1310)
    n = 6000
    x = 1.7e9 + rng.uniform(0, 1000, n)
    y = 3 * x + rng.standard_normal(n)
    t = Table([Column(rng.integers(0, 3, n).astype(np.int64)), Column(rng.permutation(n).astype(np.int64)), Column(y), Column(x)],
              ["g", "o", "y", "x"])
    frames = ["range", "rows", "partition", ("rows", -19, 0), ("rows", -500, 500), ("range_between", -40, 0)]
    fs = [(f"{f}{j}", f, "y", "x", fr) for j, fr in enumerate(frames) for f in ("corr", "regr_slope")]
    got, _ = check(t, ["g"], ["o"], fs)
    perm, P, pe, ends = bounds(t, ["g"], ["o"], [True], ["last"])
    naive_fails = False
    for j, fr in enumerate(frames):
        lo, hi = frame_bounds(t, ["o"], fr, perm, P, pe, ends)
        m, ex, _, _, _ = exact_comoments(t, perm, "y", "x", lo, hi, isinstance(fr, str))
        ok = m >= 3
        for k, f in enumerate(("corr", "regr_slope")):
            vals = got[4 + 2 * j + k][0]
            exact = np.array([(_corr_exact(e[0], e[1], e[2]) if f == "corr" else float(e[2] / e[0])) if e is not None and e[0] and e[1] else 0.0
                              for e in ex])
            assert np.all(np.abs(vals[ok] - exact[ok]) <= 1e-6 * np.abs(exact[ok])), (f, fr)
            if fr == "partition" and f == "regr_slope":  # the one-pass formula in double
                gs, xs, ys = t.columns[0].values_numpy()[perm], x[perm], y[perm]
                sx, sy, sxy, sxx, c = (np.bincount(gs, w) for w in (xs, ys, xs * ys, xs * xs, None))
                naive = ((sxy - sx * sy / c) / (sxx - sx * sx / c))[gs]
                naive_fails = bool(np.any(np.abs(naive[ok] - exact[ok]) > 1e-6 * np.abs(exact[ok])))
    assert naive_fails


def test_no_leakage_from_outside_the_frame(gpu_lib):
    y = np.array([1e15, 1.0, 2.0, 3.0])
    t = Table([Column(np.zeros(4, np.int64)), Column(np.arange(4, dtype=np.int64)), Column(y), Column(np.arange(4, dtype=np.float64))],
              ["g", "o", "y", "x"])
    got, _ = run(t, ["g"], ["o"], [True], ["last"], [("s", "regr_slope", "y", "x", ("rows", -1, 0)), ("c", "corr", "y", "x", ("rows", -1, 0)),
                                                     ("i", "regr_intercept", "y", "x", ("rows", -1, 0))])
    assert got[4][0][3] == 1.0 and got[4][0][2] == 1.0
    assert got[5][0][3] == 1.0
    assert got[6][0][3] == 0.0


@pytest.mark.parametrize("n", [2047, 2048, 2049])
def test_tile_edges(gpu_lib, n):
    rng = np.random.default_rng(1320 + n)
    i = np.arange(n)
    t = Table([Column((i // 1000).astype(np.int64)), Column((i // 3 % 7).astype(np.int64)), make_column(CTypes.INT32, n, rng, True, small=False),
               _values(CTypes.FLOAT64, n, rng, True)], ["g", "o", "x", "f"])
    fs = bivariate_funcs("f", "x", ["range", "rows", "partition", ("rows", -2047, 0), ("rows", -3, 2048)])
    for chunk in in_states(fs, 4):
        check(t, ["g"], ["o"], chunk, sizes=(TILE - 1, TILE, TILE + 1))


def test_large_input_against_torch(gpu_lib):
    """2^24 + a few tiles of device rows: covar_pop / corr / slope over the partition and covar_samp over 9 PRECEDING against
    torch float64 two-pass computations."""
    n = CHUNK + 3 * TILE + 5
    dev = torch.device("cuda", 0)
    g = torch.Generator(device=dev).manual_seed(1330)
    pk = torch.randint(0, 50, (n,), generator=g, device=dev, dtype=torch.int64)
    x = 1e4 + torch.randn(n, generator=g, device=dev, dtype=torch.float64)
    y = 2 * x + torch.randn(n, generator=g, device=dev, dtype=torch.float64)
    rid = torch.arange(n, device=dev, dtype=torch.int64)
    funcs = [("cp", "covar_pop", "y", "x", "partition"), ("co", "corr", "y", "x", "partition"), ("sl", "regr_slope", "y", "x", "partition"),
             ("c10", "covar_samp", "y", "x", ("rows", -9, 0))]
    st = W.init_window_state(-1, ["p"], ["r"], [True], ["last"], funcs, ["p", "r", "y", "x"], output_batch_size=1 << 30)
    b = 3_000_000
    for r0 in range(0, n, b):
        t = Table([Column(pk[r0:r0 + b]), Column(rid[r0:r0 + b]), Column(y[r0:r0 + b]), Column(x[r0:r0 + b])], ["p", "r", "y", "x"])
        W.window_build_consume_batch(st, t, r0 + b >= n)
    out, last = W.window_produce_output_batch(st)
    assert last and out.n_rows == n
    got = [torch.as_tensor(c.data, device=dev) for c in out.columns]
    idx = torch.sort(pk, stable=True).indices
    assert torch.equal(got[1], idx)
    sp, sx, sy = pk[idx], x[idx], y[idx]
    cnt = torch.bincount(sp, minlength=50).to(torch.float64)
    z = lambda: torch.zeros(50, dtype=torch.float64, device=dev)  # noqa: E731
    mx, my = z().index_add_(0, sp, sx) / cnt, z().index_add_(0, sp, sy) / cnt
    dx, dy = sx - mx[sp], sy - my[sp]
    sxy, sxx, syy = z().index_add_(0, sp, dx * dy), z().index_add_(0, sp, dx * dx), z().index_add_(0, sp, dy * dy)
    torch.testing.assert_close(got[4], (sxy / cnt)[sp], rtol=1e-9, atol=0)
    torch.testing.assert_close(got[5], (sxy / torch.sqrt(sxx * syy))[sp], rtol=1e-9, atol=0)
    torch.testing.assert_close(got[6], (sxy / sxx)[sp], rtol=1e-9, atol=0)
    i = torch.arange(n, device=dev, dtype=torch.int64)
    ps = torch.ones(n, dtype=torch.bool, device=dev)
    ps[1:] = torch.diff(sp) != 0
    P = torch.cummax(torch.where(ps, i, 0), 0).values
    j = i[:, None] - torch.arange(10, device=dev)[None, :]
    inside = j >= P[:, None]
    wx, wy = torch.where(inside, sx[j.clamp(min=0)], 0.0), torch.where(inside, sy[j.clamp(min=0)], 0.0)
    c = inside.sum(1).to(torch.float64)
    ux, uy = wx.sum(1) / c, wy.sum(1) / c
    v = torch.where(inside, (wx - ux[:, None]) * (wy - uy[:, None]), 0.0).sum(1) / (c - 1)
    del j, inside, wx, wy
    ok = c >= 2
    assert torch.equal(torch.as_tensor(col_mask(out.columns[7]), device=dev), ok)
    torch.testing.assert_close(got[7][ok], v[ok], rtol=1e-7, atol=1e-9)
    for k in (4, 5, 6):
        assert out.columns[k].valid_mask_numpy().all()
    W.delete_window_state(st)


def test_determinism_across_batches(gpu_lib):
    rng = np.random.default_rng(1340)
    n = 30_000
    t = Table([Column(rng.integers(0, 5, n).astype(np.int64)), Column(rng.integers(0, 50, n).astype(np.int64)),
               float_values(CTypes.FLOAT64, n, rng, True), make_column(CTypes.INT64, n, rng, True, small=False)], ["g", "o", "y", "x"])
    fs = [(f"{f}{j}", f, "y", "x", fr) for f in ("covar_samp", "corr", "regr_intercept")
          for j, fr in enumerate(["range", "rows", "partition", ("rows", -6, 0), ("rows", -300, 300), ("range_between", -3, 1)])]
    for chunk in in_states(fs, 4):
        ref, _ = run(t, ["g"], ["o"], [True], ["last"], chunk)
        again, _ = run(t, ["g"], ["o"], [True], ["last"], chunk)
        for sizes, dev in (((1000,), True), ((4096, 17), False), ((TILE,), True)):
            got, _ = run(t, ["g"], ["o"], [True], ["last"], chunk, sizes=sizes, device=dev)
            for a, b, c in zip(ref[4:], got[4:], again[4:]):
                np.testing.assert_array_equal(a[0].view(np.uint64), b[0].view(np.uint64))
                np.testing.assert_array_equal(a[0].view(np.uint64), c[0].view(np.uint64))
                np.testing.assert_array_equal(a[1], b[1])


def test_rows_sharing_a_frame_share_bits(gpu_lib):
    rng = np.random.default_rng(1350)
    n = 20_000
    t = Table([Column(rng.integers(0, 7, n).astype(np.int64)), Column(rng.integers(0, 40, n).astype(np.int64)),
               float_values(CTypes.FLOAT64, n, rng, True), Column(rng.standard_normal(n))], ["g", "o", "y", "x"])
    fs = [("r", "corr", "y", "x", "range"), ("p", "regr_slope", "y", "x", "partition")]
    got, _ = run(t, ["g"], ["o"], [True], ["last"], fs)
    perm, P, pe, ends = bounds(t, ["g"], ["o"], [True], ["last"])
    for j, fr in enumerate(("range", "partition")):
        vals, mask, _ = got[4 + j]
        e = ends[fr]
        np.testing.assert_array_equal(vals.view(np.uint64), vals[e].view(np.uint64))
        np.testing.assert_array_equal(mask, mask[e])


def test_mixed_state_keeps_old_columns(gpu_lib):
    rng = np.random.default_rng(1360)
    n = 10_000
    o = make_column(CTypes.INT32, n, rng, True)
    o.data = np.asarray(o.data) % 2000
    t = Table([make_column(CTypes.INT16, n, rng, True), o, _values(CTypes.FLOAT64, n, rng, True), make_column(CTypes.INT64, n, rng, True, small=False)],
              ["g", "o", "x", "z"])
    old = [("rn", "row_number"), ("dr", "dense_rank"), ("s", "sum", "x", "rows"), ("lg", "lag", "x", 1, 0.0), ("ms", "sum", "x", ("rows", -3, 3)),
           ("v", "var", "x", ("rows", -3, 3)), ("sd", "std", "z", "partition"), ("rs", "mean", "x", ("range_between", -20, 0)),
           ("nv", "nth_value", "o", 2)]
    new = [("k", "corr", "x", "z", ("rows", -3, 3)), ("cv", "covar_samp", "z", "x", "rows"), ("b", "regr_slope", "x", "z", "partition"),
           ("ri", "regr_intercept", "x", "o", ("range_between", -20, 0)), ("cp", "covar_pop", "x", "x", "range")]
    alone, _ = run(t, ["g"], ["o"], [True], ["last"], old)
    mixed = [old[0], new[0], old[1], old[2], new[1], old[3], old[4], new[2], old[5], old[6], new[3], old[7], new[4], old[8]]
    got, _ = run(t, ["g"], ["o"], [True], ["last"], mixed)
    for j, f in enumerate(mixed):
        if f in old:
            a, b = alone[4 + old.index(f)], got[4 + j]
            np.testing.assert_array_equal(a[0].view(f"u{a[0].itemsize}"), b[0].view(f"u{b[0].itemsize}"), err_msg=f[0])
            np.testing.assert_array_equal(a[1], b[1])
    check(t, ["g"], ["o"], new)


# ---- pandas ----
@pytest.mark.parametrize("with_na", [False, True])
def test_pandas_rolling_cov_corr(gpu_lib, with_na):
    """Series.rolling(w, min_periods=2).cov(other) / .corr(other) on one partition, where pandas is finite and the window's
    result is valid; pandas drops pairs with a NaN as the window does."""
    from bodo_b200.physical import window

    rng = np.random.default_rng(1370 + with_na)
    n = 5000
    x = rng.integers(-2000, 2000, n) / 8.0
    y = 0.5 * x + rng.standard_normal(n) * 10
    if with_na:
        x = np.where(rng.random(n) < 0.1, np.nan, x)
        y = np.where(rng.random(n) < 0.1, np.nan, y)
    df = pd.DataFrame({"p": np.zeros(n, np.int64), "o": np.arange(n), "y": y, "x": x})
    funcs = [("cv", "covar_samp", "y", "x", ("rows", -19, 0)), ("cr", "corr", "y", "x", ("rows", -19, 0))]
    got = window(df, "p", "o", funcs, batch_size=1700)
    exp = {"cv": df["y"].rolling(20, min_periods=2).cov(df["x"]), "cr": df["y"].rolling(20, min_periods=2).corr(df["x"])}
    for k, e in exp.items():
        g = got[k].to_numpy(dtype=np.float64, na_value=np.nan)
        e = e.to_numpy(dtype=np.float64)
        both = np.isfinite(g) & np.isfinite(e)
        assert both.sum() > n // 2
        np.testing.assert_allclose(g[both], e[both], rtol=1e-7, atol=1e-9, err_msg=k)


# ---- the C ABI ----
def _init(L, cts, descs, n_order=1):
    n = len(cts)
    c_types = ffi.new("int8_t[]", cts)
    a_types = ffi.new("int8_t[]", [ArrTypes.NUMPY] * n)
    one = ffi.new("int32_t[]", [1])
    fs = ffi.new("b200_window_func[]", len(descs))
    for d, (code, col, frame, arg) in zip(fs, descs):
        d.code, d.col, d.frame, d.default_valid, d.arg, d.default_bits = code, col, frame, 0, arg, 0
    return L.b200_window_state_init(-1, c_types, a_types, n, 1, n_order, one, one, fs, len(descs), 1024, 0, ffi.NULL)


def test_abi_codes_and_validation(gpu_lib):
    L = _lib.lib()
    cts = [CTypes.INT64, CTypes.INT64, CTypes.FLOAT64, CTypes.INT32, CTypes.DATETIME]
    for code in range(20, 25):
        h = _init(L, cts, [(code, 2, 2, 3)])
        assert h != ffi.NULL, ffi.string(L.b200_last_error()).decode()
        L.b200_delete_sort_state(h)
    for arg, msg in ((5, "second column index"), (-1, "second column index")):
        assert _init(L, cts, [(22, 2, 2, arg)]) == ffi.NULL
        assert msg in ffi.string(L.b200_last_error()).decode()
    for col, arg in ((4, 2), (2, 4)):
        assert _init(L, cts, [(20, col, 1, arg)]) == ffi.NULL
        assert "covar, corr and regr need integer, bool or float columns" in ffi.string(L.b200_last_error()).decode()
    assert _init(L, cts, [(23, 2, 0, 3)]) == ffi.NULL
    assert "unknown frame" in ffi.string(L.b200_last_error()).decode()
    assert _init(L, cts, [(25, 2, 2, 3)]) == ffi.NULL
    assert "unknown function code" in ffi.string(L.b200_last_error()).decode()


def test_temporal_column_at_first_consume(gpu_lib):
    n = 8
    t = Table([Column(np.zeros(n, np.int64)), Column(np.arange(n, dtype=np.int64)), Column(np.arange(n, dtype=np.float64)),
               Column(np.arange(n, dtype=np.int64), None, CTypes.DATETIME, ArrTypes.NUMPY, n)], ["g", "o", "y", "t"])
    for cols in (("y", "t"), ("t", "y")):
        st = W.init_window_state(-1, ["g"], ["o"], True, "last", [("c", "corr", *cols, "rows")], t.names)
        with pytest.raises(_lib.B200Error, match="covar, corr and regr need integer, bool or float columns"):
            W.window_build_consume_batch(st, t, True)
        W.delete_window_state(st)
