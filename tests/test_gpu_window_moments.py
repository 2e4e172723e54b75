"""VAR / STDDEV / VAR_POP / STDDEV_POP window functions on the GPU, over the cumulative frames ("range", "rows", "partition") and
bounded ROWS frames.

The oracle is exact: each cell as a double (what the device converts it to) is an integer multiple of 2^-1074, so with X the
scaled integers of a frame's m valid, finite cells, M2 = (m sum X^2 - (sum X)^2) / (m 2^2148) is a Python rational.  The device's
M2 must lie within the bound of DESIGN §3c,
    |M2 - M2*| <= sqrt(h) (gamma_{21h} M2* + gamma_{8h} |mean*| sqrt(m M2*)),
with h = min(m - 1, 10 + 3 floor(log2 W)) for a frame of W rows (the tree's combination height) and h = m - 1 for the cumulative
frames; var / std add the division and the sqrt.  Frame bounds come from tests/test_gpu_window_frames.py's lo_hi over
tests/test_gpu_window_values.py's partition boundaries, independently of the device."""

import math
from fractions import Fraction

import numpy as np
import pandas as pd
import pytest
import torch

from bodo_b200 import _lib
from bodo_b200.streaming import window as W
from bodo_b200.table import ArrTypes, Column, CTypes, Table
from tests.test_gpu_sort import KEY_TYPES, col_mask, make_column
from tests.test_gpu_window_frames import FRAMES as BOUNDED, ilog2, in_states, lo_hi
from tests.test_gpu_window_values import CHUNK, TEMPORAL, TILE, U, _sorted_col, bounds, float_values, run

pytestmark = pytest.mark.gpu

MOMENTS = ("var", "std", "var_pop", "std_pop")
CUMULATIVE = ("range", "rows", "partition")
NUM_TYPES = [ct for ct in KEY_TYPES if ct not in TEMPORAL]


@pytest.fixture(autouse=True)
def _return_device_memory():
    yield
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    _lib.lib().b200_pool_trim(torch.cuda.current_device(), 0)


def gamma(k):
    return k * U / (1 - k * U) if k > 0 else 0.0


def frame_of(fn):
    return fn[3] if len(fn) > 3 else "range"


def exact_moments(table, col, perm, fr, P, pe, ends):
    """Per row over its frame: (m, M2* as float, |mean*|, any +-inf, h), from the doubles the device reads."""
    v, mask, _ = _sorted_col(table, col, perm)
    d = v.astype(np.float64)
    good = mask & ~np.isnan(d)
    inf = good & np.isinf(d)
    fin = good & ~inf
    X = [num * ((1 << 1074) // den) for num, den in (x.as_integer_ratio() if f else (0, 1) for x, f in zip(d.tolist(), fin.tolist()))]
    S1, S2 = [0], [0]
    for x in X:
        S1.append(S1[-1] + x)
        S2.append(S2[-1] + x * x)
    cnt = np.concatenate([[0], np.cumsum(good)])
    ninf = np.concatenate([[0], np.cumsum(inf)])
    lo, hi = lo_hi(fr, P, pe, ends)
    a, b = np.where(lo <= hi, lo, 0), np.where(lo <= hi, hi + 1, 0)
    m = cnt[b] - cnt[a]
    has_inf = ninf[b] - ninf[a] > 0
    n = len(perm)
    M2, amean = np.zeros(n), np.zeros(n)
    for i in range(n):
        mi = int(m[i])
        if mi == 0 or has_inf[i]:
            continue
        s1, s2 = S1[b[i]] - S1[a[i]], S2[b[i]] - S2[a[i]]
        M2[i] = float(Fraction(mi * s2 - s1 * s1, mi << 2148))
        amean[i] = abs(float(Fraction(s1, mi << 1074)))
    h = np.maximum(m - 1, 0)
    if not isinstance(fr, str):
        h = np.minimum(h, 10 + 3 * ilog2(hi - lo + 1))
    return m, M2, amean, has_inf, h


def expected(table, fn, perm, P, pe, ends):
    """(exact value, validity, tolerance, non-finite expected) of one moment function."""
    m, M2, amean, has_inf, h = exact_moments(table, fn[2], perm, frame_of(fn), P, pe, ends)
    pop = fn[1] in ("var_pop", "std_pop")
    valid = m >= (1 if pop else 2)
    div = np.maximum(m - (0 if pop else 1), 1).astype(np.float64)
    sh = np.sqrt(h.astype(np.float64))
    tol_m2 = sh * (np.array([gamma(21 * k) for k in h]) * M2 + np.array([gamma(8 * k) for k in h]) * amean * np.sqrt(m * M2))
    var, tv = M2 / div, tol_m2 / div
    tv = tv + U * (var + tv)
    if fn[1] in ("var", "var_pop"):
        return var, valid, tv, has_inf
    sd = np.sqrt(var)
    with np.errstate(divide="ignore", invalid="ignore"):
        ts = np.minimum(np.sqrt(tv), np.where(sd > 0, tv / np.where(sd > 0, sd, 1), np.inf))
    return sd, valid, ts + U * (sd + np.sqrt(tv)), has_inf


def check(table, part, order, funcs, **kw):
    part, order = list(part), list(order)
    perm, P, pe, ends = bounds(table, part, order, [True] * len(order), ["last"] * len(order))
    got, sizes = run(table, part, order, [True] * len(order), ["last"] * len(order), funcs, **kw)
    for c, (vals, mask, _) in zip(table.columns, got):
        np.testing.assert_array_equal(vals.view(np.uint8), c.values_numpy()[perm].view(np.uint8))
    for fn, (vals, mask, oc) in zip(funcs, got[table.n_cols:]):
        assert (oc.c_type, oc.arr_type) == (CTypes.FLOAT64, ArrTypes.NULLABLE_INT_BOOL), fn
        assert vals.dtype == np.float64, fn
        exact, valid, tol, nonfinite = expected(table, fn, perm, P, pe, ends)
        np.testing.assert_array_equal(mask, valid, err_msg=str(fn))
        nan_rows = valid & nonfinite
        assert np.isnan(vals[nan_rows]).all(), fn  # a frame holding +-inf gives a valid NaN
        ok = valid & ~nonfinite
        g = vals[ok]
        assert np.all(g >= 0), fn  # M2 is never negative (so std is never NaN for finite input)
        err = np.abs(g - exact[ok])
        bad = np.flatnonzero(~(err <= tol[ok]))
        assert bad.size == 0, (fn, g[bad[:5]], exact[ok][bad[:5]], tol[ok][bad[:5]])
    return got, sizes


def moment_funcs(col, frames):
    fs = []
    for j, fr in enumerate(frames):
        fs += [(f"{f}{j}", f, col, fr) for f in MOMENTS]
    return fs


ALL_FRAMES = list(CUMULATIVE) + [("rows", s, e) for s, e in BOUNDED]


# ---- every function x every frame x every value type ----
@pytest.mark.parametrize("ct", NUM_TYPES)
@pytest.mark.parametrize("nullable", [False, True])
def test_value_types(gpu_lib, ct, nullable):
    rng = np.random.default_rng(900 + ct * 2 + nullable)
    n = 1500
    x = float_values(ct, n, rng, nullable) if ct in (CTypes.FLOAT32, CTypes.FLOAT64) else make_column(ct, n, rng, nullable, small=False)
    t = Table([make_column(CTypes.INT8, n, rng, False), make_column(CTypes.INT16, n, rng, True, na_frac=0.1), x], ["g", "o", "x"])
    for chunk in in_states(moment_funcs("x", ALL_FRAMES), 3):
        check(t, ["g"], ["o"], chunk, sizes=(777,))


def test_few_cells_nan_inf_and_constants(gpu_lib):
    """Partitions of m = 0, 1, 2 valid cells, NaN counted as NA, +-inf giving NaN, constant values giving exactly 0.0."""
    nan, inf = np.nan, np.inf
    parts = [[nan, nan], [5.0], [nan, 2.5, nan], [1.0, 4.0], [3.0, inf, 1.0], [-inf, 2.0], [7.25] * 9, [-1e300] * 3,
             [0.1] * 50, [2.0, nan, 2.0, 2.0]]
    g = np.concatenate([np.full(len(p), k) for k, p in enumerate(parts)]).astype(np.int64)
    x = np.concatenate([np.array(p) for p in parts])
    n = len(x)
    t = Table([Column(g), Column(np.arange(n, dtype=np.int64)), Column(x)], ["g", "o", "x"])
    fs = moment_funcs("x", ["partition", "rows", ("rows", -1, 0), ("rows", -2, 2)])
    got, _ = check(t, ["g"], ["o"], fs)
    res = {fn[0]: got[3 + j] for j, fn in enumerate(fs)}
    off = np.cumsum([0] + [len(p) for p in parts])
    sl = {k: slice(off[k], off[k + 1]) for k in range(len(parts))}
    # m = 0: every function NA; m = 1: var / std NA, var_pop / std_pop 0.0
    for f in MOMENTS:
        assert not res[f"{f}0"][1][sl[0]].any()
    assert not res["var0"][1][sl[1]].any() and not res["std0"][1][sl[1]].any()
    assert res["var_pop0"][1][sl[1]].all() and (res["var_pop0"][0][sl[1]] == 0.0).all() and (res["std_pop0"][0][sl[1]] == 0.0).all()
    # NaN is NA: [nan, 2.5, nan] has m = 1
    assert not res["var0"][1][sl[2]].any() and (res["var_pop0"][0][sl[2]] == 0.0).all()
    # m = 2: [1, 4] has var 4.5 and var_pop 2.25 exactly
    assert (res["var0"][0][sl[3]] == 4.5).all() and (res["var_pop0"][0][sl[3]] == 2.25).all() and (res["std_pop0"][0][sl[3]] == 1.5).all()
    # +-inf: a valid NaN over the whole partition
    for k in (4, 5):
        for f in MOMENTS:
            assert res[f"{f}0"][1][sl[k]].all() and np.isnan(res[f"{f}0"][0][sl[k]]).all()
    # equal values: exactly 0.0 in every frame with enough cells
    for k in (6, 7, 8, 9):
        for j in range(4):
            for f in MOMENTS:
                vals, mask, _ = res[f"{f}{j}"]
                assert (vals[sl[k]][mask[sl[k]]] == 0.0).all(), (k, j, f)
                assert mask[sl[k]].sum() > 0


def test_catastrophic_cancellation(gpu_lib):
    """1.7e9 + U[0, 1000): var within 1e-6 of exact in every frame, where the sum-of-squares formula loses about 3 digits."""
    rng = np.random.default_rng(91)
    n = 6000
    x = 1.7e9 + rng.uniform(0, 1000, n)
    t = Table([Column(rng.integers(0, 3, n).astype(np.int64)), Column(rng.permutation(n).astype(np.int64)), Column(x)], ["g", "o", "x"])
    frames = ["range", "rows", "partition", ("rows", -19, 0), ("rows", -500, 500)]
    fs = [(f"v{j}", "var", "x", fr) for j, fr in enumerate(frames)]
    got, _ = check(t, ["g"], ["o"], fs)
    perm, P, pe, ends = bounds(t, ["g"], ["o"], [True], ["last"])
    for j, fr in enumerate(frames):
        m, M2, _, _, _ = exact_moments(t, "x", perm, fr, P, pe, ends)
        ok = m >= 2
        exact = M2[ok] / (m[ok] - 1)
        vals = got[3 + j][0][ok]
        assert np.all(np.abs(vals - exact) <= 1e-6 * exact), fr
        if fr == "partition":  # the one-pass formula in double fails the same check
            gs, xs = t.columns[0].values_numpy()[perm], x[perm]
            s1, s2, c = np.bincount(gs, xs), np.bincount(gs, xs * xs), np.bincount(gs)
            naive = ((s2 - s1 * s1 / c) / (c - 1))[gs][ok]
            assert np.any(np.abs(naive - exact) > 1e-6 * exact)


def test_excluded_outlier(gpu_lib):
    x = np.array([1e15, 1.0, 2.0, 3.0])
    t = Table([Column(np.zeros(4, np.int64)), Column(np.arange(4, dtype=np.int64)), Column(x)], ["g", "o", "x"])
    got, _ = run(t, ["g"], ["o"], [True], ["last"], [("v", "var", "x", ("rows", -1, 0)), ("s", "std_pop", "x", ("rows", -1, 0))])
    assert got[3][0][3] == 0.5 and got[3][0][2] == 0.5
    assert got[4][0][3] == math.sqrt(0.25)


@pytest.mark.parametrize("n", [2047, 2048, 2049])
def test_tile_edges(gpu_lib, n):
    rng = np.random.default_rng(n)
    i = np.arange(n)
    t = Table([Column((i // 1000).astype(np.int64)), Column((i // 3 % 7).astype(np.int64)),
               make_column(CTypes.INT32, n, rng, True, small=False), float_values(CTypes.FLOAT64, n, rng, True)], ["g", "o", "x", "f"])
    fs = moment_funcs("f", ["range", "rows", "partition", ("rows", -2047, 0), ("rows", -3, 2048)])
    fs += [(f"i{j}_{f}", f, "x", fr) for j, fr in enumerate(["rows", ("rows", -100, 100)]) for f in ("var", "std_pop")]
    for chunk in in_states(fs, 4):
        check(t, ["g"], ["o"], chunk, sizes=(TILE - 1, TILE, TILE + 1))


def test_large_input_against_torch(gpu_lib):
    """2^24 + a few tiles of device rows: var_pop / std over the partition and var over 9 PRECEDING against torch float64 two-pass
    computations."""
    n = CHUNK + 3 * TILE + 5
    dev = torch.device("cuda", 0)
    g = torch.Generator(device=dev).manual_seed(92)
    pk = torch.randint(0, 50, (n,), generator=g, device=dev, dtype=torch.int64)
    x = 1e4 + torch.randn(n, generator=g, device=dev, dtype=torch.float64)
    rid = torch.arange(n, device=dev, dtype=torch.int64)
    funcs = [("vp", "var_pop", "x", "partition"), ("sd", "std", "x", "partition"), ("v10", "var", "x", ("rows", -9, 0))]
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
    cnt = torch.bincount(sp, minlength=50).to(torch.float64)
    mean = torch.zeros(50, dtype=torch.float64, device=dev).index_add_(0, sp, sx) / cnt
    m2 = torch.zeros(50, dtype=torch.float64, device=dev).index_add_(0, sp, (sx - mean[sp]) ** 2)
    torch.testing.assert_close(got[3], (m2 / cnt)[sp], rtol=1e-9, atol=0)
    torch.testing.assert_close(got[4], torch.sqrt(m2 / (cnt - 1))[sp], rtol=1e-9, atol=0)
    i = torch.arange(n, device=dev, dtype=torch.int64)
    ps = torch.ones(n, dtype=torch.bool, device=dev)
    ps[1:] = torch.diff(sp) != 0
    P = torch.cummax(torch.where(ps, i, 0), 0).values
    j = i[:, None] - torch.arange(10, device=dev)[None, :]
    inside = j >= P[:, None]
    w = torch.where(inside, sx[j.clamp(min=0)], 0.0)
    c = inside.sum(1).to(torch.float64)
    mu = w.sum(1) / c
    v = torch.where(inside, (w - mu[:, None]) ** 2, 0.0).sum(1) / (c - 1)
    del j, inside, w
    ok = c >= 2
    assert torch.equal(torch.as_tensor(col_mask(out.columns[5]), device=dev), ok)
    torch.testing.assert_close(got[5][ok], v[ok], rtol=1e-8, atol=0)
    for k in (3, 4):
        assert out.columns[k].valid_mask_numpy().all()
    W.delete_window_state(st)


def test_determinism_across_batches(gpu_lib):
    rng = np.random.default_rng(93)
    n = 30_000
    t = Table([Column(rng.integers(0, 5, n).astype(np.int64)), Column(rng.integers(0, 50, n).astype(np.int64)),
               float_values(CTypes.FLOAT64, n, rng, True), make_column(CTypes.INT64, n, rng, True, small=False)], ["g", "o", "x", "y"])
    fs = [(f"{f}{c}{j}", f, c, fr) for c in ("x", "y") for f in ("var", "std_pop")
          for j, fr in enumerate(["range", "rows", "partition", ("rows", -6, 0), ("rows", -300, 300), ("rows", None, 77)])]
    ref, _ = run(t, ["g"], ["o"], [True], ["last"], fs)
    again, _ = run(t, ["g"], ["o"], [True], ["last"], fs)
    for sizes, dev in (((1000,), True), ((4096, 17), False), ((TILE,), True), ((1 << 30,), False)):
        got, _ = run(t, ["g"], ["o"], [True], ["last"], fs, sizes=sizes, device=dev)
        for a, b, c in zip(ref[4:], got[4:], again[4:]):
            np.testing.assert_array_equal(a[0].view(np.uint64), b[0].view(np.uint64))
            np.testing.assert_array_equal(a[0].view(np.uint64), c[0].view(np.uint64))
            np.testing.assert_array_equal(a[1], b[1])


def test_rows_sharing_a_frame_end_share_bits(gpu_lib):
    """Peers share their "range" frame and every row of a partition its "partition" frame: bit-identical results."""
    rng = np.random.default_rng(94)
    n = 20_000
    t = Table([Column(rng.integers(0, 7, n).astype(np.int64)), Column(rng.integers(0, 40, n).astype(np.int64)),
               float_values(CTypes.FLOAT64, n, rng, True)], ["g", "o", "x"])
    fs = [("r", "var", "x", "range"), ("p", "std", "x", "partition")]
    got, _ = run(t, ["g"], ["o"], [True], ["last"], fs)
    perm, P, pe, ends = bounds(t, ["g"], ["o"], [True], ["last"])
    for j, fr in enumerate(("range", "partition")):
        vals, mask, _ = got[3 + j]
        e = ends[fr]
        np.testing.assert_array_equal(vals.view(np.uint64), vals[e].view(np.uint64))
        np.testing.assert_array_equal(mask, mask[e])


def test_mixed_state_keeps_old_columns(gpu_lib):
    rng = np.random.default_rng(95)
    n = 10_000
    t = Table([make_column(CTypes.INT16, n, rng, True), make_column(CTypes.INT32, n, rng, True), float_values(CTypes.FLOAT64, n, rng, True)],
              ["g", "o", "x"])
    old = [("rn", "row_number"), ("s", "sum", "x", "rows"), ("lg", "lag", "x", 1, 0.0), ("ms", "sum", "x", ("rows", -3, 3)),
           ("mx", "max", "o", "range"), ("nv", "nth_value", "o", 2), ("mn", "min", "x", ("rows", -10, 0))]
    new = [("v", "var", "x", ("rows", -3, 3)), ("sd", "std", "x", "rows"), ("vp", "var_pop", "o", "partition"),
           ("sp", "std_pop", "x", ("rows", -10, 0))]
    alone, _ = run(t, ["g"], ["o"], [True], ["last"], old)
    mixed = [old[0], new[0], old[1], old[2], new[1], old[3], old[4], new[2], old[5], new[3], old[6]]
    got, _ = run(t, ["g"], ["o"], [True], ["last"], mixed)
    for j, f in enumerate(mixed):
        if f in old:
            a, b = alone[3 + old.index(f)], got[3 + j]
            np.testing.assert_array_equal(a[0].view(f"u{a[0].itemsize}"), b[0].view(f"u{b[0].itemsize}"), err_msg=f[0])
            np.testing.assert_array_equal(a[1], b[1])
    check(t, ["g"], ["o"], new)


# ---- pandas ----
@pytest.mark.parametrize("with_na", [False, True])
def test_pandas(gpu_lib, with_na):
    """expanding().var() / .std() for "rows", transform("var") / transform("std", ddof=0) for "partition", rolling(w,
    min_periods=...) trailing, centred and forward for bounded frames.  pandas skips NaN as the window skips NA; where pandas
    gives NaN (too few cells) the window gives NA, and the masks are compared explicitly.  pandas' add / remove rolling update
    can leave a residue of about 1e-6 (u times the squared mean 1e6) where a window's cells are all equal; the window gives
    exactly 0.0 there, so the absolute tolerance is 1e-5."""
    from bodo_b200.physical import window

    rng = np.random.default_rng(96 + with_na)
    n = 20_000
    f = rng.integers(-2000, 2000, n) / 8.0 + 1e6
    if with_na:
        f = np.where(rng.random(n) < 0.2, np.nan, f)
    df = pd.DataFrame({"p": rng.integers(0, 300, n), "o": rng.permutation(n), "f": f})
    funcs = [("ev", "var", "f", "rows"), ("es", "std", "f", "rows"), ("tv", "var", "f", "partition"), ("ts", "std_pop", "f", "partition"),
             ("r7", "var", "f", ("rows", -6, 0)), ("rs7", "std", "f", ("rows", -6, 0)), ("rp7", "var_pop", "f", ("rows", -6, 0)),
             ("c7", "std", "f", ("rows", -3, 3)), ("f10", "var", "f", ("rows", 0, 9))]
    got = window(df, "p", "o", funcs, batch_size=7000)
    srt = df.sort_values(["p", "o"], kind="stable").reset_index(drop=True)
    gb = srt.groupby("p", sort=False)["f"]

    def per_row(r):
        return r.reset_index(level=0, drop=True).sort_index()

    fwd = pd.api.indexers.FixedForwardWindowIndexer(window_size=10)
    exp = {"ev": per_row(gb.expanding(min_periods=1).var()), "es": per_row(gb.expanding(min_periods=1).std()),
           "tv": gb.transform("var"), "ts": gb.transform("std", ddof=0),
           "r7": per_row(gb.rolling(7, min_periods=1).var()), "rs7": per_row(gb.rolling(7, min_periods=1).std()),
           "rp7": per_row(gb.rolling(7, min_periods=1).var(ddof=0)), "c7": per_row(gb.rolling(7, center=True, min_periods=1).std()),
           "f10": per_row(gb.rolling(fwd, min_periods=1).var())}
    for k, e in exp.items():
        g = got[k].to_numpy(dtype=np.float64, na_value=np.nan)
        e = e.to_numpy(dtype=np.float64)
        np.testing.assert_array_equal(np.isnan(g), np.isnan(e), err_msg=k)
        np.testing.assert_allclose(g, e, rtol=1e-7, atol=1e-5, err_msg=k)
