"""The groupby's float-valued aggregates against an exact reference, through every path a float aggregate takes.

Reference (CPU, below): a group's values are turned into integers X_i = x_i * 2^-e (e = the smallest exponent among them), so
n, sum x, sum (x - mean)^2 and sum (x - mean)^3 are exact rationals, rounded to a double once at the end.  Integer value columns
enter as float64(value), the reference's conversion.  NaN is NA.

What each aggregate must satisfy (u = 2^-53, gamma_k = k u / (1 - k u)):
  * count, min, max, first, last: bit-exact, ±inf / subnormals / ±max-finite included.  Signed zero: the device keeps min / max
    in an ordered encoding (f64_to_ordered), in which -0.0 < +0.0, so min({-0.0, 0.0}) = -0.0 and max = +0.0 whatever order the
    rows come in (pandas returns whichever zero it saw first).
  * sum / mean of dyadic values k / 1024, |k| < 2^20: every partial sum is exact in any order, so the sum is bit-exact (float32:
    float32(exact)) and the mean is exact_sum / n rounded once.
  * sum / mean with cancellation: |got - exact| <= gamma_{n-1} sum|x| (recursive summation in any order, or any summation tree:
    its depth is at most n - 1); the mean adds that bound / n and one rounding.
  * var / std / var_pop / std_pop / skew: the device accumulates S_k = sum d^k of d = x - c about a per-group shift c (one of the
    group's values) and forms M2 = S2 - S1^2 / n, M3 = S3 - 3 S2 S1 / n + 2 S1^3 / n^2.  With e_i = x_i - c, R = max|x_i - mean|,
    sigma^2 = M2 / n: |mean - c| <= R and |e_i| <= 2 R.  Each S_k is a sum of n terms whose own error is a few u, so
    |dS1| <~ (n + 1) u sum|e|, |dS2| <~ (n + 3) u sum e^2, |dS3| <~ (n + 4) u sum|e|^3; with (sum|e|)^2 <= n sum e^2 and
    sum e^2 sum|e| <= n sum|e|^3 the terms S1^2 / n and S2 S1 / n, S1^3 / n^2 carry errors of the same order, so
        |dM2| <~ 3 (n + 4) u sum e^2 = 3 (n + 4) u M2 (1 + (mean - c)^2 / sigma^2),
        |dM3| <~ 13 (n + 4) u sum|e|^3 <= 13 (n + 4) u n (rho sigma)^3,           rho = 2 R / sigma.
    The exchange re-centres partials by delta = c_s - c_t (|delta| <= 2 R, rounded once); its extra terms are O(u n R^2) in M2 and
    O(u n R^3) in M3, inside the same bounds.  Hence, stated with headroom:
        var, var_pop (and std, std_pop, whose relative error is half that plus one rounding):
            |got - exact| <= 8 (n + 4) u (1 + R^2 / sigma^2) |exact|
        skew = K M3 / M2^1.5 with K = n sqrt(n - 1) / (n - 2) <= 3 sqrt(n), so K sum|e|^3 / M2^1.5 <= 3 rho^3 and
            |got - exact| <= 40 (n + 4) u rho^2 (rho + |skew|).
    Neither grows with |mean| / spread.  The old power sums about 0 lost 2 log10(|mean| / spread) digits instead: var of
    1e5 + N(0, 1) was off by ~4e-5 relative and skew by O(1).

Every check runs through every path a float aggregate can take: host batches, device batches, 32 768-row batches, a table that
starts at expected_groups=8 (fail list, replay, rehash_kernel), 3-column keys (groupby_consume_mk_kernel), dropna=False with the NA
key and the key INT64_MIN (the special slots cap and cap + 1), and the sharded exchange (fused and NCCL forms, 2 and 3 ranks).
The single-state paths assert they stay on the direct path (metrics 8, 10, 12, 14 stay 0)."""

import functools
import math
from fractions import Fraction

import numpy as np
import pandas as pd
import pytest

U = 2.0 ** -53
INT64_MIN = np.iinfo(np.int64).min
PATHS = ["host", "device", "batch32k", "grow", "multikey", "special_slots", "fused-2", "fused-3", "nccl-2", "nccl-3"]


def gamma(k):
    k = np.asarray(k, dtype=np.float64)
    return k * U / (1 - k * U)


# ---- exact reference ---------------------------------------------------------------------------------------------------

def _scaled_ints(v):
    """finite float64 values -> (Python ints X, e) with v_i = X_i * 2^e exactly"""
    m, ex = np.frexp(v)
    mi = np.ldexp(m, 53).astype(np.int64)
    ex = ex.astype(np.int64) - 53
    e = int(ex.min())
    return [int(a) << int(s) for a, s in zip(mi.tolist(), (ex - e).tolist())], e


def _q(num, den, e2):
    """num / den * 2^e2, rounded once"""
    return float(Fraction(num, den) * Fraction(2) ** e2)


def exact_moments(vals):
    """The reference aggregates of one group's values (NaN = NA), with the NA / NaN rules of eval_output_kernel.  Returns a dict:
    n, sum, abs_sum, mean, var, var_pop, std, std_pop, skew (None = NA), and m2, r (max |x - mean|) for the error bounds."""
    v = np.asarray(vals, dtype=np.float64)
    v = v[~np.isnan(v)]
    n = len(v)
    out = dict(n=n, sum=0.0, abs_sum=0.0, mean=None, var=None, var_pop=None, std=None, std_pop=None, skew=None, m2=0.0, r=0.0)
    if n == 0:
        return out
    if not np.isfinite(v).all():  # ±inf: IEEE sums, NaN moments
        with np.errstate(invalid="ignore"):
            s = float(np.sum(v))
        out.update(sum=s, abs_sum=math.inf, mean=s / n, var_pop=math.nan, std_pop=math.nan, m2=math.nan)
        if n >= 2:
            out.update(var=math.nan, std=math.nan)
        if n >= 3:
            out["skew"] = math.nan
        return out
    X, e = _scaled_ints(v)
    Xo = np.array(X, dtype=object)
    S, Q, C = int(Xo.sum()), int((Xo * Xo).sum()), int((Xo * Xo * Xo).sum())
    A = int(np.abs(Xo).sum())
    num2 = n * Q - S * S                       # n M2 / 2^2e
    num3 = n * n * C - 3 * n * S * Q + 2 * S ** 3  # n^2 M3 / 2^3e
    out.update(sum=_q(S, 1, e), abs_sum=_q(A, 1, e), mean=_q(S, n, e), var_pop=_q(num2, n * n, 2 * e), m2=_q(num2, n, 2 * e))
    out["std_pop"] = math.sqrt(out["var_pop"])
    out["r"] = _q(max(abs(n * max(X) - S), abs(n * min(X) - S)), n, e)
    if n >= 2:
        out["var"] = _q(num2, n * (n - 1), 2 * e)
        out["std"] = math.sqrt(out["var"])
    if n >= 3:
        m2, m3 = out["m2"], _q(num3, n * n, 3 * e)
        den = m2 ** 1.5
        if m3 == 0.0 or abs(den) < 1e-14 or math.log2(abs(den)) - math.log2(abs(m3)) < -20:
            out["skew"] = 0.0
        else:
            out["skew"] = n * math.sqrt(n - 1) / (n - 2) * m3 / den
    return out


def var_tol(ref):
    """relative bound of var / var_pop / std / std_pop (module docstring)"""
    n, m2, r = ref["n"], ref["m2"], ref["r"]
    if not (m2 > 0):
        return 0.0
    return 8 * (n + 4) * U * (1 + r * r / (m2 / n))


def skew_tol(ref):
    """absolute bound of skew (module docstring)"""
    n, m2, r = ref["n"], ref["m2"], ref["r"]
    if not (m2 > 0):
        return 0.0
    rho = 2 * r / math.sqrt(m2 / n)
    return 40 * (n + 4) * U * rho * rho * (rho + abs(ref["skew"]))


def _groups(gid, G):
    order = np.argsort(gid, kind="stable")
    bounds = np.searchsorted(gid[order], np.arange(G + 1))
    return [order[bounds[g]:bounds[g + 1]] for g in range(G)]


def _total_order(v):
    """float64 -> int64 keys in IEEE total order (-0.0 < +0.0), the order of the device's f64_to_ordered"""
    b = np.asarray(v, dtype=np.float64).view(np.int64)
    return np.where(b < 0, b ^ np.int64(0x7FFFFFFFFFFFFFFF), b)


# ---- the reference pinned on the CPU ----------------------------------------------------------------------------------

def test_reference_hand_computed():
    r = exact_moments([1.0, 2.0, 3.0, 4.0])  # mean 5/2, M2 = 5, M3 = 0
    assert (r["n"], r["sum"], r["mean"], r["var"], r["var_pop"], r["skew"]) == (4, 10.0, 2.5, 5 / 3, 1.25, 0.0)
    assert r["std"] == math.sqrt(5 / 3) and r["r"] == 1.5
    r = exact_moments([1.0, 2.0, 10.0])  # mean 13/3, M2 = 438/9, M3 = 3570/27
    assert r["var"] == 73 / 3 and r["var_pop"] == float(Fraction(146, 9))
    assert r["skew"] == pytest.approx(3 * math.sqrt(2) * (3570 / 27) / (438 / 9) ** 1.5, rel=1e-15)
    # exact where naive float64 is not: 1e16 + 1 - 1e16 + 1 = 2 (the float64 sum in this order is 1, pandas' Kahan sum too)
    r = exact_moments([1e16, 1.0, -1e16, 1.0])
    assert r["sum"] == 2.0 and r["mean"] == 0.5 and r["abs_sum"] == 2e16 + 2
    assert exact_moments([0.1, 0.2, 0.3])["sum"] == float(Fraction(0.1) + Fraction(0.2) + Fraction(0.3))
    # a large common offset costs nothing: 1e9 + {0, 1, 2} has var 1 and skew 0 exactly; every value equal gives 0
    r = exact_moments([1e9 + 2, 1e9, 1e9 + 1])
    assert (r["var"], r["var_pop"], r["skew"]) == (1.0, 2 / 3, 0.0)
    r = exact_moments([1e9] * 50)
    assert (r["var"], r["std"], r["var_pop"], r["skew"]) == (0.0, 0.0, 0.0, 0.0)
    # NA rules (eval_output_kernel): var / std need 2 values, var_pop / std_pop 1, skew 3; NaN is NA; ±inf makes the moments NaN
    r = exact_moments([np.nan, 4.0, np.nan])
    assert (r["n"], r["mean"], r["var"], r["var_pop"], r["skew"]) == (1, 4.0, None, 0.0, None)
    r = exact_moments([1.0, 3.0])
    assert (r["var"], r["skew"]) == (2.0, None)
    r = exact_moments([np.nan, np.nan])
    assert (r["n"], r["mean"], r["var_pop"]) == (0, None, None)
    r = exact_moments([1.0, 2.0, np.inf, 3.0])
    assert r["mean"] == np.inf and all(math.isnan(r[k]) for k in ("var", "std", "var_pop", "std_pop", "skew"))
    r = exact_moments([-np.inf, 5.0, np.inf])
    assert math.isnan(r["mean"]) and math.isnan(r["skew"])
    # subnormals are exact too
    assert exact_moments([5e-324, 5e-324, 1.0])["sum"] == 1.0 and exact_moments([5e-324, 5e-324])["sum"] == 1e-323


def test_reference_against_pandas():
    """Well-conditioned data (offset <= 10), where pandas' Welford / moment code agrees with the exact values to ~1e-12."""
    rng = np.random.default_rng(5)
    n, G = 20_000, 37
    gid = rng.integers(0, G, n)
    x = rng.standard_normal(n) * rng.choice([0.5, 3.0], n) + rng.choice([0.0, 1.0, 10.0], G)[gid]
    refs = [exact_moments(x[ix]) for ix in _groups(gid, G)]
    g = pd.DataFrame({"g": gid, "x": x}).groupby("g").x
    for name, exp in (("sum", g.sum()), ("mean", g.mean()), ("var", g.var()), ("std", g.std()), ("var_pop", g.var(ddof=0)),
                      ("std_pop", g.std(ddof=0)), ("skew", g.skew())):
        np.testing.assert_allclose([r[name] for r in refs], exp.to_numpy(), rtol=1e-12, atol=1e-12, err_msg=name)


# ---- running a path ---------------------------------------------------------------------------------------------------

def _key_frame(gid, path):
    """key columns that put group g where the path wants it (multikey: 3 columns; special_slots: g 0 = NA key, g 1 = INT64_MIN)"""
    if path == "multikey":
        return {"k0": gid // 64, "k1": ((gid // 8) % 8).astype(np.int32), "k2": gid % 8}
    if path == "special_slots":
        k = np.where(gid == 1, INT64_MIN, gid).astype(np.int64)
        return {"k": pd.arrays.IntegerArray(k, gid == 0)}
    return {"k": gid.astype(np.int64)}


def _gid_of(out, nk, path):
    if path == "multikey":
        k = [out.iloc[:, j].to_numpy(dtype=np.int64) for j in range(3)]
        return k[0] * 64 + k[1] * 8 + k[2]
    if path == "special_slots":
        kc = out.iloc[:, 0]
        g = kc.to_numpy(dtype=np.int64, na_value=0)
        return np.where(kc.isna().to_numpy(), 0, np.where(g == INT64_MIN, 1, g))
    return out.iloc[:, 0].to_numpy(dtype=np.int64)


def _values_and_na(s):
    a = s.array
    if isinstance(a, (pd.arrays.FloatingArray, pd.arrays.IntegerArray)):
        return np.asarray(a._data), np.asarray(a._mask)
    return s.to_numpy(), np.zeros(len(s), dtype=bool)


def run_path(path, gid, G, values: dict, fn, cols):
    """Runs fn over the value columns `cols` (names in `values`) grouped by gid along `path`; returns per function (values, NA mask)
    in group order."""
    from bodo_b200.streaming.groupby import (delete_groupby_state, get_metric, groupby_build_consume_batch,
                                             groupby_produce_output_batch, init_groupby_state)
    from bodo_b200.table import Table
    from tests.helpers import table_to_device

    keys = _key_frame(gid, path)
    nk = len(keys)
    df = pd.DataFrame({**keys, **values})
    names = list(df.columns)
    phys = tuple(names.index(c) for c in cols)
    if path.startswith(("fused", "nccl")):
        from tests.test_gpu_groupby_exchange import _run, _states
        transport, R = path.split("-")
        outs, _ = _run(_states(df, nk, fn, phys, int(R)), transport)
        out = pd.concat(outs, ignore_index=True)
    else:
        batch, on_device, expected = {"host": (7_001, False, 0), "device": (100_003, True, 0), "batch32k": (32_768, True, 0),
                                      "grow": (50_000, None, 8), "multikey": (40_009, None, 0),
                                      "special_slots": (60_000, None, 0)}[path]
        st = init_groupby_state(-1, tuple(range(nk)), fn, tuple(range(len(fn) + 1)), phys, dropna=path != "special_slots",
                                expected_groups=expected, output_batch_size=1 << 30)
        t = Table.from_pandas(df)
        n = t.n_rows
        for i, r0 in enumerate(range(0, n, batch)):
            b = t.slice(r0, min(n, r0 + batch))
            dev = on_device if on_device is not None else i % 2 == 0  # None: device and host batches alternate
            groupby_build_consume_batch(st, table_to_device(b) if dev else b, r0 + batch >= n, True)
        out, last = groupby_produce_output_batch(st, True)
        assert last
        out = out.to_pandas()
        m = {w: get_metric(st, w) for w in (3, 8, 10, 12, 14)}
        delete_groupby_state(st)
        assert m[8] == m[10] == m[12] == m[14] == 0, m  # the direct path, not an SM-partitioned / low-cardinality kernel
        if expected:
            assert m[3] > 0, m  # the table grew: rows went through the fail list, the replay and rehash_kernel
    g = _gid_of(out, nk, path)
    order = np.argsort(g)
    np.testing.assert_array_equal(g[order], np.arange(G))
    return [_values_and_na(out.iloc[order, nk + j].reset_index(drop=True)) for j in range(len(fn))]


# ---- count / min / max / first / last: bit-exact ----------------------------------------------------------------------

POOL64 = np.array([np.inf, -np.inf, -0.0, 0.0, 5e-324, -5e-324, np.finfo(np.float64).max, -np.finfo(np.float64).max,
                   2.2250738585072014e-308, 1.0, -2.5, 1e-300, np.nan, np.nan])
POOL32 = np.array([np.inf, -np.inf, -0.0, 0.0, 1e-45, -1e-45, np.finfo(np.float32).max, -np.finfo(np.float32).max,
                   np.finfo(np.float32).tiny, 1.5, -3.0, np.nan], dtype=np.float32)


@functools.lru_cache(maxsize=None)
def _extremes_data():
    rng = np.random.default_rng(71)
    G, n = 300, 60_000
    gid = rng.integers(0, G, n)
    # each group draws from 3 entries of the pools, so min / max / first / last land on every special value, and some groups are
    # all NaN
    p64, p32 = rng.integers(0, len(POOL64), (G, 3)), rng.integers(0, len(POOL32), (G, 3))
    pick = rng.integers(0, 3, n)
    x64, x32 = POOL64[p64[gid, pick]], POOL32[p32[gid, pick]]
    # groups 0 and 1 hold only zeros, +0.0 first in group 0 and -0.0 first in group 1 (rows are in order on every path)
    z0, z1 = np.flatnonzero(gid == 0), np.flatnonzero(gid == 1)
    x64[z0], x64[z1] = np.where(np.arange(len(z0)) % 2 == 0, 0.0, -0.0), np.where(np.arange(len(z1)) % 2 == 0, -0.0, 0.0)
    x32[z0], x32[z1] = x64[z0], x64[z1]
    return gid, G, x64, x32


def _expect_extremes(gid, G, x):
    cnt, mn, mx, first, last = np.zeros(G, np.int64), np.full(G, np.nan), np.full(G, np.nan), np.full(G, np.nan), np.full(G, np.nan)
    for g, ix in enumerate(_groups(gid, G)):
        v = x[ix].astype(np.float64)
        v = v[~np.isnan(v)]
        cnt[g] = len(v)
        if len(v):
            key = _total_order(v)
            mn[g], mx[g], first[g], last[g] = v[np.argmin(key)], v[np.argmax(key)], v[0], v[-1]
    return {"count": cnt, "min": mn, "max": mx, "first": first, "last": last}


def _assert_bits(got, exp, what):
    got = np.asarray(got)
    exp = exp.astype(got.dtype)
    nan = np.isnan(exp)
    assert (np.isnan(got) == nan).all(), (what, np.flatnonzero(np.isnan(got) != nan)[:5])
    bits = got.view(np.int64 if got.dtype == np.float64 else np.int32), exp.view(np.int64 if got.dtype == np.float64 else np.int32)
    bad = np.flatnonzero((bits[0] != bits[1]) & ~nan)
    assert len(bad) == 0, (what, bad[:5], got[bad[:5]], exp[bad[:5]])


@pytest.mark.gpu
@pytest.mark.parametrize("path", PATHS)
def test_count_min_max_first_last_bit_exact(gpu_lib, path):
    gid, G, x64, x32 = _extremes_data()
    fn = ("count", "min", "max", "first", "last", "min", "max", "first", "last")
    cols = ("x64",) * 5 + ("x32",) * 4
    if path == "multikey":  # first / last take single-column keys
        fn, cols = ("count", "min", "max", "min", "max"), ("x64",) * 3 + ("x32",) * 2
    got = run_path(path, gid, G, {"x64": x64, "x32": x32}, fn, cols)
    exp = {"x64": _expect_extremes(gid, G, x64), "x32": _expect_extremes(gid, G, x32)}
    for (vals, na), f, c in zip(got, fn, cols):
        if f == "count":
            np.testing.assert_array_equal(vals, exp[c]["count"])
            continue
        assert vals.dtype == (np.float64 if c == "x64" else np.float32), (f, c, vals.dtype)
        assert not na.any()  # numpy input: a group without values gives NaN, not NA
        _assert_bits(vals, exp[c][f], (f, c))
    # the device's signed-zero rule, stated explicitly: min({-0.0, +0.0}) = -0.0 and max = +0.0 in either row order
    for (vals, _), f in zip(got, fn):
        if f in ("min", "max"):
            assert vals[0] == 0 and vals[1] == 0
            assert (np.signbit(vals[:2]) == (f == "min")).all(), (f, vals[:2])
        if f == "first":  # (first / last keep the bits of the row: pandas' rule)
            assert list(np.signbit(vals[:2])) == [False, True]


# ---- sum / mean -------------------------------------------------------------------------------------------------------

CANCEL = np.array([1e16, -1e16, 1.0, 1.0, 3.0, -7e15, 7e15, 0.1, 2.5e-3, -1e-3])


@functools.lru_cache(maxsize=None)
def _sum_data():
    rng = np.random.default_rng(72)
    G, n = 257, 200_000
    gid = rng.integers(0, G, n)
    k = rng.integers(-(2 ** 20) + 1, 2 ** 20, n)
    dy64 = k / 1024.0
    dy64[rng.random(n) < 0.03] = np.nan  # NA rows are skipped
    dy32 = (k / 1024.0).astype(np.float32)
    c = CANCEL[rng.integers(0, len(CANCEL), n)]
    g2 = np.flatnonzero(gid == 2)[:4]  # group 2 starts with 1e16, 1, -1e16, 1 (exact sum 2, pandas' Kahan sum 1)
    c[np.flatnonzero(gid == 2)] = 0.0
    c[g2] = [1e16, 1.0, -1e16, 1.0]
    return gid, G, k, dy64, dy32, c


@pytest.mark.gpu
@pytest.mark.parametrize("path", PATHS)
def test_sum_mean_dyadic_exact_and_cancellation_bounded(gpu_lib, path):
    gid, G, k, dy64, dy32, c = _sum_data()
    fn, cols = ("sum", "mean", "sum", "mean", "sum", "mean"), ("dy64", "dy64", "dy32", "dy32", "c", "c")
    got = run_path(path, gid, G, {"dy64": dy64, "dy32": dy32, "c": c}, fn, cols)
    # dyadic: exact integer sums of k
    ok64 = ~np.isnan(dy64)
    ks64, n64 = np.zeros(G, np.int64), np.bincount(gid[ok64], minlength=G)
    np.add.at(ks64, gid[ok64], k[ok64])
    ks32 = np.zeros(G, np.int64)
    np.add.at(ks32, gid, k)
    n32 = np.bincount(gid, minlength=G)
    s64, s32 = ks64 / 1024.0, ks32 / 1024.0
    (g_s64, na_s64), (g_m64, na_m64), (g_s32, na_s32), (g_m32, na_m32) = got[:4]
    assert g_s32.dtype == np.float32 and not (na_s64.any() or na_s32.any() or na_m64.any() or na_m32.any())
    _assert_bits(g_s64, s64, "sum float64")
    _assert_bits(g_m64, s64 / n64, "mean float64")
    _assert_bits(g_s32, s32.astype(np.float32), "sum float32")
    _assert_bits(g_m32, s32 / n32, "mean float32")
    # cancellation: any summation order
    refs = [exact_moments(c[ix]) for ix in _groups(gid, G)]
    n = np.array([r["n"] for r in refs])
    exact, abs_sum = np.array([r["sum"] for r in refs]), np.array([r["abs_sum"] for r in refs])
    (g_sc, _), (g_mc, _) = got[4:]
    bound = gamma(n - 1) * abs_sum
    assert (np.abs(g_sc - exact) <= bound).all(), np.max(np.abs(g_sc - exact) / bound)
    mean = np.array([r["mean"] for r in refs])
    assert (np.abs(g_mc - mean) <= bound / n * (1 + U) + U * np.abs(mean)).all()


# ---- var / std / var_pop / std_pop / skew -----------------------------------------------------------------------------

OFFSETS = [0.0, 1e3, 1e5, 1e6, 1e9, 1.7e9, 1e12]
SIZES = [3, 4, 7, 31, 1000, 100_000]


@functools.lru_cache(maxsize=None)
def _moment_data():
    rng = np.random.default_rng(73)
    gx, gi = [], []
    for o in OFFSETS:  # spread 1 about the offset; the int column: int64 offset + integers in [-1000, 1000)
        for s in SIZES:
            x = o + rng.standard_normal(s)
            x[rng.random(s) < 0.01] = np.nan
            gx.append(x)
            gi.append(np.int64(o) + rng.integers(-1000, 1000, s))
    special = [np.full(50, 1e9), np.array([1.0, 2.0, np.inf, 3.0]), np.array([-np.inf, 5.0, np.inf, 7.0]), np.full(3, np.inf),
               np.full(3, np.nan), np.array([4.0]), np.array([1.0, 3.0]), np.array([2.0, np.nan, 3.0])]
    gx += special
    gi += [np.full(len(s), 1_000_000_000, np.int64) if j == 0 else rng.integers(-5, 5, len(s)) for j, s in enumerate(special)]
    G = len(gx)
    gid = np.concatenate([np.full(len(x), g) for g, x in enumerate(gx)])
    x, i = np.concatenate(gx), np.concatenate(gi)
    perm = rng.permutation(len(gid))  # rows of all groups interleave: which row sets a group's shift varies
    gid, x, i = gid[perm], x[perm], i[perm]
    groups = _groups(gid, G)
    return gid, G, x, i, [exact_moments(x[ix]) for ix in groups], [exact_moments(i[ix].astype(np.float64)) for ix in groups]


def _check_moment(got, na, refs, name, what):
    for g, r in enumerate(refs):
        e = r[name]
        ctx = (what, name, g, r["n"], got[g], e)
        if e is None:
            assert na[g], ctx
            continue
        assert not na[g], ctx
        if not math.isfinite(e):
            assert got[g] == e or (math.isnan(e) and math.isnan(got[g])), ctx
        elif name == "mean":
            b = gamma(r["n"] - 1) * r["abs_sum"] / r["n"] * (1 + U) + U * abs(e)
            assert abs(got[g] - e) <= b, ctx + (b,)
        elif name == "skew":
            assert abs(got[g] - e) <= skew_tol(r), ctx + (skew_tol(r),)
        else:
            assert abs(got[g] - e) <= var_tol(r) * abs(e), ctx + (var_tol(r),)


@pytest.mark.gpu
@pytest.mark.parametrize("path", PATHS)
def test_var_std_skew_against_exact_moments(gpu_lib, path):
    gid, G, x, i, rx, ri = _moment_data()
    fn = ("var", "std", "var_pop", "std_pop", "skew", "mean", "count", "var", "std", "skew")
    cols = ("x",) * 7 + ("i",) * 3
    got = run_path(path, gid, G, {"x": x, "i": i}, fn, cols)
    for (vals, na), f, c in zip(got, fn, cols):
        refs = rx if c == "x" else ri
        if f == "count":
            np.testing.assert_array_equal(vals, [r["n"] for r in refs])
        else:
            _check_moment(vals, na, refs, f, c)
    # every value equal at offset 1e9: exactly 0 (group 0 of the special groups, in both columns)
    g0 = len(OFFSETS) * len(SIZES)
    for (vals, _), f in zip(got, fn):
        if f in ("var", "std", "var_pop", "std_pop", "skew"):
            assert vals[g0] == 0.0, f
