"""prod, kurtosis, the boolean and bitwise aggregates and count_if on the CPU: their function numbers, the Python-side argument
errors, and two references for kurtosis that tests/test_gpu_groupby_reductions.py checks the device against.

  * `kurt_update` / `kurt_combine` / `kurt_eval` restate the device's kurtosis in the groupby's update -> combine -> eval shape:
    power sums S1..S4 of d = x - c about a per-group shift c (the group's first value), partials re-centred by the binomial
    expansion when they combine, and pandas' nankurt on the central moments M2 = S2 - S1^2 / n,
    M4 = S4 - 4 S3 S1 / n + 6 S2 S1^2 / n^2 - 3 S1^4 / n^3.  Pinned against pandas `Series.kurt`.
  * `exact_kurt` computes the same statistic from exact rational moments, rounded once, and `kurt_tol` bounds the device's error
    against it (derived below), in the manner of tests/test_gpu_groupby_float_values.py's skew bound.

Error bound.  With e_i = x_i - c, R = max |x_i - mean|, sigma^2 = M2 / n and rho = 2 R / sigma: |e_i| <= 2 R, each S_k is a sum of
n terms of a few roundings each, so |dS_k| <~ (n + 4) u sum |e|^k; the four terms of M4 are each at most sum e^4 in size (power
means), so |dM4| <~ 20 (n + 4) u sum e^4 <= 20 (n + 4) u n rho^4 sigma^4, and |dM2| <~ 3 (n + 4) u M2 (1 + rho^2).  kurtosis =
q n M4 / M2^2 - a with q = (n + 1)(n - 1) / ((n - 2)(n - 3)) and a = 3 (n - 1)^2 / ((n - 2)(n - 3)), so
    |got - exact| <~ 20 (n + 4) u q rho^4 + 6 (n + 4) u (1 + rho^2) (|exact| + a);
the test allows 4 times that.  It does not grow with |mean| / spread: power sums about 0 lose 4 log10(|mean| / spread) digits."""

import math
from fractions import Fraction

import numpy as np
import pandas as pd
import pytest

from bodo_b200 import _lib
from bodo_b200.streaming.groupby import FTYPES, init_groupby_state

from .test_gpu_groupby_float_values import _scaled_ints

U = 2.0 ** -53
NEW = {"prod": 17, "kurtosis": 26, "boolor_agg": 28, "booland_agg": 29, "boolxor_agg": 30, "bitor_agg": 31, "bitand_agg": 32,
       "bitxor_agg": 33, "count_if": 34}


# ---- the device's algorithm, restated ----------------------------------------------------------------------------------

def kurt_update(vals):
    """One partial: (n, c, S1, S2, S3, S4) of the non-NaN values of `vals` in row order, c = the first of them (None: no value)."""
    v = [float(x) for x in vals if not math.isnan(x)]
    if not v:
        return (0, None, 0.0, 0.0, 0.0, 0.0)
    c = v[0]
    d = [x - c for x in v]
    return (len(v), c, sum(d), sum(x * x for x in d), sum(x * x * x for x in d), sum((x * x) * (x * x) for x in d))


def kurt_combine(t, s):
    """Partial s merged into t: s's sums re-centred on t's shift (delta = c_s - c_t), as combine_apply does."""
    if s[1] is None:
        return t
    if t[1] is None:
        return s
    n, c, t1, t2, t3, t4 = t
    m, cs, s1, s2, s3, s4 = s
    dl = cs - c
    return (n + m, c, t1 + s1 + m * dl, t2 + s2 + 2 * dl * s1 + m * dl * dl, t3 + s3 + 3 * dl * s2 + 3 * dl * dl * s1 + m * dl ** 3,
            t4 + s4 + 4 * dl * s3 + 6 * dl * dl * s2 + 4 * dl ** 3 * s1 + m * dl ** 4)


def kurt_eval(st):
    """pandas' nankurt on the shifted power sums; None for NA (fewer than 4 values)."""
    n, _, s1, s2, s3, s4 = st
    if n < 4:
        return None
    if not all(math.isfinite(x) for x in (s1, s2, s3, s4)):
        return math.nan
    mean = s1 / n
    m2 = s2 - s1 * mean
    m4 = s4 - 4.0 * s3 * mean + 6.0 * s2 * mean * mean - 3.0 * s1 * mean * mean * mean
    num, den = n * (n + 1.0) * (n - 1.0) * m4, (n - 2.0) * (n - 3.0) * m2 * m2
    num, den = (0.0 if abs(num) < 1e-14 else num), (0.0 if abs(den) < 1e-14 else den)
    return 0.0 if den == 0.0 else num / den - 3.0 * (n - 1.0) ** 2 / ((n - 2.0) * (n - 3.0))


def kurt_batches(vals, batch):
    st = (0, None, 0.0, 0.0, 0.0, 0.0)
    for r0 in range(0, len(vals), batch):
        st = kurt_combine(st, kurt_update(vals[r0:r0 + batch]))
    return kurt_eval(st)


# ---- exact reference ----------------------------------------------------------------------------------------------------

def exact_kurt(vals):
    """(kurtosis from exact rational moments rounded once, None for NA, with nankurt's rules; n; M2; R = max |x - mean|).  The values
    are scaled to integers X_i = x_i 2^-e, so n^3 M4 2^-4e = n^3 sum X^4 - 4 n^2 S sum X^3 + 6 n S^2 sum X^2 - 3 S^4 (S = sum X) and
    n M2 2^-2e = n sum X^2 - S^2 are exact integers."""
    v = np.asarray(vals, dtype=np.float64)
    v = v[~np.isnan(v)]
    n = len(v)
    if n < 4:
        return None, n, 0.0, 0.0
    if not np.isfinite(v).all():
        return math.nan, n, math.nan, math.nan
    X, e = _scaled_ints(v)
    Xo = np.array(X, dtype=object)
    X2 = Xo * Xo
    S, Q, C, F = int(Xo.sum()), int(X2.sum()), int((X2 * Xo).sum()), int((X2 * X2).sum())
    num2 = n * Q - S * S
    num4 = n ** 3 * F - 4 * n * n * S * C + 6 * n * S * S * Q - 3 * S ** 4
    m2, m4 = Fraction(num2, n) * Fraction(2) ** (2 * e), Fraction(num4, n ** 3) * Fraction(2) ** (4 * e)
    num, den = n * (n + 1) * (n - 1) * m4, (n - 2) * (n - 3) * m2 * m2
    num, den = (0 if abs(num) < Fraction(1e-14) else num), (0 if abs(den) < Fraction(1e-14) else den)
    k = 0.0 if den == 0 else float(num / den - Fraction(3 * (n - 1) ** 2, (n - 2) * (n - 3)))
    r = Fraction(max(abs(n * max(X) - S), abs(n * min(X) - S)), n) * Fraction(2) ** e
    return k, n, float(m2), float(r)


def kurt_tol(k, n, m2, r):
    """absolute bound of the device's kurtosis against exact_kurt (module docstring)"""
    if not (m2 > 0):
        return 0.0
    rho = 2 * r / math.sqrt(m2 / n)
    qn = (n + 1) * (n - 1) / ((n - 2) * (n - 3))
    a = 3 * (n - 1) ** 2 / ((n - 2) * (n - 3))
    return 4 * (n + 4) * U * (20 * qn * rho ** 4 + 6 * (1 + rho * rho) * (abs(k) + a))


# ---- tests --------------------------------------------------------------------------------------------------------------

def test_function_numbers():
    for name, num in NEW.items():
        assert FTYPES[name] == num, name
    assert len(set(FTYPES.values())) == len(FTYPES)
    # the neighbours that fix 17 and 26
    assert (FTYPES["max"], FTYPES["first"], FTYPES["std"], FTYPES["skew"]) == (16, 18, 25, 27)
    # no pandas aliases: any / all return False for an all-NA group, which is not boolor_agg's / booland_agg's NA
    for alias in ("any", "all", "kurt", "product", "median"):
        assert alias not in FTYPES


@pytest.mark.parametrize("name", ["any", "all", "kurt", "product", "BOOLOR_AGG", "bit_or"])
def test_aliases_are_unsupported(name):
    with pytest.raises(_lib.B200Error, match=f"unsupported aggregate function '{name}'"):
        init_groupby_state(-1, (0,), (name,), (0, 1), (1,))


def test_new_names_take_the_usual_arguments():
    st = init_groupby_state(-1, (0,), tuple(NEW), tuple(range(len(NEW) + 1)), (1,) * len(NEW))
    assert st.fnames == tuple(NEW) and st.handle is None  # (the C state is created at the first batch)
    with pytest.raises(_lib.B200Error, match="f_in_offsets must have len"):
        init_groupby_state(-1, (0,), ("prod", "count_if"), (0, 1), (1,))
    with pytest.raises(_lib.B200Error, match="min_row_number_filter cannot be combined"):
        init_groupby_state(-1, (0,), ("bitor_agg", "min_row_number_filter"), (0, 1, 2), (1, 2), (2,), (True,), (True,), (1,))


def test_exact_kurt_hand_computed():
    # {1, 2, 3, 4}: mean 5/2, M2 = 5, M4 = 41/4 -> 4*5*3 * 41/4 / (2*1*25) - 27/2 = -1.2
    k, n, m2, r = exact_kurt([1.0, 2.0, 3.0, 4.0])
    assert (k, n, m2, r) == (-1.2, 4, 5.0, 1.5)
    # exact at any offset
    assert exact_kurt([1e9 + 1, 1e9 + 2, 1e9 + 3, 1e9 + 4])[0] == -1.2
    assert exact_kurt([7.0, 7.0, 7.0, 7.0, 7.0])[0] == 0.0  # constant: the denominator is 0
    assert exact_kurt([1.0, 2.0, 3.0])[0] is None and exact_kurt([1.0, np.nan, 2.0, 3.0])[0] is None
    assert math.isnan(exact_kurt([1.0, 2.0, np.inf, 3.0])[0])


@pytest.mark.parametrize("batch", [1, 3, 7, 1000])
def test_restatement_follows_pandas(batch):
    rng = np.random.default_rng(11)
    groups = [rng.standard_normal(s) * sc + o for s, sc, o in
              [(4, 1.0, 0.0), (5, 2.0, 3.0), (7, 0.5, -4.0), (31, 1.0, 10.0), (200, 3.0, 0.0), (1000, 1.0, 1.0)]]
    groups += [rng.exponential(1.0, 300), rng.standard_t(5, 400), np.array([1.0, 2.0, 3.0, 4.0]), np.array([2.0, 2.0, 2.0, 9.0])]
    for g in groups:
        g = g.copy()
        if len(g) > 10:
            g[rng.random(len(g)) < 0.1] = np.nan
        exp = pd.Series(g).kurt()
        got = kurt_batches(g, batch)
        assert got == pytest.approx(exp, rel=1e-9, abs=1e-9), (len(g), batch)
        k, n, m2, r = exact_kurt(g)
        assert abs(got - k) <= kurt_tol(k, n, m2, r), (len(g), got, k)


def test_restatement_edge_cases_follow_pandas():
    for g in ([1.0, 2.0, 3.0], [1.0, np.nan, 2.0, 3.0], [np.nan] * 5, []):  # fewer than 4 values: NA
        assert kurt_batches(np.array(g), 2) is None and math.isnan(pd.Series(g, dtype=float).kurt())
    for g in ([5.0] * 4, [1e9] * 50, [-3.25] * 7):  # constant: 0
        assert kurt_batches(np.array(g), 3) == 0.0 == pd.Series(g).kurt()
    for g in ([1.0, 2.0, 4.0, 8.0], [0.0, 0.0, 1.0, 5.0]):  # n = 4 exactly
        assert kurt_batches(np.array(g), 1) == pytest.approx(pd.Series(g).kurt(), rel=1e-12)
    assert math.isnan(kurt_batches(np.array([1.0, 2.0, np.inf, 3.0, 4.0]), 2))


@pytest.mark.parametrize("offset", [1e6, 1e9, 1.7e9])
def test_restatement_keeps_its_digits_at_an_offset(offset):
    """About a per-group shift, a large common offset costs nothing; power sums about 0 would lose every digit at 1e9."""
    rng = np.random.default_rng(int(offset) % 1000)
    x = offset + rng.standard_normal(2000)
    k, n, m2, r = exact_kurt(x)
    for batch in (1, 64, 2000):
        got = kurt_batches(x, batch)
        assert abs(got - k) <= kurt_tol(k, n, m2, r), (batch, got, k)
    # pandas' two-pass nankurt agrees with the exact value here too
    assert pd.Series(x).kurt() == pytest.approx(k, abs=1e-6)
    # the same sums about 0 (c = 0) are useless at this offset
    s = [sum(float(v) ** p for v in x) for p in (1, 2, 3, 4)]
    naive = kurt_eval((len(x), 0.0, *s))
    assert not abs(naive - k) <= 1e-3
