"""mode, percentile_cont and percentile_disc without a GPU: their function numbers, every refusal of percentiles= and of the input
columns, the C header's contract, physical.groupby_agg's 4-tuples, and the numpy restatement of the three definitions that
tests/test_gpu_groupby_holistic.py checks the device against, pinned here against pandas and numpy."""

import math
import os

import numpy as np
import pandas as pd
import pytest

from bodo_b200 import _lib, physical
from bodo_b200.streaming import groupby as G

HEADER = os.path.join(os.path.dirname(__file__), "..", "include", "bodo_b200.h")
TINY = 5e-324
ONE_MINUS_ULP = 1.0 - 2.0 ** -53
QS = (0.0, TINY, 1 / 3, 0.5, ONE_MINUS_ULP, 1.0)


# ================================================================================================ the restatement
def present(values, valid=None):
    """V sorted: the values whose cell is valid, NaN skipped in a float column, -0.0 as +0.0 (one value with 0.0)."""
    v = np.asarray(values)
    keep = np.ones(len(v), dtype=bool) if valid is None else np.asarray(valid, dtype=bool).copy()
    if v.dtype.kind == "f":
        keep &= ~np.isnan(v)
    v = v[keep]
    if v.dtype.kind == "f":
        v = np.where(v == 0, np.zeros((), v.dtype), v)
    return np.sort(v, kind="stable")


def _f64(x):
    return float(np.float64(x))  # (numpy's conversion rounds to nearest, as the device's)


def percentile_cont(V, q):
    """h = q (m - 1), lo = floor(h), f = h - lo; v_lo when f == 0, else a + (b - a) f in float64; None when m == 0."""
    m = len(V)
    if m == 0:
        return None
    h = float(q) * float(m - 1)
    lo = math.floor(h)
    f = h - lo
    a = _f64(V[lo])
    if f == 0.0:
        return a
    return a + (_f64(V[lo + 1]) - a) * f


def percentile_disc(V, q):
    """v_i with i = clamp(ceil(q m) - 1, 0, m - 1); None when m == 0."""
    m = len(V)
    if m == 0:
        return None
    i = math.ceil(float(q) * float(m)) - 1
    return V[min(max(i, 0), m - 1)]


def mode(V):
    """The most frequent value, ties to the least; None when m == 0."""
    if len(V) == 0:
        return None
    vals, counts = np.unique(V, return_counts=True)
    return vals[int(np.argmax(counts))]


def reference(f, V, q=None):
    return percentile_cont(V, q) if f == "percentile_cont" else percentile_disc(V, q) if f == "percentile_disc" else mode(V)


def bits(x):
    """The float64 bit pattern of x (ints pass through), for bit-exact comparisons."""
    if x is None:
        return None
    if isinstance(x, (float, np.floating)):
        return int(np.float64(x).view(np.int64))
    return int(x)


# ================================================================================================ function numbers
def test_function_numbers():
    assert (G.FTYPES["mode"], G.FTYPES["percentile_cont"], G.FTYPES["percentile_disc"]) == (38, 39, 40)
    assert len(set(G.FTYPES.values())) == len(G.FTYPES)
    assert "median" not in G.FTYPES


# ================================================================================================ refusals
def _init(fnames, n_in=None, **kw):
    n_in = n_in or [1] * len(fnames)
    offs = tuple(np.concatenate([[0], np.cumsum(n_in)]).astype(int).tolist())
    return G.init_groupby_state(-1, (0,), tuple(fnames), offs, tuple(range(1, 1 + offs[-1])), **kw)


@pytest.mark.parametrize("fnames, kw, needle", [
    (("percentile_cont",), {}, "percentiles must give one fraction"),
    (("percentile_disc", "mode"), {}, "percentiles must give one fraction"),
    (("percentile_cont", "percentile_disc"), {"percentiles": (0.5,)}, "percentiles must be a sequence"),
    (("percentile_cont",), {"percentiles": (0.5, 0.9)}, "percentiles must be a sequence"),
    (("percentile_cont",), {"percentiles": 0.5}, "percentiles must be a sequence"),
    (("percentile_cont",), {"percentiles": "5"}, "percentiles must be a sequence"),
    (("percentile_cont",), {"percentiles": (True,)}, "percentiles entries must be numbers in [0, 1]"),
    (("percentile_cont",), {"percentiles": (float("nan"),)}, "percentiles entries must be numbers in [0, 1]"),
    (("percentile_disc",), {"percentiles": (-1e-300,)}, "percentiles entries must be numbers in [0, 1]"),
    (("percentile_disc",), {"percentiles": (1.0000000000000002,)}, "percentiles entries must be numbers in [0, 1]"),
    (("percentile_cont",), {"percentiles": ("0.5",)}, "percentiles entries must be numbers in [0, 1]"),
    (("mode",), {"percentiles": (0.5,)}, "percentiles needs a percentile_cont or percentile_disc"),
    (("sum", "mean"), {"percentiles": ()}, "percentiles needs a percentile_cont or percentile_disc"),
])
def test_percentiles_refusals(fnames, kw, needle):
    with pytest.raises(_lib.B200Error, match="percentiles") as e:
        _init(fnames, **kw)
    assert needle in str(e.value)


@pytest.mark.parametrize("f", G.HOLISTIC)
@pytest.mark.parametrize("n_in", [0, 2])
def test_one_input_column(f, n_in):
    kw = {"percentiles": (0.5,)} if f in G.PERCENTILES else {}
    with pytest.raises(_lib.B200Error, match=f"{f} takes exactly one input column"):
        _init((f,), n_in=[n_in], **kw)


def test_mixed_state_and_median_still_unsupported():
    st = _init(("sum", "percentile_cont", "mode", "percentile_disc", "nunique"), percentiles=(0.25, np.float32(0.75)))
    assert st.fractions[1:4:2] == (0.25, 0.75) and math.isnan(st.fractions[0]) and math.isnan(st.fractions[2])
    assert st.handle is None  # (the C state comes with the first batch)
    with pytest.raises(_lib.B200Error, match="unsupported aggregate function 'median'"):
        _init(("median",))


def test_mrnf_takes_no_percentiles():
    with pytest.raises(_lib.B200Error, match="percentiles"):
        G.init_groupby_state(-1, (0,), (G.MRNF,), (0, 0), (), (1,), (True,), (True,), (1,), percentiles=(0.5,))


# ================================================================================================ header
def test_header_documents_the_entry():
    text = open(HEADER).read()
    for needle in ("b200_groupby_state_init_percentiles", "const double* fractions", "mode=38", "percentile_cont=39",
                   "percentile_disc=40", "recalled", "b200_groupby_state_init is this entry with fractions = NULL",
                   "at most 2^31 rows", "2^32 groups", "inverted_cdf", "Series.mode().iloc[0]", "a + (b - a) f",
                   "no fused multiply-add", "MEDIAN(x) is q = 0.5", "20 the values appended", "21 the digit passes"):
        assert needle in text, needle
    assert "b200_groupby_state_init_percentiles" in _lib.declared_symbols()


# ================================================================================================ physical.groupby_agg
class _Captured(Exception):
    pass


def test_groupby_agg_forwards_percentile_tuples(monkeypatch):
    seen = {}

    def fake_init(operator_id, key_inds, fnames, f_in_offsets, f_in_cols, *a, **kw):
        seen.update(key_inds=key_inds, fnames=fnames, f_in_offsets=f_in_offsets, f_in_cols=f_in_cols, kw=kw)
        raise _Captured

    monkeypatch.setattr(G, "init_groupby_state", fake_init)
    df = pd.DataFrame({"k": [1, 2], "x": [1.0, 2.0], "y": [3, 4]})
    aggs = [("p50", "x", "percentile_cont", 0.5), ("s", "y", "sum"), ("d", "y", "percentile_disc", 0.9), ("m", "x", "mode")]
    for fn, arg in ((physical.groupby_agg, df), (physical.groupby_agg_parquet, "unused.parquet")):
        seen.clear()
        with pytest.raises(_Captured):
            fn(arg, "k", aggs)
        assert seen["fnames"] == ("percentile_cont", "sum", "percentile_disc", "mode")
        assert seen["f_in_cols"] == (1, 2, 2, 1) and seen["f_in_offsets"] == (0, 1, 2, 3, 4)
        assert seen["kw"]["percentiles"] == (0.5, 0.9)


@pytest.mark.parametrize("aggs, needle", [
    ([("p", "x", "percentile_cont")], "a percentile \\(out_name, column, func, q\\)"),
    ([("s", "x", "sum", 0.5)], "only percentile_cont / percentile_disc take a fraction"),
    ([("p", "x")], "an aggregate is"),
])
def test_groupby_agg_refuses_malformed_tuples(aggs, needle):
    with pytest.raises(_lib.B200Error, match=needle):
        physical.groupby_agg(pd.DataFrame({"k": [1], "x": [1.0]}), "k", aggs)


# ================================================================================================ the restatement, pinned
def _cases():
    """(name, values) of one group each; float64 unless the values say otherwise."""
    inf = np.inf
    return [
        ("m0", np.array([], dtype=np.float64)),
        ("m0_all_nan", np.array([np.nan, np.nan])),
        ("m1", np.array([3.5])),
        ("m2", np.array([2.0, -1.0])),
        ("signed_zero", np.array([-0.0, 0.0, -0.0, 1.0])),
        ("inf", np.array([-inf, 1.0, 2.0, inf])),
        ("inf_only", np.array([inf, -inf])),
        ("inf_same", np.array([inf, inf, 1.0])),
        ("nan_mixed", np.array([np.nan, 4.0, 1.0, np.nan, 2.0, 8.0])),
        ("uniform", np.linspace(-3.0, 7.0, 31)),
        ("dup", np.array([5.0, 1.0, 5.0, 1.0, 2.0, 2.0, 2.0])),
        ("i64_big", np.array([2 ** 53 + 1, 2 ** 62 + 3, -(2 ** 63), 2 ** 63 - 1, 2 ** 53 + 3], dtype=np.int64)),
        ("u64_big", np.array([2 ** 64 - 1, 2 ** 63 + 1, 7], dtype=np.uint64)),
        ("i32", np.array([-7, 3, 3, 100, -7, -7], dtype=np.int32)),
        ("f32", np.array([0.1, -2.5, 3.25, np.nan, -0.0], dtype=np.float32)),
    ]


# pandas' linear group_quantile computes v_lo + (v_hi - v_lo) * f as the restatement does (NaN too, from inf - inf).  The one
# difference: a zero result keeps the sign of the cell pandas read (-0.0), where the restatement decodes every zero as +0.0.
def _same_as_pandas(g, want):
    return bits(g) == bits(want) or (math.isnan(g) and math.isnan(want)) or (g == 0.0 and want == 0.0)


@pytest.mark.parametrize("q", QS)
def test_percentile_cont_matches_pandas_groupby_quantile(q):
    for name, v in _cases():
        V = present(v)
        want = percentile_cont(V, q)
        df = pd.DataFrame({"k": np.zeros(len(v), dtype=np.int64), "v": v})
        got = df.groupby("k")["v"].quantile(q)
        if len(V) == 0:
            assert want is None and (len(got) == 0 or np.isnan(got.iloc[0])), name
            continue
        g = float(got.iloc[0])
        assert _same_as_pandas(g, want), (name, q, g, want)


@pytest.mark.parametrize("q", QS)
def test_percentile_disc_matches_numpy_inverted_cdf(q):
    for name, v in _cases():
        V = present(v)
        want = percentile_disc(V, q)
        if len(V) == 0:
            assert want is None
            continue
        got = np.quantile(V, q, method="inverted_cdf")
        assert bits(got.item()) == bits(want.item()), (name, q, got, want)


def test_mode_matches_series_mode():
    for name, v in _cases() + [("bool", np.array([True, False, True, False])), ("bool1", np.array([True, True, False]))]:
        V = present(v)
        want = mode(V)
        if len(V) == 0:
            assert want is None
            continue
        s = pd.Series(v).mode(dropna=True)
        got = s.iloc[0]
        if v.dtype.kind == "f" and got == 0:
            got = abs(got)  # (pandas may report the -0.0 it saw first; the restatement returns +0.0)
        assert bits(got.item() if hasattr(got, "item") else got) == bits(want.item()), (name, got, want)


def test_restatement_edge_values():
    V = present(np.array([1.0, 2.0]))
    assert percentile_cont(V, TINY) == 1.0 + (2.0 - 1.0) * TINY  # f = TINY: a + (b - a) f rounds back to a
    assert percentile_cont(V, ONE_MINUS_ULP) == 1.0 + ONE_MINUS_ULP
    assert percentile_disc(V, 0.0) == 1.0 and percentile_disc(V, TINY) == 1.0 and percentile_disc(V, 0.5) == 1.0
    assert percentile_disc(V, 0.5000000000000001) == 2.0 and percentile_disc(V, 1.0) == 2.0
    assert bits(percentile_cont(present(np.array([-0.0, -0.0])), 0.5)) == 0  # +0.0
    assert math.isnan(percentile_cont(present(np.array([np.inf, np.inf])), 0.5))  # (inf - inf) * f
    assert percentile_cont(present(np.array([np.inf, np.inf])), 1.0) == np.inf  # f == 0: v_lo
    V = present(np.array([2 ** 53 + 1, 2 ** 53 + 3], dtype=np.int64))
    assert percentile_cont(V, 0.0) == float(2 ** 53) and percentile_disc(V, 1.0) == 2 ** 53 + 3
    assert mode(present(np.array([3, 1, 3, 1], dtype=np.int64))) == 1
