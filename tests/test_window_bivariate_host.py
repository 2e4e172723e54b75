"""Host-side checks of the COVAR_SAMP / COVAR_POP / CORR / REGR_SLOPE / REGR_INTERCEPT window functions: parsing of every form
and frame spelling, descriptors carrying the second column in arg, errors naming the entry, the header's codes and the bivariate
entry, and PhysicalWindow plumbing (no GPU needed)."""

import re
import struct

import pytest

from bodo_b200 import _lib
from bodo_b200._lib import B200Error
from bodo_b200.physical import PhysicalWindow
from bodo_b200.streaming import window as W
from bodo_b200.table import CTypes

COLS = ["a", "b", "c", "d", "e"]
TYPES = [CTypes.INT64, CTypes.FLOAT32, CTypes.DATETIME, CTypes.UINT8, CTypes.BOOL]  # a, b, c, d, e
UP, UF = W.UNBOUNDED_PRECEDING, W.UNBOUNDED_FOLLOWING
BIG = (1 << 31) - 1
BIVARIATE = ("covar_samp", "covar_pop", "corr", "regr_slope", "regr_intercept")


def init(funcs, **kw):
    args = dict(operator_id=-1, partition_by=["a"], order_by=["b"], ascending=True, na_position="last", funcs=funcs, col_names=COLS)
    args.update(kw)
    return W.init_window_state(**args)


def test_codes():
    assert W.BIVARIATE_FUNCS == {"covar_samp": 20, "covar_pop": 21, "corr": 22, "regr_slope": 23, "regr_intercept": 24}
    assert not set(BIVARIATE) & (set(W.FUNCS) | set(W.VALUE_FUNCS) | set(W.FRAME_FUNCS) | set(W.MOMENT_FUNCS) | set(W.BOUNDED_FUNCS))
    others = [*W.FUNCS.values(), *W.VALUE_FUNCS.values(), *W.FRAME_FUNCS.values(), *W.MOMENT_FUNCS.values()]
    assert not set(W.BIVARIATE_FUNCS.values()) & set(others)


@pytest.mark.parametrize("fname", BIVARIATE)
def test_every_frame_spelling(fname):
    code = W.BIVARIATE_FUNCS[fname]
    st = init([("d0", fname, "d", "a"), ("r", fname, "b", "d", "range"), ("w", fname, "a", "a", "rows"), ("p", fname, "e", "b", "partition"),
               ("w2", fname, "a", "e", ("rows", None, 0)), ("p2", fname, "e", "d", ["rows", None, None]),
               ("m", fname, "d", "b", ("rows", -59, 0)), ("ce", fname, "b", "a", ("rows", -3, 3)), ("x", fname, "d", "e", ("rows", -BIG, BIG)),
               ("rb", fname, "a", "d", ("range_between", -2, 0)), ("rf", fname, "d", "a", ("range_between", 0, 5)),
               ("r2", fname, "a", "d", ("range_between", None, 0)), ("p3", fname, "a", "d", ("range_between", None, None))])
    assert st.funcs == [("d0", code, "a", "d", 1, None), ("r", code, "d", "b", 1, None), ("w", code, "a", "a", 2, None),
                        ("p", code, "b", "e", 3, None), ("w2", code, "e", "a", 2, None), ("p2", code, "d", "e", 3, None),
                        ("m", code, "b", "d", 4, None, (-59, 0)), ("ce", code, "a", "b", 4, None, (-3, 3)),
                        ("x", code, "e", "d", 4, None, (-BIG, BIG)), ("rb", code, "d", "a", 5, None, (-2, 0)),
                        ("rf", code, "a", "d", 5, None, (0, 5)), ("r2", code, "d", "a", 1, None), ("p3", code, "d", "a", 3, None)]
    # (code, col = y, frame, default_valid, arg = x, default_bits), columns by physical index
    assert st.descriptors(TYPES) == [(code, 3, 1, 0, 0, 0), (code, 1, 1, 0, 3, 0), (code, 0, 2, 0, 0, 0), (code, 4, 3, 0, 1, 0),
                                     (code, 0, 2, 0, 4, 0), (code, 4, 3, 0, 3, 0), (code, 3, 4, 0, 1, 0), (code, 1, 4, 0, 0, 0),
                                     (code, 3, 4, 0, 4, 0), (code, 0, 5, 0, 3, 0), (code, 3, 5, 0, 0, 0), (code, 0, 1, 0, 3, 0),
                                     (code, 0, 3, 0, 3, 0)]
    assert st.frames() == [(UP, UF)] * 6 + [(-59, 0), (-3, 3), (-BIG, BIG)] + [(UP, UF)] * 4
    two, five = (struct.unpack("<Q", struct.pack("<d", v))[0] for v in (2.0, 5.0))  # offsets on the FLOAT32 key b
    assert st.ranges(TYPES)[9:11] == [(1, 2, two, 0), (2, 3, 0, five)]


def test_mixed_with_other_functions():
    st = init([("rn", "row_number"), ("s", "sum", "d", ("rows", -2, 0)), ("k", "corr", "d", "a", ("rows", -2, 0)), ("lg", "lag", "a", 1),
               ("v", "var", "a", "partition"), ("bt", "regr_slope", "a", "d", "partition")])
    assert [f[1] for f in st.funcs] == [0, 6, 22, 13, 16, 23]
    assert st.descriptors(TYPES) == [(0, -1, 0, 0, 0, 0), (6, 3, 4, 0, 0, 0), (22, 3, 4, 0, 0, 0), (13, 0, 0, 0, 1, 0), (16, 0, 3, 0, 0, 0),
                                     (23, 0, 3, 0, 3, 0)]


@pytest.mark.parametrize("f,msg", [
    (("x", "corr", None, "d"), "unknown column None"),
    (("x", "covar_samp", "zz", "d"), "unknown column 'zz'"),
    (("x", "corr", "d", None), "unknown second column None"),
    (("x", "regr_slope", "d", "zz"), "unknown second column 'zz'"),
    (("x", "covar_pop", "d"), "unknown second column None"),
    (("x", "corr", "d", "a", "groups"), "bad frame"),
    (("x", "corr", "d", "a", 3), "bad frame"),
    (("x", "regr_intercept", "d", "a", "rows", 1), "takes \\(out_name, 'regr_intercept', column1, column2\\[, frame\\]\\)"),
    (("x", "covar_samp", "d", "a", ("rows", 2, 1)), "frame start 2 is after frame end 1"),
    (("x", "corr", "d", "a", ("rows", -(1 << 31), 0)), "bad frame bound"),
    (("x", "corr", "d", "a", ("range_between", 3, -3)), "frame start 3 is after frame end -3"),
    (("x", "regr_slope", "d", "a", ("range_between", "x", 0)), "bad frame bound"),
])
def test_errors_name_the_entry(f, msg):
    with pytest.raises(B200Error, match=msg) as e:
        init([f])
    assert repr(f) in str(e.value)


def test_unknown_function_message_lists_the_bivariate_form():
    with pytest.raises(B200Error) as e:
        init([("x", "cov", "d", "a")])
    m = str(e.value)
    assert "unknown window function" in m and all(repr(f) in m for f in BIVARIATE)
    assert "(out_name, fname, column1, column2[, frame])" in m
    assert "(out_name, fname, column[, frame])" in m and "'nth_value', column, n[, frame]" in m
    with pytest.raises(B200Error, match="unknown window function"):
        init([("x", "corr")])


@pytest.mark.parametrize("fname", BIVARIATE)
@pytest.mark.parametrize("frame", ["range", ("rows", -59, 0), ("range_between", -2, 0)])
@pytest.mark.parametrize("cols", [("c", "a"), ("a", "c"), ("c", "c")])
def test_temporal_column_names_the_entry(fname, frame, cols):
    st = init([("x", fname, *cols, frame)])
    with pytest.raises(B200Error, match=re.escape(repr(("x", fname, *cols, frame))) + ".*covar, corr and regr need integer, bool or float columns"):
        st.descriptors(TYPES)
    # every other pair of types is accepted
    fs = [(f"x{y}{x}", fname, y, x, frame) for y in "abde" for x in "abde"]
    assert [d[0] for d in init(fs).descriptors(TYPES)] == [W.BIVARIATE_FUNCS[fname]] * 16


def test_var_message_is_unchanged():
    with pytest.raises(B200Error, match="var and std need an integer, bool or float column"):
        init([("x", "var", "c")]).descriptors(TYPES)


def test_header_documents_the_codes_and_declares_the_entry():
    with open(_lib.HEADER) as f:
        text = f.read()
    header = " ".join(re.sub(r"\n\s*\*", " ", text).split())
    assert "20 covar_samp, 21 covar_pop, 22 corr, 23 regr_slope, 24 regr_intercept" in header
    assert "20 covar_samp = Sxy / (m - 1), NA when m < 2" in header and "21 covar_pop = Sxy / m, NA when m = 0" in header
    assert "22 corr = Sxy / sqrt(Sxx Syy), NA when m < 2, Sxx = 0 or Syy = 0" in header
    assert "23 regr_slope = Sxy / Sxx, NA when Sxx = 0" in header and "24 regr_intercept = my - regr_slope mx" in header
    assert [s for s in _lib.declared_symbols() if s.startswith("b200_window_state_init")] == ["b200_window_state_init"]
    # the earlier entries' sentences stay as they were
    assert "16 var, 17 std, 18 var_pop, 19 std_pop" in header


def test_physical_window_plumbing():
    funcs = [("beta", "regr_slope", "b", "d", ("rows", -59, 0)), ("rho", "corr", "b", "d", ("rows", -59, 0)),
             ("cv", "covar_samp", "a", "b", "partition")]
    op = PhysicalWindow("a", ["b"], funcs)
    assert op.state is None
    assert op.args == ("a", ["b"], True, "last", funcs, False)
    op.Finalize()
