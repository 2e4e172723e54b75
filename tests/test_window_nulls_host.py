"""Host-side checks of IGNORE NULLS on FIRST_VALUE / LAST_VALUE / NTH_VALUE / LAG / LEAD: parsing of the trailing marker in every
entry form and frame, "respect_nulls" as the default, refusal on every other function with the entry named, unchanged errors,
the header's definitions and the new entry (no GPU needed)."""

import re

import pytest

from bodo_b200 import _lib
from bodo_b200._lib import B200Error, ffi
from bodo_b200.physical import PhysicalWindow
from bodo_b200.streaming import window as W
from bodo_b200.table import CTypes

COLS = ["a", "b", "c", "d", "ignore_nulls"]
TYPES = [CTypes.INT64, CTypes.FLOAT64, CTypes.DATETIME, CTypes.INT32, CTypes.FLOAT32]
FRAMES = [None, "range", "rows", "partition", ("rows", None, 0), ("rows", None, None), ("rows", -3, 0), ("rows", 0, None),
          ("rows", 2, 5), ("rows", -(1 << 31) + 1, (1 << 31) - 1), ("range_between", -2, 0), ("range_between", 0, None),
          ("range_between", None, 0), ("range_between", None, None), ("range_between", 1.5, 4)]


def init(funcs, **kw):
    args = dict(operator_id=-1, partition_by=["a"], order_by=["b"], ascending=True, na_position="last", funcs=funcs, col_names=COLS)
    args.update(kw)
    return W.init_window_state(**args)


def entries():
    """Every entry form of the five functions, without a marker."""
    fs = []
    for j, fr in enumerate(FRAMES):
        tail = () if fr is None else (fr,)
        fs += [(f"f{j}", "first_value", "d", *tail), (f"l{j}", "last_value", "b", *tail), (f"n{j}", "nth_value", "d", 1 + j, *tail)]
    fs += [("lg", "lag", "d"), ("lg2", "lag", "b", 2), ("lg3", "lag", "d", 0, 7), ("ld", "lead", "b"), ("ld2", "lead", "d", 3, None),
           ("ld3", "lead", "b", 1 << 20, -2.5)]
    return fs


@pytest.mark.parametrize("marker", ["ignore_nulls", "respect_nulls"])
@pytest.mark.parametrize("part", [0, 1])
def test_marker_in_every_form_and_frame(marker, part):
    fs = entries()[part::2]  # a state holds at most 32 columns
    plain = init(fs)
    marked = init([f + (marker,) for f in fs])
    assert marked.funcs == plain.funcs
    assert marked.descriptors(TYPES) == plain.descriptors(TYPES)
    assert marked.frames() == plain.frames() and marked.ranges(TYPES) == plain.ranges(TYPES)
    assert marked.ignore_nulls == [marker == "ignore_nulls"] * len(fs)
    assert plain.ignore_nulls == [False] * len(fs)


def test_issue_examples_and_mixed_flags():
    st = init([("ffill", "last_value", "d", "rows", "ignore_nulls"), ("prev", "lag", "d", 1, None, "ignore_nulls"),
               ("second", "nth_value", "d", 2, "partition", "ignore_nulls"), ("f", "first_value", "d", "ignore_nulls"),
               ("rn", "row_number"), ("s", "sum", "d", "rows"), ("r", "last_value", "d", "rows"), ("k", "corr", "b", "d")])
    assert st.funcs == [("ffill", 12, 0, "d", 2, None), ("prev", 13, 1, "d", 0, None), ("second", 15, 2, "d", 3, None),
                        ("f", 11, 0, "d", 1, None), ("rn", 0, 0), ("s", 6, 0, "d", 2, None), ("r", 12, 0, "d", 2, None),
                        ("k", 22, "d", "b", 1, None)]
    assert st.ignore_nulls == [True, True, True, True, False, False, False, False]


def test_a_column_named_ignore_nulls_is_a_column():
    st = init([("x", "last_value", "ignore_nulls"), ("y", "lag", "ignore_nulls"), ("z", "sum", "ignore_nulls", "rows"),
               ("w", "first_value", "ignore_nulls", "rows", "ignore_nulls")])
    assert [f[3] for f in st.funcs] == ["ignore_nulls"] * 4
    assert st.ignore_nulls == [False, False, False, True]
    assert st.descriptors(TYPES)[0][:3] == (12, 4, 1)


OTHERS = [("x", "rank", "a", "ignore_nulls"), ("x", "row_number", "b", "respect_nulls"), ("x", "ntile", 3, "ignore_nulls"),
          ("x", "sum", "d", "ignore_nulls"), ("x", "count", None, "ignore_nulls"), ("x", "mean", "d", "rows", "respect_nulls"),
          ("x", "min", "d", ("rows", -1, 1), "ignore_nulls"), ("x", "max", "d", "ignore_nulls"), ("x", "var", "d", "ignore_nulls"),
          ("x", "std_pop", "d", "partition", "ignore_nulls"), ("x", "corr", "b", "d", "ignore_nulls"),
          ("x", "regr_slope", "b", "d", "rows", "respect_nulls"), ("x", "covar_samp", "b", "ignore_nulls")]


@pytest.mark.parametrize("f", OTHERS)
def test_marker_on_any_other_function_names_the_entry(f):
    with pytest.raises(B200Error, match="takes one of \\['first_value', 'last_value', 'nth_value', 'lag', 'lead'\\]") as e:
        init([f])
    assert repr(f) in str(e.value)


@pytest.mark.parametrize("f,msg", [
    (("x", "lag", "d", 1, 0, 0), "lag takes"),
    (("x", "nth_value", "d", 1, "rows", 0), "nth_value takes"),
    (("x", "nth_value", "d", "ignore_nulls"), "nth_value takes"),
    (("x", "nth_value", "d", 0, "ignore_nulls"), "nth_value takes"),
    (("x", "lag", "d", "rows", "ignore_nulls"), "lag takes no frame"),
    (("x", "lead", "d", -1, "ignore_nulls"), "needs an integer k"),
    (("x", "lag", "d", 1, 0, 0, "ignore_nulls"), "lag takes"),
    (("x", "first_value", "zz", "ignore_nulls"), "unknown column 'zz'"),
    (("x", "last_value", "d", "groups", "ignore_nulls"), "bad frame"),
    (("x", "first_value", "d", "rows", "rows", "ignore_nulls"), "bad frame"),
    (("x", "last_value", "d", ("rows", 2, 1), "respect_nulls"), "frame start 2 is after frame end 1"),
    (("x", "first_value", "d", ("range_between", "x", 0), "ignore_nulls"), "bad frame bound"),
])
def test_errors_name_the_entry_as_written(f, msg):
    with pytest.raises(B200Error, match=msg) as e:
        init([f])
    assert repr(f) in str(e.value)
    if f[-1] not in W.NULLS_MARKERS:  # the same message as before
        with pytest.raises(B200Error, match=msg):
            init([f + ("ignore_nulls",)])


def test_marker_does_not_make_an_unknown_function_known():
    for f in [("x", "median", "d", "ignore_nulls"), ("x", "ignore_nulls"), ("x", "ignore_nulls", "d", "ignore_nulls")]:
        with pytest.raises(B200Error, match="unknown window function"):
            init([f])


def test_unknown_function_message_names_the_marker():
    with pytest.raises(B200Error) as e:
        init([("x", "ffill", "d")])
    m = str(e.value)
    assert "(out_name, fname, column[, frame])" in m and "'lag' | 'lead', column[, k[, default]]" in m
    assert "'ignore_nulls' or 'respect_nulls'" in m


def test_later_errors_show_the_marker():
    st = init([("x", "lag", "d", 1, 0.5, "ignore_nulls")])
    with pytest.raises(B200Error, match=re.escape(repr(("x", "lag", "d", 1, 0.5, "ignore_nulls"))) + ".*not exactly representable"):
        st.descriptors(TYPES)
    with pytest.raises(B200Error, match=re.escape(repr(("x", "lag", "d", 1, 0.5))) + ".*not exactly representable"):
        init([("x", "lag", "d", 1, 0.5)]).descriptors(TYPES)
    st = init([("x", "first_value", "d", ("range_between", 0.5, 1), "ignore_nulls")], order_by=["d"])
    with pytest.raises(B200Error, match=re.escape(repr(("x", "first_value", "d", ("range_between", 0.5, 1), "ignore_nulls")))):
        st.ranges(TYPES)
    with pytest.raises(B200Error, match=re.escape("'nth_value', 'd', 2, ('range_between', -1, 0), 'ignore_nulls')") + ".*exactly one ORDER"):
        init([("x", "nth_value", "d", 2, ("range_between", -1, 0), "ignore_nulls")], order_by=["b", "c"])


def test_header_defines_ignore_nulls_and_declares_the_entry():
    with open(_lib.HEADER) as f:
        text = f.read()
    header = " ".join(re.sub(r"\n\s*\*", " ", text).split())
    assert [s for s in _lib.declared_symbols() if s.startswith("b200_window_state_init")] == ["b200_window_state_init"]
    assert "codes 11 first_value, 12 last_value, 13 lag, 14 lead and 15 nth_value only" in header
    assert "its validity is clear or it is a float NaN" in header
    for d in ("first_value the first non-null cell in [lo, hi]; NA if none", "last_value the last non-null cell in [lo, hi]; NA if none",
              "nth_value the n-th non-null cell in [lo, hi] (FROM FIRST)", "lag the k-th non-null cell before row i within [P, i)",
              "lead the k-th non-null cell after row i within (i, pe)"):
        assert d in header, d
    decl = re.search(r"void\* b200_window_state_init\(([^;]*)\);", text).group(1)
    assert "const b200_window_func* funcs, int32_t n_funcs" in " ".join(decl.split())
    assert dict(ffi.typeof("b200_window_func").fields)["ignore_nulls"].type is ffi.typeof("int32_t")
    # the RESPECT NULLS sentences stay as they were
    assert "first_value, last_value the cell at P / e as it is (bits and validity: a NaN stays a valid NaN)" in header


def test_physical_window_passes_the_marker_through():
    funcs = [("ffill", "last_value", "b", "rows", "ignore_nulls"), ("bfill", "first_value", "b", ("rows", 0, None), "ignore_nulls")]
    op = PhysicalWindow("a", ["d"], funcs)
    assert op.state is None
    assert op.args == ("a", ["d"], True, "last", funcs, False)
    op.Finalize()
