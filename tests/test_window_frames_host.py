"""Host-side checks of bounded ROWS frames (("rows", start, end)) and NTH_VALUE: parsing, the two spellings of the unbounded
frames, the errors and the entries they name, the header's codes and sentinels, the ABI entry and frame struct, and PhysicalWindow
plumbing (no GPU needed)."""

import re

import pytest

from bodo_b200 import _lib
from bodo_b200._lib import B200Error, ffi
from bodo_b200.physical import PhysicalWindow
from bodo_b200.streaming import window as W
from bodo_b200.table import CTypes

COLS = ["a", "b", "c", "d"]
TYPES = [CTypes.INT64, CTypes.FLOAT32, CTypes.DATETIME, CTypes.INT8]  # a, b, c, d
UP, UF = W.UNBOUNDED_PRECEDING, W.UNBOUNDED_FOLLOWING
BIG = (1 << 31) - 1


def init(funcs, **kw):
    args = dict(operator_id=-1, partition_by=["a"], order_by=["b"], ascending=True, na_position="last", funcs=funcs, col_names=COLS)
    args.update(kw)
    return W.init_window_state(**args)


def test_frame_forms():
    st = init([("m7", "mean", "d", ("rows", -6, 0)), ("sc", "sum", "b", ("rows", -3, 3)), ("mx", "max", "c", ("rows", 0, 9)),
               ("lb", "min", "a", ("rows", None, 3)), ("fw", "first_value", "d", ("rows", 2, None)), ("cz", "count", None, ("rows", -5, -2)),
               ("cx", "count", "c", ["rows", -BIG, BIG]), ("lv", "last_value", "b", ("rows", 0, 0))])
    assert st.funcs == [("m7", 8, 0, "d", 4, None, (-6, 0)), ("sc", 6, 0, "b", 4, None, (-3, 3)), ("mx", 10, 0, "c", 4, None, (0, 9)),
                        ("lb", 9, 0, "a", 4, None, (UP, 3)), ("fw", 11, 0, "d", 4, None, (2, UF)), ("cz", 7, 0, None, 4, None, (-5, -2)),
                        ("cx", 7, 0, "c", 4, None, (-BIG, BIG)), ("lv", 12, 0, "b", 4, None, (0, 0))]
    assert st.descriptors(TYPES) == [(8, 3, 4, 0, 0, 0), (6, 1, 4, 0, 0, 0), (10, 2, 4, 0, 0, 0), (9, 0, 4, 0, 0, 0), (11, 3, 4, 0, 0, 0),
                                     (7, -1, 4, 0, 0, 0), (7, 2, 4, 0, 0, 0), (12, 1, 4, 0, 0, 0)]
    assert st.frames() == [(-6, 0), (-3, 3), (0, 9), (UP, 3), (2, UF), (-5, -2), (-BIG, BIG), (0, 0)]


def test_nth_value_forms():
    st = init([("n1", "nth_value", "d", 1), ("n2", "nth_value", "b", 2, "rows"), ("n3", "nth_value", "c", BIG, "partition"),
               ("n4", "nth_value", "a", 3, ("rows", -2, 2))])
    assert st.funcs == [("n1", 15, 1, "d", 1, None), ("n2", 15, 2, "b", 2, None), ("n3", 15, BIG, "c", 3, None),
                        ("n4", 15, 3, "a", 4, None, (-2, 2))]
    assert st.descriptors(TYPES) == [(15, 3, 1, 0, 1, 0), (15, 1, 2, 0, 2, 0), (15, 2, 3, 0, BIG, 0), (15, 0, 4, 0, 3, 0)]
    assert st.frames() == [(UP, UF), (UP, UF), (UP, UF), (-2, 2)]


def test_unbounded_spellings_normalise():
    """(UNBOUNDED PRECEDING, CURRENT ROW) is "rows" and (UNBOUNDED PRECEDING, UNBOUNDED FOLLOWING) is "partition"."""
    a = init([("r", "sum", "d", ("rows", None, 0)), ("p", "max", "b", ("rows", None, None)), ("n", "nth_value", "d", 2, ("rows", None, 0))])
    b = init([("r", "sum", "d", "rows"), ("p", "max", "b", "partition"), ("n", "nth_value", "d", 2, "rows")])
    assert a.funcs == b.funcs and a.descriptors(TYPES) == b.descriptors(TYPES) and a.frames() == b.frames()
    # other unbounded frames keep frame 4
    assert init([("x", "sum", "d", ("rows", 0, None))]).descriptors(TYPES)[0][2] == 4
    assert init([("x", "sum", "d", ("rows", None, 1))]).descriptors(TYPES)[0][2] == 4


@pytest.mark.parametrize("f,msg", [
    (("x", "sum", "d", ("rows", 2, 1)), "frame start 2 is after frame end 1"),
    (("x", "sum", "d", ("rows", 0, -1)), "after frame end"),
    (("x", "sum", "d", ("rows", -(1 << 31), 0)), "bad frame bound"),
    (("x", "sum", "d", ("rows", 0, 1 << 31)), "bad frame bound"),
    (("x", "sum", "d", ("rows", True, 1)), "bad frame bound"),
    (("x", "sum", "d", ("rows", 0, 1.0)), "bad frame bound"),
    (("x", "sum", "d", ("rows", "a", 1)), "bad frame bound"),
    (("x", "sum", "d", ("range", -1, 0)), "bad frame"),
    (("x", "sum", "d", ("rows", -1)), "bad frame"),
    (("x", "sum", "d", ("rows", -1, 0, 1)), "bad frame"),
    (("x", "sum", "d", ("rows", -1, 0), "rows"), "bad frame"),
    (("x", "lag", "d", ("rows", -1, 0)), "0 <= k < 2\\^31"),
    (("x", "nth_value", "d"), "nth_value takes"),
    (("x", "nth_value", "d", 0), "1 <= n < 2\\^31"),
    (("x", "nth_value", "d", 1 << 31), "1 <= n < 2\\^31"),
    (("x", "nth_value", "d", True), "1 <= n < 2\\^31"),
    (("x", "nth_value", "d", 2.0), "1 <= n < 2\\^31"),
    (("x", "nth_value", "d", 1, "rows", 0), "nth_value takes"),
    (("x", "nth_value", "d", 1, "groups"), "bad frame"),
    (("x", "nth_value", "d", 1, ("rows", 3, 1)), "after frame end"),
    (("x", "nth_value", None, 1), "unknown column None"),
])
def test_errors_name_the_entry(f, msg):
    with pytest.raises(B200Error, match=msg) as e:
        init([f])
    assert repr(f) in str(e.value)


def test_existing_frame_errors_are_unchanged():
    for f in (("x", "sum", "d", 3), ("x", "max", "d", "rows", 1), ("x", "sum", "d", "groups")):
        with pytest.raises(B200Error, match="bad frame"):
            init([f])
    with pytest.raises(B200Error) as e:
        init([("x", "nth_value")])
    m = str(e.value)
    assert "unknown window function" in m and "(out_name, fname)" in m and "(out_name, fname, column[, frame])" in m
    assert "'lag' | 'lead', column[, k[, default]]" in m and "'nth_value', column, n[, frame]" in m


def test_temporal_sum_names_the_bounded_entry():
    st = init([("x", "sum", "c", ("rows", None, 2))])
    with pytest.raises(B200Error, match=r"\('x', 'sum', 'c', \('rows', None, 2\)\).*sum and mean need"):
        st.descriptors(TYPES)
    assert init([("x", "nth_value", "c", 2, ("rows", -1, 1))]).descriptors(TYPES) == [(15, 2, 4, 0, 2, 0)]


def test_header_codes_and_sentinels():
    with open(_lib.HEADER) as f:
        text = f.read()
    header = " ".join(re.sub(r"\n\s*\*", " ", text).split())
    assert "13 lag, 14 lead, 15 nth_value" in header and "4 rows between" in header
    assert re.search(r"#define B200_WINDOW_UNBOUNDED_PRECEDING INT64_MIN\b", text)
    assert re.search(r"#define B200_WINDOW_UNBOUNDED_FOLLOWING INT64_MAX\b", text)
    assert (UP, UF) == (-(1 << 63), (1 << 63) - 1)
    assert W.FRAME_FUNCS == {"nth_value": 15} and W.ROWS_BETWEEN == 4
    assert "nth_value" not in W.VALUE_FUNCS and 4 not in W.FRAMES.values()


def test_abi_declares_the_frame_entry_and_struct():
    assert [s for s in _lib.declared_symbols() if s.startswith("b200_window_state_init")] == ["b200_window_state_init"]
    assert ffi.sizeof("b200_window_frame") == 16
    assert [name for name, _ in ffi.typeof("b200_window_frame").fields] == ["start", "end"]
    assert ffi.sizeof("b200_window_func") == 80
    assert dict(ffi.typeof("b200_window_func").fields)["rows"].type is ffi.typeof("b200_window_frame")


def test_physical_window_plumbing():
    funcs = [("ma7", "mean", "b", ("rows", -6, 0)), ("n2", "nth_value", "a", 2, ("rows", None, 3))]
    op = PhysicalWindow("a", ["b"], funcs)
    assert op.state is None
    assert op.args == ("a", ["b"], True, "last", funcs, False)
    op.Finalize()
