"""Host-side checks of the VAR / STDDEV / VAR_POP / STDDEV_POP window functions: parsing of every form and frame spelling,
descriptors and codes, the temporal error naming the entry, the header's codes and the moments entry, and PhysicalWindow plumbing
(no GPU needed)."""

import re

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
MOMENTS = ("var", "std", "var_pop", "std_pop")


def init(funcs, **kw):
    args = dict(operator_id=-1, partition_by=["a"], order_by=["b"], ascending=True, na_position="last", funcs=funcs, col_names=COLS)
    args.update(kw)
    return W.init_window_state(**args)


def test_codes():
    assert W.MOMENT_FUNCS == {"var": 16, "std": 17, "var_pop": 18, "std_pop": 19}
    assert all(f in W.BOUNDED_FUNCS for f in MOMENTS)
    assert not set(MOMENTS) & (set(W.FUNCS) | set(W.VALUE_FUNCS) | set(W.FRAME_FUNCS))


@pytest.mark.parametrize("fname", MOMENTS)
def test_every_frame_spelling(fname):
    code = W.MOMENT_FUNCS[fname]
    st = init([("d0", fname, "d"), ("r", fname, "b", "range"), ("w", fname, "a", "rows"), ("p", fname, "e", "partition"),
               ("w2", fname, "a", ("rows", None, 0)), ("p2", fname, "e", ["rows", None, None]), ("m", fname, "d", ("rows", -19, 0)),
               ("ce", fname, "b", ("rows", -3, 3)), ("f", fname, "a", ("rows", 0, None)), ("x", fname, "d", ("rows", -BIG, BIG))])
    assert st.funcs == [("d0", code, 0, "d", 1, None), ("r", code, 0, "b", 1, None), ("w", code, 0, "a", 2, None),
                        ("p", code, 0, "e", 3, None), ("w2", code, 0, "a", 2, None), ("p2", code, 0, "e", 3, None),
                        ("m", code, 0, "d", 4, None, (-19, 0)), ("ce", code, 0, "b", 4, None, (-3, 3)), ("f", code, 0, "a", 4, None, (0, UF)),
                        ("x", code, 0, "d", 4, None, (-BIG, BIG))]
    assert st.descriptors(TYPES) == [(code, 3, 1, 0, 0, 0), (code, 1, 1, 0, 0, 0), (code, 0, 2, 0, 0, 0), (code, 4, 3, 0, 0, 0),
                                     (code, 0, 2, 0, 0, 0), (code, 4, 3, 0, 0, 0), (code, 3, 4, 0, 0, 0), (code, 1, 4, 0, 0, 0),
                                     (code, 0, 4, 0, 0, 0), (code, 3, 4, 0, 0, 0)]
    assert st.frames() == [(UP, UF)] * 6 + [(-19, 0), (-3, 3), (0, UF), (-BIG, BIG)]


def test_mixed_with_other_functions():
    st = init([("rn", "row_number"), ("s", "sum", "d", ("rows", -2, 0)), ("v", "var", "d", ("rows", -2, 0)), ("lg", "lag", "a", 1),
               ("sd", "std", "a", "partition")])
    assert [f[1] for f in st.funcs] == [0, 6, 16, 13, 17]
    assert st.descriptors(TYPES) == [(0, -1, 0, 0, 0, 0), (6, 3, 4, 0, 0, 0), (16, 3, 4, 0, 0, 0), (13, 0, 0, 0, 1, 0), (17, 0, 3, 0, 0, 0)]


@pytest.mark.parametrize("f,msg", [
    (("x", "var", None), "unknown column None"),
    (("x", "std", "zz"), "unknown column 'zz'"),
    (("x", "var", "d", "groups"), "bad frame"),
    (("x", "var", "d", 3), "bad frame"),
    (("x", "std_pop", "d", "rows", 1), "bad frame"),
    (("x", "var_pop", "d", ("rows", 2, 1)), "frame start 2 is after frame end 1"),
    (("x", "std", "d", ("rows", -(1 << 31), 0)), "bad frame bound"),
    (("x", "var", "d", ("range", -1, 0)), "bad frame"),
])
def test_errors_name_the_entry(f, msg):
    with pytest.raises(B200Error, match=msg) as e:
        init([f])
    assert repr(f) in str(e.value)


def test_unknown_function_message_lists_the_moments():
    with pytest.raises(B200Error) as e:
        init([("x", "variance", "d")])
    m = str(e.value)
    assert "unknown window function" in m and all(repr(f) in m for f in MOMENTS)
    assert "(out_name, fname, column[, frame])" in m and "'nth_value', column, n[, frame]" in m
    with pytest.raises(B200Error, match="unknown window function"):
        init([("x", "var")])


@pytest.mark.parametrize("fname", MOMENTS)
@pytest.mark.parametrize("frame", ["range", ("rows", -19, 0), ("rows", None, 0)])
def test_temporal_column_names_the_entry(fname, frame):
    st = init([("x", fname, "c", frame)])
    shown = ("rows", *[None if b in (UP, UF) else b for b in frame[1:]]) if isinstance(frame, tuple) else frame
    if shown == ("rows", None, 0):
        shown = "rows"
    with pytest.raises(B200Error, match=re.escape(repr(("x", fname, "c", shown))) + ".*var and std need an integer, bool or float column"):
        st.descriptors(TYPES)
    # every other type is accepted
    assert [d[0] for d in init([(f"x{c}", fname, c, frame) for c in "abde"]).descriptors(TYPES)] == [W.MOMENT_FUNCS[fname]] * 4


def test_sum_message_is_unchanged():
    with pytest.raises(B200Error, match="sum and mean need an integer, bool or float column"):
        init([("x", "mean", "c")]).descriptors(TYPES)


def test_header_documents_the_codes_and_declares_the_entry():
    with open(_lib.HEADER) as f:
        text = f.read()
    header = " ".join(re.sub(r"\n\s*\*", " ", text).split())
    assert "16 var, 17 std, 18 var_pop, 19 std_pop" in header
    assert "16 var = M2 / (m - 1), NA when m < 2" in header and "18 var_pop = M2 / m, NA when m = 0" in header
    assert "17 std = sqrt(var)" in header and "19 std_pop = sqrt(var_pop)" in header
    assert [s for s in _lib.declared_symbols() if s.startswith("b200_window_state_init")] == ["b200_window_state_init"]
    assert "13 lag, 14 lead, 15 nth_value" in header


def test_physical_window_plumbing():
    funcs = [("sd20", "std", "b", ("rows", -19, 0)), ("v", "var", "a", "rows"), ("sp", "std_pop", "d", "partition")]
    op = PhysicalWindow("a", ["b"], funcs)
    assert op.state is None
    assert op.args == ("a", ["b"], True, "last", funcs, False)
    op.Finalize()
