"""Host-side checks of RANGE frames with value offsets (("range_between", start, end)): parsing and normalisation of every
bound form, the b200_window_range kinds and bits per ORDER BY key type, errors naming the entry, the header's codes, struct and
entry, and PhysicalWindow plumbing (no GPU needed)."""

import datetime
import re
import struct

import numpy as np
import pandas as pd
import pytest

from bodo_b200 import _lib
from bodo_b200._lib import B200Error, ffi
from bodo_b200.physical import PhysicalWindow
from bodo_b200.streaming import window as W
from bodo_b200.table import CTypes

COLS = ["a", "t", "x"]
RB = W.RANGE_BETWEEN
UP, UF = W.UNBOUNDED_PRECEDING, W.UNBOUNDED_FOLLOWING
K = W.RANGE_KINDS


def init(funcs, order=("t",), **kw):
    args = dict(operator_id=-1, partition_by=["a"], order_by=list(order), ascending=True, na_position="last", funcs=funcs, col_names=COLS)
    args.update(kw)
    return W.init_window_state(**args)


def dbits(x):
    return struct.unpack("<Q", struct.pack("<d", x))[0]


def test_codes():
    assert W.RANGE_BETWEEN == 5 and W.ROWS_BETWEEN == 4
    assert W.FRAMES == {"range": 1, "rows": 2, "partition": 3}
    assert W.RANGE_KINDS == {"unbounded_preceding": 0, "preceding": 1, "current_row": 2, "following": 3, "unbounded_following": 4}


@pytest.mark.parametrize("fname", W.BOUNDED_FUNCS)
def test_every_function_parses(fname):
    f = ("o", fname, "x", 3, ("range_between", -2, 5)) if fname == "nth_value" else ("o", fname, "x", ("range_between", -2, 5))
    st = init([f])
    assert st.funcs[0][4] == RB and st.funcs[0][-1] == (-2, 5)
    assert st.ranges([CTypes.INT64, CTypes.INT32, CTypes.FLOAT64]) == [(K["preceding"], K["following"], 2, 5)]
    assert st.frames() == [(UP, UF)]


def test_normalisation():
    st = init([("r", "sum", "x", ("range_between", None, 0)), ("r2", "sum", "x", ("range_between", None, -0.0)),
               ("r3", "sum", "x", ("range_between", None, np.timedelta64(0, "ns"))), ("p", "sum", "x", ("range_between", None, None)),
               ("c", "sum", "x", ("range_between", 0, 0)), ("c2", "sum", "x", ("range_between", -0.0, datetime.timedelta(0))),
               ("u", "sum", "x", ("range_between", 0, None))])
    assert [f[4] for f in st.funcs] == [1, 1, 1, 3, RB, RB, RB]
    assert st.funcs[4][-1] == (0, 0) and st.funcs[5][-1] == (0, 0) and st.funcs[6][-1] == (0, None)
    r = st.ranges([CTypes.INT64, CTypes.BOOL, CTypes.FLOAT64])  # no offsets: any key type, the bool key included
    assert r[4:] == [(2, 2, 0, 0), (2, 2, 0, 0), (2, 4, 0, 0)]
    assert r[:4] == [(0, 4, 0, 0)] * 4


@pytest.mark.parametrize("ct,start,end,bits", [
    (CTypes.INT64, -(1 << 63) + 1, (1 << 63) - 1, ((1 << 63) - 1, (1 << 63) - 1)),
    (CTypes.UINT64, np.int64(-5), np.uint8(7), (5, 7)),
    (CTypes.INT8, -300, 0, (300, 0)),
    (CTypes.FLOAT64, -0.5, 1e16, (dbits(0.5), dbits(1e16))),
    (CTypes.FLOAT32, -3, np.float32(2.5), (dbits(3.0), dbits(2.5))),
    (CTypes.FLOAT64, -(2 ** 53), 2 ** 60, (dbits(2.0 ** 53), dbits(2.0 ** 60))),
    (CTypes.DATETIME, -pd.Timedelta("1h"), np.timedelta64(3, "us"), (3_600 * 10 ** 9, 3000)),
    (CTypes.TIMEDELTA, -datetime.timedelta(days=1, microseconds=5), np.timedelta64(7000, "ps"), (86_400 * 10 ** 9 + 5000, 7)),
    (CTypes.DATE, -np.timedelta64(2, "W"), pd.Timedelta(days=3), (14, 3)),
    (CTypes.DATE, -np.timedelta64(48, "h"), datetime.timedelta(days=1), (2, 1)),
])
def test_bits_per_key_type(ct, start, end, bits):
    st = init([("s", "count", "x", ("range_between", start, end))])
    assert st.ranges([CTypes.INT64, ct, CTypes.FLOAT64])[0][2:] == bits


def test_descending_and_kinds():
    st = init([("a1", "sum", "x", ("range_between", 2, 5)), ("a2", "min", "x", ("range_between", -5, -2)),
               ("a3", "count", None, ("range_between", None, -1)), ("a4", "max", "x", ("range_between", 1, None))], ascending=False)
    assert st.ranges([CTypes.INT64, CTypes.INT64, CTypes.INT64]) == [(3, 3, 2, 5), (1, 1, 5, 2), (0, 1, 0, 1), (3, 4, 1, 0)]


@pytest.mark.parametrize("f,msg", [
    (("y", "sum", "x", ("range_between", 2, 1)), "frame start 2 is after frame end 1"),
    (("y", "sum", "x", ("range_between", 1, 0)), "frame start 1 is after frame end 0"),
    (("y", "sum", "x", ("range_between", 0, -pd.Timedelta("1s"))), "is after frame end"),
    (("y", "sum", "x", ("range_between", "7D", 0)), "bad frame bound '7D'"),
    (("y", "sum", "x", ("range_between", True, 0)), "bad frame bound True"),
    (("y", "sum", "x", ("range_between", -np.inf, 0)), "bad frame bound"),
    (("y", "sum", "x", ("range_between", np.nan, 0)), "bad frame bound"),
    (("y", "sum", "x", ("range_between", np.timedelta64("NaT"), 0)), "bad frame bound"),
    (("y", "sum", "x", ("range_between", -np.timedelta64(1, "M"), 0)), "bad frame bound"),
    (("y", "sum", "x", ("range_between", -np.timedelta64(1, "ps"), 0)), "bad frame bound"),
    (("y", "sum", "x", ("range_between", -(1 << 63), 0)), "bad frame bound"),
    (("y", "sum", "x", ("range_between", -1)), "bad frame"),
    (("y", "sum", "x", ("range", -1, 0)), "bad frame"),
    (("y", "lag", "x", ("range_between", -1, 0)), "lag takes no frame"),
])
def test_errors_name_the_entry(f, msg):
    with pytest.raises(B200Error, match=re.escape(msg) if "'" in msg else msg) as e:
        init([f])
    assert repr(f) in str(e.value)


def test_ranking_function_takes_no_frame():
    with pytest.raises(B200Error, match="takes no argument"):
        init([("r", "row_number", ("range_between", -1, 0))])


@pytest.mark.parametrize("order", [(), ("t", "x")])
def test_offsets_need_exactly_one_order_key(order):
    f = ("s", "sum", "x", ("range_between", -1, 0))
    with pytest.raises(B200Error, match="needs exactly one ORDER BY key") as e:
        init([f], order=order)
    assert repr(f) in str(e.value)
    # CURRENT ROW and UNBOUNDED need no key, or take several
    init([("c", "sum", "x", ("range_between", 0, None)), ("d", "count", None, ("range_between", 0, 0))], order=order)


@pytest.mark.parametrize("ct,bound", [
    (CTypes.INT64, -1.5), (CTypes.INT32, -pd.Timedelta("1s")), (CTypes.UINT8, -2.0), (CTypes.BOOL, -1),
    (CTypes.FLOAT64, -pd.Timedelta("1s")), (CTypes.FLOAT64, -(2 ** 53 + 1)),
    (CTypes.DATETIME, -5), (CTypes.TIMEDELTA, -5.0), (CTypes.DATE, -3), (CTypes.DATE, -pd.Timedelta("36h")),
])
def test_offset_type_errors_name_the_entry(ct, bound):
    f = ("s", "count", "x", ("range_between", bound, 0))
    st = init([f])
    with pytest.raises(B200Error, match="does not fit ORDER BY key 't'") as e:
        st.ranges([CTypes.INT64, ct, CTypes.FLOAT64])
    assert repr(f) in str(e.value)


def test_temporal_sum_message_shows_the_range_frame():
    st = init([("s", "sum", "x", ("range_between", -1, 0))])
    with pytest.raises(B200Error, match=re.escape(repr(("s", "sum", "x", ("range_between", -1, 0)))) + ".*sum and mean need"):
        st.descriptors([CTypes.INT64, CTypes.INT64, CTypes.DATETIME])


def test_mixed_with_other_frames():
    st = init([("rn", "row_number"), ("m", "sum", "x", ("rows", -2, 0)), ("r", "sum", "x", ("range_between", -2, 0)), ("lg", "lag", "x", 1)])
    assert st.descriptors([CTypes.INT64, CTypes.INT64, CTypes.INT64]) == [(0, -1, 0, 0, 0, 0), (6, 2, 4, 0, 0, 0), (6, 2, 5, 0, 0, 0),
                                                                         (13, 2, 0, 0, 1, 0)]
    assert st.frames() == [(UP, UF), (-2, 0), (UP, UF), (UP, UF)]
    assert st.ranges([CTypes.INT64] * 3) == [(0, 4, 0, 0), (0, 4, 0, 0), (1, 2, 2, 0), (0, 4, 0, 0)]


def test_header_declares_the_struct_and_entry():
    with open(_lib.HEADER) as f:
        text = f.read()
    header = " ".join(re.sub(r"\n\s*\*", " ", text).split())
    assert "0 UNBOUNDED PRECEDING, 1 PRECEDING, 2 CURRENT ROW, 3 FOLLOWING, 4 UNBOUNDED FOLLOWING" in header
    assert "5 range between" in header and "4 rows between" in header
    assert ffi.sizeof("b200_window_range") == 24
    assert ffi.sizeof("b200_window_frame") == 16 and ffi.sizeof("b200_window_func") == 80
    assert dict(ffi.typeof("b200_window_func").fields)["range"].type is ffi.typeof("b200_window_range")
    assert [s for s in _lib.declared_symbols() if s.startswith("b200_window_state_init")] == ["b200_window_state_init"]


def test_physical_window_plumbing():
    funcs = [("s1h", "sum", "amount", ("range_between", -pd.Timedelta("1h"), 0)), ("c", "count", None, ("range_between", -0.5, 0.5))]
    op = PhysicalWindow("acct", ["ts"], funcs)
    assert op.state is None
    assert op.args == ("acct", ["ts"], True, "last", funcs, False)
    op.Finalize()
