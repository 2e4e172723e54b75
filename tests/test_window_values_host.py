"""Host-side checks of the window operator's value functions: the tuple forms and their errors, the value codes against the
header, the ABI entry and descriptor, the descriptors built from the column types, and PhysicalWindow plumbing (no GPU needed)."""

import re

import numpy as np
import pytest

from bodo_b200 import _lib
from bodo_b200._lib import B200Error, ffi
from bodo_b200.physical import PhysicalWindow
from bodo_b200.streaming import window as W
from bodo_b200.table import Column, CTypes, Table

COLS = ["a", "b", "c", "d"]
TYPES = [CTypes.INT64, CTypes.FLOAT32, CTypes.DATETIME, CTypes.INT8]  # a, b, c, d


def init(funcs, **kw):
    args = dict(operator_id=-1, partition_by=["a"], order_by=["b"], ascending=True, na_position="last", funcs=funcs, col_names=COLS)
    args.update(kw)
    return W.init_window_state(**args)


def test_tuple_forms():
    st = init([("rn", "row_number"), ("s", "sum", "d"), ("r", "sum", "b", "rows"), ("p", "max", "c", "partition"),
               ("n", "count", None), ("f", "first_value", "a", "range"), ("l1", "lag", "d"), ("l2", "lead", "b", 0),
               ("l3", "lag", "c", (1 << 31) - 1, 5)])
    assert st.funcs == [("rn", 0, 0), ("s", 6, 0, "d", 1, None), ("r", 6, 0, "b", 2, None), ("p", 10, 0, "c", 3, None),
                        ("n", 7, 0, None, 1, None), ("f", 11, 0, "a", 1, None), ("l1", 13, 1, "d", 0, None), ("l2", 14, 0, "b", 0, None),
                        ("l3", 13, (1 << 31) - 1, "c", 0, 5)]
    assert st.out_names[4:] == ["rn", "s", "r", "p", "n", "f", "l1", "l2", "l3"]
    assert [st.out_names[i] for i in st.out_order] == COLS + ["rn", "s", "r", "p", "n", "f", "l1", "l2", "l3"]
    # physical column indices: keys first (a, b), then c, d
    assert st.descriptors(TYPES) == [(0, -1, 0, 0, 0, 0), (6, 3, 1, 0, 0, 0), (6, 1, 2, 0, 0, 0), (10, 2, 3, 0, 0, 0), (7, -1, 1, 0, 0, 0),
                                     (11, 0, 1, 0, 0, 0), (13, 3, 0, 0, 1, 0), (14, 1, 0, 0, 0, 0), (13, 2, 0, 1, (1 << 31) - 1, 5)]


@pytest.mark.parametrize("ct,default,bits", [
    (CTypes.INT8, -1, 0xFF), (CTypes.INT64, -(1 << 63), 1 << 63), (CTypes.UINT64, (1 << 64) - 1, (1 << 64) - 1),
    (CTypes.FLOAT32, 0.5, 0x3F000000), (CTypes.FLOAT64, -2.0, 0xC000000000000000), (CTypes.FLOAT64, float("nan"), 0x7FF8000000000000),
    (CTypes.BOOL, True, 1), (CTypes.INT16, 3.0, 3), (CTypes.DATE, 19000, 19000),
])
def test_default_bits(ct, default, bits):
    st = init([("l", "lead", "d", 1, default)])
    assert st.descriptors([CTypes.INT64, CTypes.INT64, CTypes.INT64, ct])[0] == (14, 3, 0, 1, 1, bits)


@pytest.mark.parametrize("ct,default", [(CTypes.INT8, 128), (CTypes.INT8, 0.5), (CTypes.UINT8, -1), (CTypes.INT64, 1 << 63),
                                        (CTypes.UINT64, 1 << 64), (CTypes.FLOAT32, 0.1), (CTypes.FLOAT32, 1e300), (CTypes.INT32, "x")])
def test_default_must_round_trip(ct, default):
    st = init([("l", "lag", "d", 2, default)])
    with pytest.raises(B200Error, match="not exactly representable"):
        st.descriptors([CTypes.INT64, CTypes.INT64, CTypes.INT64, ct])


@pytest.mark.parametrize("fname", ["sum", "mean"])
def test_sum_and_mean_of_a_temporal_column(fname):
    st = init([("x", fname, "c", "rows")])
    with pytest.raises(B200Error, match=r"\('x', '%s', 'c', 'rows'\).*sum and mean need" % fname):
        st.descriptors(TYPES)
    assert init([("x", "min", "c")]).descriptors(TYPES) == [(9, 2, 1, 0, 0, 0)]


def test_type_errors_surface_at_the_first_consume_without_a_device():
    n = 3
    t = Table([Column(np.zeros(n, np.int64)), Column(np.zeros(n, np.float32)), Column(np.zeros(n, np.int64), None, CTypes.DATETIME),
               Column(np.zeros(n, np.int8))], COLS)
    st = init([("s", "sum", "c")])
    with pytest.raises(B200Error, match="sum and mean need"):
        W.window_build_consume_batch(st, t, True)
    assert st.handle is None


@pytest.mark.parametrize("f,msg", [
    (("x", "sum", "zz"), "unknown column 'zz'"),
    (("x", "sum", None), "unknown column None"),
    (("x", "lag", None), "unknown column None"),
    (("x", "sum", "d", "groups"), "bad frame"),
    (("x", "sum", "d", 3), "bad frame"),
    (("x", "max", "d", "rows", 1), "bad frame"),
    (("x", "lag", "d", "rows"), "lag takes no frame"),
    (("x", "lead", "d", "partition"), "lead takes no frame"),
    (("x", "lag", "d", -1), "0 <= k < 2\\^31"),
    (("x", "lead", "d", 1 << 31), "0 <= k < 2\\^31"),
    (("x", "lag", "d", 1.0), "0 <= k < 2\\^31"),
    (("x", "lag", "d", True), "0 <= k < 2\\^31"),
    (("x", "lag", "d", 1, 0, 0), "lag takes"),
    (("x", "sum"), "unknown window function"),
    (("x", "lag"), "unknown window function"),
    (("x", "median", "d"), "unknown window function"),
])
def test_entry_errors_name_the_entry(f, msg):
    with pytest.raises(B200Error, match=msg) as e:
        init([f])
    assert repr(f) in str(e.value)


def test_unknown_function_message_names_both_forms():
    with pytest.raises(B200Error) as e:
        init([("x", "sum")])
    m = str(e.value)
    assert "unknown window function" in m and "(out_name, fname)" in m and "(out_name, fname, column[, frame])" in m
    assert "'lag' | 'lead', column[, k[, default]]" in m


def test_names_and_column_limit_count_value_functions():
    with pytest.raises(B200Error, match="duplicate output names"):
        init([("x", "sum", "d"), ("x", "rank")])
    with pytest.raises(B200Error, match="clash with input columns"):
        init([("d", "sum", "d")])
    with pytest.raises(B200Error, match="exceed 32 output columns"):
        init([(f"f{i}", "lag", "d") for i in range(29)])
    assert len(init([(f"f{i}", "lag", "d") for i in range(28)]).funcs) == 28


def test_value_codes_match_the_header():
    with open(_lib.HEADER) as f:
        header = " ".join(re.sub(r"\n\s*\*", " ", f.read()).split())  # comment lines joined without their leading " * "
    assert ("0 row_number, 1 rank, 2 dense_rank, 3 percent_rank, 4 cume_dist, 5 ntile (the ranking functions above), then the value "
            "functions 6 sum, 7 count, 8 mean, 9 min, 10 max, 11 first_value, 12 last_value, 13 lag, 14 lead") in header
    assert "1 range" in header and "2 rows" in header and "3 partition" in header
    assert W.VALUE_FUNCS == {"sum": 6, "count": 7, "mean": 8, "min": 9, "max": 10, "first_value": 11, "last_value": 12, "lag": 13, "lead": 14}
    assert W.FRAMES == {"range": 1, "rows": 2, "partition": 3}
    assert W.FUNCS == {"row_number": 0, "rank": 1, "dense_rank": 2, "percent_rank": 3, "cume_dist": 4, "ntile": 5}


def test_abi_declares_the_entry_and_descriptor():
    assert [s for s in _lib.declared_symbols() if s.startswith("b200_window_state_init")] == ["b200_window_state_init"]
    assert ffi.sizeof("b200_window_func") == 80
    assert [name for name, _ in ffi.typeof("b200_window_func").fields] == ["code", "col", "frame", "default_valid", "arg", "default_bits",
                                                                          "rows", "range", "ignore_nulls"]


def test_physical_window_plumbing():
    funcs = [("rn", "row_number"), ("s", "sum", "b", "rows"), ("l", "lead", "a", 2, 0)]
    op = PhysicalWindow("a", ["b"], funcs, ascending=False, na_position="first")
    assert op.state is None
    assert op.args == ("a", ["b"], False, "first", funcs, False)
    op.Finalize()
