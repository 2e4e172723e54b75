"""The fused filter + projection kernel (csrc/expr.cu: filter_project_kernel behind b200_filter_project) and dictionary
unification (dictionary.py + remap_i32_kernel) against an exact reference.

`ref_eval` below evaluates an Expr TREE with numpy (not the compiled postfix program, so compile_program is checked as well)
and states the semantics of the VM:

* column loads: integers widen exactly to int64, a uint64 column keeps its value (kind "u"); floats widen to float64 and NaN
  read from a float column is NA; NaT in a datetime / timedelta column is NA (the host turns it into a null);
* + - * and negation of integers are int64 and wrap; `/` is true division in float64; a NaN or +-inf made by arithmetic is a
  valid value; a uint64 operand of arithmetic is its int64 bit pattern;
* comparisons with a float operand are done in float64 (a float32 column compares as its exact double); integer comparisons
  are exact, uint64 values >= 2^63 included;
* arithmetic and comparisons propagate NA; and / or / not are Kleene with truthiness value != 0 (-0.0 is false, NaN true);
  a NA or false predicate drops the row; isnull is always valid;
* astype(int) truncates toward zero (NaN and out-of-range values are left untested: the device saturates, numpy's result is
  undefined);
* the value stored to an output is converted to the output's type (physical._infer_ctype) as numpy astype converts it.

Kernel results are compared bit-exactly (float64 included: one IEEE operation per VM instruction, no fast-math), NA masks
exactly, data under NA ignored.  Output order across 1024-row tiles is unspecified (each tile claims its place with an atomic
cursor), so every kernel test passes a row id through and sorts both sides by it, which also checks that the output columns
stay row-aligned.
"""

import datetime
import functools

import numpy as np
import pandas as pd
import pyarrow as pa
import pytest

from bodo_b200 import _lib
from bodo_b200._lib import B200Error, ffi
from bodo_b200.dictionary import DictionaryBuilder
from bodo_b200.expr import OPS, col, lit
from bodo_b200.physical import (OperatorResult, PhysicalAggregate, PhysicalFilterProject, PhysicalReadArrowDevice, ResultCollector,
                                _infer_ctype, filter_project_table, run_pipeline)
from bodo_b200.table import ArrTypes, Column, CTable, CTypes, Table, column_to_pandas, np_dtype_of
from tests.helpers import table_to_device

I64_MIN, I64_MAX = -(1 << 63), (1 << 63) - 1
FLOATS = (CTypes.FLOAT32, CTypes.FLOAT64)
TILE = 1024


# ---------------------------------------------------------------------------------------------------------------- reference
def _load(ct, values, valid):
    if ct in FLOATS:
        v = values.astype(np.float64)
        return "f", v, valid & ~np.isnan(v)
    if ct == CTypes.UINT64:
        return "u", values.astype(np.uint64), valid.copy()
    return "i", values.astype(np.int64), valid.copy()


def _f64(kind, v):
    return v if kind == "f" else v.astype(np.float64)


def _i64(kind, v):
    return v.view(np.int64) if kind == "u" else v


def _int_lt_eq(kx, x, ky, y):
    """(x < y, x == y) of two integer operands by value (int64 or uint64)."""
    if kx == ky:
        return x < y, x == y
    if kx == "u":
        lt, eq = _int_lt_eq(ky, y, kx, x)
        return ~lt & ~eq, eq
    nonneg = x >= 0
    xu = np.where(nonneg, x, 0).astype(np.uint64)
    return ~nonneg | (xu < y), nonneg & (xu == y)


def ref_eval(e, cols):
    """(kind, values, valid) of Expr `e` over `cols` = {name: (ctype, storage values, valid bool array)}; kind is "i" (int64),
    "u" (a uint64 column's value) or "f" (float64)."""
    n = len(next(iter(cols.values()))[1])
    op = e.op
    if op == "col":
        return _load(*cols[e.value])
    if op == "const_i64":
        return "i", np.full(n, e.value, np.int64), np.ones(n, bool)
    if op == "const_f64":
        return "f", np.full(n, e.value, np.float64), np.ones(n, bool)
    args = [ref_eval(a, cols) for a in e.args]
    with np.errstate(all="ignore"):
        if op in ("add", "sub", "mul", "div"):
            (kx, x, vx), (ky, y, vy) = args
            f = {"add": np.add, "sub": np.subtract, "mul": np.multiply, "div": np.divide}[op]
            if op == "div" or "f" in (kx, ky):
                return "f", f(_f64(kx, x), _f64(ky, y)), vx & vy
            return "i", f(_i64(kx, x), _i64(ky, y)), vx & vy
        if op in ("lt", "le", "gt", "ge", "eq", "ne"):
            (kx, x, vx), (ky, y, vy) = args
            if "f" in (kx, ky):
                p, q = _f64(kx, x), _f64(ky, y)
                lt, eq = p < q, p == q
            else:
                lt, eq = _int_lt_eq(kx, x, ky, y)
            t = {"lt": lt, "le": lt | eq, "gt": ~(lt | eq), "ge": ~lt, "eq": eq, "ne": ~eq}[op]
            if "f" in (kx, ky):  # NaN is unordered: only != holds
                nan = np.isnan(p) | np.isnan(q)
                t = np.where(nan, op == "ne", t)
            return "i", t.astype(np.int64), vx & vy
        if op in ("and", "or"):
            (kx, x, vx), (ky, y, vy) = args
            xt, yt = vx & (x != 0), vy & (y != 0)
            xf, yf = vx & (x == 0), vy & (y == 0)
            if op == "and":
                return "i", (xt & yt).astype(np.int64), xf | yf | (vx & vy)
            return "i", (xt | yt).astype(np.int64), xt | yt | (vx & vy)
        (k, x, v), = args
        if op == "not":
            return "i", (x == 0).astype(np.int64), v
        if op == "neg":
            return ("f", -x, v) if k == "f" else ("i", 0 - _i64(k, x), v)
        if op == "to_f64":
            return "f", _f64(k, x), v
        if op == "to_i64":
            return "i", (np.trunc(x).astype(np.int64) if k == "f" else _i64(k, x)), v
        if op == "is_null":
            return "i", (~v).astype(np.int64), np.ones(n, bool)
    raise ValueError(op)


def ref_store(kind, x, ct):
    """A value converted to output type `ct` as numpy astype does (for values the type holds)."""
    dt = np_dtype_of(ct)
    with np.errstate(all="ignore"):
        if ct == CTypes.BOOL:
            return x != 0
        if dt.kind == "f" or kind != "f":
            return x.astype(dt)
        return np.trunc(x).astype(np.uint64 if ct == CTypes.UINT64 else np.int64).astype(dt)


def ref_filter_project(cols, predicate, outputs):
    """(kept row mask, [(ctype, stored values, valid) per output]) over every input row."""
    n = len(next(iter(cols.values()))[1])
    keep = np.ones(n, bool)
    if predicate is not None:
        k, x, v = ref_eval(predicate, cols)
        keep = v & (x != 0)
    cts = {nm: c[0] for nm, c in cols.items()}
    outs = []
    for _, e in outputs:
        ct = _infer_ctype(e, cts)
        k, x, v = ref_eval(e, cols)
        outs.append((ct, ref_store(k, x, ct), v))
    return keep, outs


# ------------------------------------------------------------------------------------------------------------ comparisons
def _same_values(got, exp):
    """Element-wise bit equality (NaN equals NaN whatever its payload; -0.0 differs from 0.0)."""
    got, exp = np.asarray(got), np.asarray(exp)
    if exp.dtype == bool:
        return got.view(np.uint8) == exp.view(np.uint8)
    if exp.dtype.kind == "f":
        bits = np.dtype(f"i{exp.dtype.itemsize}")
        return (got.view(bits) == exp.view(bits)) | (np.isnan(got) & np.isnan(exp))
    return got == exp


def _assert_column(name, got_vals, got_valid, exp_vals, exp_valid):
    got_valid = np.ones(len(got_vals), bool) if got_valid is None else got_valid
    np.testing.assert_array_equal(got_valid, exp_valid, err_msg=f"{name}: NA mask")
    assert got_vals.dtype == exp_vals.dtype, (name, got_vals.dtype, exp_vals.dtype)
    bad = np.flatnonzero(~_same_values(got_vals[exp_valid], exp_vals[exp_valid]))
    assert bad.size == 0, f"{name}: {bad.size} values differ, first at valid row {bad[0]}: got {got_vals[exp_valid][bad[0]]!r}, " \
                          f"expected {exp_vals[exp_valid][bad[0]]!r}"


def check_filter_project(table, cols, predicate, outputs, rid="rid", op=None):
    """Run `table` (host or device) through PhysicalFilterProject and compare with the reference over `cols`; `rid` is the name
    of an output that passes the row id (0..n-1) through."""
    op = op or PhysicalFilterProject(predicate, outputs)
    res, _ = op.ProcessBatch(table, OperatorResult.NEED_MORE_INPUT)
    keep, exp = ref_filter_project(cols, predicate, outputs)
    names = [nm for nm, _ in outputs]
    assert res.n_rows == int(keep.sum()), (res.n_rows, int(keep.sum()))
    got = {nm: (c.values_numpy(), c.valid_mask_numpy()) for nm, c in zip(names, res.columns)}
    order = np.argsort(got[rid][0], kind="stable")
    np.testing.assert_array_equal(got[rid][0][order], np.flatnonzero(keep), err_msg="kept row ids")
    for nm, c, (ct, vals, valid) in zip(names, res.columns, exp):
        assert c.c_type == ct, (nm, c.c_type, ct)
        gv, gm = got[nm]
        _assert_column(nm, gv[order], None if gm is None else gm[order], vals[keep], valid[keep])
    return res


# ------------------------------------------------------------------------------------------------------------ test inputs
DTYPES = ["int8", "int16", "int32", "int64", "uint8", "uint16", "uint32", "uint64", "float32", "float64", "bool", "date32",
          "datetime", "timedelta"]
_CT = {"date32": CTypes.DATE, "datetime": CTypes.DATETIME, "timedelta": CTypes.TIMEDELTA}


def gen_values(dt, n, rng):
    """Storage values of a column of dtype `dt` spanning its range, its edge values first."""
    if dt == "bool":
        return rng.random(n) < 0.5
    if dt in ("float32", "float64"):
        f = np.dtype(dt)
        fi = np.finfo(f)
        v = (rng.standard_normal(n) * 10.0 ** rng.integers(-3, 4, n)).astype(f)
        v[rng.random(n) < 0.05] = np.nan
        edge = np.array([0.0, -0.0, np.inf, -np.inf, np.nan, fi.smallest_subnormal, -fi.max, 0.1, 0.5, -2.7], dtype=f)
    elif dt == "date32":
        v = rng.integers(-20000, 40000, n).astype(np.int32)
        edge = np.array([0, -1, -20000, 39999], np.int32)
    elif dt in ("datetime", "timedelta"):
        v = rng.integers(-(1 << 62), 1 << 62, n, dtype=np.int64)
        edge = np.array([0, -1, 1, I64_MAX], np.int64)
    else:
        info = np.iinfo(dt)
        v = rng.integers(info.min, info.max, n, dtype=dt, endpoint=True)
        edge = np.array(sorted({info.min, info.max, 0, 1, info.max // 2, info.max // 2 + 1} | ({-1} if info.min < 0 else set())), dt)
    m = min(n, len(edge))
    v[:m] = edge[:m]
    return v


def threshold(dt):
    return {"bool": 1, "float32": 0.0, "float64": 0.0, "uint8": 128, "uint16": 1 << 15, "uint32": 1 << 31, "uint64": 1 << 62}.get(dt, 0)


def make_column(dt, values, valid, source):
    """Host Column of `values` with NA where not `valid`, built the way a user would: pandas numpy dtype, pandas nullable
    dtype, or an Arrow array sliced at an offset that is not a multiple of 8.  Datetime / timedelta NA is NaT in pandas."""
    n = len(values)
    if dt in ("datetime", "timedelta") and source != "arrow_offset":
        raw = np.where(valid, values, np.int64(I64_MIN))  # NaT
        s = pd.Series(raw.view("datetime64[ns]" if dt == "datetime" else "timedelta64[ns]"))
        return Table.from_pandas(pd.DataFrame({"x": s})).columns[0]
    if dt == "date32" or source == "arrow_offset":
        pad = 5
        vals = np.concatenate([np.zeros(pad, values.dtype), values])
        mask = np.concatenate([np.zeros(pad, bool), ~valid])
        a = pa.array(vals, mask=mask if mask.any() else None)
        if dt in _CT:
            a = a.view({"date32": pa.date32(), "datetime": pa.timestamp("ns"), "timedelta": pa.duration("ns")}[dt])
        return Table.from_arrow(pa.RecordBatch.from_arrays([a.slice(pad)], ["x"])).columns[0]
    if source == "numpy":
        assert valid.all()
        return Table.from_pandas(pd.DataFrame({"x": values})).columns[0]
    cls = {"b": pd.arrays.BooleanArray, "f": pd.arrays.FloatingArray}.get(values.dtype.kind, pd.arrays.IntegerArray)
    return Table.from_pandas(pd.DataFrame({"x": cls(values.copy(), ~valid)})).columns[0]


def _ref_valid(dt, values, valid):
    """What the reference sees as valid: NaN in a float column is handled by the load, NaT is NA."""
    return valid & (values != I64_MIN) if dt in ("datetime", "timedelta") else valid.copy()


def build_inputs(spec, n, seed):
    """spec: [(name, dtype, source, null fraction)] -> (host Table with a leading int64 'rid' column, reference columns)."""
    rng = np.random.default_rng(seed)
    cols = {"rid": (CTypes.INT64, np.arange(n, dtype=np.int64), np.ones(n, bool))}
    tcols = [Column(np.arange(n, dtype=np.int64), None, CTypes.INT64)]
    for name, dt, source, pnull in spec:
        v = gen_values(dt, n, rng)
        valid = rng.random(n) >= pnull if source != "numpy" else np.ones(n, bool)
        if dt in ("datetime", "timedelta") and source == "numpy":
            valid = rng.random(n) >= 0.05   # NaT in a numpy column
        c = make_column(dt, v, valid, source)
        cols[name] = (c.c_type, v, _ref_valid(dt, v, valid))
        tcols.append(c)
    return Table(tcols, ["rid"] + [s[0] for s in spec]), cols


def G():
    import torch

    return torch.cuda.get_device_properties(0).multi_processor_count * 8 * TILE


# ============================================================================================ CPU: the reference itself
def _pd_cols(df):
    cts = {"Int64": CTypes.INT64, "Float64": CTypes.FLOAT64, "boolean": CTypes.BOOL}
    return {c: (cts[str(df[c].dtype)], df[c].array._data.copy(), ~df[c].isna().to_numpy()) for c in df.columns}


def test_reference_evaluator_matches_pandas_nullable():
    """Where the semantics coincide (no NaN, no overflow, no division by zero), ref_eval equals pandas' nullable arrays."""
    rng = np.random.default_rng(5)
    n = 5000
    na = lambda: rng.random(n) < 0.15  # noqa: E731
    df = pd.DataFrame({"a": pd.arrays.IntegerArray(rng.integers(-1000, 1000, n), na()),
                       "b": pd.arrays.IntegerArray(rng.integers(-1000, 1000, n), na()),
                       "x": pd.arrays.FloatingArray(rng.uniform(0.5, 4.0, n) * rng.choice([-1, 1], n), na()),
                       "p": pd.arrays.BooleanArray(rng.random(n) < 0.5, na()),
                       "q": pd.arrays.BooleanArray(rng.random(n) < 0.5, na())})
    cols = _pd_cols(df)
    a, b, x, p, q = (df[c] for c in "abxpq")
    cases = [(col("a") + col("b") * 3 - 2, a + b * 3 - 2), (-col("a"), -a), (col("a") / col("x"), a / x),
             (col("x") * 2.5 + col("a"), x * 2.5 + a), (col("a") / 4, a / 4), (col("a") < col("b"), a < b),
             (col("x") >= 0.5, x >= 0.5), (col("a") == 3, a == 3), (col("a") != col("b"), a != b), (col("x") <= col("a"), x <= a),
             ((col("a") < col("b")) & col("p"), (a < b) & p), (col("p") | col("q"), p | q), (~col("p"), ~p),
             (~(col("x") > 0) | (col("a") > 500), ~(x > 0) | (a > 500)), (col("a").isnull(), a.isna()),
             (col("a").astype(float), a.astype("Float64")), (col("p") & (col("q") | (col("b") > 0)), p & (q | (b > 0)))]
    for e, s in cases:
        k, v, valid = ref_eval(e, cols)
        exp_valid = ~s.isna().to_numpy()
        np.testing.assert_array_equal(valid, exp_valid)
        ev = s.to_numpy(dtype="float64", na_value=np.nan)[exp_valid]
        np.testing.assert_array_equal(v[valid].astype(np.float64), ev)


def test_reference_evaluator_on_hand_computed_rows():
    """Where the project differs from pandas' nullable arrays, ref_eval gives the values stated in the module docstring."""
    f = np.array([np.nan, -0.0, 0.0, 1.5, np.inf])
    i = np.array([I64_MAX, I64_MIN, -1, 0, 3], np.int64)
    f32 = np.array([0.1, 0.5, -0.0, 1.0, 2.0], np.float32)
    u = np.array([1 << 63, (1 << 64) - 1, 0, 5, (1 << 63) - 1], np.uint64)
    ones = np.ones(5, bool)
    cols = {"f": (CTypes.FLOAT64, f, ones), "i": (CTypes.INT64, i, ones), "f32": (CTypes.FLOAT32, f32, ones), "u": (CTypes.UINT64, u, ones)}
    ev = lambda e: ref_eval(e, cols)  # noqa: E731
    _, _, valid = ev(col("f"))
    assert valid.tolist() == [False, True, True, True, True]                       # NaN read from a float column is NA
    assert ev(col("f").isnull())[1].tolist() == [1, 0, 0, 0, 0]
    _, v, valid = ev(col("f") - col("f"))                                          # inf - inf: a valid NaN
    assert valid[4] and np.isnan(v[4]) and not ev((col("f") - col("f")).isnull())[1][4]
    assert ev(col("i") + 1)[1][0] == I64_MIN and ev(-col("i"))[1][1] == I64_MIN   # int64 wraps
    assert ev(col("i") * 2)[1].tolist() == [-2, 0, -2, 0, 6]
    assert ev(~col("f"))[1].tolist()[1:] == [1, 1, 0, 0]                          # -0.0 and 0.0 are false
    assert ev(col("f") | lit(False))[1].tolist()[1:] == [0, 0, 1, 1]
    assert ev(col("f32") == 0.1)[1][0] == 0 and ev(col("f32") == float(np.float32(0.1)))[1][0] == 1 and ev(col("f32") > 0.1)[1][0] == 1
    assert ev(col("u") > 0)[1].tolist() == [1, 1, 0, 1, 1] and ev(col("u") == -1)[1].tolist() == [0] * 5
    assert ev(col("u") > col("i"))[1].tolist() == [1, 1, 1, 1, 1]                  # 2^63 > INT64_MAX, 2^64 - 1 > INT64_MIN
    assert ev(lit(I64_MAX) < col("u"))[1].tolist() == [1, 1, 0, 0, 0]
    assert ev(lit(-2.7).astype(int))[1][0] == -2 and ev(lit(2.7).astype(int))[1][0] == 2
    k, v, _ = ev(col("i") / 0)
    assert k == "f" and v[0] == np.inf and v[1] == -np.inf and np.isnan(v[3])
    assert ref_store("f", np.array([-3.7, 2.9, -0.0, 0.5]), CTypes.INT8).tolist() == [-3, 2, 0, 0]
    assert ref_store("f", np.array([-3.7, 0.0, -0.0, 0.5]), CTypes.BOOL).tolist() == [True, False, False, True]
    assert ref_store("i", np.array([5, 0, 70000]), CTypes.BOOL).tolist() == [True, False, True]
    assert ref_store("i", np.array([70000]), CTypes.INT16).tolist() == [4464]


# ============================================================================================ CPU: host-side conversions
def test_nat_in_numpy_temporal_columns_is_na():
    df = pd.DataFrame({"ts": pd.to_datetime(["2020-01-01", None, "1969-12-31"]), "td": pd.to_timedelta(["1s", "2s", None])})
    t = Table.from_pandas(df)
    for c, exp in zip(t.columns, ([True, False, True], [True, True, False])):
        assert c.arr_type == ArrTypes.NULLABLE_INT_BOOL
        assert c.valid_mask_numpy().tolist() == exp
    back = t.to_pandas()
    assert back["ts"].isna().tolist() == [False, True, False] and back["td"].isna().tolist() == [False, False, True]
    assert Table.from_pandas(df.iloc[[0, 2]]).columns[0].validity is None     # no NaT: stays a NUMPY column


def test_nullable_bool_column_reads_back_with_its_nas():
    c = Column(np.array([True, False, True, False]), np.packbits(np.array([1, 1, 0, 0], bool), bitorder="little"), CTypes.BOOL,
               ArrTypes.NULLABLE_INT_BOOL, 4)
    s = pd.Series(column_to_pandas(c))
    assert str(s.dtype) == "boolean" and s.isna().tolist() == [False, False, True, True] and s[:2].tolist() == [True, False]
    assert column_to_pandas(Column(np.array([True, False]), None, CTypes.BOOL)).dtype == bool   # NUMPY bools stay numpy


def test_filter_project_without_outputs_is_rejected():
    with pytest.raises(ValueError, match="at least one output"):
        PhysicalFilterProject(col("a") > 0, [])


# ============================================================================================ GPU: launch shape
ROW_COUNTS = ["0", "1", "31", "32", "33", "1023", "1024", "1025", "G-1", "G", "G+1", "3G+517"]
PREDICATES = ["none", "all", "nothing", "one_per_tile", "lane31", "slot3", "random"]


def _rows(spec):
    if "G" not in spec:
        return int(spec)
    g = G()
    return {"G-1": g - 1, "G": g, "G+1": g + 1, "3G+517": 3 * g + 517}[spec]


@functools.lru_cache(maxsize=None)
def _shape_inputs(n):
    rng = np.random.default_rng(n)
    rid = np.arange(n, dtype=np.int64)
    k = rng.integers(-(1 << 31), (1 << 31) - 1, n, dtype=np.int32)
    kv = rng.random(n) >= 0.1
    x = rng.standard_normal(n)
    x[rng.random(n) < 0.05] = np.nan
    pat = {"one_per_tile": rid % TILE == 517, "lane31": rid % 32 == 31, "slot3": (rid % TILE) // 256 == 3}
    pr, prv = rng.random(n) < 0.5, rng.random(n) >= 0.1
    df = pd.DataFrame({"rid": rid, "k": pd.arrays.IntegerArray(k, ~kv), "x": x, **{p: m.astype(np.uint8) for p, m in pat.items()},
                       "random": pd.arrays.BooleanArray(pr, ~prv)})
    cols = {"rid": (CTypes.INT64, rid, np.ones(n, bool)), "k": (CTypes.INT32, k, kv), "x": (CTypes.FLOAT64, x, np.ones(n, bool)),
            **{p: (CTypes.UINT8, m.astype(np.uint8), np.ones(n, bool)) for p, m in pat.items()}, "random": (CTypes.BOOL, pr, prv)}
    return table_to_device(Table.from_pandas(df)), cols


@pytest.mark.gpu
@pytest.mark.parametrize("pred", PREDICATES)
@pytest.mark.parametrize("rows", ROW_COUNTS)
def test_launch_shape_and_tile_edges(gpu_lib, rows, pred):
    """Row counts around the warp, tile and grid edges (G = SMs x 8 CTAs x 1024 rows: beyond it the grid-stride loop runs and
    wsum / tile_base are reused) under predicates that keep everything, nothing, one row per tile, one lane per warp, one row
    slot per tile, or a random half."""
    table, cols = _shape_inputs(_rows(rows))
    predicate = {"none": None, "all": col("rid") >= 0, "nothing": col("rid") < 0, "random": col("random")}.get(pred, col(pred))
    outs = [("rid", col("rid")), ("k", col("k")), ("x", col("x")), ("kk", col("k") * 3 - 1), ("xk", col("x") * 2.5 + col("k")),
            ("big", col("x") > 0.5), ("kn", col("k").isnull())]
    check_filter_project(table, cols, predicate, outs)


# ============================================================================================ GPU: every input dtype
def _sweep_outputs(dt):
    x, thr = col("x"), threshold(dt)
    outs = [("rid", col("rid")), ("x", x), ("add", x + 1), ("mul", x * 3), ("fmul", x * 2.5), ("div", x / 3), ("neg", -x),
            ("gt", x > lit(thr)), ("flt", x <= 0.5), ("isn", x.isnull()), ("not", ~x), ("or", x | col("m")), ("tof", x.astype(float))]
    if dt not in ("float32", "float64"):
        outs.append(("toi", x.astype(int)))
    return (x >= lit(thr)) | col("m"), outs


SOURCES = [(dt, s) for dt in DTYPES for s in ("numpy", "nullable", "arrow_offset") if not (dt == "bool" and s == "arrow_offset")]


@pytest.mark.gpu
@pytest.mark.parametrize("dt,source", SOURCES, ids=[f"{d}-{s}" for d, s in SOURCES])
def test_every_input_dtype(gpu_lib, dt, source):
    """Each dtype table.py accepts, as a NUMPY column, as a nullable one and as an Arrow array at offset 5, through arithmetic,
    comparisons, Kleene logic, casts and is-null, over a few tiles."""
    table, cols = build_inputs([("x", dt, source, 0.1), ("m", "bool", "nullable", 0.2)], 3001, seed=DTYPES.index(dt))
    predicate, outs = _sweep_outputs(dt)
    check_filter_project(table_to_device(table), cols, predicate, outs)


@pytest.mark.gpu
def test_every_dtype_passes_through_beyond_the_grid(gpu_lib):
    """All dtypes in one table of G + 1 rows: passthrough of every column while the grid-stride loop runs."""
    spec = [(f"c_{dt}", dt, "nullable" if dt != "date32" else "arrow_offset", 0.1) for dt in DTYPES] + [("m", "bool", "nullable", 0.3)]
    table, cols = build_inputs(spec, G() + 1, seed=11)
    outs = [("rid", col("rid"))] + [(nm, col(nm)) for nm, *_ in spec]
    check_filter_project(table_to_device(table), cols, col("m") | (col("c_int64") > 0), outs)


# ============================================================================================ GPU: values where kernels go wrong
def _value_table():
    f = np.array([0.0, -0.0, np.inf, -np.inf, np.nan, -2.7, 2.7, 1.5, -1.5, 1e300], np.float64)
    n = len(f)
    i = np.array([I64_MIN, I64_MAX, (1 << 53) + 1, -(1 << 53) - 1, 0, -1, 1, 7, -7, 1 << 62], np.int64)
    u = np.array([1 << 63, (1 << 64) - 1, 0, 1, (1 << 63) - 1, 5, (1 << 63) + 1, 1 << 62, 2, (1 << 64) - 2], np.uint64)
    w = np.array([(1 << 64) - 1, 1 << 63, 0, 1, 1 << 63, 5, 1 << 63, 7, 3, (1 << 64) - 1], np.uint64)
    u32 = np.array([1 << 31, (1 << 32) - 1, 0, 1, (1 << 31) - 1, 5, 3, 2, 1 << 31, 9], np.uint32)
    f32 = np.array([0.1, -0.0, 0.5, np.nan, -2.7, 1.0, np.inf, 3.0, 0.1, 2.0], np.float32)
    data = {"rid": np.arange(n, dtype=np.int64), "f": f, "i": i, "u": u, "w": w, "u32": u32, "f32": f32}
    ones = np.ones(n, bool)
    cols = {k: (Column(v).c_type, v, ones) for k, v in data.items()}
    return Table([Column(v) for v in data.values()], list(data)), cols


VALUE_OUTPUTS = [
    ("rid", col("rid")),
    ("i_add", col("i") + 1), ("i_sub", col("i") - 1), ("i_mul", col("i") * 3), ("i_sq", col("i") * col("i")), ("i_neg", -col("i")),
    ("i_eq_2p53", col("i") == 9007199254740992.0), ("i_gt_2p53", col("i") > 9007199254740992.0), ("i_gt_int", col("i") > (1 << 53)),
    ("u32_gt", col("u32") > (1 << 31) - 1), ("u32_add", col("u32") + 1), ("u32_f", col("u32") * 1.0),
    ("u_gt0", col("u") > 0), ("u_eq_m1", col("u") == -1), ("u_lt_i", col("u") < col("i")), ("u_ge_w", col("u") >= col("w")),
]
VALUE_OUTPUTS_2 = [
    ("rid", col("rid")),
    ("u_gt_f", col("u") > 9.2e18), ("u_f", col("u").astype(float)), ("u_eq_w", col("u") == col("w")), ("u_toi", col("u").astype(int)),
    ("f_not", ~col("f")), ("f_and", col("f") & lit(True)), ("f_or", col("f") | lit(False)), ("f_div0", col("f") / 0),
    ("i_div0", col("i") / 0), ("zz", (col("i") * 0) / 0), ("zz_null", ((col("i") * 0) / 0).isnull()), ("f_neg", -col("f")),
    ("f32_eq", col("f32") == 0.1), ("f32_eq32", col("f32") == float(np.float32(0.1))), ("f32_gt", col("f32") > 0.1),
]


@pytest.mark.gpu
@pytest.mark.parametrize("outs", [VALUE_OUTPUTS, VALUE_OUTPUTS_2], ids=["ints", "uint64-floats"])
def test_edge_values(gpu_lib, outs):
    """INT64_MIN / MAX under + x and negation, 2^53 + 1 against a float literal, uint32 >= 2^31, uint64 >= 2^63 against int
    literals, int64 and another uint64 column, +-0.0 / +-inf / NaN truthiness, x / 0 and 0 / 0, float32 0.1 against 0.1."""
    table, cols = _value_table()
    res = check_filter_project(table_to_device(table), cols, None, outs)
    got = res.to_pandas().set_index("rid").sort_index()
    if "u_gt0" in got:  # the hand-checked rows behind the reference (uint64 >= 2^63 is above every int64)
        assert got["u_gt0"].tolist() == [True, True, False, True, True, True, True, True, True, True]
        assert not got["u_eq_m1"].any() and got["u_lt_i"].tolist()[:2] == [False, False]
    else:
        assert got["f_not"].tolist()[:4] == [True, True, False, False] and pd.isna(got["f_not"].iloc[4])  # -0.0 is false


@pytest.mark.gpu
def test_astype_int_truncates_toward_zero(gpu_lib):
    f = np.array([-2.7, 2.7, -0.5, 0.5, -1e15 - 0.5, 3.0], np.float64)
    table = Table([Column(np.arange(6, dtype=np.int64)), Column(f)], ["rid", "f"])
    cols = {"rid": (CTypes.INT64, np.arange(6, dtype=np.int64), np.ones(6, bool)), "f": (CTypes.FLOAT64, f, np.ones(6, bool))}
    res = check_filter_project(table_to_device(table), cols, None, [("rid", col("rid")), ("t", col("f").astype(int))])
    assert sorted(res.columns[1].values_numpy().tolist()) == sorted([-2, 2, 0, 0, -1000000000000000, 3])


@pytest.mark.gpu
def test_predicate_truthiness_of_floats(gpu_lib):
    """A float predicate keeps a row when its value is != 0: -0.0 and 0.0 drop it, NaN read from the column is NA and drops it."""
    f = np.array([0.0, -0.0, 1.0, -1.0, np.nan, np.inf], np.float64)
    table = Table([Column(np.arange(6, dtype=np.int64)), Column(f)], ["rid", "f"])
    cols = {"rid": (CTypes.INT64, np.arange(6, dtype=np.int64), np.ones(6, bool)), "f": (CTypes.FLOAT64, f, np.ones(6, bool))}
    res = check_filter_project(table_to_device(table), cols, col("f"), [("rid", col("rid"))])
    assert sorted(res.columns[0].values_numpy().tolist()) == [2, 3, 5]


# ============================================================================================ GPU: program shapes
def _small_device_table(n_cols=1, n=100):
    rng = np.random.default_rng(3)
    data = {f"a{j}" if j else "rid": (rng.integers(-100, 100, n) if j else np.arange(n)).astype(np.int64) for j in range(max(n_cols, 1))}
    cols = {k: (CTypes.INT64, v, np.ones(n, bool)) for k, v in data.items()}
    return table_to_device(Table([Column(v) for v in data.values()], list(data))), cols


def _chain(e, k):
    for _ in range(k):
        e = e + 1
    return e


def _deep(depth):
    """A right-nested sum of `depth` leaves: the VM stack holds `depth` values at its deepest."""
    e = col("rid")
    for _ in range(depth - 1):
        e = col("rid") + e
    return e


@pytest.mark.gpu
def test_program_limits_accept_the_limit(gpu_lib):
    """Stack depth 8, 64 instructions, 16 outputs and 32 input columns all run."""
    table, cols = _small_device_table()
    check_filter_project(table, cols, None, [("rid", col("rid")), ("d", _deep(8))])
    check_filter_project(table, cols, None, [("rid", col("rid")), ("c", _chain(col("rid"), 30))])   # 2 + 62 = 64 instructions
    check_filter_project(table, cols, None, [("rid", col("rid"))] + [(f"o{j}", col("rid") * j) for j in range(15)])
    t32, c32 = _small_device_table(32)
    check_filter_project(t32, c32, col("a31") > 0, [("rid", col("rid"))] + [(f"a{j}", col(f"a{j}")) for j in range(1, 16)])


@pytest.mark.gpu
def test_program_limits_reject_beyond_the_limit(gpu_lib):
    """Stack depth 9, 65 instructions, 17 outputs and 33 input columns are refused by the host check with B200Error."""
    import torch

    table, _ = _small_device_table()
    run = lambda t, p, o: PhysicalFilterProject(p, o).ProcessBatch(t, OperatorResult.NEED_MORE_INPUT)  # noqa: E731
    with pytest.raises(B200Error, match="too deep"):
        run(table, None, [("d", _deep(9))])
    with pytest.raises(B200Error, match="1 to 64 instructions"):
        run(table, ~(col("rid") < 0), [("rid", _chain(col("rid"), 29))])                  # 5 + 60 = 65 instructions
    with pytest.raises(B200Error, match="more than 16 output"):
        run(table, None, [(f"o{j}", col("rid") + j) for j in range(17)])
    t33, _ = _small_device_table(33)
    with pytest.raises(B200Error, match="more than 32 columns"):
        run(t33, None, [("rid", col("rid"))])
    keep = table.columns[0].data.to(dtype=torch.uint8)
    wide = Table([table.columns[0]] * 17, [f"c{j}" for j in range(17)])
    with pytest.raises(B200Error, match="more than 16 output"):                            # the runtime join filter's limit
        filter_project_table(wide, keep)


# ============================================================================================ GPU: the C ABI directly
def _raw(table, prog, pred_start, out_specs, out_starts=None, n_instr=None):
    """b200_filter_project on a device `table` with a hand-written program [(op name, arg)]; out_specs = [(ctype, with bitmap)]."""
    import torch

    cprog = ffi.new("b200_expr_instr[]", max(len(prog), 1))
    for j, (op, arg) in enumerate(prog):
        cprog[j].op, cprog[j].arg = OPS[op], arg
    n = table.n_rows
    outs = []
    for ct, with_bitmap in out_specs:   # raw byte buffers (0x55 where nothing was written), read back as np_dtype_of(ct)
        v = torch.zeros((n + 31) // 32 * 4 + 8, dtype=torch.uint8, device="cuda:0") if with_bitmap else None
        d = torch.full((max(n, 1) * np_dtype_of(ct).itemsize,), 0x55, dtype=torch.uint8, device="cuda:0")
        outs.append(Column(d, v, ct, ArrTypes.NUMPY, n))
    cin, cout = CTable(table), CTable(Table(outs, [f"o{j}" for j in range(len(outs))]))
    starts = out_starts if out_starts is not None else [0] * len(out_specs)
    rc = int(_lib.lib().b200_filter_project(cin.ptr, cprog, len(prog) if n_instr is None else n_instr, pred_start,
                                            ffi.new("int32_t[]", starts or [0]), len(starts), cout.ptr, ffi.NULL))
    return rc, outs


@pytest.mark.gpu
@pytest.mark.parametrize("ct", [CTypes.INT8, CTypes.UINT8, CTypes.INT16, CTypes.UINT16, CTypes.INT32, CTypes.UINT32, CTypes.INT64,
                                CTypes.UINT64, CTypes.FLOAT32, CTypes.BOOL])
@pytest.mark.parametrize("src", ["float", "int"])
def test_abi_store_to_every_output_type(gpu_lib, ct, src):
    """A float (or integer) expression stored to a narrow integer / BOOL / FLOAT32 output converts the VALUE (truncation toward
    zero, low bytes of an integer, BOOL = value != 0), not the raw bits."""
    fv = np.array([-3.7, 2.9, 0.0, -0.0, 100.5, 0.5, -100.2, 1.0, 7.0, -1.0], np.float64)
    iv = np.array([5, 0, -1, 70000, 300, -129, 255, 1 << 40, 2, -(1 << 31) - 3], np.int64)
    x = fv if src == "float" else iv
    if ct in (CTypes.UINT8, CTypes.UINT16, CTypes.UINT32, CTypes.UINT64) and src == "float":
        x = np.abs(x)   # a negative float has no unsigned value (numpy leaves it undefined)
    table = table_to_device(Table([Column(x)], ["x"]))
    rc, outs = _raw(table, [("col", 0), ("const_f64" if src == "float" else "const_i64", _bits(1.0) if src == "float" else 1),
                            ("mul", 0), ("end", 0)], -1, [(ct, True)])
    _lib.check(rc, "filter_project")
    assert rc == len(x)
    got = _out_values(outs[0], rc)
    exp = ref_store("f" if src == "float" else "i", x, ct)
    np.testing.assert_array_equal(got.view(np.uint8) if ct == CTypes.BOOL else got, exp.view(np.uint8) if ct == CTypes.BOOL else exp)


def _out_values(c, n):
    return c.data.cpu().numpy().view(np_dtype_of(c.c_type))[:n]


def _bits(v):
    return int(np.float64(v).view(np.int64))


@pytest.mark.gpu
def test_abi_count_only_and_output_without_bitmap(gpu_lib):
    """n_out == 0 returns the kept count; an output without a validity buffer receives its data and no bitmap."""
    n = 5000
    x = np.random.default_rng(9).integers(-50, 50, n).astype(np.int64)
    table = table_to_device(Table([Column(x)], ["x"]))
    pred = [("col", 0), ("const_i64", 10), ("gt", 0), ("end", 0)]
    rc, _ = _raw(table, pred, 0, [], out_starts=[])
    assert rc == int((x > 10).sum())
    rc, outs = _raw(table, pred + [("col", 0), ("const_i64", 2), ("mul", 0), ("end", 0)], 0, [(CTypes.INT64, False)], out_starts=[4])
    assert rc == int((x > 10).sum()) and outs[0].validity is None
    np.testing.assert_array_equal(np.sort(_out_values(outs[0], rc)), np.sort(x[x > 10] * 2))


@pytest.mark.gpu
def test_abi_malformed_programs_are_rejected(gpu_lib):
    table = table_to_device(Table([Column(np.arange(10, dtype=np.int64))], ["x"]))
    cases = [([("col", 0), ("add", 0), ("end", 0)], "underflow"), ([("col", 0)], "not terminated"),
             ([("col", 0), ("col", 0), ("end", 0)], "exactly one value"), ([("col", 1), ("end", 0)], "bad column index")]
    for prog, msg in cases:
        rc, _ = _raw(table, prog, -1, [(CTypes.INT64, True)])
        assert rc < 0
        with pytest.raises(B200Error, match=msg):
            _lib.check(rc)


@pytest.mark.gpu
def test_abi_bad_start_is_rejected(gpu_lib):
    """pred_start / out_starts[j] must be 0 or follow an END; anything else is refused before the launch."""
    table = table_to_device(Table([Column(np.arange(10, dtype=np.int64))], ["x"]))
    prog = [("col", 0), ("const_i64", 1), ("add", 0), ("end", 0), ("col", 0), ("end", 0)]
    for pred_start, out_starts in [(1, [4]), (2, [4]), (-2, [4]), (6, [4]), (-1, [1]), (-1, [3]), (-1, [6]), (-1, [-1]), (0, [4, 5])]:
        rc, _ = _raw(table, prog, pred_start, [(CTypes.INT64, True)] * len(out_starts), out_starts=out_starts)
        assert rc < 0, (pred_start, out_starts)
        with pytest.raises(B200Error, match="does not start an expression"):
            _lib.check(rc)
    rc, outs = _raw(table, prog, -1, [(CTypes.INT64, True)] * 2, out_starts=[0, 4])
    assert rc == 10


# ============================================================================================ GPU: operators around the kernel
@pytest.mark.gpu
def test_multiple_batches_through_one_operator(gpu_lib):
    """The program is compiled from the first batch and reused: every later batch (other sizes, other nulls) stays exact."""
    spec = [("a", "int32", "nullable", 0.2), ("x", "float64", "nullable", 0.1), ("t", "datetime", "numpy", 0.0)]
    predicate = (col("a") > 0) | (col("x") < -0.5) | col("t").isnull()
    outs = [("rid", col("rid")), ("a", col("a")), ("e", col("a") * 2 + col("x")), ("t", col("t")), ("c", col("a") == 7)]
    op = PhysicalFilterProject(predicate, outs)
    for seed, n in enumerate([4000, 0, 1, 70000, 1025]):
        table, cols = build_inputs(spec, n, seed)
        check_filter_project(table_to_device(table) if n else table, cols, predicate, outs, op=op)


@pytest.mark.gpu
def test_filter_project_table_keeps_rows_bit_for_bit(gpu_lib):
    """The runtime join filter's compaction: every column of a mixed-dtype table with nulls passes through unchanged for the
    rows whose keep byte is non-zero (any non-zero byte keeps): c-type, array type, bitmap presence, validity and bits, so a
    float NaN stays a valid NaN with its payload."""
    import torch

    spec = [(f"c_{dt}", dt, "nullable" if dt != "date32" else "arrow_offset", 0.15) for dt in DTYPES]
    n = 40_000
    table, cols = build_inputs(spec, n, seed=21)
    keep = np.random.default_rng(2).choice(np.array([0, 1, 2, 255], np.uint8), n)
    dt = table_to_device(table)
    out = filter_project_table(dt, torch.from_numpy(keep).to("cuda:0"))
    assert out.names == dt.names and out.n_rows == int((keep != 0).sum())
    order = np.argsort(out.columns[0].values_numpy())
    np.testing.assert_array_equal(out.columns[0].values_numpy()[order], np.flatnonzero(keep))
    as_bits = lambda x: x.view(np.uint8) if x.dtype == bool else x.view(f"i{x.dtype.itemsize}") if x.dtype.kind == "f" else x  # noqa: E731
    for nm, c, inc in zip(out.names[1:], out.columns[1:], dt.columns[1:]):
        ct, v, valid = cols[nm]
        assert (c.c_type, c.arr_type, c.validity is not None) == (inc.c_type, inc.arr_type, inc.validity is not None), nm
        got = c.values_numpy()[order]
        _assert_column(nm, as_bits(got), c.valid_mask_numpy()[order], as_bits(v)[keep != 0], valid[keep != 0])


@pytest.mark.gpu
def test_nat_rows_are_na_through_filter_and_groupby(gpu_lib):
    from bodo_b200.physical import groupby_agg

    ts = pd.to_datetime(["2020-01-01", None, "2019-06-01", None, "2021-03-04", "2020-01-01"])
    df = pd.DataFrame({"ts": ts, "v": np.arange(6, dtype=np.int64)})
    op = PhysicalFilterProject(col("ts") <= lit(datetime.datetime(2020, 6, 1)), [("v", col("v")), ("ts", col("ts"))])
    got, _ = op.ProcessBatch(table_to_device(Table.from_pandas(df)), OperatorResult.FINISHED)
    assert sorted(got.columns[0].values_numpy().tolist()) == [0, 2, 5]                   # NaT <= x is NA: dropped
    for dropna in (True, False):
        g = groupby_agg(df, "ts", [("s", "v", "sum")], dropna=dropna)
        e = df.groupby("ts", dropna=dropna, as_index=False).agg(s=("v", "sum"))
        key = lambda d: sorted(zip([-1 if pd.isna(t) else pd.Timestamp(t).value for t in d["ts"]], d["s"].astype("int64").tolist()))  # noqa: E731
        assert key(g) == key(e), (g, e)


@pytest.mark.gpu
def test_comparison_outputs_keep_their_nas(gpu_lib):
    df = pd.DataFrame({"c": pd.array([7, None, 3, 7, None], dtype="Int32")})
    op = PhysicalFilterProject(None, [("eq", col("c") == 7), ("n", col("c").isnull())])
    got, _ = op.ProcessBatch(table_to_device(Table.from_pandas(df)), OperatorResult.FINISHED)
    out = got.to_pandas()
    assert str(out["eq"].dtype) == "boolean"
    assert sorted(map(str, out["eq"].tolist())) == sorted(["True", "<NA>", "False", "True", "<NA>"])
    assert out["n"].sum() == 2 and not out["n"].isna().any()


# ============================================================================================ GPU: dictionary unification
def _dict_batches():
    d = pa.array(["a", "b", None, "a", "c"])
    return [
        pa.array(["x", "y", None, "x"]),
        pa.array(["w", None, "x", "w"], type=pa.large_string()),
        pa.DictionaryArray.from_arrays(pa.array([0, 1, 2, 1, None, 0], pa.int8()), pa.array(["y", "q", "z"])),
        pa.DictionaryArray.from_arrays(pa.array([3, 2, 1, 0, 3], pa.int16()), pa.array(["r", "x", "s", "t"])),
        pa.DictionaryArray.from_arrays(pa.array([0, 1, 2, 3, 4, 0, 2, None, 1, 4, 3], pa.int32()), d).slice(3),   # offset 3
        pa.DictionaryArray.from_arrays(pa.array([0, 1, 2, 1, 0], pa.int32()), pa.array(["a", "a", "b"])),          # repeated entries
        pa.DictionaryArray.from_arrays(pa.array([0, 1, 2, 1], pa.int32()), pa.array(["a", None, "a"])),           # null entry
        pa.DictionaryArray.from_arrays(pa.array([None, None, None], pa.int32()), pa.array([], pa.string())),     # all null
        pa.chunked_array([pa.array(["k", "l"]).dictionary_encode(), pa.array(["m", None, "k"]).dictionary_encode(),
                          pa.DictionaryArray.from_arrays(pa.array([1, 0], pa.int32()), pa.array(["n", None]))]),
    ]


@pytest.mark.gpu
def test_dictionary_unification_matches_to_pylist(gpu_lib):
    b = DictionaryBuilder()
    for j, arr in enumerate(_dict_batches()):
        c = b.unify(arr, 0)
        assert c.c_type == CTypes.INT32 and c.length == len(arr)
        assert list(b.decode(c.values_numpy(), c.valid_mask_numpy())) == arr.to_pylist(), j
    assert None not in b.values and len(set(b.values)) == len(b.values)
    assert b.values[:4] == ["x", "y", "w", "q"]     # first-appearance order across batches


@pytest.mark.gpu
def test_dictionary_unification_of_a_large_batch(gpu_lib):
    """2 M rows over 100 k distinct strings: remap_i32_kernel runs its grid-stride loop."""
    rng = np.random.default_rng(4)
    n, k = 2_000_000, 100_000
    b = DictionaryBuilder()
    b.unify(pa.array([f"s{i}" for i in rng.permutation(k)[:5000]]), 0)          # global ids differ from the batch's
    dictionary = pa.array([f"s{i}" for i in range(k)])
    idx = rng.integers(0, k, n).astype(np.int32)
    arr = pa.DictionaryArray.from_arrays(pa.array(idx, mask=rng.random(n) < 0.05), dictionary)
    c = b.unify(arr, 0)
    ids, valid = c.values_numpy(), c.valid_mask_numpy()
    gid = np.array([b.index[s] for s in dictionary.to_pylist()], np.int32)
    exp_valid = np.asarray(arr.is_valid())
    np.testing.assert_array_equal(valid, exp_valid)
    np.testing.assert_array_equal(ids[exp_valid], gid[idx[exp_valid]])


@pytest.mark.gpu
@pytest.mark.parametrize("dropna", [True, False])
def test_dictionary_key_groupby_matches_pandas(gpu_lib, dropna):
    """A dictionary-encoded key with null indices and null dictionary entries, unified batch by batch, grouped on the device:
    both kinds of null are one NA group (dropped with dropna=True), as pandas groups the decoded strings."""
    rng = np.random.default_rng(8)
    n = 10_000
    dictionary = pa.array(["a", None, "b", "c", None, "a", "d"])
    idx = rng.integers(0, len(dictionary), n).astype(np.int32)
    s = pa.DictionaryArray.from_arrays(pa.array(idx, mask=rng.random(n) < 0.05), dictionary)
    v = rng.integers(-1000, 1000, n).astype(np.int64)
    b = DictionaryBuilder()
    src = PhysicalReadArrowDevice(pa.table({"s": s, "v": v}), 1537, 0, {"s": b})
    agg = PhysicalAggregate((0,), [("sum", 1), ("size", None)], dropna=dropna)
    run_pipeline(src, [], agg)
    coll = ResultCollector()
    run_pipeline(agg, [], coll)
    agg.Finalize()
    got = coll.result()
    got.columns = ["s", "sum", "size"]
    keys = b.decode(got["s"].to_numpy(dtype="int64", na_value=-1))
    g = sorted(zip(map(str, keys), got["sum"].astype("int64"), got["size"].astype("int64")))
    e = pd.DataFrame({"s": s.to_pylist(), "v": v}).groupby("s", dropna=dropna).agg(sum=("v", "sum"), size=("v", "size")).reset_index()
    exp = sorted(zip(map(lambda x: str(None) if pd.isna(x) else str(x), e["s"]), e["sum"].astype("int64"), e["size"].astype("int64")))
    assert g == exp
