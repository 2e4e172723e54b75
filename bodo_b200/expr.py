"""Expression trees for the fused filter + projection kernel (csrc/expr.cu) — the Python face of the reference's
PhysicalExpression hierarchy (bodo/pandas/physical/expression.h: column refs, constants, arithmetic, comparison,
conjunction, cast, null test), compiled to the postfix program b200_filter_project interprets.

    e = (col("L_SHIPDATE") <= lit(datetime.date(1998, 9, 2))) & ~col("L_DISCOUNT").isnull()
    p = col("L_EXTENDEDPRICE") * (lit(1.0) - col("L_DISCOUNT"))

A join's non-equi condition names the side of each column (streaming.join.init_join_state, non_equi_condition):

    c = (probe_col("ts") >= build_col("start")) & (probe_col("ts") < build_col("end"))
"""

from __future__ import annotations

import datetime
import struct

import numpy as np

OPS = {"col": 0, "const_i64": 1, "const_f64": 2, "add": 3, "sub": 4, "mul": 5, "div": 6, "lt": 7, "le": 8, "gt": 9, "ge": 10, "eq": 11,
       "ne": 12, "and": 13, "or": 14, "not": 15, "to_f64": 16, "to_i64": 17, "is_null": 18, "neg": 19, "end": 20}


class Expr:
    def __init__(self, op, args=(), value=None):
        self.op, self.args, self.value = op, tuple(args), value

    def _bin(self, op, other, rev=False):
        other = other if isinstance(other, Expr) else lit(other)
        return Expr(op, (other, self) if rev else (self, other))

    def __add__(self, o): return self._bin("add", o)
    def __radd__(self, o): return self._bin("add", o, True)
    def __sub__(self, o): return self._bin("sub", o)
    def __rsub__(self, o): return self._bin("sub", o, True)
    def __mul__(self, o): return self._bin("mul", o)
    def __rmul__(self, o): return self._bin("mul", o, True)
    def __truediv__(self, o): return self._bin("div", o)
    def __rtruediv__(self, o): return self._bin("div", o, True)
    def __lt__(self, o): return self._bin("lt", o)
    def __le__(self, o): return self._bin("le", o)
    def __gt__(self, o): return self._bin("gt", o)
    def __ge__(self, o): return self._bin("ge", o)
    def __eq__(self, o): return self._bin("eq", o)  # noqa: comparison builds an expression node, like pandas / polars
    def __ne__(self, o): return self._bin("ne", o)
    def __and__(self, o): return self._bin("and", o)
    def __or__(self, o): return self._bin("or", o)
    def __invert__(self): return Expr("not", (self,))
    def __neg__(self): return Expr("neg", (self,))
    __hash__ = None

    def isnull(self): return Expr("is_null", (self,))
    def astype(self, kind):
        return Expr("to_f64" if np.dtype(kind).kind == "f" else "to_i64", (self,))

    def columns(self):
        if self.op == "col":
            return {self.value}
        out = set()
        for a in self.args:
            out |= a.columns()
        return out


def col(name) -> Expr:
    return Expr("col", value=name)


def build_col(name) -> Expr:
    """Column `name` of a join's build side (the right table of merge), for a join's non_equi_condition."""
    return Expr("col", value=("build", name))


def probe_col(name) -> Expr:
    """Column `name` of a join's probe side (the left table of merge), for a join's non_equi_condition."""
    return Expr("col", value=("probe", name))


def lit(v) -> Expr:
    """Constant: ints, floats, bools, datetime.date (days since epoch, the storage of DATE columns), datetime / np.datetime64
    (nanoseconds, the storage of DATETIME columns)."""
    if isinstance(v, Expr):
        return v
    if isinstance(v, (bool, np.bool_)):
        return Expr("const_i64", value=int(v))
    if isinstance(v, datetime.datetime):
        return Expr("const_i64", value=int(np.datetime64(v, "ns").astype("int64")))
    if isinstance(v, datetime.date):
        return Expr("const_i64", value=(v - datetime.date(1970, 1, 1)).days)
    if isinstance(v, np.datetime64):
        return Expr("const_i64", value=int(v.astype("datetime64[ns]").astype("int64")))
    if isinstance(v, (int, np.integer)):
        return Expr("const_i64", value=int(v))
    if isinstance(v, (float, np.floating)):
        return Expr("const_f64", value=float(v))
    raise TypeError(f"bodo_b200.expr: unsupported constant {v!r}")


def compile_program(exprs, col_index: dict):
    """exprs: list of Expr.  Returns (list of (op, arg) instructions, start offset of every expression)."""
    prog, starts = [], []

    def emit(e: Expr):
        if e.op == "col":
            if e.value not in col_index:
                raise KeyError(f"bodo_b200.expr: unknown column {e.value!r}")
            prog.append((OPS["col"], col_index[e.value]))
        elif e.op == "const_i64":
            prog.append((OPS["const_i64"], e.value))
        elif e.op == "const_f64":
            prog.append((OPS["const_f64"], struct.unpack("<q", struct.pack("<d", e.value))[0]))
        else:
            for a in e.args:
                emit(a)
            prog.append((OPS[e.op], 0))

    for e in exprs:
        starts.append(len(prog))
        emit(e)
        prog.append((OPS["end"], 0))
    return prog, starts
