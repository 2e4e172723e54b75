"""The join's non-equi condition on the host: build_col / probe_col, the program init_join_state compiles (columns resolved to
their physical, keys-first index; probe columns offset by 32), every refusal and its message, and that nothing reaches the GPU
before the first build batch."""

import pytest

from bodo_b200 import _lib
from bodo_b200._lib import B200Error
from bodo_b200.expr import OPS, Expr, build_col, col, lit, probe_col
from bodo_b200.streaming.join import EX_MAX_INSTR, EX_MAX_STACK, J_MAX_COLS, compile_condition, init_join_state


def state(cond, bkeys=(0,), pkeys=(0,), bnames=("k", "start", "end"), pnames=("k", "ts"), **kw):
    return init_join_state(-1, bkeys, pkeys, bnames, pnames, False, False, non_equi_condition=cond, **kw)


def test_side_references():
    b, p = build_col("start"), probe_col("ts")
    assert isinstance(b, Expr) and b.op == "col" and b.value == ("build", "start")
    assert p.op == "col" and p.value == ("probe", "ts")
    assert (p >= b).columns() == {("build", "start"), ("probe", "ts")}


def test_program_uses_physical_columns_and_the_probe_offset():
    """Keys come first on each side: build (a, k, b) keyed on k is physical (k, a, b); probe (x, y, k) keyed on k is (k, x, y)."""
    cond = (probe_col("y") > build_col("b")) & (probe_col("k") + 1 <= build_col("a") * 2.5) | build_col("k").isnull()
    prog = compile_condition(cond, (1,), (2,), ["a", "k", "b"], ["x", "y", "k"])
    cols = [arg for op, arg in prog if op == OPS["col"]]
    assert cols == [J_MAX_COLS + 2, 2, J_MAX_COLS + 0, 1, 0]
    assert prog[-1] == (OPS["end"], 0) and sum(op == OPS["end"] for op, _ in prog) == 1
    assert [op for op, _ in prog] == [OPS[o] for o in ("col", "col", "gt", "col", "const_i64", "add", "col", "const_f64", "mul", "le",
                                                      "and", "col", "is_null", "or", "end")]


def test_program_with_two_key_columns():
    prog = compile_condition(probe_col("v") < build_col("w"), (2, 0), (1, 0), ["k0", "w", "k1"], ["k0", "k1", "v"])
    assert prog == [(OPS["col"], J_MAX_COLS + 2), (OPS["col"], 2), (OPS["lt"], 0), (OPS["end"], 0)]  # build (k1, k0, w), probe (k1, k0, v)


def test_state_keeps_the_program_and_touches_no_gpu(monkeypatch):
    def no_gpu(*a, **k):
        raise AssertionError("the library was reached before the first build batch")

    monkeypatch.setattr(_lib, "lib", no_gpu)
    monkeypatch.setattr(_lib, "require_gpu", no_gpu)
    st = state((probe_col("ts") >= build_col("start")) & (probe_col("ts") < build_col("end")))
    assert st.handle is None
    assert st.condition == compile_condition((probe_col("ts") >= build_col("start")) & (probe_col("ts") < build_col("end")), (0,), (0,),
                                             ["k", "start", "end"], ["k", "ts"])
    assert state(None).condition is None


def test_physical_join_forwards_the_condition():
    from bodo_b200.physical import PhysicalJoin

    cond = probe_col("ts") >= build_col("start")
    for how in ("inner", "left", "right", "outer", "anti", "mark"):
        st = PhysicalJoin(0, 0, ("k", "start"), ("k", "ts"), how=how, non_equi_condition=cond).state
        assert st.condition == [(OPS["col"], J_MAX_COLS + 1), (OPS["col"], 1), (OPS["ge"], 0), (OPS["end"], 0)]


def test_unknown_column_is_named():
    with pytest.raises(B200Error, match=r"the build side has no column 'stop'"):
        state(probe_col("ts") < build_col("stop"))
    with pytest.raises(B200Error, match=r"the probe side has no column 'start'"):
        state(probe_col("start") < build_col("end"))


def test_ambiguous_column_is_refused():
    with pytest.raises(B200Error, match=r"more than one column 'x'"):
        state(probe_col("x") < build_col("end"), pnames=("k", "x", "x"))


def test_colnames_none_is_refused():
    with pytest.raises(B200Error, match=r"build_colnames is None"):
        state(probe_col("ts") < build_col("end"), bnames=None)
    with pytest.raises(B200Error, match=r"probe_colnames is None"):
        state(probe_col("ts") < build_col("end"), pnames=None)


def test_column_without_a_side_is_refused():
    with pytest.raises(B200Error, match=r"column 'ts' names no join side: use build_col\('ts'\) or probe_col\('ts'\)"):
        state(col("ts") < build_col("end"))


def test_string_condition_is_refused():
    with pytest.raises(B200Error, match=r"must be a bodo_b200.expr.Expr .*\(string conditions are not supported\)"):
        state("left.`ts` < right.`end`")


def _chain(m):
    """probe ts + 1 + 1 ... (m additions, left-nested: stack depth 2) > 0: 2 m + 4 instructions."""
    e = probe_col("ts")
    for _ in range(m):
        e = e + 1
    return e > 0


def _nest(leaves):
    """1 + (1 + (... + ts)) with `leaves` leaves, compared with a build column: stack depth `leaves`."""
    e = probe_col("ts")
    for _ in range(leaves - 1):
        e = lit(1) + e
    return e > build_col("start")


def test_program_limits():
    assert len(state(_chain(30)).condition) == EX_MAX_INSTR
    with pytest.raises(B200Error, match=r"compiles to 66 instructions; the limit is 64"):
        state(_chain(31))
    assert state(_nest(EX_MAX_STACK)).condition is not None
    with pytest.raises(B200Error, match=r"needs a stack of 9 values while it runs; the limit is 8"):
        state(_nest(EX_MAX_STACK + 1))


def test_nested_loop_join_is_refused():
    with pytest.raises(B200Error, match=r"without an equi-join key \(a nested-loop join\) is not supported"):
        state(probe_col("ts") < build_col("end"), bkeys=(), pkeys=())


def test_interval_join_is_still_refused():
    with pytest.raises(B200Error, match=r"interval joins \(interval_build_columns\) are not supported"):
        init_join_state(-1, (0,), (0,), ("k", "s", "e"), ("k", "t"), False, False, interval_build_columns=(1, 2))
    with pytest.raises(B200Error, match=r"interval joins"):
        init_join_state(-1, (0,), (0,), ("k", "s", "e"), ("k", "t"), False, False, interval_build_columns=(1, 2),
                        non_equi_condition=probe_col("t") < build_col("e"))


def test_header_declares_set_condition():
    assert "b200_join_set_condition" in set(_lib.declared_symbols())
