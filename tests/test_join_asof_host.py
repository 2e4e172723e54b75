"""The as-of join on the host: asof_on resolved to physical columns (keys first; without keys, after the constant key column),
every refusal of init_join_state and PhysicalJoin before any device is touched, the tolerance in the column's units, the C entry
point's declaration, and merge_asof's output layout against pandas.merge_asof's on small frames."""

import math

import numpy as np
import pandas as pd
import pytest

from bodo_b200 import _lib
from bodo_b200._lib import B200Error
from bodo_b200.expr import build_col, probe_col
from bodo_b200.physical import PhysicalJoin, asof_output_layout
from bodo_b200.streaming.join import asof_tolerance_units, init_join_state
from bodo_b200.table import CTypes


@pytest.fixture(autouse=True)
def no_gpu(monkeypatch):
    def refuse(*a, **k):
        raise AssertionError("the library was reached before the first build batch")

    monkeypatch.setattr(_lib, "lib", refuse)
    monkeypatch.setattr(_lib, "require_gpu", refuse)


def state(bkeys=(0,), pkeys=(0,), bnames=("k", "ts", "bid"), pnames=("px", "k", "ts"), on=("ts", "ts"), **kw):
    return init_join_state(-1, bkeys, pkeys, bnames, pnames, False, kw.pop("probe_outer", True), asof_on=on, **kw)


def test_on_resolves_to_physical_columns():
    st = state(bkeys=(0,), pkeys=(1,))
    # build (k, ts, bid) keyed on k: physical (k, ts, bid); probe (px, k, ts) keyed on k: physical (k, px, ts)
    assert st.asof == (1, 2, 0, True, None) and not st.const_key
    st = state(bkeys=(2, 0), pkeys=(1, 0), bnames=("k0", "ts", "k1"), pnames=("k0", "k1", "ts"), asof_direction="nearest",
               asof_allow_exact_matches=False, asof_tolerance=5)
    assert st.asof == (2, 2, 2, False, 5)


def test_no_keys_appends_a_constant_key():
    st = state(bkeys=(), pkeys=(), asof_direction="forward")
    assert st.const_key and st.build_key_inds == (3,) and st.probe_key_inds == (3,)
    assert st.asof[:3] == (2, 3, 1)  # physical (key, k, ts, bid) and (key, px, k, ts)
    assert st.handle is None


@pytest.mark.parametrize("kw, msg", [
    (dict(build_outer=True), r"a build-outer asof join is not supported"),
    (dict(is_mark_join=True), r"an asof join is not a mark, anti or non_equi_condition join"),
    (dict(is_anti_join=True), r"not a mark, anti or non_equi_condition join"),
    (dict(non_equi_condition=probe_col("ts") >= build_col("bid")), r"not a mark, anti or non_equi_condition join"),
    (dict(build_parallel=True), r"a sharded asof join is not supported"),
    (dict(probe_parallel=True), r"a sharded asof join is not supported"),
    (dict(asof_direction="closest"), r"asof_direction must be one of \['backward', 'forward', 'nearest'\]"),
    (dict(asof_tolerance=-1), r"asof_tolerance must be finite and >= 0"),
    (dict(asof_tolerance=-0.5), r"finite and >= 0"),
    (dict(asof_tolerance=math.inf), r"finite and >= 0"),
    (dict(asof_tolerance=math.nan), r"finite and >= 0"),
    (dict(asof_tolerance=pd.Timedelta("-1s")), r"asof_tolerance must be >= 0"),
    (dict(asof_tolerance="1s"), r"must be an int, a float or a pd.Timedelta \(got str\)"),
    (dict(asof_tolerance=True), r"got bool"),
])
def test_refusals_at_init(kw, msg):
    build_outer = kw.pop("build_outer", False)
    with pytest.raises(B200Error, match=msg):
        init_join_state(-1, (0,), (1,), ("k", "ts", "bid"), ("px", "k", "ts"), build_outer, True, asof_on=("ts", "ts"), **kw)


def test_bad_on_names_are_refused():
    with pytest.raises(B200Error, match=r"the build side has no column 't'"):
        state(on=("t", "ts"))
    with pytest.raises(B200Error, match=r"the probe side has more than one column 'ts'"):
        state(pnames=("k", "ts", "ts"))
    with pytest.raises(B200Error, match=r"build column 'k' is an equi-join key"):
        state(on=("k", "ts"))
    with pytest.raises(B200Error, match=r"build_colnames is None"):
        state(bnames=None)
    with pytest.raises(B200Error, match=r"asof_on must be \(build column name, probe column name\)"):
        state(on="ts")


def test_zero_keys_without_asof_on_is_refused():
    with pytest.raises(B200Error, match=r"1 to 4 equi-join keys per side"):
        init_join_state(-1, (), (), ("ts",), ("ts",), False, True)


def test_physical_join_takes_left_and_inner_only():
    for how in ("left", "inner"):
        assert PhysicalJoin((), (), ("ts", "v"), ("ts", "w"), how=how, asof_on=("ts", "ts")).state.const_key
    for how in ("right", "outer", "anti", "mark"):
        with pytest.raises(B200Error, match=rf"how='left' or how='inner', not '{how}'"):
            PhysicalJoin(0, 0, ("k", "ts"), ("k", "ts"), how=how, asof_on=("ts", "ts"))


def test_tolerance_units():
    assert asof_tolerance_units(None, CTypes.INT64) == (0, 0, 0.0)
    assert asof_tolerance_units(pd.Timedelta("1500ms"), CTypes.DATETIME) == (1, 1_500_000_000, 0.0)
    assert asof_tolerance_units(pd.Timedelta("2us"), CTypes.TIMEDELTA) == (1, 2000, 0.0)
    assert asof_tolerance_units(pd.Timedelta("3D"), CTypes.DATE) == (1, 3, 0.0)
    assert asof_tolerance_units(7, CTypes.DATE) == (1, 7, 0.0)
    assert asof_tolerance_units(np.int64(9), CTypes.UINT8) == (1, 9, 0.0)
    assert asof_tolerance_units(4.0, CTypes.INT32) == (1, 4, 0.0)
    assert asof_tolerance_units(0.25, CTypes.FLOAT32) == (1, 0, 0.25)
    assert asof_tolerance_units(3, CTypes.FLOAT64) == (1, 0, 3.0)
    with pytest.raises(B200Error, match=r"not a whole number of days"):
        asof_tolerance_units(pd.Timedelta("36h"), CTypes.DATE)
    with pytest.raises(B200Error, match=r"needs a date, datetime or timedelta `on` column"):
        asof_tolerance_units(pd.Timedelta("1s"), CTypes.INT64)
    with pytest.raises(B200Error, match=r"is not an integer"):
        asof_tolerance_units(0.5, CTypes.INT64)


def test_set_asof_is_declared():
    assert "b200_join_set_asof" in set(_lib.declared_symbols())


L = pd.DataFrame({"t": [1, 2, 3], "k": [1, 1, 2], "v": [1.0, 2, 3], "a": [0, 0, 0]})
R = pd.DataFrame({"t": [1, 2], "k": [1, 2], "v": [5.0, 6], "b": [1, 1]})


@pytest.mark.parametrize("left, right, kw", [
    (L, R, dict(on="t", by="k")),
    (L, R, dict(on="t")),
    (L, R, dict(left_on="t", right_on="t")),
    (L, R, dict(left_on="t", right_on="t", by="k")),
    (L, R, dict(on="t", left_by="k", right_by="k")),
    (L, R, dict(on="t", left_by="k", right_by="b")),
    (L, R, dict(on="t", by="k", suffixes=("_l", "_r"))),
    (L, R.assign(a=1), dict(on="t", by=["k", "a"])),
    (L, R.assign(a=1), dict(on="t", by="k")),
    (L, R.assign(a=1), dict(left_on="t", right_on="t", left_by="k", right_by="b")),
    (L.rename(columns={"v": "s"}), R.rename(columns={"t": "s"}), dict(left_on="t", right_on="s")),
])
def test_merge_asof_layout_matches_pandas(left, right, kw):
    *_, names = asof_output_layout(list(left.columns), list(right.columns), **kw)
    assert names == list(pd.merge_asof(left, right, **kw).columns)


def test_merge_asof_layout_refusals():
    with pytest.raises(ValueError, match=r"give on=, or both left_on= and right_on="):
        asof_output_layout(["t"], ["t"], on="t", left_on="t", right_on="t")
    with pytest.raises(ValueError, match=r"give on=, or both"):
        asof_output_layout(["t"], ["t"], left_on="t")
    with pytest.raises(ValueError, match=r"the same number of columns"):
        asof_output_layout(["t", "k"], ["t", "k"], on="t", left_by=["k"], right_by=[])
    with pytest.raises(ValueError, match=r"the right frame has no column 'x'"):
        asof_output_layout(["t", "x"], ["t"], on="t", by="x")
