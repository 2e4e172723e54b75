"""Host side of the nested-loop join (a join without an equi-join key): the argument refusals of init_nested_loop_join_state,
PhysicalJoin(how="cross") and merge(how="cross"), the condition's names resolved to physical columns without keys, and
PhysicalJoin building a nested-loop state for every kind.  Nothing here touches the device: the C state is created at the first
build batch."""

import pandas as pd
import pytest

from bodo_b200._lib import B200Error
from bodo_b200.expr import build_col, lit, probe_col
from bodo_b200.physical import PhysicalJoin, merge
from bodo_b200.streaming.join import J_MAX_COLS, init_nested_loop_join_state

BANDS = ("lo", "hi", "bid")
EVENTS = ("x", "eid")
BAND = (probe_col("x") >= build_col("lo")) & (probe_col("x") < build_col("hi"))


def state(cond=BAND, bnames=BANDS, pnames=EVENTS, build_outer=False, probe_outer=False, **kw):
    return init_nested_loop_join_state(-1, bnames, pnames, build_outer, probe_outer, cond, **kw)


@pytest.mark.parametrize("kw,msg", [
    (dict(build_parallel=True), r"a sharded nested-loop join is not supported"),
    (dict(probe_parallel=True), r"a sharded nested-loop join is not supported"),
    (dict(asof_on=("lo", "x")), r"a nested-loop join has no as-of form"),
    (dict(interval_build_columns=(0, 1)), r"interval joins \(interval_build_columns\) are not supported"),
    (dict(is_mark_join=True, build_outer=True), r"mark / anti joins do not emit build rows"),
    (dict(is_anti_join=True, build_outer=True), r"mark / anti joins do not emit build rows"),
    (dict(is_mark_join=True, is_anti_join=True), r"a mark join or an anti join, not both"),
])
def test_init_refusals(kw, msg):
    with pytest.raises(B200Error, match=msg):
        state(**kw)


def test_condition_names_resolve_without_keys():
    st = state(BAND, bnames=("hi", "bid", "lo"), pnames=("eid", "x"))
    assert st.build_key_inds == () and st.probe_key_inds == () and st.nested_loop
    cols = [arg for op, arg in st.condition if op == 0]
    # probe x is probe column 1, build lo build column 2, build hi build column 0: logical order is physical order without keys
    assert cols == [J_MAX_COLS + 1, 2, J_MAX_COLS + 1, 0]
    assert state(None).condition is None


def test_condition_name_errors():
    with pytest.raises(B200Error, match=r"the build side has no column 'nope'"):
        state(probe_col("x") < build_col("nope"))
    with pytest.raises(B200Error, match=r"probe_colnames is None"):
        state(probe_col("x") < build_col("lo"), pnames=None)
    with pytest.raises(B200Error, match=r"string conditions are not supported"):
        state("left.x < right.lo")
    assert state(probe_col("x") > lit(3)).condition is not None


@pytest.mark.parametrize("how,flags", [("inner", (False, False, False, False)), ("left", (False, True, False, False)),
                                       ("right", (True, False, False, False)), ("outer", (True, True, False, False)),
                                       ("anti", (False, False, False, True)), ("mark", (False, False, True, False)),
                                       ("cross", (False, False, False, False))])
@pytest.mark.parametrize("with_cond", [False, True])
def test_physical_join_builds_a_nested_loop_state_for_every_kind(how, flags, with_cond):
    if how == "cross" and with_cond:
        return
    kw = dict(non_equi_condition=BAND) if with_cond else {}
    st = PhysicalJoin((), (), BANDS, EVENTS, how=how, **kw).state
    assert st.nested_loop and st.build_key_inds == () and st.probe_key_inds == ()
    assert (st.build_outer, st.probe_outer, st.is_mark_join, st.is_anti_join) == flags
    assert (st.condition is not None) == with_cond


def test_physical_join_cross_refusals():
    with pytest.raises(B200Error, match=r"a cross join \(how='cross'\) takes no key columns"):
        PhysicalJoin(0, 0, BANDS, EVENTS, how="cross")
    with pytest.raises(B200Error, match=r"a cross join \(how='cross'\) takes no non_equi_condition"):
        PhysicalJoin((), (), BANDS, EVENTS, how="cross", non_equi_condition=BAND)
    with pytest.raises(B200Error, match=r"a join without keys is how= one of"):
        PhysicalJoin((), (), BANDS, EVENTS, how="semi")
    with pytest.raises(B200Error, match=r"a sharded nested-loop join is not supported"):
        PhysicalJoin((), (), BANDS, EVENTS, how="inner", build_parallel=True)


def test_physical_join_with_keys_is_still_a_hash_join():
    st = PhysicalJoin(0, 0, BANDS, EVENTS, how="inner").state
    assert not st.nested_loop and st.build_key_inds == (0,)


def test_merge_refusals():
    left, right = pd.DataFrame({"x": [1, 2]}), pd.DataFrame({"lo": [0], "hi": [3]})
    with pytest.raises(ValueError, match=r"how='cross' takes no left_on / right_on"):
        merge(left, right, "x", "lo", how="cross")
    with pytest.raises(ValueError, match=r"how='cross' takes no non_equi_condition"):
        merge(left, right, how="cross", non_equi_condition=BAND)
    with pytest.raises(ValueError, match=r"no key columns: give left_on and right_on, how='cross', or a non_equi_condition"):
        merge(left, right)
    with pytest.raises(ValueError, match=r"give both left_on and right_on, or neither"):
        merge(left, right, "x", None)
