"""Host-side checks of the streaming top-k operator: argument validation and PhysicalSort plumbing (no GPU needed)."""

import pytest

from bodo_b200._lib import B200Error
from bodo_b200.physical import OperatorResult, PhysicalSort
from bodo_b200.streaming import sort as S

COLS = ["a", "b", "c", "d", "e"]


def init(**kw):
    args = dict(operator_id=-1, limit=10, offset=0, by=["a"], asc=[True], na_position=["last"], col_names=COLS)
    args.update(kw)
    return S.init_stream_sort_state(**args)


def test_valid_arguments_create_a_lazy_state():
    st = init(by=["b", "a"], asc=[False, True], na_position=["first", "last"], limit=5, offset=3)
    assert st.handle is None
    assert st.phys == [1, 0, 2, 3, 4] and st.out_order == [1, 0, 2, 3, 4]
    assert st.na_last == [False, True] and st.asc == [False, True]
    st = init(by="c", asc=False, na_position="first")
    assert st.by == ["c"] and st.asc == [False] and st.na_last == [False]
    assert st.phys == [2, 0, 1, 3, 4] and [st.phys[i] for i in st.out_order] == [0, 1, 2, 3, 4]


@pytest.mark.parametrize("kw,msg", [
    (dict(limit=None), "limit is required"),
    (dict(limit=-1), "non-negative"),
    (dict(offset=-3), "non-negative"),
    (dict(limit=S.MAX_LIMIT_PLUS_OFFSET), None),
    (dict(limit=S.MAX_LIMIT_PLUS_OFFSET - 5, offset=6), "exceeds the top-k cap"),
    (dict(limit=S.MAX_LIMIT_PLUS_OFFSET + 1), "exceeds the top-k cap"),
    (dict(by=[], asc=[], na_position=[]), "1 to 4 sort keys"),
    (dict(by=COLS, asc=[True] * 5, na_position=["last"] * 5), "1 to 4 sort keys"),
    (dict(by=["a"], na_position=["middle"]), "na_position"),
    (dict(by=["a"], na_position="nowhere"), "na_position"),
    (dict(by=["a", "b"], asc=[True]), "one entry per sort key"),
    (dict(by=["a", "b"], asc=[True, False], na_position=["last"]), "one entry per sort key"),
    (dict(by=["zz"]), "must be distinct columns"),
    (dict(by=["a", "a"], asc=[True, True], na_position=["last", "last"]), "must be distinct columns"),
])
def test_argument_checks(kw, msg):
    if msg is None:
        assert init(**kw).limit == S.MAX_LIMIT_PLUS_OFFSET
        return
    with pytest.raises(B200Error, match=msg):
        init(**kw)


def test_produce_before_consume_raises():
    with pytest.raises(B200Error, match="before the last batch"):
        S.produce_output_batch(init())


def test_physical_sort_plumbing():
    with pytest.raises(B200Error, match="limit is required"):
        PhysicalSort(["a"])
    op = PhysicalSort(["a", "b"], [True, False], "first", limit=7, offset=2)
    assert op.state is None and op.args == (["a", "b"], [True, False], "first", 7, 2, False)
    op.Finalize()  # nothing to free before the first batch
    assert OperatorResult.FINISHED.value == 2
