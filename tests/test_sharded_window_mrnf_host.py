"""Host-side checks of the sharded window (streaming.window.init_sharded_window_state) and the sharded min_row_number_filter
(streaming.groupby.init_sharded_mrnf_state), no GPU needed: argument checks, lazy creation, the verbs' dispatch, the operators
building the new states, the count agreement's window form, and the key-class partition's C entry point."""

import numpy as np
import pytest

from bodo_b200 import _lib
from bodo_b200._lib import B200Error
from bodo_b200.physical import OperatorResult, PhysicalAggregate, PhysicalWindow
from bodo_b200.streaming import groupby as G
from bodo_b200.streaming import sort as S
from bodo_b200.streaming import window as W
from bodo_b200.table import ArrTypes, Column, CTypes, Table

COLS = ["a", "b", "c"]


def _table(n=4):
    return Table([Column(np.arange(n, dtype=np.int64), None, CTypes.INT64, ArrTypes.NUMPY, n) for _ in COLS], list(COLS))


def test_the_key_class_partition_is_declared_and_exported():
    assert "b200_shuffle_partition_classes" in _lib.declared_symbols()
    import inspect

    from bodo_b200 import shuffle

    assert "by_class" in inspect.signature(shuffle.partition_device).parameters


# ---- sharded window ----
def test_window_validates_like_init_window_state():
    for args, match in (((["a"], ["a"], True, "last", [("r", "row_number")]), "distinct"),
                        ((["a", "b"], ["c", "x"], True, "last", [("r", "row_number")]), "1 to 4 keys|distinct"),
                        (("a", "b", True, "middle", [("r", "row_number")]), "na_position"),
                        (("a", "b", True, "last", [("r", "nope")]), "unknown window function"),
                        (("a", "b", True, "last", [("a", "row_number")]), "clash")):
        with pytest.raises(B200Error, match=match):
            W.init_window_state(-1, *args, COLS)
        with pytest.raises(B200Error, match=match):
            W.init_sharded_window_state(-1, *args, COLS)


def test_window_state_is_created_lazily():
    st = W.init_sharded_window_state(-1, "a", "b", True, "last", [("r", "row_number"), ("s", "sum", "c", "rows")], COLS,
                                     output_batch_size=77)
    assert isinstance(st, W.ShardedWindowState) and isinstance(st.local, W.WindowState)
    assert st.local.handle is None and st.n_ranks is None and not st.done
    assert st.local.phys[:1] == [0] and st.local.output_batch_size == 77 and not st.local.parallel  # the partition key leads
    W.delete_window_state(st)  # nothing to free


def test_window_verbs_dispatch(monkeypatch):
    st = W.init_sharded_window_state(-1, "a", "b", True, "last", [("r", "row_number")], COLS)
    seen = []
    monkeypatch.setattr(W.ShardedWindowState, "consume", lambda self, t, last: seen.append(("consume", last)) or True)
    assert W.window_build_consume_batch(st, _table(), False) == (False, True)
    with pytest.raises(B200Error, match="before the last batch"):
        W.window_produce_output_batch(st)
    st.done = True
    with pytest.raises(B200Error, match="after is_last"):
        W.window_build_consume_batch(st, _table(), True)
    assert seen == [("consume", False)]


def test_the_parallel_local_window_still_refuses_more_than_one_rank(monkeypatch):
    import torch.distributed as dist

    monkeypatch.setattr(dist, "is_initialized", lambda: True)
    monkeypatch.setattr(dist, "get_world_size", lambda group=None: 2)
    st = W.init_window_state(-1, "a", "b", True, "last", [("r", "row_number")], COLS, parallel=True)
    with pytest.raises(B200Error, match="a sharded window is not supported"):
        W.window_build_consume_batch(st, _table(), False)


def test_physical_window_builds_the_sharded_state(monkeypatch):
    built = []
    monkeypatch.setattr(W.ShardedWindowState, "consume", lambda self, t, last: built.append(self) or True)
    op = PhysicalWindow("a", ["b"], [("r", "row_number")], parallel=True, output_batch_size=5)
    op.ConsumeBatch(_table(), OperatorResult.NEED_MORE_INPUT)
    assert isinstance(op.state, W.ShardedWindowState) and built == [op.state] and op.state.local.output_batch_size == 5
    op2 = PhysicalWindow("a", ["b"], [("r", "row_number")])
    monkeypatch.setattr(W.WindowState, "_ensure", lambda self, t, *a: None)
    monkeypatch.setattr(W.WindowState, "_consume", lambda self, t, last: True)
    op2.ConsumeBatch(_table(), OperatorResult.NEED_MORE_INPUT)
    assert type(op2.state) is W.WindowState


def test_the_count_agreement_counts_rows_already_received(monkeypatch):
    """agree_receive_rows with received= and a cap: the window's form of the sort's count agreement (one rank: no collective)."""
    import torch
    import torch.distributed as dist

    monkeypatch.setattr(dist, "is_initialized", lambda: False)
    monkeypatch.setattr(dist, "all_reduce", lambda t, group=None: None)
    m = S.agree_receive_rows([5], torch.device("cpu"), received=[3], cap=9, what="Streaming Window: sharded window",
                             cap_name="the window's cap")
    assert m.tolist() == [[5]]
    with pytest.raises(B200Error, match=r"Streaming Window: sharded window: rank 0 would receive 9 rows, at or above the window's cap of 9"):
        S.agree_receive_rows([5], torch.device("cpu"), received=[4], cap=9, what="Streaming Window: sharded window",
                             cap_name="the window's cap")
    with pytest.raises(B200Error, match="sharded full sort: rank 0 would receive 7 rows, at or above the full sort's cap of 6 rows"):
        monkeypatch.setattr(S, "MAX_SHARDED_RECEIVE_ROWS", 6)
        S.agree_receive_rows([7], torch.device("cpu"))


# ---- sharded min_row_number_filter ----
def _mrnf(**kw):
    args = dict(key_inds=[0], mrnf_sort_col_inds=[1], mrnf_sort_col_asc=[True], mrnf_sort_col_na=[True], mrnf_col_inds_keep=[2])
    args.update(kw)
    return G.init_sharded_mrnf_state(-1, args.pop("key_inds"), args.pop("mrnf_sort_col_inds"), args.pop("mrnf_sort_col_asc"),
                                     args.pop("mrnf_sort_col_na"), args.pop("mrnf_col_inds_keep"), **args)


def test_mrnf_argument_checks():
    with pytest.raises(B200Error, match="mrnf_sort_col_inds must have 1 to 4"):
        _mrnf(mrnf_sort_col_inds=[], mrnf_sort_col_asc=[], mrnf_sort_col_na=[])
    with pytest.raises(B200Error, match="mrnf_sort_col_asc must have one entry per sort column"):
        _mrnf(mrnf_sort_col_asc=[True, False])
    with pytest.raises(B200Error, match="lists a column twice"):
        _mrnf(mrnf_col_inds_keep=[2, 2])
    with pytest.raises(B200Error, match="mrnf_col_inds_keep must have 1 to 26"):
        _mrnf(mrnf_col_inds_keep=[])
    for bad in (0, True, 1.5, 1 << 31):
        with pytest.raises(B200Error, match="mrnf_limit"):
            _mrnf(mrnf_limit=bad)


def test_mrnf_kept_union_limit():
    keep = list(range(3, 27))  # 24 kept columns: with key 0 and sort 1, 2 the union has 27 columns
    with pytest.raises(B200Error, match=r"union of the keys \[0\], the sort columns \[1, 2\].*27 columns"):
        _mrnf(mrnf_sort_col_inds=[1, 2], mrnf_sort_col_asc=[True, True], mrnf_sort_col_na=[True, True], mrnf_col_inds_keep=keep)
    st = _mrnf(mrnf_sort_col_inds=[1], mrnf_col_inds_keep=keep)  # 26 columns: accepted
    assert st.union == list(range(27))[:1] + [1] + keep and len(st.union) == 26


def test_mrnf_state_is_created_lazily():
    st = _mrnf(key_inds=[3], mrnf_col_inds_keep=[2, 0], mrnf_limit=4, output_batch_size=99, dropna=False)
    assert isinstance(st, G.ShardedMrnfState) and st.local.handle is None and st.final is None and st.n_ranks is None
    assert st.union == [0, 1, 2, 3]
    assert st.local.mrnf == ((1,), (True,), (True,), (0, 1, 2, 3)) and st.local.mrnf_limit == 4 and not st.local.dropna
    assert st.local.output_batch_size == 0 and not st.local.parallel  # the winners leave the local state as one batch
    G.delete_groupby_state(st)


def test_mrnf_verbs_dispatch(monkeypatch):
    st = _mrnf()
    monkeypatch.setattr(G.ShardedMrnfState, "consume", lambda self, t, last: (last, True))
    assert G.groupby_build_consume_batch(st, _table(), False) == (False, True)
    with pytest.raises(B200Error, match="before the last batch"):
        G.groupby_produce_output_batch(st)
    st.final = st.local
    with pytest.raises(B200Error, match="after is_last"):
        G.groupby_build_consume_batch(st, _table(), True)


def test_the_parallel_groupby_mrnf_still_refuses_more_than_one_rank(monkeypatch):
    import torch.distributed as dist

    monkeypatch.setattr(dist, "is_initialized", lambda: True)
    monkeypatch.setattr(dist, "get_world_size", lambda group=None: 2)
    st = G.init_groupby_state(-1, [0], (G.MRNF,), (0, 0), (), mrnf_sort_col_inds=[1], mrnf_sort_col_asc=[True], mrnf_sort_col_na=[True],
                              mrnf_col_inds_keep=[2], parallel=True)
    with pytest.raises(B200Error, match="a sharded min_row_number_filter is not supported"):
        G.groupby_build_consume_batch(st, _table(), False)


def test_physical_aggregate_builds_the_sharded_mrnf():
    op = PhysicalAggregate([0], [], dropna=False, parallel=True, mrnf=([1], [False], [True], [2, 0]), mrnf_limit=3, output_batch_size=8)
    st = op.state
    assert isinstance(st, G.ShardedMrnfState) and st.spec == ((1,), (False,), (True,), (2, 0)) and st.output_batch_size == 8
    assert st.args[2:] == (3, False)
    local = PhysicalAggregate([0], [], parallel=False, mrnf=([1], [True], [True], [2])).state
    assert type(local) is G.GroupbyState and local.mrnf is not None
    with pytest.raises(B200Error, match="cannot be combined"):
        PhysicalAggregate([0], [("sum", 1)], parallel=True, mrnf=([1], [True], [True], [2]))
