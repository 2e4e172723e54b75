"""Host-side checks of the streaming window operator: argument validation, the key plan it hands the sort state, PhysicalWindow
plumbing and the sharded refusal (no GPU needed)."""

import os
import socket

import numpy as np
import pytest

from bodo_b200 import _lib
from bodo_b200._lib import B200Error
from bodo_b200.physical import PhysicalWindow
from bodo_b200.streaming import window as W

COLS = ["a", "b", "c", "d"]


def init(**kw):
    args = dict(operator_id=-1, partition_by=["a"], order_by=["b"], ascending=True, na_position="last",
                funcs=[("rn", "row_number")], col_names=COLS)
    args.update(kw)
    return W.init_window_state(**args)


def test_state_is_lazy_and_keeps_the_key_plan():
    st = init(partition_by=["c", "a"], order_by=["d"], ascending=False, na_position="first",
              funcs=[("rn", "row_number"), ("nt", "ntile", 4), ("pr", "percent_rank")])
    assert st.handle is None and st.full
    assert st.by == ["c", "a", "d"] and st.partition_by == ["c", "a"] and st.order_by == ["d"]
    assert st.asc == [True, True, False] and st.na_last == [True, True, False]  # PARTITION BY: ascending, NA last
    assert st.phys == [2, 0, 3, 1]
    assert st.out_names == ["c", "a", "d", "b", "rn", "nt", "pr"]
    assert [st.out_names[i] for i in st.out_order] == COLS + ["rn", "nt", "pr"]
    assert st.funcs == [("rn", 0, 0), ("nt", 5, 4), ("pr", 3, 0)]


def test_key_forms():
    assert init(partition_by="a", order_by=None).by == ["a"]
    assert init(partition_by=[], order_by="b").by == ["b"]
    st = init(partition_by=None, order_by=["b", "c"], ascending=[True, False], na_position=["first", "last"])
    assert st.asc == [True, False] and st.na_last == [False, True]
    assert init(partition_by=["a", "b", "c"], order_by=[], ascending=[], na_position=[]).by == ["a", "b", "c"]


@pytest.mark.parametrize("kw,msg", [
    (dict(partition_by=[], order_by=[]), "1 to 4 keys"),
    (dict(partition_by=["a", "b", "c"], order_by=["d", "x"]), "1 to 4 keys"),
    (dict(order_by=["zz"]), "must be distinct columns"),
    (dict(partition_by=["a"], order_by=["a"]), "must be distinct columns"),
    (dict(partition_by=["a", "a"]), "must be distinct columns"),
    (dict(order_by=["b", "c"], ascending=[True]), "one value or one entry per ORDER BY key"),
    (dict(order_by=["b"], na_position=["last", "last"]), "one value or one entry per ORDER BY key"),
    (dict(na_position="middle"), "na_position must be"),
    (dict(funcs=[]), "at least one window function"),
    (dict(funcs=[("x", "lag")]), "unknown window function"),
    (dict(funcs=[("x", "sum")]), "unknown window function"),
    (dict(funcs=[("x",)]), "unknown window function"),
    (dict(funcs=[(3, "rank")]), "unknown window function"),
    (dict(funcs=[("x", "ntile", 0)]), "ntile needs an integer n >= 1"),
    (dict(funcs=[("x", "ntile", -2)]), "ntile needs an integer n >= 1"),
    (dict(funcs=[("x", "ntile")]), "ntile needs an integer n >= 1"),
    (dict(funcs=[("x", "ntile", 2.5)]), "ntile needs an integer n >= 1"),
    (dict(funcs=[("x", "rank", 3)]), "rank takes no argument"),
    (dict(funcs=[("x", "rank"), ("x", "dense_rank")]), "duplicate output names"),
    (dict(funcs=[("b", "rank")]), "clash with input columns"),
    (dict(funcs=[(f"f{i}", "rank") for i in range(29)]), "exceed 32 output columns"),
])
def test_argument_checks(kw, msg):
    with pytest.raises(B200Error, match=msg):
        init(**kw)


def test_column_limit_is_inclusive():
    assert len(init(funcs=[(f"f{i}", "rank") for i in range(28)]).funcs) == 28


def test_produce_before_consume_raises():
    with pytest.raises(B200Error, match="before the last batch"):
        W.window_produce_output_batch(init())


def test_function_codes_match_the_header():
    with open(_lib.HEADER) as f:
        header = f.read()
    assert "0 row_number, 1 rank, 2 dense_rank, 3 percent_rank, 4 cume_dist, 5 ntile" in header
    assert W.FUNCS == {"row_number": 0, "rank": 1, "dense_rank": 2, "percent_rank": 3, "cume_dist": 4, "ntile": 5}


def test_abi_declares_the_window_entry():
    assert "b200_window_state_init" in _lib.declared_symbols()
    assert W.MAX_WINDOW_ROWS == 1 << 31 and W.MAX_COLS == 32


def test_physical_window_plumbing():
    op = PhysicalWindow("a", ["b"], [("rn", "row_number"), ("nt", "ntile", 2)], ascending=False, na_position="first")
    assert op.state is None
    assert op.args == ("a", ["b"], False, "first", [("rn", "row_number"), ("nt", "ntile", 2)], False)
    op.Finalize()  # nothing was created


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _sharded_worker(rank, world, port, q):
    import torch.distributed as dist

    from bodo_b200.table import ArrTypes, Column, CTypes, Table

    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        n = 10
        t = Table([Column(np.arange(n, dtype=np.int64), None, CTypes.INT64, ArrTypes.NUMPY, n)], ["k"])
        st = W.init_window_state(-1, ["k"], [], True, "last", [("rn", "row_number")], ["k"], parallel=True)
        try:
            W.window_build_consume_batch(st, t, True)
            q.put((rank, "no error"))
        except B200Error as e:
            q.put((rank, str(e)))
    finally:
        dist.destroy_process_group()


@pytest.mark.timeout(300)
def test_sharded_window_is_refused():
    """A parallel window state on a process group of 2 ranks raises at its first consume call, before touching a device."""
    import torch.multiprocessing as mp

    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_sharded_worker, args=(r, 2, port, q)) for r in range(2)]
    for p in procs:
        p.start()
    res = dict(q.get(timeout=240) for _ in range(2))
    for p in procs:
        p.join(timeout=60)
    for r in range(2):
        assert "a sharded window is not supported" in res[r], res[r]
