"""Host-side checks of the full streaming sort (ORDER BY without LIMIT): the opt-in keyword, argument validation, PhysicalSort
plumbing and the sharded refusal (no GPU needed)."""

import os
import socket

import numpy as np
import pytest

from bodo_b200 import _lib
from bodo_b200._lib import B200Error
from bodo_b200.physical import PhysicalSort
from bodo_b200.streaming import sort as S

COLS = ["a", "b", "c"]


def init(**kw):
    args = dict(operator_id=-1, limit=None, offset=0, by=["a"], asc=[True], na_position=["last"], col_names=COLS, full=True)
    args.update(kw)
    return S.init_stream_sort_state(**args)


def test_full_state_is_lazy_and_keeps_the_key_plan():
    st = init(by=["c", "a"], asc=[False, True], na_position=["first", "last"])
    assert st.full and st.handle is None
    assert st.phys == [2, 0, 1] and [st.phys[i] for i in st.out_order] == [0, 1, 2]
    assert st.asc == [False, True] and st.na_last == [False, True]
    assert init(offset=None).full


@pytest.mark.parametrize("kw", [dict(limit=10), dict(limit=0), dict(offset=3), dict(limit=5, offset=2)])
def test_full_sort_takes_no_limit_or_offset(kw):
    with pytest.raises(B200Error, match="full sort takes no limit or offset"):
        init(**kw)


@pytest.mark.parametrize("kw,msg", [
    (dict(by=[], asc=[], na_position=[]), "1 to 4 sort keys"),
    (dict(by=["a", "b"], asc=[True]), "one entry per sort key"),
    (dict(by=["zz"]), "must be distinct columns"),
    (dict(na_position="middle"), "na_position"),
])
def test_full_sort_argument_checks(kw, msg):
    with pytest.raises(B200Error, match=msg):
        init(**kw)


def test_limit_none_without_full_still_raises():
    with pytest.raises(B200Error, match="limit is required"):
        S.init_stream_sort_state(-1, None, 0, ["a"], [True], ["last"], COLS)
    with pytest.raises(B200Error, match="limit is required"):
        PhysicalSort(["a"])


def test_produce_before_consume_raises():
    with pytest.raises(B200Error, match="before the last batch"):
        S.produce_output_batch(init())


def test_physical_sort_full_plumbing():
    op = PhysicalSort(["a", "b"], [True, False], "first", full=True)
    assert op.full and op.state is None and op.args == (["a", "b"], [True, False], "first", None, 0, False)
    op.Finalize()
    for kw in (dict(limit=7), dict(offset=2)):
        with pytest.raises(B200Error, match="full sort takes no limit or offset"):
            PhysicalSort(["a"], full=True, **kw)


def test_abi_declares_the_full_sort_entry():
    assert "b200_sort_state_init_full" in _lib.declared_symbols()
    assert S.MAX_FULL_SORT_ROWS == 1 << 31


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
        st = S.init_stream_sort_state(-1, None, 0, ["k"], [True], ["last"], ["k"], parallel=True, full=True)
        try:
            S.sort_build_consume_batch(st, t, True)
            q.put((rank, "no error"))
        except B200Error as e:
            q.put((rank, str(e)))
    finally:
        dist.destroy_process_group()


@pytest.mark.timeout(300)
def test_sharded_full_sort_is_refused():
    """A parallel full-sort state on a process group of 2 ranks raises at its first consume call, before touching a device."""
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
        assert "a sharded full sort is not supported" in res[r], res[r]
