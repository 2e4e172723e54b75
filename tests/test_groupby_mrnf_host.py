"""CPU tests (no GPU) of the groupby's min_row_number_filter: argument validation and its messages, the C header's entry and
rules, the physical helper's plumbing, and that consume refuses to run without a device or on more than one rank."""

import os
import socket

import numpy as np
import pandas as pd
import pytest

from bodo_b200 import B200Error, _lib
from bodo_b200.streaming import groupby as G
from bodo_b200.table import ArrTypes, Column, CTypes, Table

MRNF = ("min_row_number_filter",)


def mrnf_state(sort=(1,), asc=(True,), na=(True,), keep=(0, 1), key_inds=(0,), fnames=MRNF, offs=(0, 1), fcols=(1,), **kw):
    return G.init_groupby_state(-1, key_inds, fnames, offs, fcols, mrnf_sort_col_inds=sort, mrnf_sort_col_asc=asc,
                                mrnf_sort_col_na=na, mrnf_col_inds_keep=keep, **kw)


def test_valid_arguments_build_an_mrnf_state():
    st = mrnf_state(sort=(2, 0), asc=(False, True), na=(0, 1), keep=(3, 0), fcols=(1, 2, 3), offs=(0, 3))
    assert st.mrnf == ((2, 0), (False, True), (False, True), (3, 0))
    assert st.fnames == () and st.handle is None and st.f_in_cols == (1, 2, 3)
    # the reference may list no input columns at all; a sort column may be a key
    assert mrnf_state(sort=(0,), fcols=(), offs=(0, 0)).mrnf[0] == (0,)


@pytest.mark.parametrize("kw, arg", [
    (dict(sort=()), "mrnf_sort_col_inds"),
    (dict(sort=(1, 2, 3, 4, 5), asc=(True,) * 5, na=(True,) * 5), "mrnf_sort_col_inds"),
    (dict(sort=(1, 1), asc=(True, True), na=(True, True)), "mrnf_sort_col_inds"),
    (dict(sort=(-1,)), "mrnf_sort_col_inds"),
    (dict(sort=(1.5,)), "mrnf_sort_col_inds"),
    (dict(asc=(True, False)), "mrnf_sort_col_asc"),
    (dict(na=()), "mrnf_sort_col_na"),
    (dict(keep=()), "mrnf_col_inds_keep"),
    (dict(keep=(0, 0)), "mrnf_col_inds_keep"),
    (dict(keep=(-2,)), "mrnf_col_inds_keep"),
    (dict(keep=tuple(range(27))), "mrnf_col_inds_keep"),
    (dict(offs=(0, 2)), "f_in_offsets"),
    (dict(offs=(0, 1, 1)), "f_in_offsets"),
    (dict(fcols=(0,)), "f_in_cols"),
])
def test_bad_arguments_name_the_argument(kw, arg):
    with pytest.raises(B200Error, match=arg):
        mrnf_state(**kw)


def test_mrnf_with_other_functions_or_without_its_arguments():
    # the message of the ordinary state (MRNF arguments beside another function) names min_row_number_filter
    with pytest.raises(B200Error, match="min_row_number_filter"):
        G.init_groupby_state(-1, (0,), ("sum",), (0, 1), (1,), mrnf_sort_col_inds=(1,))
    with pytest.raises(B200Error, match="min_row_number_filter cannot be combined"):
        mrnf_state(fnames=("min_row_number_filter", "sum"), offs=(0, 1, 2), fcols=(1, 1))
    with pytest.raises(B200Error, match="needs mrnf_sort_col_inds, mrnf_sort_col_asc, mrnf_sort_col_na, mrnf_col_inds_keep"):
        G.init_groupby_state(-1, (0,), MRNF, (0, 1), (1,))
    with pytest.raises(B200Error, match="needs mrnf_col_inds_keep"):
        G.init_groupby_state(-1, (0,), MRNF, (0, 1), (1,), mrnf_sort_col_inds=(1,), mrnf_sort_col_asc=(True,), mrnf_sort_col_na=(True,))


def test_physical_aggregate_routes_mrnf():
    from bodo_b200.physical import PhysicalAggregate

    op = PhysicalAggregate([0], [], dropna=False, mrnf=([2], [False], [True], [1, 0]))
    assert op.state.mrnf == ((2,), (False,), (True,), (1, 0)) and not op.state.dropna
    with pytest.raises(B200Error, match="min_row_number_filter cannot be combined"):
        PhysicalAggregate([0], [("sum", 1)], mrnf=([2], [True], [True], [1]))
    op.Finalize()  # nothing was created


def test_header_declares_the_entry_and_its_rules():
    src = open(_lib.HEADER).read()
    assert "b200_groupby_state_init_mrnf" in _lib.declared_symbols()
    i = src.index("void* b200_groupby_state_init_mrnf(")
    doc = src[src.rindex("/*", 0, i):i]
    for needle in ("groupby_state_init_py_entry (_groupby.cpp:4917-4970)", "sort_asc / sort_na / n_sort_keys / cols_to_keep",
                   "1 <= n_sort <= 4", "-0.0 ties with 0.0", "arrival", "bit-identical", "at most 26", "n_pes > 1",
                   "NaN is the NA key", "winner's -0.0", "metric 0: groups"):
        assert needle in doc, needle
    assert _lib.lib().b200_abi_version() == 1


def test_consume_without_gpu_raises():
    L = _lib.lib()
    if L.b200_device_count() > 0:
        pytest.skip("a GPU is visible")
    st = mrnf_state()
    t = Table.from_pandas(pd.DataFrame({"k": [1, 1, 2], "o": [3.0, 1.0, 2.0]}))
    with pytest.raises(B200Error, match="no CUDA device|no CPU fallback|CUDA-only"):
        G.groupby_build_consume_batch(st, t, True, True)
    # the C entry refuses too: there is no CPU path behind it
    ffi = _lib.ffi
    h = L.b200_groupby_state_init_mrnf(-1, ffi.new("int8_t[]", [CTypes.INT64, CTypes.FLOAT64]), ffi.new("int8_t[]", [0, 0]), 2, 1,
                                       ffi.new("int32_t[]", [1]), ffi.new("int32_t[]", [1]), ffi.new("int32_t[]", [1]), 1,
                                       ffi.new("int32_t[]", [1, 1]), 32768, 0, 0, 0, 1, 0, 0, ffi.NULL)
    assert h == ffi.NULL and "no CUDA device" in ffi.string(L.b200_last_error()).decode()


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _sharded_worker(rank, world, port, q):
    import torch.distributed as dist

    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        n = 10
        t = Table([Column(np.arange(n, dtype=np.int64), None, CTypes.INT64, ArrTypes.NUMPY, n),
                   Column(np.arange(n, dtype=np.int64), None, CTypes.INT64, ArrTypes.NUMPY, n)], ["k", "o"])
        st = mrnf_state(parallel=True)
        try:
            G.groupby_build_consume_batch(st, t, True, True)
            q.put((rank, "no error"))
        except B200Error as e:
            q.put((rank, str(e)))
    finally:
        dist.destroy_process_group()


@pytest.mark.timeout(300)
def test_sharded_mrnf_is_refused():
    """A parallel MRNF state on a process group of 2 ranks raises at its first consume call, before touching a device."""
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
        assert "a sharded min_row_number_filter is not supported" in res[r], res[r]
