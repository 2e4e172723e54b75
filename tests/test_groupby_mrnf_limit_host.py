"""CPU tests (no GPU) of the min_row_number_filter's row limit (mrnf_limit, QUALIFY ROW_NUMBER() <= n): argument validation and its
messages, the state's attributes, the physical helper's plumbing, the C header's entry and rules, and that consume refuses to run
without a device or on more than one rank."""

import numpy as np
import pandas as pd
import pytest

from bodo_b200 import B200Error, _lib
from bodo_b200.streaming import groupby as G
from bodo_b200.table import CTypes, Table
from tests.test_gpu_join_sharded import LockstepGroup, RankError
from tests.test_groupby_mrnf_host import mrnf_state


@pytest.fixture
def lockstep(monkeypatch):
    """lockstep(R) -> a LockstepGroup of R ranks, installed as torch.distributed for this test."""
    return lambda n: LockstepGroup(n).install(monkeypatch)


def test_the_limit_is_stored_beside_the_unchanged_mrnf_tuple():
    st = mrnf_state(sort=(2, 0), asc=(False, True), na=(0, 1), keep=(3, 0), fcols=(1, 2, 3), offs=(0, 3), mrnf_limit=3)
    assert st.mrnf == ((2, 0), (False, True), (False, True), (3, 0))
    assert st.mrnf_limit == 3 and st.handle is None
    assert mrnf_state().mrnf_limit == 1
    assert mrnf_state(mrnf_limit=np.int64(7)).mrnf_limit == 7
    assert mrnf_state(mrnf_limit=(1 << 31) - 1).mrnf_limit == (1 << 31) - 1


@pytest.mark.parametrize("bad", [True, False, 0, -1, 2.0, 2.5, "3", None, 1 << 31, 1 << 40])
def test_bad_limits_name_mrnf_limit(bad):
    with pytest.raises(B200Error, match="mrnf_limit"):
        mrnf_state(mrnf_limit=bad)


def test_a_limit_needs_min_row_number_filter():
    with pytest.raises(B200Error, match="mrnf_limit=3 needs min_row_number_filter"):
        G.init_groupby_state(-1, (0,), ("sum",), (0, 1), (1,), mrnf_limit=3)
    with pytest.raises(B200Error, match="mrnf_limit"):
        G.init_groupby_state(-1, (0,), ("sum",), (0, 1), (1,), mrnf_limit=0)
    st = G.init_groupby_state(-1, (0,), ("sum",), (0, 1), (1,), mrnf_limit=1)  # the default, spelled out
    assert st.mrnf is None and st.mrnf_limit == 1


def test_physical_helpers_forward_the_limit(monkeypatch):
    from bodo_b200 import physical
    from bodo_b200.physical import PhysicalAggregate

    op = PhysicalAggregate([0], [], dropna=False, mrnf=([2], [False], [True], [1, 0]), mrnf_limit=4)
    assert op.state.mrnf == ((2,), (False,), (True,), (1, 0)) and op.state.mrnf_limit == 4
    op.Finalize()
    df = pd.DataFrame({"k": [1, 1, 2], "o": [3.0, 1.0, 2.0]})
    with pytest.raises(B200Error, match="mrnf_limit"):
        physical.min_row_number_filter(df, "k", "o", n=0)
    seen, real = [], G.init_groupby_state

    def spy(*args, **kw):  # the state min_row_number_filter asks for, without running it
        seen.append(real(*args, **kw).mrnf_limit)
        raise StopIteration

    monkeypatch.setattr(G, "init_groupby_state", spy)
    for n in (1, 5):
        with pytest.raises(StopIteration):
            physical.min_row_number_filter(df, "k", "o", n=n)
    assert seen == [1, 5]


def test_header_declares_the_entry_and_its_rules():
    src = open(_lib.HEADER).read()
    assert "b200_groupby_state_init_mrnf_limit" in _lib.declared_symbols()
    i = src.index("void* b200_groupby_state_init_mrnf_limit(")
    doc = src[src.rindex("/*", 0, i):i]
    for needle in ("rows_per_group", "rank order", "arrival", "at most 26", "2^31", "groups x rows_per_group", "beyond",
                   "ROW_NUMBER()", "head(rows_per_group)", "bit-identical", "18", "19"):
        assert needle in doc, needle
    decl = src[i:src.index(";", i)]
    assert decl.rstrip(")").endswith("int64_t rows_per_group")


def test_consume_without_gpu_raises():
    L = _lib.lib()
    if L.b200_device_count() > 0:
        pytest.skip("a GPU is visible")
    st = mrnf_state(mrnf_limit=3)
    t = Table.from_pandas(pd.DataFrame({"k": [1, 1, 2], "o": [3.0, 1.0, 2.0]}))
    with pytest.raises(B200Error, match="no CUDA device|no CPU fallback|CUDA-only"):
        G.groupby_build_consume_batch(st, t, True, True)
    ffi = _lib.ffi
    h = L.b200_groupby_state_init_mrnf_limit(-1, ffi.new("int8_t[]", [CTypes.INT64, CTypes.FLOAT64]), ffi.new("int8_t[]", [0, 0]), 2, 1,
                                             ffi.new("int32_t[]", [1]), ffi.new("int32_t[]", [1]), ffi.new("int32_t[]", [1]), 1,
                                             ffi.new("int32_t[]", [1, 1]), 32768, 0, 0, 0, 1, 0, 0, ffi.NULL, 3)
    assert h == ffi.NULL and "no CUDA device" in ffi.string(L.b200_last_error()).decode()


def test_sharded_state_with_a_limit_is_refused(lockstep):
    """A parallel state with mrnf_limit=3 on a 2-rank group raises the sharded refusal at its first consume call."""
    from tests.test_gpu_join_exact import col

    t = Table([col(CTypes.INT64, np.arange(10)), col(CTypes.INT64, np.arange(10))], ["k", "o"])
    with pytest.raises(RankError) as ei:
        lockstep(2).run(lambda r: G.groupby_build_consume_batch(mrnf_state(parallel=True, mrnf_limit=3), t, True, True))
    assert ei.value.rank == 0 and isinstance(ei.value.error, B200Error)
    assert "a sharded min_row_number_filter is not supported" in str(ei.value.error)
