"""CPU-side checks added in round 2: what the shipped cubins contain (cuobjdump is part of the CUDA toolkit, no GPU needed) and
host-side plumbing of the join kinds / bench arguments."""

import os
import re
import shutil
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "bodo_b200", "libbodo_b200.so")


def _cuobjdump():
    """cuobjdump on PATH, else the one beside the nvcc the library was built with."""
    found = shutil.which("cuobjdump")
    if found:
        return found
    from bodo_b200 import build

    try:
        cand = os.path.join(os.path.dirname(build._nvcc()), "cuobjdump")
    except RuntimeError:
        return None
    return cand if os.path.exists(cand) else None


@pytest.mark.skipif(_cuobjdump() is None or not os.path.exists(LIB), reason="needs cuobjdump and the built library")
def test_cubins_are_sm90a_only_and_the_partition_kernels_use_tma():
    """The library holds sm_90a code only; the three K1 kernels of the SM-partitioned path stage their tiles with TMA bulk copies
    completed on an mbarrier (SASS UBLKCP + SYNCS), the low-cardinality kernel reduces uniform warps with REDUX."""
    sass = subprocess.run([_cuobjdump(), "-sass", LIB], capture_output=True, text=True, check=True).stdout
    assert set(re.findall(r"arch = (sm_\w+)", sass)) == {"sm_90a"}
    per_kernel, cur = {}, None
    for line in sass.splitlines():
        m = re.search(r"Function : (\S+)", line)
        if m:
            cur = m.group(1)
            per_kernel[cur] = {"UBLKCP": 0, "SYNCS": 0, "REDUX": 0, "ATOMS": 0}
            continue
        if cur:
            for k in per_kernel[cur]:
                if f" {k}" in line or f"\t{k}" in line:
                    per_kernel[cur][k] += 1
    def kernels(sub):
        return {k: v for k, v in per_kernel.items() if sub in k}
    for sub in ("spg_partition_tma_kernel", "spgn_partition_kernel", "spgg_partition_kernel"):
        ks = kernels(sub)
        assert ks, sub
        for name, c in ks.items():
            assert c["UBLKCP"] >= 1 and c["SYNCS"] >= 1 and c["ATOMS"] >= 1, (name, c)
    for sub in ("spg_aggregate_kernel", "spgn_aggregate_kernel", "spgg_aggregate_kernel"):
        for name, c in kernels(sub).items():
            assert c["ATOMS"] >= 2, (name, c)
    assert any(c["REDUX"] >= 4 for name, c in kernels("groupby_lowcard_kernel").items())


def test_join_kind_plumbing_needs_no_gpu_until_the_first_batch():
    from bodo_b200 import B200Error
    from bodo_b200.physical import PhysicalJoin
    from bodo_b200.streaming.join import init_join_state, runtime_join_filter
    from bodo_b200.table import Table
    import pandas as pd

    st = init_join_state(-1, (0,), (0,), ("k", "b"), ("k", "p"), False, False, is_mark_join=True)
    assert st.is_mark_join and not st.is_anti_join and st.handle is None
    assert PhysicalJoin(0, 0, ("k",), ("k",), how="anti").state.is_anti_join
    assert PhysicalJoin(0, 0, ("k",), ("k",), how="mark").state.is_mark_join
    assert PhysicalJoin(0, 0, ("k",), ("k",), how="left").state.probe_outer
    with pytest.raises(B200Error, match="device resident"):
        runtime_join_filter((st,), Table.from_pandas(pd.DataFrame({"k": [1, 2]})), ((0,),))


def test_bench_arguments_select_the_workloads(monkeypatch):
    sys.path.insert(0, ROOT)
    import bench

    monkeypatch.setattr(sys, "argv", ["bench.py", "--workload", "shuffle", "--n-dest", "4", "--rows", "1000"])
    a = bench.parse_args()
    assert a.workload == "shuffle" and a.n_dest == 4 and a.rows == 1000 and a.gpus == 1 and a.warmup >= 3
    monkeypatch.setattr(sys, "argv", ["bench.py", "--aggs", "mean,min,max", "--nullable", "--key-dtype", "int32", "--no-hint"])
    a = bench.parse_args()
    assert a.aggs == "mean,min,max" and a.nullable and a.key_dtype == "int32" and a.no_hint and a.workload == "groupby"
