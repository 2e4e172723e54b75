"""Sharded full sort (streaming.sort.init_sharded_sort_state): the receiver's merge of sorted runs against a radix re-sort, and
the sharded operator's step time.

    python benchmarks/sharded_sort_bench.py [--rows 268435456] [--reps 5]
    python -m torch.distributed.run --nproc-per-node G benchmarks/sharded_sort_bench.py [--rows 268435456] [--reps 3]

Data, resident in HBM: a float64 key (uniform doubles in [0, 1)) and two int64 columns (the row id and a copy of it).

One GPU (no torch.distributed): the rows are cut into P = 2, 4 and 8 runs of equal length, each sorted by the key (torch, not
timed), as a receiving rank holds them after the exchange.  Every timed call is the is_last call (with an empty batch) after
the rows were consumed, so it holds the sort or merge, the gather of every column into the output and the bitmap packing:
  resort_ms   a full sort (b200_sort_state_init_full) of the same rows: the radix sort the merge replaces
  merge_ms    a merge state (b200_sort_state_init_runs) with the P run lengths: ceil(log2 P) merge-path rounds
The two are alternated, `--reps` times each, after one warm-up of each; medians are reported.  The phases of one sharded step
at these rows per rank are also timed: local_sort_ms (the full sort above), sample_split_ms (b200_sort_sample of 4096 samples
plus b200_sort_count_below of P - 1 splitters on the sorted rows) and merge_ms.  Checks: the merged key column is
nondecreasing, and the row-id column equals the re-sort's.

Under torch.distributed.run (one process per GPU, NCCL): per-step time of the sharded sort at `--rows` rows per rank (init ->
consume -> is_last -> produce every batch -> delete, all ranks), against a full sort of one rank's rows on one GPU.  Rank 0
prints the result.

The card's name and power limit are printed with the numbers, one JSON line per case."""

from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def card(dev=0):
    try:
        return subprocess.run(["nvidia-smi", f"--id={dev}", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                              text=True, timeout=30).stdout.strip()
    except Exception as e:  # noqa: BLE001
        return f"nvidia-smi unavailable ({e})"


def make_rows(torch, n, dev, seed=1234):
    from bodo_b200.table import ArrTypes, Column, CTypes, Table

    g = torch.Generator(device=dev)
    g.manual_seed(seed)
    key = torch.rand(n, dtype=torch.float64, device=dev, generator=g)
    rid = torch.arange(n, dtype=torch.int64, device=dev)
    return key, rid, lambda k, a, b: Table([Column(k, None, CTypes.FLOAT64, ArrTypes.NUMPY, n), Column(a, None, CTypes.INT64, ArrTypes.NUMPY, n),
                                            Column(b, None, CTypes.INT64, ArrTypes.NUMPY, n)], ["k", "a", "b"])


def timed_finish(torch, S, t, runs=None):
    """A state that consumed t: returns (state, ms of the is_last call)."""
    st = S.SortState(-1, None, 0, ["k"], [True], ["last"], t.names, False, 1 << 30, None, 0, None, full=True)
    st.runs = runs
    st._ensure(t)
    st._consume(t, False)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    st._consume(_empty(t), True)
    torch.cuda.synchronize()
    st.done = True
    return st, (time.perf_counter() - t0) * 1e3


def _empty(t):
    from bodo_b200.table import Column, Table

    return Table([Column(c.data[:0], None, c.c_type, c.arr_type, 0) for c in t.columns], list(t.names))


def sample_split_ms(torch, S, st, P, n):
    import numpy as np

    from bodo_b200 import _lib
    from bodo_b200._lib import ffi

    L = _lib.lib()
    s = min(S.SAMPLES_PER_RANK, n)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    rec = np.zeros((s, 4), dtype=np.uint64)
    _lib.check(L.b200_sort_sample(st.handle, s, 0, ffi.cast("uint64_t*", rec.ctypes.data)), "sample")
    spl = np.ascontiguousarray(S.choose_splitters(rec, np.diff(np.arange(s + 1) * n // s), P))
    cnt = np.zeros(len(spl), dtype=np.int64)
    _lib.check(L.b200_sort_count_below(st.handle, ffi.cast("uint64_t*", spl.ctypes.data), len(spl), 0,
                                       ffi.cast("int64_t*", cnt.ctypes.data)), "count below")
    return (time.perf_counter() - t0) * 1e3


def one_gpu(args):
    import torch

    from bodo_b200 import _lib
    from bodo_b200.streaming import sort as S

    _lib.require_gpu()
    dev = torch.device("cuda", 0)
    n = args.rows
    key, rid, mk = make_rows(torch, n, dev)
    name = card()
    for P in (2, 4, 8):
        runs = [n // P] * P
        runs[-1] += n - sum(runs)
        k2, a2 = key.clone(), rid.clone()
        off = 0
        for m in runs:  # each run sorted by the key, stably, as the exchange delivers it
            v, i = torch.sort(key[off: off + m], stable=True)
            k2[off: off + m] = v
            a2[off: off + m] = rid[off: off + m][i]
            off += m
        t = mk(k2, a2, a2.clone())
        merge, resort, split = [], [], []
        for rep in range(args.reps + 1):
            st_m, ms_m = timed_finish(torch, S, t, runs)
            st_r, ms_r = timed_finish(torch, S, t)
            ms_s = sample_split_ms(torch, S, st_r, P, n)
            if rep == 0:  # check once: merged keys nondecreasing, row ids equal to the re-sort's
                om, _ = st_m._produce_phys(True)
                orr, _ = st_r._produce_phys(True)
                km = torch.as_tensor(om.columns[0].data, device=dev)
                ok = bool((km[1:] >= km[:-1]).all()) and torch.equal(torch.as_tensor(om.columns[1].data, device=dev),
                                                                     torch.as_tensor(orr.columns[1].data, device=dev))
                if not ok:
                    print(json.dumps({"case": f"merge_P{P}", "check": "FAILED"}), flush=True)
                    sys.exit(1)
            else:
                merge.append(ms_m)
                resort.append(ms_r)
                split.append(ms_s)
            S.delete_stream_sort_state(st_m)
            S.delete_stream_sort_state(st_r)
            torch.cuda.synchronize()
        del t, k2, a2
        torch.cuda.empty_cache()
        mm, rm = statistics.median(merge), statistics.median(resort)
        print(json.dumps({"case": f"merge_P{P}", "rows": n, "merge_ms": round(mm, 2), "resort_ms": round(rm, 2),
                          "speedup": round(rm / mm, 2), "local_sort_ms": round(rm, 2),
                          "sample_split_ms": round(statistics.median(split), 2), "merge_spread_ms": [round(x, 2) for x in sorted(merge)],
                          "resort_spread_ms": [round(x, 2) for x in sorted(resort)], "check": "ok", "card": name}), flush=True)


def distributed(args):
    import torch
    import torch.distributed as dist

    from bodo_b200.streaming import sort as S

    rank, world = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"])
    local = int(os.environ.get("LOCAL_RANK", rank))
    torch.cuda.set_device(local)
    dev = torch.device("cuda", local)
    dist.init_process_group("nccl", device_id=dev)
    n = args.rows
    key, rid, mk = make_rows(torch, n, dev, seed=1234 + rank)
    t = mk(key, rid + rank * n, rid.clone())

    def step(sharded):
        dist.barrier()
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        if sharded:
            st = S.init_sharded_sort_state(-1, ["k"], True, "last", t.names, output_batch_size=1 << 24)
        else:
            st = S.init_stream_sort_state(-1, None, 0, ["k"], True, "last", t.names, output_batch_size=1 << 24, full=True)
        S.sort_build_consume_batch(st, t, True)
        while not S.produce_output_batch(st)[1]:
            pass
        torch.cuda.synchronize()
        ms = (time.perf_counter() - t0) * 1e3
        S.delete_stream_sort_state(st)
        torch.cuda.synchronize()
        return ms

    sharded, local_ms = [], []
    for rep in range(args.reps + 1):
        a, b = step(True), step(False)
        if rep:
            sharded.append(a)
            local_ms.append(b)
    mx = torch.tensor([statistics.median(sharded)], device=dev)
    dist.all_reduce(mx, op=dist.ReduceOp.MAX)
    if rank == 0:
        print(json.dumps({"case": f"sharded_{world}gpu", "rows_per_rank": n, "step_ms": round(float(mx), 2),
                          "one_gpu_full_sort_ms": round(statistics.median(local_ms), 2), "card": card(local)}), flush=True)
    dist.destroy_process_group()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=1 << 28)
    ap.add_argument("--reps", type=int, default=5)
    args = ap.parse_args()
    if "WORLD_SIZE" in os.environ and int(os.environ["WORLD_SIZE"]) > 1:
        distributed(args)
    else:
        one_gpu(args)


if __name__ == "__main__":
    main()
