"""Sharded window and min_row_number_filter: the key-class partition against the reference partition, the local window at one
rank's share of the rows, and the sharded operators' step time.

    python benchmarks/sharded_window_bench.py [--rows 268435456] [--reps 5]
    python -m torch.distributed.run --nproc-per-node G benchmarks/sharded_window_bench.py [--rows 268435456] [--reps 3]

One GPU (no torch.distributed):
  partition   b200_shuffle_partition_classes (classes_ms) against b200_shuffle_partition (reference_ms) on the same `--rows` int64
              keys (uniform over int64, one column, 8 destinations: one NVLink box), alternated `--reps` times each after one warm-up
              of each; medians.  The two must place every row alike on these keys (no NaN): the send counts and the partitioned
              key columns are compared.
  narrow_keys the key-class partition of `--rows` int16 keys (the reference partition refuses them) and of `--rows` float64 keys
              with 1 % NaN (the reference partition places a NaN by its value, so it is timed beside it, not compared).
  local_step  the window step (init -> consume -> produce -> delete) of benchmarks/window_bench.py's data and rn_rank_dense
              functions at N / P rows, P = 2, 4, 8: what one rank computes after the exchange.
Under torch.distributed.run (one process per GPU, NCCL): the per-step time of the sharded window (window_bench.py's data, N rows per
rank in 2^24-row batches, rn_rank_dense OVER (PARTITION BY p ORDER BY o)) and of the sharded min_row_number_filter (mrnf_bench.py's
data and query, keeping (k, o, r)), init -> consume every batch -> produce -> delete on every rank, between barriers; rank 0 prints.
Run without it, the multi-GPU numbers are printed as not measured.

Every line carries the card's name and power limit; a step is timed with a host clock around work that ends in a device
synchronise."""

from __future__ import annotations

import argparse
import json
import os
import statistics
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from benchmarks.sharded_sort_bench import card  # noqa: E402
from benchmarks.window_bench import FUNCS3  # noqa: E402


def timed(torch, fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    r = fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) * 1e3, r


def window_data(torch, synth, n, dev, seed=61):
    """window_bench.py's columns: p int64 in [0, 10^6), o uniform float64 in [0, 1), r the row id."""
    g = torch.Generator(device=dev).manual_seed(seed)
    pk = torch.randint(0, 10**6, (n,), generator=g, device=dev, dtype=torch.int64)
    ok = torch.empty(n, dtype=torch.float64, device=dev)
    synth.device_fill(None, ok, 0, 1, seed + 1, torch.cuda.current_stream(dev).cuda_stream)
    return pk, ok, torch.arange(n, dtype=torch.int64, device=dev)


def batches(Table, Column, cols, names, n, batch):
    for r0 in range(0, n, batch):
        r1 = min(n, r0 + batch)
        yield Table([Column(c[r0:r1]) for c in cols], names), r1 == n


def one_gpu(args, torch, info):
    from bodo_b200 import synth
    from bodo_b200.shuffle import partition_device
    from bodo_b200.streaming import window as W
    from bodo_b200.table import Column, Table

    dev = torch.device("cuda", 0)
    n, P = args.rows, 8
    g = torch.Generator(device=dev).manual_seed(7)
    keys = torch.randint(-(1 << 62), 1 << 62, (n,), generator=g, device=dev, dtype=torch.int64)
    t = Table([Column(keys)], ["k"])
    runs = {"classes": lambda: partition_device(t, 1, P, by_class=True), "reference": lambda: partition_device(t, 1, P)}
    for f in runs.values():
        f()
    ms = {k: [] for k in runs}
    for _ in range(args.reps):
        for k, f in runs.items():
            ms[k].append(timed(torch, f)[0])
    a, b = runs["classes"](), runs["reference"]()
    same = a[1] == b[1] and bool(torch.equal(a[0].columns[0].data, b[0].columns[0].data))
    del a, b
    print(json.dumps({"case": "partition", "rows": n, "n_pes": P, "classes_ms": statistics.median(ms["classes"]),
                      "reference_ms": statistics.median(ms["reference"]), "same_placement": same, **info}), flush=True)
    del keys, t
    i16 = torch.randint(-(1 << 15), 1 << 15, (n,), generator=g, device=dev, dtype=torch.int32).to(torch.int16)
    f64 = torch.rand(n, generator=g, device=dev, dtype=torch.float64)
    f64[torch.rand(n, generator=g, device=dev) < 0.01] = float("nan")
    t16, t64 = Table([Column(i16)], ["k"]), Table([Column(f64)], ["k"])
    cases = {"int16_classes": lambda: partition_device(t16, 1, P, by_class=True), "float64_classes": lambda: partition_device(t64, 1, P, by_class=True),
             "float64_reference": lambda: partition_device(t64, 1, P)}
    for f in cases.values():
        f()
    ms = {k: [] for k in cases}
    for _ in range(args.reps):
        for k, f in cases.items():
            ms[k].append(timed(torch, f)[0])
    print(json.dumps({"case": "narrow_keys", "rows": n, "n_pes": P, **{f"{k}_ms": statistics.median(v) for k, v in ms.items()}, **info}),
          flush=True)
    del i16, f64, t16, t64
    torch.cuda.empty_cache()
    for p in (2, 4, 8):
        m = n // p
        cols = window_data(torch, synth, m, dev)

        def step():
            st = W.init_window_state(-1, ["p"], ["o"], True, "last", FUNCS3, ["p", "o", "r"], output_batch_size=1 << 30, device=0)
            for b, last in batches(Table, Column, cols, ["p", "o", "r"], m, 1 << 24):
                W.window_build_consume_batch(st, b, last)
            W.window_produce_output_batch(st)
            W.delete_window_state(st)
        step()
        v = [timed(torch, step)[0] for _ in range(args.reps)]
        print(json.dumps({"case": "local_step", "ranks": p, "rows": m, "ms_per_step": statistics.median(v), **info}), flush=True)
        del cols
        torch.cuda.empty_cache()


def sharded(args, torch, info):
    import torch.distributed as dist

    from bodo_b200 import synth
    from bodo_b200.streaming import groupby as G
    from bodo_b200.streaming import window as W
    from bodo_b200.table import Column, Table

    rank, world = dist.get_rank(), dist.get_world_size()
    dev = torch.device("cuda", rank)
    n = args.rows
    cols = window_data(torch, synth, n, dev, seed=61 + rank)

    def window_step():
        st = W.init_sharded_window_state(-1, ["p"], ["o"], True, "last", FUNCS3, ["p", "o", "r"], output_batch_size=1 << 30, device=rank)
        for b, last in batches(Table, Column, cols, ["p", "o", "r"], n, 1 << 24):
            W.window_build_consume_batch(st, b, last)
        W.window_produce_output_batch(st)
        W.delete_window_state(st)

    def mrnf_step():
        st = G.init_sharded_mrnf_state(-1, (0,), (1,), (False,), (True,), (0, 1, 2), output_batch_size=1 << 30, device=rank)
        for b, last in batches(Table, Column, cols, ["k", "o", "r"], n, 1 << 24):
            G.groupby_build_consume_batch(st, b, last)
        G.groupby_produce_output_batch(st)
        G.delete_groupby_state(st)

    for name, step in (("sharded_window", window_step), ("sharded_mrnf", mrnf_step)):
        step()
        v = []
        for _ in range(args.reps):
            dist.barrier()
            ms, _ = timed(torch, step)
            v.append(ms)
        if rank == 0:
            print(json.dumps({"case": name, "ranks": world, "rows_per_rank": n, "ms_per_step": statistics.median(v), **info}), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=1 << 28)
    ap.add_argument("--reps", type=int, default=5)
    args = ap.parse_args()

    import torch

    from bodo_b200 import _lib

    _lib.require_gpu()
    if int(os.environ.get("WORLD_SIZE", "1")) > 1:
        import torch.distributed as dist

        rank = int(os.environ["LOCAL_RANK"])
        torch.cuda.set_device(rank)
        dist.init_process_group("nccl", device_id=torch.device("cuda", rank))
        try:
            sharded(args, torch, {"card": card(rank)})
        finally:
            dist.destroy_process_group()
        return
    torch.cuda.set_device(0)
    info = {"card": card(0)}
    one_gpu(args, torch, info)
    for name in ("sharded_window", "sharded_mrnf"):
        print(json.dumps({"case": name, "ms_per_step": "not measured", "reason": "needs torch.distributed.run over 2 or more GPUs",
                          **info}), flush=True)


if __name__ == "__main__":
    main()
