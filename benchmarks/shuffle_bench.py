"""bench.py --workload shuffle: the RAW-ROW variant of BASELINE.json configs[3] — every rank hash-partitions its slice of the
`--rows`-row (int64 key, int64 value) table by hash_to_rank(key) (b200_shuffle_partition, csrc/shuffle.cu) and, at N > 1,
exchanges the partitions with one all-to-all-v per buffer (bodo_b200.shuffle.shuffle_table -> NCCL).  The groupby of the
headline line shuffles PARTIAL AGGREGATES instead (~16 MB per rank); this is the number for the rows themselves
(rows / N x 16 B per rank, 7/8 of it leaving the rank at N = 8), the path a high-cardinality groupby or a join takes.

  value     rows/s partitioned (and exchanged at N > 1), inputs resident in HBM, CUDA events, max over ranks
  roofline  the partition pass (dest_hist + scan + scatter kernels, timed together with CUDA events on their stream):
            algorithmic 32 B/row (16 B read + 16 B written), the 8 B/row key re-read of the histogram pass and the
            1 + 1 B/row destination bytes are overhead on top
  parity    untimed, at full size: rows per destination == bincount of the device hash_to_rank; per destination segment
            the sum mod 2^64 of keys and values equals the sum over the rows routed there; the source-row permutation is
            strictly increasing inside every segment (stable, like the reference's fill_send_array); at N > 1 every received key
            hashes to this rank and the global row count / key sum / value sum are preserved.
"""

from __future__ import annotations

import json
import os
import sys

METRIC = "shuffle rows/sec"
UNIT = "rows/s"


def run(args, ClockSampler, peaks):
    if args.impl == "reference":  # the CPU arm exists for the headline workload (bench.py) and the join only
        if int(os.environ.get("RANK", "0")) == 0:
            print(json.dumps({"impl": "reference", "unavailable": "no CPU arm for the shuffle workload; see bench.py --impl reference"}), flush=True)
        return
    import torch
    import torch.distributed as dist

    from bodo_b200 import _lib, synth
    from bodo_b200 import shuffle as S
    from bodo_b200.table import Column, Table

    world = int(os.environ.get("WORLD_SIZE", "1"))
    rank = int(os.environ.get("RANK", "0"))
    local_rank = int(os.environ.get("LOCAL_RANK", "0"))
    _lib.require_gpu()
    torch.cuda.set_device(local_rank)
    dev = torch.device("cuda", local_rank)
    if world > 1:
        dist.init_process_group("nccl", device_id=dev)
    stream = torch.cuda.current_stream(dev)
    sp = stream.cuda_stream
    n_dest = world if world > 1 else args.n_dest
    chunk = (args.rows + world - 1) // world
    row0 = min(rank * chunk, args.rows)
    n = min(chunk, args.rows - row0)
    keys = torch.empty(n, dtype=torch.int64, device=dev)
    vals = torch.empty(n, dtype=torch.int64, device=dev)
    synth.device_fill(keys, vals, row0, args.groups, args.seed, sp)
    torch.cuda.synchronize(dev)
    table = Table([Column(keys), Column(vals)], ["key", "val"])
    M = (1 << 64) - 1

    def barrier():
        if world > 1:
            dist.barrier()
        torch.cuda.synchronize(dev)

    def one_step():
        if world > 1:
            return S.shuffle_table(table, 1, True, stream=sp)
        return S.partition_device(table, 1, n_dest, sp)

    sampler = ClockSampler(local_rank) if rank == 0 else None
    for _ in range(max(args.warmup, 0)):
        one_step()
    barrier()
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    ev0.record(stream)
    for _ in range(args.steps):
        one_step()
    ev1.record(stream)
    barrier()
    ms = ev0.elapsed_time(ev1)
    clocks = sampler.stop() if sampler else None

    # partition pass alone (the dominant kernels), same launches
    p0, p1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    p0.record(stream)
    for _ in range(args.steps):
        S.partition_device(table, 1, n_dest, sp)
    p1.record(stream)
    torch.cuda.synchronize(dev)
    part_ms = p0.elapsed_time(p1) / args.steps

    # ---- parity (untimed) ----
    part, counts, perm = S.partition_device(table, 1, n_dest, sp, want_perm=True)
    _, dest = S.hash_keys_table(table, 1, n_dest, sp)
    torch.cuda.synchronize(dev)
    dest = dest.to(torch.int64)
    ok = counts == torch.bincount(dest, minlength=n_dest).tolist()
    pk = torch.as_tensor(part.columns[0].data, device=dev)
    pv = torch.as_tensor(part.columns[1].data, device=dev)
    off = 0
    for d in range(n_dest):
        c = counts[d]
        m = dest == d
        ok &= (int(pk[off:off + c].sum().item()) & M) == (int(keys[m].sum().item()) & M)
        ok &= (int(pv[off:off + c].sum().item()) & M) == (int(vals[m].sum().item()) & M)
        if c > 1:
            seg = perm[off:off + c]
            ok &= bool((seg[1:] > seg[:-1]).all().item())
            ok &= bool((dest[seg] == d).all().item())
        off += c
    del part, perm, pk, pv
    if world > 1:
        recv = S.shuffle_table(table, 1, True, stream=sp)
        rk = torch.as_tensor(recv.columns[0].data, device=dev)
        rv = torch.as_tensor(recv.columns[1].data, device=dev)
        _, rdest = S.hash_keys_table(Table([Column(rk.contiguous())], ["key"]), 1, world, sp)
        torch.cuda.synchronize(dev)
        ok &= bool((rdest == rank).all().item()) if rk.numel() else True
        tot = torch.tensor([rk.numel(), int(rk.sum().item()), int(rv.sum().item()), n, int(keys.sum().item()), int(vals.sum().item())],
                           dtype=torch.int64, device=dev)
        dist.all_reduce(tot)
        t = tot.tolist()
        ok &= t[0] == t[3] and (t[1] & M) == (t[4] & M) and (t[2] & M) == (t[5] & M)
        flag = torch.tensor([0 if ok else 1, 0], dtype=torch.float64, device=dev)
        flag[1] = ms
        mx = flag.clone()
        dist.all_reduce(mx, op=dist.ReduceOp.MAX)
        ok = mx[0].item() == 0
        ms = float(mx[1].item())
    peak, peak_kind = peaks()
    achieved = 32.0 * n / 1e9 / (part_ms * 1e-3)
    if rank == 0:
        print(json.dumps({
            "metric": METRIC, "value": args.rows * args.steps / (ms * 1e-3), "unit": UNIT, "n_gpus": world, "steps": args.steps,
            "warmup": args.warmup, "ms_per_step": ms / args.steps, "higher_is_better": True, "scaling": "strong", "vs_baseline": None,
            "dtype": "int64", "data": "synthetic",
            "config": {"workload": f"raw-row hash shuffle of a {args.rows}-row int64 2-col table over {world}xH100 "
                                   f"({'partition into ' + str(n_dest) + ' destinations, no exchange' if world == 1 else 'radix partition + NCCL all-to-all-v'}; "
                                   "raw-row variant of BASELINE.json configs[3])",
                       "rows": args.rows, "rows_per_gpu": n, "n_dest": n_dest, "l2": "inputs exceed the 50 MB L2; no flush needed",
                       "step": "partition (hist + scan + scatter)" + (" + count exchange + all-to-all-v of 2 buffers" if world > 1 else ""),
                       "result_check": "counts, per-destination key/value sums, stable order, placement ok" if ok else "MISMATCH"},
            "roofline": {"bound": "hbm", "achieved": achieved, "peak": peak, "unit": "GB/s", "frac": achieved / peak, "traffic": None,
                         "peak_kind": peak_kind, "kernel": "dest_hist_kernel + scan_hist_kernel + scatter_kernel (one partition pass)",
                         "avg_launch_ms": part_ms, "algorithmic_bytes_per_launch": 32.0 * n},
            "cpu_baseline": None, "e2e": None, "clocks": clocks, "gpu_launches": 3 * args.steps,
        }), flush=True)
    if world > 1:
        dist.destroy_process_group()
    if not ok:
        sys.exit(3)
