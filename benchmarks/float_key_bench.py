"""Float-key groupby against the same groupby on int64 keys, 1 x H100.

    python benchmarks/float_key_bench.py [--rows 2000000000] [--groups 1000000,30] [--reps 3]

Shape: BASELINE.json configs[1] (`--rows` rows, SUM + COUNT of an int64 value column) with float64 keys k_int * 0.5 + 0.25,
where k_int is the int64 key column of the same seeded rows (bench.py's generator), once per `--groups` value.  Both key
columns and the value column are resident in HBM.  One step = init state -> consume one device batch -> finalize -> produce,
as bench.py's step.  Per group count:
  ms_per_step   int64-key and float64-key steps alternated in one process, median of `--reps` (CUDA events, one warm-up each)
  path          SM-partitioned launches (metric 8), of them narrow-row ones (metric 14), low-cardinality launches (metric 10)
  prepass       the canonicalisation kernel (canon_float_key_kernel) alone, from a torch.profiler run of its own: kernel
                time per step and its rate over the 16 B/row it moves (8 read, 8 written)
  check         every group of both outputs against a torch bincount / index_add_ over k_int; integers bit-exact
The card's name and power limit are printed with the numbers.
"""

from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30).stdout.strip()
    except Exception as e:
        q = f"nvidia-smi unavailable ({e})"
    return q


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=2_000_000_000)
    ap.add_argument("--groups", default="1000000,30")
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--seed", type=int, default=1)
    args = ap.parse_args()

    import torch

    from bodo_b200 import _lib, synth
    from bodo_b200.streaming import groupby as G
    from bodo_b200.table import Column, CTypes, Table

    _lib.require_gpu()
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    stream = torch.cuda.current_stream(dev)
    sp = stream.cuda_stream
    n = args.rows
    print(json.dumps({"card": card(), "torch_device": torch.cuda.get_device_name(dev)}), flush=True)
    ok_all = True
    for ng in (int(x) for x in args.groups.split(",")):
        kint = torch.empty(n, dtype=torch.int64, device=dev)
        vals = torch.empty(n, dtype=torch.int64, device=dev)
        synth.device_fill(kint, vals, 0, ng, args.seed, sp)
        kflt = torch.empty(n, dtype=torch.float64, device=dev)
        for r0 in range(0, n, 1 << 27):  # (in slices: no full-size temporary)
            kflt[r0:r0 + (1 << 27)] = kint[r0:r0 + (1 << 27)].to(torch.float64).mul_(0.5).add_(0.25)
        torch.cuda.synchronize(dev)
        tables = {"int64": Table([Column(kint, None, CTypes.INT64), Column(vals, None, CTypes.INT64)], ["key", "val"]),
                  "float64": Table([Column(kflt, None, CTypes.FLOAT64), Column(vals, None, CTypes.INT64)], ["key", "val"])}

        def reference():  # per k_int, the row count and the (wrapping) int64 sum (a function: no slice outlives it)
            cnt = torch.zeros(ng, dtype=torch.int64, device=dev)
            ssum = torch.zeros(ng, dtype=torch.int64, device=dev)
            for r0 in range(0, n, 1 << 27):
                kk = kint[r0:r0 + (1 << 27)]
                cnt += torch.bincount(kk, minlength=ng)
                ssum.index_add_(0, kk, vals[r0:r0 + (1 << 27)])
            return cnt, ssum

        cnt, ssum = reference()
        n_exp = int((cnt > 0).sum().item())

        def check(kind, out):
            m = out.n_rows
            ok_ = torch.as_tensor(out.columns[0].data, device=dev)[:m]
            ki = ok_.to(torch.int64) if kind == "int64" else ((ok_ - 0.25) * 2.0).to(torch.int64)
            if kind == "float64":  # the key must come back as exactly k_int * 0.5 + 0.25
                bad_key = int((ki.to(torch.float64) * 0.5 + 0.25 != ok_).sum().item())
            else:
                bad_key = 0
            inr = (ki >= 0) & (ki < ng)
            safe = torch.where(inr, ki, torch.zeros_like(ki))
            s = torch.as_tensor(out.columns[1].data, device=dev)[:m]
            c = torch.as_tensor(out.columns[2].data, device=dev)[:m]
            bad = int((~inr | (s != ssum[safe]) | (c != cnt[safe])).sum().item()) + bad_key + (m - torch.unique(ki).numel())
            return bad == 0 and m == n_exp, bad

        def step(kind, collect=False):
            st = G.init_groupby_state(-1, (0,), ("sum", "count"), (0, 1, 2), (1, 1), expected_groups=ng, output_batch_size=1 << 40,
                                      device=0, stream=sp)
            G.groupby_build_consume_batch(st, tables[kind], True, True)
            out, last = G.groupby_produce_output_batch(st, True)
            assert last
            res = None
            if collect:
                res = {"check": check(kind, out), "spg": G.get_metric(st, 8), "spgn": G.get_metric(st, 14), "lc": G.get_metric(st, 10)}
            G.delete_groupby_state(st)
            return res

        def timed(kind):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(stream)
            step(kind)
            e1.record(stream)
            torch.cuda.synchronize(dev)
            return e0.elapsed_time(e1)

        for kind in tables:  # warm-up
            step(kind)
        times = {k: [] for k in tables}
        for _ in range(args.reps):
            for kind in tables:
                times[kind].append(timed(kind))
        info = {kind: step(kind, collect=True) for kind in tables}

        # the pre-pass alone: kernel time from a profiled float-key step
        from torch.profiler import ProfilerActivity, profile
        torch.cuda.synchronize(dev)
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            step("float64")
            torch.cuda.synchronize(dev)
        def dev_us(e):
            return getattr(e, "self_device_time_total", None) or getattr(e, "self_cuda_time_total", 0.0)
        ka = prof.key_averages()
        pre = [e for e in ka if "canon_float_key_kernel" in e.key]
        pre_us, n_pre = sum(dev_us(e) for e in pre), sum(e.count for e in pre)
        all_us = sum(dev_us(e) for e in ka)

        med = {k: sorted(v)[len(v) // 2] for k, v in times.items()}
        ok = all(info[k]["check"][0] for k in info)
        ok_all = ok_all and ok
        print(json.dumps({
            "rows": n, "groups": ng, "aggs": ["sum", "count"], "card": card(),
            "ms_per_step": {k: round(v, 3) for k, v in med.items()}, "runs_ms": {k: [round(x, 3) for x in v] for k, v in times.items()},
            "float_over_int": round(med["float64"] / med["int64"], 3),
            "path": {k: {m: info[k][m] for m in ("spg", "spgn", "lc")} for k in info},
            "prepass": {"launches": n_pre, "ms": round(pre_us / 1e3, 3), "share_of_kernel_time": round(pre_us / all_us, 3) if all_us else None,
                        "GB_per_s": round(16 * n / (pre_us * 1e-6) / 1e9, 1) if pre_us else None},
            "check": {k: ("every group equal to the torch recomputation" if info[k]["check"][0] else f"MISMATCH ({info[k]['check'][1]} bad)")
                      for k in info},
        }), flush=True)
        del tables, kint, vals, kflt, cnt, ssum
        torch.cuda.empty_cache()
    if not ok_all:
        sys.exit(3)


if __name__ == "__main__":
    main()
