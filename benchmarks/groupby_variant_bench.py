"""bench.py --aggs ... [--nullable] [--key-dtype int32] [--val-dtype int32]: the groupby hot path on signatures OTHER than the
headline one (BASELINE.json configs[1] shape — `--rows` rows, `--groups` groups — with other aggregate functions, nullable
columns, 4-byte columns), 1 x H100.

One step = init state -> consume one device-resident batch -> finalize -> produce, as bench.py's headline step.
  value     rows/s with the inputs resident in HBM (CUDA events around `--steps` steps)
  roofline  consume launches (K1g + K2g pairs of the generic SM-partitioned path, or the direct kernel) timed by the library's
            CUDA events; algorithmic bytes = key + value bytes per row (+ 1/8 B per nullable column)
  parity    untimed, at full size: EVERY group against an independent torch recomputation (dense by key: scatter-add / amin /
            amax / bincount over the non-NA rows); integers bit-exact, mean within rtol 1e-9 (the device adds exact integer
            partial sums, the check divides the exact int64 sum)
No cpu_baseline / e2e legs: this line documents kernel generality, the headline line carries those.
"""

from __future__ import annotations

import json
import os
import sys

METRIC = "groupby rows/sec"
UNIT = "rows/s"
FT = {"sum", "count", "size", "mean", "min", "max"}


def run(args, ClockSampler, peaks):
    if args.impl == "reference":  # the CPU arm exists for the headline workload (bench.py) and the join only
        if int(os.environ.get("RANK", "0")) == 0:
            print(json.dumps({"impl": "reference", "unavailable": "no CPU arm for the groupby variant workload; see bench.py --impl reference"}), flush=True)
        return
    import torch

    from bodo_b200 import _lib, synth
    from bodo_b200.streaming import groupby as G
    from bodo_b200.table import ArrTypes, Column, CTypes, Table

    if int(os.environ.get("WORLD_SIZE", "1")) > 1:
        raise SystemExit("bench.py --aggs/--nullable variants run on one GPU")
    aggs = tuple(a.strip() for a in args.aggs.split(",") if a.strip())
    assert aggs and all(a in FT for a in aggs), f"--aggs takes a comma list of {sorted(FT)}"
    _lib.require_gpu()
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    stream = torch.cuda.current_stream(dev)
    sp = stream.cuda_stream
    n, ng = args.rows, args.groups
    keys = torch.empty(n, dtype=torch.int64, device=dev)
    vals = torch.empty(n, dtype=torch.int64, device=dev)
    synth.device_fill(keys, vals, 0, ng, args.seed, sp)
    kdt = torch.int32 if args.key_dtype == "int32" else torch.int64
    vdt = torch.int32 if args.val_dtype == "int32" else torch.int64
    if kdt == torch.int32:
        keys = keys.to(torch.int32)
    if vdt == torch.int32:
        vals = vals.to(torch.int32)
    kvalid = vvalid = None
    kmask = vmask = None
    if args.nullable:
        g = torch.Generator(device=dev); g.manual_seed(args.seed)
        nb = (n + 7) // 8 + 8

        def bitmap(p_null):
            # byte-wise random validity: bit = 1 with probability 1 - p_null
            bits = torch.rand(nb * 8, device=dev, generator=g) >= p_null
            w = (bits.view(-1, 8).to(torch.uint8) << torch.arange(8, device=dev, dtype=torch.uint8)).sum(1).to(torch.uint8)
            return w, bits[:n]

        kvalid, kmask = bitmap(0.01)
        vvalid, vmask = bitmap(0.10)
        del g
    torch.cuda.synchronize(dev)
    kct = CTypes.INT32 if kdt == torch.int32 else CTypes.INT64
    vct = CTypes.INT32 if vdt == torch.int32 else CTypes.INT64
    arr = ArrTypes.NULLABLE_INT_BOOL if args.nullable else ArrTypes.NUMPY
    table = Table([Column(keys, kvalid, kct, arr, n), Column(vals, vvalid, vct, arr, n)], ["key", "val"])
    offs, cols, c = [0], [], 0
    for f in aggs:
        if f != "size":
            cols.append(1); c += 1
        offs.append(c)
    hint = 0 if args.no_hint else ng
    stats = {}

    def one_step(collect=False, profile=False):
        st = G.init_groupby_state(-1, (0,), aggs, tuple(offs), tuple(cols), expected_groups=hint, output_batch_size=1 << 40, device=0, stream=sp)
        st._ensure(table)
        if profile:
            G.get_metric(st, 100)
        G.groupby_build_consume_batch(st, table, True, True)
        out, last = G.groupby_produce_output_batch(st, True)
        assert last
        if collect:
            stats["out"] = out
            stats["launches"] = G.get_metric(st, 4)
            stats["consume_us"] = G.get_metric(st, 6)
            stats["consume_launches"] = G.get_metric(st, 7)
            stats["spgg_launches"] = G.get_metric(st, 12)
            stats["spg_launches"] = G.get_metric(st, 8)
            stats["check"] = check(out)
        G.delete_groupby_state(st)

    def valid_bits(col, n_out):
        if col.validity is None:
            return torch.ones(n_out, dtype=torch.bool, device=dev)
        vb = torch.as_tensor(col.validity, device=dev)
        idx = torch.arange(n_out, device=dev)
        return ((vb[idx >> 3] >> (idx & 7).to(torch.uint8)) & 1).bool()

    def check(out):
        """every produced group against a dense torch recomputation; returns (ok, n_bad, n_expected)"""
        n_out = out.n_rows
        k64 = keys.to(torch.int64)
        rows_ok = kmask if kmask is not None else torch.ones(n, dtype=torch.bool, device=dev)
        val_ok = rows_ok & vmask if vmask is not None else rows_ok
        size = torch.zeros(ng, dtype=torch.int64, device=dev)
        cnt = torch.zeros(ng, dtype=torch.int64, device=dev)
        ssum = torch.zeros(ng, dtype=torch.int64, device=dev)
        mn = torch.full((ng,), torch.iinfo(torch.int64).max, dtype=torch.int64, device=dev)
        mx = torch.full((ng,), torch.iinfo(torch.int64).min, dtype=torch.int64, device=dev)
        step_rows = 1 << 26
        for r0 in range(0, n, step_rows):
            kk = k64[r0:r0 + step_rows]
            ro = rows_ok[r0:r0 + step_rows]
            vo = val_ok[r0:r0 + step_rows]
            vv = vals[r0:r0 + step_rows].to(torch.int64)
            size += torch.bincount(kk[ro], minlength=ng)
            cnt += torch.bincount(kk[vo], minlength=ng)
            ssum.index_add_(0, kk[vo], vv[vo])
            mn.scatter_reduce_(0, kk[vo], vv[vo], "amin")
            mx.scatter_reduce_(0, kk[vo], vv[vo], "amax")
        n_expected = int((size > 0).sum().item())
        okeys = torch.as_tensor(out.columns[0].data, device=dev)[:n_out].to(torch.int64)
        in_range = (okeys >= 0) & (okeys < ng)
        safe = torch.where(in_range, okeys, torch.zeros_like(okeys))
        bad = ~in_range
        for j, f in enumerate(aggs):
            col = out.columns[1 + j]
            d = torch.as_tensor(col.data, device=dev)[:n_out]
            ok = valid_bits(col, n_out)
            has = cnt[safe] > 0
            if f == "size":
                bad |= d != size[safe]
            elif f == "count":
                bad |= d != cnt[safe]
            elif f == "sum":
                # sum of an all-NA group: 0 (valid) for nullable outputs, as the reference's sum
                bad |= d.to(torch.int64) != ssum[safe]
            elif f == "mean":
                exp = ssum[safe].to(torch.float64) / cnt[safe].clamp(min=1).to(torch.float64)
                bad |= has & ok & ((d - exp).abs() > 1e-9 * exp.abs().clamp(min=1.0))
                bad |= ok != has
            else:
                ref = (mn if f == "min" else mx)[safe]
                bad |= has & ok & (d.to(torch.int64) != ref)
                if col.validity is not None:
                    bad |= ok != has
        dup = okeys.numel() - torch.unique(okeys).numel()
        n_bad = int(bad.sum().item()) + dup
        return n_bad == 0 and n_out == n_expected, n_bad, n_expected

    sampler = ClockSampler(0)
    for _ in range(max(args.warmup, 0)):
        one_step()
    torch.cuda.synchronize(dev)
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    ev0.record(stream)
    for _ in range(args.steps):
        one_step()
    ev1.record(stream)
    torch.cuda.synchronize(dev)
    ms = ev0.elapsed_time(ev1)
    clocks = sampler.stop()
    one_step(collect=True, profile=True)
    ok, n_bad, n_expected = stats["check"]
    peak, peak_kind = peaks()
    bpr = keys.element_size() + vals.element_size() + (0.25 if args.nullable else 0.0)
    kern_us = stats.get("consume_us", 0)
    n_launch = max(stats.get("consume_launches", 1), 1)
    achieved = (bpr * n / 1e9) / (kern_us * 1e-6) if kern_us else None
    path = "spgg_partition_kernel + spgg_aggregate_kernel (one launch = the pair)" if stats.get("spgg_launches") else (
        "spg/lc fast path" if stats.get("spg_launches") else "groupby_consume_kernel (direct)")
    line = {
        "metric": METRIC, "value": n * args.steps / (ms * 1e-3), "unit": UNIT, "n_gpus": 1, "steps": args.steps, "warmup": args.warmup,
        "ms_per_step": ms / args.steps, "higher_is_better": True, "scaling": "strong", "vs_baseline": None,
        "dtype": f"{args.key_dtype} key / {args.val_dtype} value", "data": "synthetic",
        "config": {"workload": f"{n}-row {ng}-group groupby {','.join(aggs)} ({'nullable' if args.nullable else 'non-null'} "
                               f"{args.key_dtype} key, {args.val_dtype} value{', 1 % NA keys, 10 % NA values' if args.nullable else ''}) on 1xH100 "
                               "— a VARIANT of BASELINE.json configs[1], not the headline signature",
                   "rows": n, "groups": ng, "aggs": list(aggs), "nullable": bool(args.nullable), "expected_groups_hint": hint,
                   "l2": "inputs exceed the 50 MB L2; no flush needed", "step": "init state + consume + finalize + produce",
                   "result_groups": stats["out"].n_rows,
                   "result_check": ("per-group ok: every group's aggregates equal an independent device recomputation" if ok
                                    else f"MISMATCH ({n_bad} bad groups, {n_expected} expected)")},
        "roofline": {"bound": "hbm", "achieved": achieved, "peak": peak, "unit": "GB/s", "frac": (achieved / peak) if achieved else None,
                     "traffic": None, "peak_kind": peak_kind, "kernel": path, "launches_per_step": n_launch,
                     "avg_launch_ms": kern_us / 1e3 / n_launch, "algorithmic_bytes_per_launch": bpr * n / n_launch},
        "cpu_baseline": None, "e2e": None, "clocks": clocks, "gpu_launches": int(stats.get("launches", 0)) * args.steps,
    }
    print(json.dumps(line), flush=True)
    if not ok:
        sys.exit(3)
