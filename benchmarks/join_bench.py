"""bench.py --workload join: BASELINE.json configs[2] — hash inner join 1 B x 100 M int64 key, 4 payload columns (2 per side)
on 1 x H100, through the streaming join operator API (bodo_b200.streaming.join).

One step = one whole operator lifetime: init state -> build (one 100 M-row batch) -> probe in `--probe-batch`-row batches,
every batch materialising its joined rows (kept columns: k, b1, b2 of the build side, p1, p2 of the probe side).

  value     probe rows/s with both inputs resident in HBM (CUDA events around the step)
  e2e       the same through the same API with HOST (pinned) inputs and every output batch copied back to pinned host memory
  roofline  dominant kernel join_probe_inline_kernel (Slot32 table: key + payload in one sector; join_probe_fast_kernel when the
            schema does not qualify): (24 B probe row + 40 B output row) x rows of a launch / its launch time
            (CUDA events on the operator's stream), against MEASURED_PEAKS.json hbm_gbs; the random slot + payload sectors a
            probe touches (>= 64 B/row) are NOT in the algorithmic figure (SURVEY.md §8d)
  parity    untimed, at full size: row count; sum mod 2^64 of EVERY output column against an independent torch computation
            (inverse permutation + gathers); sorted row-set equality on a sampled key range
  cpu_baseline  the oracle's hash join (reference algorithm shape, bodo/libs/streaming/_join.cpp:381-512, 729-827) on a
            bounded sample, one thread (the oracle join is a scalar port)
"""

from __future__ import annotations

import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
METRIC = "hash-join probe rows/sec"
UNIT = "rows/s"


def workload_name(args):
    return (f"hash inner join {args.probe_rows} x {args.build_rows} int64 key, 2 payload cols per side on 1xH100 "
            "(BASELINE.json configs[2])")


def _u64sum(t):
    """sum mod 2^64 of an int64 / float64 tensor (floats by bit pattern)."""
    import torch

    return int(t.view(torch.int64).sum().item()) & ((1 << 64) - 1)


def reference_arm(args):
    rank = int(os.environ.get("RANK", "0"))
    if rank != 0:
        return
    import numpy as np

    from oracle import oracle as O

    nb = min(args.build_rows, 20_000_000)
    npr = min(args.probe_rows, 100_000_000)
    rng = np.random.default_rng(3)
    bk = rng.permutation(nb).astype(np.int64)
    pk = rng.integers(0, nb, npr).astype(np.int64)
    for _ in range(max(args.warmup, 0)):
        O.hash_join(bk, None, pk[: npr // 10], None)
    t0 = time.perf_counter()
    for _ in range(args.steps):
        bi, pi = O.hash_join(bk, None, pk, None)
    dt = time.perf_counter() - t0
    value = npr * args.steps / dt
    sample = f"{npr} probe rows x {nb} build rows per step (index pairs only, no payload gather), 1 thread"
    print(json.dumps({
        "impl": "reference", "metric": METRIC, "value": value, "unit": UNIT, "n_gpus": args.gpus, "steps": args.steps, "warmup": args.warmup,
        "ms_per_step": dt / args.steps * 1e3, "higher_is_better": True, "scaling": "strong", "vs_baseline": None, "dtype": "int64",
        "data": "synthetic", "config": {"workload": workload_name(args), "sample": sample},
        "cpu_baseline": {"value": value, "unit": UNIT, "cores": 1, "kind": "port", "sample": sample},
        "e2e": {"value": value, "unit": UNIT, "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0}, "gpu_launches": 0}), flush=True)


def run(args, ClockSampler, peaks):
    if args.impl == "reference":
        reference_arm(args)
        return
    import torch

    from bodo_b200 import _lib, synth
    from bodo_b200.streaming import join as J
    from bodo_b200.table import Column, Table

    if int(os.environ.get("WORLD_SIZE", "1")) > 1:
        raise SystemExit("bench.py --workload join measures configs[2], a 1-GPU configuration (the sharded join is covered by tests/test_gpu_multi.py)")
    _lib.require_gpu()
    torch.cuda.set_device(0)
    dev = torch.device("cuda", 0)
    stream = torch.cuda.current_stream(dev)
    sp = stream.cuda_stream
    nb, npr, batch = args.build_rows, args.probe_rows, args.probe_batch

    # build: unique keys = a random permutation of [0, nb); probe keys uniform in [0, nb): exactly one match per probe row
    bk = torch.randperm(nb, device=dev, dtype=torch.int64, generator=torch.Generator(device=dev).manual_seed(3))
    b1 = torch.empty(nb, dtype=torch.int64, device=dev)
    b2 = torch.empty(nb, dtype=torch.float64, device=dev)
    synth.device_fill(None, b1, 0, 1, 31, sp)
    synth.device_fill(None, b2, 0, 1, 32, sp)
    pk = torch.empty(npr, dtype=torch.int64, device=dev)
    p1 = torch.empty(npr, dtype=torch.int64, device=dev)
    p2 = torch.empty(npr, dtype=torch.float64, device=dev)
    synth.device_fill(pk, p1, 0, nb, 41, sp)
    synth.device_fill(None, p2, 0, 1, 42, sp)
    torch.cuda.synchronize(dev)
    build = Table([Column(bk), Column(b1), Column(b2)], ["k", "b1", "b2"])
    kept = ([0, 1, 2], [1, 2])
    stats = {}

    def one_step(bt, pcols, host_out=None, verify=False, profile=False):
        st = J.init_join_state(-1, (0,), (0,), ("k", "b1", "b2"), ("k", "p1", "p2"), False, False, expected_build_rows=nb, device=0, stream=sp)
        J.join_build_consume_batch(st, bt, True)
        out_rows = 0
        sums = [0] * 5
        sample_rows = []
        evs = []
        for r0 in range(0, npr, batch):
            r1 = min(npr, r0 + batch)
            t = Table([Column(c[r0:r1]) for c in pcols], ["k", "p1", "p2"])
            if profile:
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record(stream)
            out, _, _ = J.join_probe_consume_batch(st, t, r1 == npr, True, kept)
            if profile:
                e1.record(stream)
                evs.append((e0, e1, r1 - r0))
            out_rows += out.n_rows
            if host_out is not None:  # e2e: every output batch goes back to pinned host memory
                for j, c in enumerate(out.columns):
                    src = torch.as_tensor(c.data, device=dev)
                    host_out[j][: out.n_rows].copy_(src[: out.n_rows], non_blocking=True)
                stream.synchronize()
            if verify:
                cols = [torch.as_tensor(c.data, device=dev)[: out.n_rows] for c in out.columns]
                for j in range(5):
                    sums[j] = (sums[j] + _u64sum(cols[j])) & ((1 << 64) - 1)
                m = (cols[0] >= args.sample_lo) & (cols[0] < args.sample_hi)
                sample_rows.append(torch.stack([c.view(torch.int64)[m] for c in cols], 1).cpu())
        stats["launches"] = J.get_metric(st, 4)
        stats["fast_probes"] = J.get_metric(st, 5)
        stats["inline_probes"] = J.get_metric(st, 6)
        J.delete_join_state(st)
        if profile:
            torch.cuda.synchronize(dev)
            stats["probe_ms"] = [e0.elapsed_time(e1) for e0, e1, _ in evs]
            stats["probe_rows"] = [n for _, _, n in evs]
        return out_rows, sums, sample_rows

    pdev = (pk, p1, p2)
    sampler = ClockSampler(0)  # started before the warm-up: same workload, every sample is under load
    for _ in range(max(args.warmup, 0)):
        one_step(build, pdev)
    torch.cuda.synchronize(dev)
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    ev0.record(stream)
    for _ in range(args.steps):
        one_step(build, pdev)
    ev1.record(stream)
    torch.cuda.synchronize(dev)
    ms = ev0.elapsed_time(ev1)
    clocks = sampler.stop()

    # ---- untimed: profiled step + parity at full size ----
    out_rows, sums, sample_rows = one_step(build, pdev, verify=True, profile=True)
    inv = torch.empty(nb, dtype=torch.int64, device=dev)
    inv[bk] = torch.arange(nb, dtype=torch.int64, device=dev)
    exp_sums = [0] * 5
    exp_sample = []
    for r0 in range(0, npr, batch):  # independent recomputation: inverse permutation + torch gathers
        r1 = min(npr, r0 + batch)
        kk = pk[r0:r1]
        bi = inv[kk]
        cols = [kk, b1[bi], b2[bi], p1[r0:r1], p2[r0:r1]]
        for j in range(5):
            exp_sums[j] = (exp_sums[j] + _u64sum(cols[j])) & ((1 << 64) - 1)
        m = (kk >= args.sample_lo) & (kk < args.sample_hi)
        exp_sample.append(torch.stack([c.view(torch.int64)[m] for c in cols], 1).cpu())
    del inv
    got_s = torch.cat(sample_rows) if sample_rows else torch.zeros((0, 5), dtype=torch.int64)
    exp_s = torch.cat(exp_sample)

    def sort_rows(t):
        idx = sorted(range(t.shape[0]), key=lambda i: tuple(t[i].tolist()))
        return t[idx]
    sample_ok = got_s.shape == exp_s.shape and bool((sort_rows(got_s) == sort_rows(exp_s)).all())
    check_ok = out_rows == npr and sums == exp_sums and sample_ok

    value = npr * args.steps / (ms * 1e-3)
    peak, peak_kind = peaks()
    pms, prow = stats["probe_ms"], stats["probe_rows"]
    alg_bytes = [n * 64 for n in prow]
    achieved = sum(alg_bytes) / 1e9 / (sum(pms) * 1e-3)
    stream_gb = (nb * 24 + npr * 24 + out_rows * 40) / 1e9
    roofline = {"bound": "hbm", "achieved": achieved, "peak": peak, "unit": "GB/s", "frac": achieved / peak, "traffic": None, "peak_kind": peak_kind,
                "kernel": ("join_probe_inline_kernel<2,2>" if stats.get("inline_probes") else "join_probe_fast_kernel") + " (one launch per probe batch)", "launches_per_step": len(pms), "avg_launch_ms": sum(pms) / len(pms),
                "algorithmic_bytes_per_launch": alg_bytes[0], "algorithmic_bytes_per_row": "24 B probe row in + 40 B joined row out",
                "compulsory_stream_gb_per_step": stream_gb, "whole_step_frac": stream_gb / (ms / args.steps * 1e-3) / peak}

    e2e = None
    if not args.no_e2e:
        try:
            hb = [torch.empty_like(c, device="cpu").pin_memory() for c in (bk, b1, b2)]
            hp = [torch.empty_like(c, device="cpu").pin_memory() for c in (pk, p1, p2)]
            for h, d in zip(hb + hp, (bk, b1, b2, pk, p1, p2)):
                h.copy_(d)
            hout = [torch.empty(batch, dtype=torch.int64).pin_memory() for _ in range(5)]
            hout[2] = hout[2].view(torch.float64); hout[4] = hout[4].view(torch.float64)
            torch.cuda.synchronize(dev)
            hbuild = Table([Column(h.numpy()) for h in hb], ["k", "b1", "b2"])
            hprobe = tuple(h.numpy() for h in hp)
            t0 = time.perf_counter()
            for _ in range(args.e2e_steps):
                one_step(hbuild, hprobe, host_out=hout)
            torch.cuda.synchronize(dev)
            wall = time.perf_counter() - t0
            e2e = {"value": npr * args.e2e_steps / wall, "unit": UNIT, "h2d_bytes_per_step": 24 * (nb + npr), "d2h_bytes_per_step": 40 * out_rows,
                   "steps": args.e2e_steps, "ms_per_step": wall * 1e3 / args.e2e_steps, "host_memory": "pinned"}
        except Exception as ex:
            e2e = {"value": None, "unit": UNIT, "error": str(ex)[:200]}

    cpu = None
    if not args.no_cpu:
        from oracle import oracle as O

        ns_b, ns_p = min(nb, 20_000_000), min(npr, 50_000_000)
        bkn = torch.randperm(ns_b, dtype=torch.int64).numpy()
        pkn = (pk[:ns_p] % ns_b).cpu().numpy()
        t0 = time.perf_counter()
        bi, pi = O.hash_join(bkn, None, pkn, None)
        dt = time.perf_counter() - t0
        cpu = {"value": ns_p / dt, "unit": UNIT, "cores": 1, "kind": "port", "seconds": dt,
               "sample": f"{ns_p} probe rows x {ns_b} build rows, index pairs only (oracle hash join, scalar port of the reference's build + probe)"}

    print(json.dumps({
        "metric": METRIC, "value": value, "unit": UNIT, "n_gpus": 1, "steps": args.steps, "warmup": args.warmup, "ms_per_step": ms / args.steps,
        "higher_is_better": True, "scaling": "strong", "vs_baseline": None, "dtype": "int64", "data": "synthetic",
        "config": {"workload": workload_name(args), "build_rows": nb, "probe_rows": npr, "probe_batch": batch, "out_rows": out_rows,
                   "l2": "inputs and outputs (66 GB per step) exceed the 50 MB L2; no flush needed",
                   "step": "init state + build (insert, CSR, payload pack) + probe batches with output materialisation",
                   "result_check": ("ok: row count, sum mod 2^64 of all 5 output columns vs inverse-permutation gathers, sorted row-set equality for keys in "
                                    f"[{args.sample_lo}, {args.sample_hi}) ({got_s.shape[0]} rows)") if check_ok else "MISMATCH"},
        "roofline": roofline, "cpu_baseline": cpu, "e2e": e2e, "clocks": clocks, "gpu_launches": int(stats["launches"]) * args.steps}), flush=True)
    if not check_ok:
        sys.exit(3)
