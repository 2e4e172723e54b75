"""Float64-key hash join against the same join on int64 keys, 1 x H100.

    python benchmarks/float_join_bench.py [--build-rows 100000000] [--probe-rows 1000000000] [--probe-batch 250000000] [--reps 3]

Shape: BASELINE.json configs[2], the join of bench.py --workload join (`--probe-rows` probe rows against `--build-rows` unique
build keys, 2 payload columns per side, kept columns k, b1, b2 of the build side and p1, p2 of the probe side), once with the
int64 keys k of bench.py's generator and once with float64 keys k * 0.5 + 0.25 (exact for these k).  All inputs are resident in
HBM.  One step = init state -> build (one batch) -> probe in `--probe-batch`-row batches, every batch materialising its rows.
  ms_per_step   int64-key and float64-key steps alternated in one process, median of `--reps` (CUDA events, one warm-up each)
  probe_ms      per probe call (one probe kernel launch + the output-cursor read), CUDA events on the operator's stream, median
                over the calls of one step
  path          join metrics 5 (unique-key probe launches), 6 (inline-payload probe launches), 7 (inline builds)
  check         row count, and the sum mod 2^64 of every output column against torch gathers over k (inverse permutation)
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


def u64sum(t):
    import torch

    return int(t.contiguous().view(torch.int64).sum().item()) & ((1 << 64) - 1)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--build-rows", type=int, default=100_000_000)
    ap.add_argument("--probe-rows", type=int, default=1_000_000_000)
    ap.add_argument("--probe-batch", type=int, default=250_000_000)
    ap.add_argument("--reps", type=int, default=3)
    args = ap.parse_args()

    import torch

    from bodo_b200 import _lib, synth
    from bodo_b200.streaming import join as J
    from bodo_b200.table import Column, Table

    _lib.require_gpu()
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    stream = torch.cuda.current_stream(dev)
    sp = stream.cuda_stream
    nb, npr, batch = args.build_rows, args.probe_rows, args.probe_batch
    print(json.dumps({"card": card(), "torch_device": torch.cuda.get_device_name(dev)}), flush=True)

    # bench.py --workload join's inputs: unique build keys (a permutation of [0, nb)), probe keys uniform in [0, nb)
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
    to_f = lambda k: k.to(torch.float64).mul_(0.5).add_(0.25)
    bkf = to_f(bk)
    pkf = torch.empty(npr, dtype=torch.float64, device=dev)
    for r0 in range(0, npr, batch):
        pkf[r0:r0 + batch] = to_f(pk[r0:r0 + batch])
    torch.cuda.synchronize(dev)
    keys = {"int64": (bk, pk), "float64": (bkf, pkf)}
    kept = ([0, 1, 2], [1, 2])

    def step(kind, collect=False):
        kb, kp = keys[kind]
        st = J.init_join_state(-1, (0,), (0,), ("k", "b1", "b2"), ("k", "p1", "p2"), False, False, expected_build_rows=nb, device=0, stream=sp)
        J.join_build_consume_batch(st, Table([Column(kb), Column(b1), Column(b2)], ["k", "b1", "b2"]), True)
        rows, sums, evs = 0, [0] * 5, []
        for r0 in range(0, npr, batch):
            r1 = min(npr, r0 + batch)
            t = Table([Column(kp[r0:r1]), Column(p1[r0:r1]), Column(p2[r0:r1])], ["k", "p1", "p2"])
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(stream)
            out, _, _ = J.join_probe_consume_batch(st, t, r1 == npr, True, kept)
            e1.record(stream)
            evs.append((e0, e1))
            rows += out.n_rows
            if collect:
                for j, c in enumerate(out.columns):
                    sums[j] = (sums[j] + u64sum(torch.as_tensor(c.data, device=dev)[: out.n_rows])) & ((1 << 64) - 1)
        torch.cuda.synchronize(dev)
        res = {"rows": rows, "sums": sums, "probe_ms": sorted(a.elapsed_time(b) for a, b in evs), "path": [J.get_metric(st, m) for m in (5, 6, 7)]}
        J.delete_join_state(st)
        return res

    def timed(kind):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(stream)
        r = step(kind)
        e1.record(stream)
        torch.cuda.synchronize(dev)
        return e0.elapsed_time(e1), r

    for kind in keys:  # warm-up
        step(kind)
    times = {k: [] for k in keys}
    probe_ms = {k: [] for k in keys}
    for _ in range(args.reps):
        for kind in keys:
            ms, r = timed(kind)
            times[kind].append(ms)
            probe_ms[kind].append(r["probe_ms"][len(r["probe_ms"]) // 2])
    info = {kind: step(kind, collect=True) for kind in keys}

    # independent recomputation: inverse permutation + torch gathers over the int64 k
    inv = torch.empty(nb, dtype=torch.int64, device=dev)
    inv[bk] = torch.arange(nb, dtype=torch.int64, device=dev)
    exp = {k: [0] * 5 for k in keys}
    for r0 in range(0, npr, batch):
        kk = pk[r0:r0 + batch]
        bi = inv[kk]
        tail = [b1[bi], b2[bi], p1[r0:r0 + batch], p2[r0:r0 + batch]]
        for kind, kcol in (("int64", kk), ("float64", pkf[r0:r0 + batch])):
            for j, c in enumerate([kcol] + tail):
                exp[kind][j] = (exp[kind][j] + u64sum(c)) & ((1 << 64) - 1)
        del bi, tail
    check = {k: info[k]["rows"] == npr and info[k]["sums"] == exp[k] for k in keys}

    med = {k: sorted(v)[len(v) // 2] for k, v in times.items()}
    pmed = {k: sorted(v)[len(v) // 2] for k, v in probe_ms.items()}
    print(json.dumps({
        "build_rows": nb, "probe_rows": npr, "probe_batch": batch, "card": card(),
        "ms_per_step": {k: round(v, 3) for k, v in med.items()}, "runs_ms": {k: [round(x, 3) for x in v] for k, v in times.items()},
        "float_over_int": round(med["float64"] / med["int64"], 4),
        "probe_ms": {k: round(v, 3) for k, v in pmed.items()}, "probe_runs_ms": {k: [round(x, 3) for x in v] for k, v in probe_ms.items()},
        "path_metrics_5_6_7": {k: info[k]["path"] for k in keys},
        "check": {k: ("ok: row count and sum mod 2^64 of all 5 output columns" if check[k] else f"MISMATCH {info[k]['rows']} {info[k]['sums']} {exp[k]}")
                  for k in keys},
    }), flush=True)
    if not all(check.values()):
        sys.exit(3)


if __name__ == "__main__":
    main()
