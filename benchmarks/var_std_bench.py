"""var / std / mean of a float64 column on the direct groupby path, 1 x H100.

    python benchmarks/var_std_bench.py [--rows 268435456] [--groups 1000000] [--reps 5]

Shape: `--rows` rows of a non-null int64 key with `--groups` groups (bench.py's seeded generator) and a non-null float64 value
1.7e9 + y, y = (v mod 4096) / 1024 for the generator's int64 value v (epoch seconds with a spread of about 1), both resident in HBM,
aggregated as ("var", "std", "mean") of the value column.  var / std accumulate moments about a per-group shift (K_SHIFT in
groupby.cu): one more accumulator column, read (and CASed once per group) by every row.  One step = init state -> consume one
device batch -> finalize -> produce, as bench.py's step.
  ms_per_step   CUDA events around a step, median / min / max of `--reps` after one warm-up
  check         every group against a torch recomputation from y (exact shift-free data: var is shift invariant):
                var and std to rtol 1e-9, mean to rtol 1e-12
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
    ap.add_argument("--rows", type=int, default=1 << 28)
    ap.add_argument("--groups", type=int, default=1_000_000)
    ap.add_argument("--reps", type=int, default=5)
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
    n, ng = args.rows, args.groups
    key = torch.empty(n, dtype=torch.int64, device=dev)
    x = torch.empty(n, dtype=torch.int64, device=dev)
    synth.device_fill(key, x, 0, ng, args.seed, sp)
    x = x.remainder_(4096).to(torch.float64).div_(1024.0)  # y (exact)
    cnt = torch.bincount(key, minlength=ng).to(torch.float64)
    sy = torch.zeros(ng, dtype=torch.float64, device=dev).index_add_(0, key, x)
    syy = torch.zeros(ng, dtype=torch.float64, device=dev).index_add_(0, key, x * x)
    x.add_(1.7e9)  # the value column: exact, y is below 4 and 1.7e9 has 2^-22 resolution
    torch.cuda.synchronize(dev)
    table = Table([Column(key, None, CTypes.INT64), Column(x, None, CTypes.FLOAT64)], ["key", "val"])

    def step(collect=False):
        st = G.init_groupby_state(-1, (0,), ("var", "std", "mean"), (0, 1, 2, 3), (1, 1, 1), expected_groups=ng,
                                  output_batch_size=1 << 40, device=0, stream=sp)
        G.groupby_build_consume_batch(st, table, True, True)
        out, last = G.groupby_produce_output_batch(st, True)
        assert last
        res = None
        if collect:
            res = {"check": check(out), "direct": all(G.get_metric(st, m) == 0 for m in (8, 10, 12, 14))}
        G.delete_groupby_state(st)
        return res

    def check(out):
        m = out.n_rows
        k = torch.as_tensor(out.columns[0].data, device=dev)[:m]
        var, std, mean = (torch.as_tensor(out.columns[j].data, device=dev)[:m] for j in (1, 2, 3))
        c = cnt[k]
        ev = (syy[k] - sy[k] * sy[k] / c) / (c - 1)  # y lies in [0, 4): no cancellation to speak of
        em = sy[k] / c + 1.7e9
        multi = c > 1
        bad = int((~torch.isclose(var[multi], ev[multi], rtol=1e-9, atol=0)).sum().item())
        bad += int((~torch.isclose(std[multi], ev[multi].sqrt(), rtol=1e-9, atol=0)).sum().item())
        bad += int((~torch.isclose(mean, em, rtol=1e-12, atol=0)).sum().item())
        return bad == 0 and m == int((cnt > 0).sum().item()), bad

    step()  # warm-up
    times = []
    for _ in range(args.reps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(stream)
        step()
        e1.record(stream)
        torch.cuda.synchronize(dev)
        times.append(e0.elapsed_time(e1))
    info = step(collect=True)
    s = sorted(times)
    print(json.dumps({
        "rows": n, "groups": ng, "aggs": ["var", "std", "mean"], "card": card(),
        "ms_per_step": {"median": round(s[len(s) // 2], 3), "min": round(s[0], 3), "max": round(s[-1], 3)},
        "runs_ms": [round(t, 3) for t in times], "grows_per_s": round(n / (s[len(s) // 2] * 1e-3) / 1e9, 3),
        "direct_path": info["direct"],
        "check": "every group equal to the torch recomputation" if info["check"][0] else f"MISMATCH ({info['check'][1]} bad)",
    }), flush=True)
    if not info["check"][0]:
        sys.exit(3)


if __name__ == "__main__":
    main()
