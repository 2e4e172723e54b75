"""prod, boolor_agg + count_if, bitand_agg, kurtosis and skew on the direct groupby path, 1 x H100, against min as a baseline.

    python benchmarks/reduction_agg_bench.py [--rows 268435456] [--batch 16777216] [--groups 1000000,30] [--reps 3]

Shape: `--rows` rows of a non-null int64 key (bench.py's seeded generator) with 10^6, 30 and 1 groups, resident in HBM and fed
as device batches of `--batch` rows.  Value columns, derived from the generator's int64 value v: v itself (int64), vo = v | 1 (odd,
so that a product never reaches 0, where a CAS that cannot change the word is skipped), y = 1 + ((v mod
4096) - 2048) 2^-30 (float64, so products stay finite), b = (v mod 5 == 0) (bool) and x = 1.7e9 + (v mod 4096) / 1024 (float64 at
an epoch-seconds offset).  One step = init state -> consume every batch -> finalize -> produce, as bench.py's step.
  ms_per_step   CUDA events around a step, median / min / max of `--reps` after one warm-up
  check         every group against a torch recomputation where torch has one: int64 prod at 10^6 groups through
                scatter_reduce("prod") (bit-exact; its CAS loop per row is far too slow at few groups), float64 prod as
                exp(sum log y) (rtol 1e-7: n u is 3e-8 at one group), boolor / count_if through
                bincount, kurtosis / skew from two-pass central moments of x - 1.7e9 (rtol 1e-6), min through
                scatter_reduce("amin"); bitand_agg has no torch recomputation
The baseline `min` runs with B200_SPG_GEN=0 (set for the whole process; none of the other signatures takes the SM-partitioned
generic path anyway), so every case is the direct kernel (asserted).  The card's name and power limit are printed with the numbers.
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

CASES = {  # name -> (functions, value column of each)
    "prod_int64": (("prod",), ("vo",)),
    "prod_float64": (("prod",), ("y",)),
    "boolor_count_if": (("boolor_agg", "count_if"), ("b", "b")),
    "bitand_agg": (("bitand_agg",), ("v",)),
    "kurtosis": (("kurtosis",), ("x",)),
    "skew": (("skew",), ("x",)),
    "min_baseline": (("min",), ("v",)),
}


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
    ap.add_argument("--batch", type=int, default=1 << 24)
    ap.add_argument("--groups", default="1000000,30,1")
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--seed", type=int, default=1)
    ap.add_argument("--cases", default=",".join(CASES))
    args = ap.parse_args()
    os.environ["B200_SPG_GEN"] = "0"

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
    names = ["key", "v", "vo", "y", "b", "x"]
    for ng in (int(g) for g in args.groups.split(",")):
        key = torch.empty(n, dtype=torch.int64, device=dev)
        v = torch.empty(n, dtype=torch.int64, device=dev)
        synth.device_fill(key, v, 0, ng, args.seed, sp)
        r = v.remainder(4096)
        y = 1.0 + (r - 2048).to(torch.float64) * 2.0 ** -30
        b = v.remainder(5) == 0
        xs = r.to(torch.float64) / 1024.0  # x - 1.7e9, exact
        x = xs + 1.7e9
        del r
        vo = v.bitwise_or(1)
        cols = {"key": Column(key, None, CTypes.INT64), "v": Column(v, None, CTypes.INT64), "vo": Column(vo, None, CTypes.INT64),
                "y": Column(y, None, CTypes.FLOAT64),
                "b": Column(b.view(torch.uint8), None, CTypes.BOOL), "x": Column(x, None, CTypes.FLOAT64)}
        batches = []
        for r0 in range(0, n, args.batch):
            r1 = min(n, r0 + args.batch)
            batches.append(Table([Column(cols[c].data[r0:r1], None, cols[c].c_type) for c in names], names))
        cnt = torch.bincount(key, minlength=ng)

        def reference(f, c):
            if f == "prod" and c == "vo":  # (torch's scatter_reduce("prod") runs one CAS loop per row: far too slow at few groups)
                return torch.ones(ng, dtype=torch.int64, device=dev).scatter_reduce(0, key, vo, "prod", include_self=False) if ng >= 1000 else None
            if f == "prod":  # (y > 0)
                return torch.zeros(ng, dtype=torch.float64, device=dev).index_add_(0, key, torch.log(y)).exp()
            if f == "boolor_agg":
                return torch.bincount(key[b], minlength=ng) > 0
            if f == "count_if":
                return torch.bincount(key[b], minlength=ng)
            if f == "min":
                return torch.full((ng,), 2 ** 63 - 1, dtype=torch.int64, device=dev).scatter_reduce(0, key, v, "amin", include_self=False)
            if f in ("kurtosis", "skew"):
                c64 = cnt.to(torch.float64)
                mean = torch.zeros(ng, dtype=torch.float64, device=dev).index_add_(0, key, xs) / c64
                d = xs - mean[key]
                m2, m3, m4 = (torch.zeros(ng, dtype=torch.float64, device=dev).index_add_(0, key, d ** p) for p in (2, 3, 4))
                if f == "skew":
                    return c64 * (c64 - 1).sqrt() / (c64 - 2) * m3 / m2 ** 1.5
                return c64 * (c64 + 1) * (c64 - 1) * m4 / ((c64 - 2) * (c64 - 3) * m2 * m2) - 3 * (c64 - 1) ** 2 / ((c64 - 2) * (c64 - 3))
            return None

        def step(fns, in_cols, collect=False):
            st = G.init_groupby_state(-1, (0,), fns, tuple(range(len(fns) + 1)), tuple(names.index(c) for c in in_cols),
                                      expected_groups=ng, output_batch_size=1 << 40, device=0, stream=sp)
            for i, t in enumerate(batches):
                G.groupby_build_consume_batch(st, t, i == len(batches) - 1, True)
            out, last = G.groupby_produce_output_batch(st, True)
            assert last
            res = None
            if collect:
                res = {"check": check(out, fns, in_cols), "direct": all(G.get_metric(st, m) == 0 for m in (8, 10, 12, 14))}
            G.delete_groupby_state(st)
            return res

        def check(out, fns, in_cols):
            m = out.n_rows
            k = torch.as_tensor(out.columns[0].data, device=dev)[:m]
            bad, checked = 0, []
            for j, (f, c) in enumerate(zip(fns, in_cols)):
                ref = reference(f, c)
                if ref is None:
                    continue
                checked.append(f)
                got = torch.as_tensor(out.columns[1 + j].data, device=dev)[:m]
                e = ref[k]
                if f in ("kurtosis", "skew"):
                    ok = cnt[k] >= (4 if f == "kurtosis" else 3)
                    bad += int((~torch.isclose(got[ok], e[ok], rtol=1e-6, atol=1e-9)).sum().item())
                elif e.dtype == torch.float64:
                    bad += int((~torch.isclose(got, e, rtol=1e-7, atol=0)).sum().item())
                else:
                    bad += int((got.to(e.dtype) != e).sum().item())
            return bad == 0 and m == int((cnt > 0).sum().item()), bad, checked

        for name in args.cases.split(","):
            fns, in_cols = CASES[name]
            step(fns, in_cols)  # warm-up
            times = []
            for _ in range(args.reps):
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record(stream)
                step(fns, in_cols)
                e1.record(stream)
                torch.cuda.synchronize(dev)
                times.append(e0.elapsed_time(e1))
            info = step(fns, in_cols, collect=True)
            s = sorted(times)
            ok, nbad, checked = info["check"]
            print(json.dumps({
                "case": name, "aggs": list(fns), "rows": n, "batch_rows": args.batch, "groups": ng, "card": card(),
                "ms_per_step": {"median": round(s[len(s) // 2], 3), "min": round(s[0], 3), "max": round(s[-1], 3)},
                "grows_per_s": round(n / (s[len(s) // 2] * 1e-3) / 1e9, 3), "direct_path": info["direct"],
                "check": (f"every group equal to torch ({', '.join(checked)})" if checked else "no torch recomputation") if ok
                else f"MISMATCH ({nbad} bad)",
            }), flush=True)
            if not ok or not info["direct"]:
                sys.exit(3)
        del batches, cols, key, v, vo, y, b, x, xs
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
