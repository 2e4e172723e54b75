#!/usr/bin/env python
"""Secondary benchmark (not the bench.py contract): the Zipf variant of BASELINE.json configs[1] named in SURVEY.md §8(d) —
hash-aggregate SUM+COUNT over int64 (key, value) rows whose keys follow Zipf(s) over n_groups groups (a few hot keys
carry most of the rows), 1 x H100, inputs resident in HBM.

    python benchmarks/bench_skew.py [--rows 536870912] [--groups 1000000] [--s 1.1] [--batch 134217728]

Keys are drawn on the device by inverting the Zipf CDF (torch.searchsorted; torch is only the input generator and the
independent checker here).  The result is checked against torch.bincount / index_add_ on the same rows.
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=1 << 29)
    ap.add_argument("--groups", type=int, default=1_000_000)
    ap.add_argument("--s", type=float, default=1.1)
    ap.add_argument("--batch", type=int, default=1 << 27)
    ap.add_argument("--reps", type=int, default=3)
    args = ap.parse_args()
    import torch

    from bodo_b200.streaming import groupby as G
    from bodo_b200.table import Column, Table

    dev = torch.device("cuda", 0)
    n, g = args.rows, args.groups
    w = torch.arange(1, g + 1, dtype=torch.float64, device=dev).pow_(-args.s)
    cdf = torch.cumsum(w, 0)
    cdf /= cdf[-1].clone()
    # rank r -> key: scramble the ranks so hot keys are not the small integers (odd multiplier modulo a power of two >= g)
    gen = torch.Generator(device=dev)
    gen.manual_seed(7)
    perm = torch.randperm(g, device=dev, generator=gen)
    keys = torch.empty(n, dtype=torch.int64, device=dev)
    vals = torch.empty(n, dtype=torch.int64, device=dev)
    for r0 in range(0, n, 1 << 26):
        r1 = min(n, r0 + (1 << 26))
        u = torch.rand(r1 - r0, dtype=torch.float64, device=dev, generator=gen)
        rank = torch.searchsorted(cdf, u).clamp_(max=g - 1)
        keys[r0:r1] = perm[rank]
        vals[r0:r1] = torch.randint(-500, 500, (r1 - r0,), dtype=torch.int64, device=dev, generator=gen)
        del u, rank
    top_share = float((keys[: 1 << 24] == perm[0]).double().mean().item())
    torch.cuda.synchronize()

    times, ok = [], True
    for rep in range(args.reps):
        st = G.init_groupby_state(-1, (0,), ("sum", "count"), (0, 1, 2), (1, 1), expected_groups=g, device=0)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for r0 in range(0, n, args.batch):
            r1 = min(n, r0 + args.batch)
            t = Table([Column(keys[r0:r1]), Column(vals[r0:r1])], ["k", "v"])
            G.groupby_build_consume_batch(st, t, r1 == n, True)
        e1.record()
        torch.cuda.synchronize()
        times.append(e0.elapsed_time(e1))
        if rep == 0:
            outs = []
            while True:
                out, last = G.groupby_produce_output_batch(st, True)
                outs.append(out)
                if last:
                    break
            ok_k = torch.cat([torch.as_tensor(o.columns[0].data, device=dev) for o in outs if o.n_rows])
            ok_s = torch.cat([torch.as_tensor(o.columns[1].data, device=dev) for o in outs if o.n_rows])
            ok_c = torch.cat([torch.as_tensor(o.columns[2].data, device=dev) for o in outs if o.n_rows])
            cnt = torch.bincount(keys, minlength=g)
            sm = torch.zeros(g, dtype=torch.int64, device=dev).index_add_(0, keys, vals)
            ok = bool(ok_k.numel() == int((cnt > 0).sum().item()) and torch.equal(cnt[ok_k], ok_c) and torch.equal(sm[ok_k], ok_s))
            metrics = {name: G.get_metric(st, i) for name, i in (("spg_launches", 8), ("retry_rows", 9), ("lc_launches", 10), ("fail_rows", 5))}
        G.delete_groupby_state(st)
    ms = min(times)
    print(json.dumps({"metric": "groupby_agg_rows_per_sec_zipf", "value": n / ms * 1e3, "unit": "rows/s", "ms": ms, "all_ms": times,
                      "config": {"workload": f"{n} rows, {g} groups, Zipf(s={args.s}) keys, SUM+COUNT int64", "top_key_share": top_share},
                      "result_check": "ok" if ok else "MISMATCH", "metrics": metrics, "roofline_frac": n * 16 / ms / 1e6 / 3350.0}))


if __name__ == "__main__":
    main()
