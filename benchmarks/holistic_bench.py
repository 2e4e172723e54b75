"""Groupby holistic aggregates (percentile_cont, percentile_disc, mode) against the full sort and a SUM groupby of the same data,
1 x H100.

    python benchmarks/holistic_bench.py [--rows 268435456] [--batch 16777216] [--reps 3] [--check 4096]
                                        [--cases p50,p3,mode,g30,g2e27,zipf]

`--rows` device-resident rows of an int64 key k and a float64 value v (synth.device_fill's uniform doubles in [0, 1)), fed in
`--batch`-row batches.  Cases (key in [0, 10^6) unless said otherwise):
  p50    percentile_cont(0.5) of v
  p3     percentile_cont(0.5), percentile_cont(0.9) and percentile_disc(0.99) of v: three results from one store and one sort
  mode   mode of an int64 value in [0, 100)
  g30    percentile_cont(0.5) with k in [0, 30)
  g2e27  percentile_cont(0.5) with k in [0, 2^27)
  zipf   percentile_cont(0.5) with a Zipf(1.2) key folded into [0, 10^6)
Each case alternates, in this process, three steps: the holistic state, a full sort state over (k, v) (ORDER BY k, v: the same
two columns, the yardstick the holistic state should not exceed, since it sorts (id, value) and gathers no payload) and a SUM
groupby of v by k.  One step = init -> consume every batch -> produce -> delete, timed with CUDA events; the median of `--reps`
rounds after one warm-up round.  The holistic results of `--check` random groups (and the largest) are compared, bit for bit,
with a torch recomputation (a stable sort by (k, value), then the definitions' positions); the process exits non-zero on a
mismatch.  Printed per case: ms per step of the three, rows/s, groups, store values and digit passes (metrics 20 / 21), and the
card's name and power limit read in the same run.
"""

from __future__ import annotations

import argparse
import json
import math
import os
import statistics
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from benchmarks.sort_bench import card  # noqa: E402

CASES = {"p50": (("percentile_cont",), (0.5,), "uniform"), "p3": (("percentile_cont", "percentile_cont", "percentile_disc"), (0.5, 0.9, 0.99), "uniform"),
         "mode": (("mode",), (), "uniform"), "g30": (("percentile_cont",), (0.5,), "g30"), "g2e27": (("percentile_cont",), (0.5,), "g2e27"),
         "zipf": (("percentile_cont",), (0.5,), "zipf")}


def ref_value(f, V, q):
    """The definitions on V (sorted ascending, a float64 or int64 numpy array)."""
    m = len(V)
    if f == "percentile_cont":
        h = q * float(m - 1)
        lo = math.floor(h)
        a = float(V[lo])
        return a if h - lo == 0.0 else a + (float(V[lo + 1]) - a) * (h - lo)
    if f == "percentile_disc":
        return V[min(max(math.ceil(q * float(m)) - 1, 0), m - 1)]
    vals, counts = __import__("numpy").unique(V, return_counts=True)
    return vals[int(counts.argmax())]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=1 << 28)
    ap.add_argument("--batch", type=int, default=1 << 24)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--check", type=int, default=4096)
    ap.add_argument("--cases", type=str, default=",".join(CASES))
    args = ap.parse_args()

    import numpy as np
    import torch

    from bodo_b200 import _lib, synth
    from bodo_b200.streaming import groupby as G
    from bodo_b200.streaming import sort as S
    from bodo_b200.table import Column, Table

    _lib.require_gpu()
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    stream = torch.cuda.current_stream(dev)
    sp = stream.cuda_stream
    n = args.rows
    print(json.dumps({"card": card(), "torch_device": torch.cuda.get_device_name(dev)}), flush=True)
    g = torch.Generator(device=dev).manual_seed(71)
    v = torch.empty(n, dtype=torch.float64, device=dev)
    synth.device_fill(None, v, 0, 1, 72, sp)
    vi = torch.randint(0, 100, (n,), generator=g, device=dev, dtype=torch.int64)
    keys = {}

    def key(kind):
        if kind not in keys:
            if kind == "uniform":
                keys[kind] = torch.randint(0, 10**6, (n,), generator=g, device=dev, dtype=torch.int64)
            elif kind == "g30":
                keys[kind] = torch.randint(0, 30, (n,), generator=g, device=dev, dtype=torch.int64)
            elif kind == "g2e27":
                keys[kind] = torch.randint(0, 1 << 27, (n,), generator=g, device=dev, dtype=torch.int64)
            else:  # Zipf(1.2) by inverse transform of a continuous power law, folded into [0, 10^6)
                u = torch.rand(n, generator=g, device=dev, dtype=torch.float64)
                keys[kind] = (torch.floor(u.pow(-1.0 / 0.2)) - 1).clamp(max=2**62).to(torch.int64) % 10**6
        return keys[kind]

    def source(k, x):
        for r0 in range(0, n, args.batch):
            r1 = min(n, r0 + args.batch)
            yield Table([Column(k[r0:r1]), Column(x[r0:r1])], ["k", "v"]), r1 == n

    def holistic_step(k, x, fnames, qs, keep=False):
        st = G.init_groupby_state(-1, (0,), fnames, tuple(range(len(fnames) + 1)), (1,) * len(fnames), device=0, stream=sp,
                                  output_batch_size=1 << 30, percentiles=qs or None)
        for t, last in source(k, x):
            G.groupby_build_consume_batch(st, t, last, True)
        out, _ = G.groupby_produce_output_batch(st, True)
        res = [torch.as_tensor(c.data, device=dev).clone() for c in out.columns] if keep else None
        m = {"groups": G.get_metric(st, 0), "store_values": G.get_metric(st, 20), "digit_passes": G.get_metric(st, 21)}
        G.delete_groupby_state(st)
        return res, m

    def sort_step(k, x):
        st = S.init_stream_sort_state(-1, None, None, ["k", "v"], True, "last", ["k", "v"], output_batch_size=1 << 30, device=0,
                                      stream=sp, full=True)
        for t, last in source(k, x):
            S.sort_build_consume_batch(st, t, last)
        S.produce_output_batch(st, True)
        S.delete_stream_sort_state(st)

    def sum_step(k, x):
        st = G.init_groupby_state(-1, (0,), ("sum",), (0, 1), (1,), device=0, stream=sp, output_batch_size=1 << 30)
        for t, last in source(k, x):
            G.groupby_build_consume_batch(st, t, last, True)
        G.groupby_produce_output_batch(st, True)
        G.delete_groupby_state(st)

    def timed(fn):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(stream)
        r = fn()
        e1.record(stream)
        torch.cuda.synchronize(dev)
        return e0.elapsed_time(e1), r

    failed = []
    for case in args.cases.split(","):
        fnames, qs, kind = CASES[case]
        k = key(kind)
        x = vi if case == "mode" else v
        res, m = holistic_step(k, x, fnames, qs, keep=True)
        # check against torch: stable sort by (k, x), per group the definitions' positions
        p = torch.sort(x, stable=True).indices
        p = p[torch.sort(k[p], stable=True).indices]
        ks, xs = k[p], x[p]
        uk, cnt = torch.unique_consecutive(ks, return_counts=True)
        start = torch.cumsum(cnt, 0) - cnt
        rng = np.random.default_rng(0)
        pick = np.unique(np.concatenate([[int(cnt.argmax())], rng.integers(0, len(uk), args.check)]))
        out_keys = res[0].cpu().numpy()
        where = {int(a): i for i, a in enumerate(out_keys)}
        ok = len(where) == len(uk)
        uk_h, st_h, cnt_h = uk.cpu().numpy(), start.cpu().numpy(), cnt.cpu().numpy()
        outs = [r.cpu().numpy() for r in res[1:]]
        qit = iter(qs)
        fq = [(f, next(qit) if f != "mode" else None) for f in fnames]
        for j in pick:
            V = xs[int(st_h[j]):int(st_h[j] + cnt_h[j])].cpu().numpy()
            i = where.get(int(uk_h[j]))
            if i is None:
                ok = False
                break
            for (f, q), o in zip(fq, outs):
                w = ref_value(f, V, q)
                if np.float64(o[i]).view(np.int64) != np.float64(w).view(np.int64):
                    ok = False
        del p, ks, xs
        if not ok:
            failed.append(case)
        for _ in range(1):  # warm-up round
            holistic_step(k, x, fnames, qs)
            sort_step(k, x)
            sum_step(k, x)
        th, ts, tg = [], [], []
        for _ in range(args.reps):
            th.append(timed(lambda: holistic_step(k, x, fnames, qs))[0])
            ts.append(timed(lambda: sort_step(k, x))[0])
            tg.append(timed(lambda: sum_step(k, x))[0])
        h, s, sm = statistics.median(th), statistics.median(ts), statistics.median(tg)
        print(json.dumps({"case": case, "rows": n, "holistic_ms": round(h, 2), "full_sort_ms": round(s, 2), "sum_groupby_ms": round(sm, 2),
                          "holistic_over_sort": round(h / s, 3), "holistic_rows_per_s": round(n / h * 1e3), **m, "checked_groups": len(pick),
                          "exact": ok}), flush=True)
    print(json.dumps({"card": card()}), flush=True)
    if failed:
        print(f"MISMATCH in {failed}", flush=True)
        sys.exit(1)


if __name__ == "__main__":
    main()
