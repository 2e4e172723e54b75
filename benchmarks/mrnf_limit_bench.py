"""Groupby min_row_number_filter with a row limit (QUALIFY ROW_NUMBER() OVER (PARTITION BY k ORDER BY o DESC) <= n), 1 x H100.

    python benchmarks/mrnf_limit_bench.py [--rows 268435456] [--batch 16777216] [--reps 3]
                                          [--cases n1,n3,n10,n100,window3,adversarial3,heavy1000,growth3] [--profile]

Data of benchmarks/mrnf_bench.py, resident in HBM: `--rows` rows of an int64 key k in [0, 10^6), a float64 order key o
(synth.device_fill's uniform doubles in [0, 1)) and an int64 row id r, fed in `--batch`-row batches; every case keeps (k, o, r).
Cases:
  n1, n3, n10, n100  mrnf_limit = 1 (the one-winner-record path), 3, 10, 100 on that data (random arrival)
  window3            the same query for n = 3 as window row_number OVER (PARTITION BY k ORDER BY o DESC) plus the filter rn <= 3
                     (torch), which stores and sorts every row
  adversarial3       n = 3 with o = r: every row ranks above every earlier row of its group, so every row is a candidate
  heavy1000          k in [0, 30), n = 1000
  growth3            n = 3, k = (r * odd) mod 2^25: 2^25 groups of eight rows, the table grows from its default 2^21 slots
One step = init -> consume every batch (is_last on the last) -> produce -> delete, timed with CUDA events on the operator's
stream; the median of `--reps` steps after one warm-up step.  Every case is checked against a torch computation (stable sort by
o descending, then a stable sort by k, the first n rows per k) as a multiset of (k, o, r) rows; the process exits non-zero on a
mismatch.  Printed per case: ms_per_step, rows_per_s, output rows, table rebuilds, candidate rows admitted and store reduces
(metrics 18 / 19), the card's name and power limit.  --profile adds, per case, a separate step under torch.profiler and prints
the device time per kernel name (the timed steps run without the profiler).
"""

from __future__ import annotations

import argparse
import json
import os
import re
import statistics
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from benchmarks.sort_bench import card  # noqa: E402

MRNF = ("min_row_number_filter",)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=1 << 28)
    ap.add_argument("--batch", type=int, default=1 << 24)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--cases", type=str, default="n1,n3,n10,n100,window3,adversarial3,heavy1000,growth3")
    ap.add_argument("--profile", action="store_true")
    args = ap.parse_args()

    import torch

    from bodo_b200 import _lib, synth
    from bodo_b200.streaming import groupby as G
    from bodo_b200.streaming import window as W
    from bodo_b200.table import Column, Table

    _lib.require_gpu()
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    stream = torch.cuda.current_stream(dev)
    sp = stream.cuda_stream
    n = args.rows
    print(json.dumps({"card": card(), "torch_device": torch.cuda.get_device_name(dev)}), flush=True)

    g = torch.Generator(device=dev).manual_seed(61)
    pk = torch.randint(0, 10**6, (n,), generator=g, device=dev, dtype=torch.int64)
    ok = torch.empty(n, dtype=torch.float64, device=dev)
    synth.device_fill(None, ok, 0, 1, 62, sp)
    rid = torch.arange(n, dtype=torch.int64, device=dev)
    torch.cuda.synchronize(dev)
    names = ["k", "o", "r"]
    failed = []

    def source(k, o):
        def gen():
            for r0 in range(0, n, args.batch):
                r1 = min(n, r0 + args.batch)
                yield Table([Column(k[r0:r1]), Column(o[r0:r1]), Column(rid[r0:r1])], names), r1 == n
        return gen

    def mrnf_step(src, limit, keep=False):
        st = G.init_groupby_state(-1, (0,), MRNF, (0, 0), (), mrnf_sort_col_inds=(1,), mrnf_sort_col_asc=(False,), mrnf_sort_col_na=(True,),
                                  mrnf_col_inds_keep=(0, 1, 2), output_batch_size=1 << 30, device=0, stream=sp, mrnf_limit=limit)
        for t, last in src():
            G.groupby_build_consume_batch(st, t, last, True)
        out, _ = G.groupby_produce_output_batch(st, True)
        res = [torch.as_tensor(c.data, device=dev).clone() for c in out.columns] if keep else None
        m = {"out_rows": G.get_metric(st, 0), "rebuilds": G.get_metric(st, 3), "admitted": G.get_metric(st, 18), "reduces": G.get_metric(st, 19)}
        G.delete_groupby_state(st)
        return res, m

    def window_step(src, limit, keep=False):
        st = W.init_window_state(-1, ["k"], ["o"], False, "last", [("rn", "row_number")], names, output_batch_size=1 << 30, device=0, stream=sp)
        for t, last in src():
            W.window_build_consume_batch(st, t, last)
        out, _ = W.window_produce_output_batch(st)
        sel = torch.as_tensor(out.columns[3].data, device=dev) <= limit
        res = [torch.as_tensor(c.data, device=dev)[sel].clone() for c in out.columns[:3]] if keep else None
        m = {"out_rows": int(sel.sum())}
        W.delete_window_state(st)
        return res, m

    def timed(fn):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(stream)
        r = fn()
        e1.record(stream)
        torch.cuda.synchronize(dev)
        return e0.elapsed_time(e1), r

    def first_n_per_key(k, o, limit):
        """torch: stable sort by o descending, then stably by k; the first `limit` rows of each k, as row ids."""
        p = torch.sort(o, descending=True, stable=True).indices
        p = p[torch.sort(k[p], stable=True).indices]
        ks = k[p]
        start = torch.ones(n, dtype=torch.bool, device=dev)
        start[1:] = ks[1:] != ks[:-1]
        pos = torch.arange(n, device=dev)
        first = torch.cummax(torch.where(start, pos, torch.zeros_like(pos)), 0).values
        return p[(pos - first) < limit]

    def same(res, k, o, exp):
        got = torch.sort(res[2]).values
        want = torch.sort(exp).values
        return bool(torch.equal(got, want)) and bool(torch.equal(res[0], k[res[2]])) and bool(torch.equal(res[1], o[res[2]]))

    def profile(fn):
        from torch.profiler import ProfilerActivity
        from torch.profiler import profile as prof

        with prof(activities=[ProfilerActivity.CUDA]) as p:
            fn()
            torch.cuda.synchronize(dev)
        rows = [(e.key, e.device_time_total / 1e3, e.count) for e in p.key_averages() if e.device_time_total > 0]
        rows.sort(key=lambda x: -x[1])
        return {key[:60]: [round(ms, 2), cnt] for key, ms, cnt in rows[:12]}

    for case in args.cases.split(","):
        if case.startswith("window"):
            limit, k, o, step = int(case[6:]), pk, ok, window_step
        else:
            limit = int(re.search(r"\d+$", case).group())
            k = pk % 30 if case.startswith("heavy") else ((rid * 0x9E3779B1) & ((1 << 25) - 1) if case.startswith("growth") else pk)
            o = rid.to(torch.float64) if case.startswith("adversarial") else ok
            step = mrnf_step
        src = source(k, o)
        res, m = step(src, limit, keep=True)
        check_ok = same(res, k, o, first_n_per_key(k, o, limit))
        del res
        torch.cuda.empty_cache()
        ms = []
        for _ in range(args.reps):
            t, (_, m) = timed(lambda: step(src, limit))
            ms.append(t)
        if not check_ok:
            failed.append(case)
        rec = {"case": case, "limit": limit, "rows": n, "batch": args.batch, "ms_per_step": round(statistics.median(ms), 2),
               "all_ms": [round(x, 2) for x in ms], "rows_per_s": round(n / (statistics.median(ms) / 1e3)), **m,
               "result_check": "pass" if check_ok else "FAIL", "card": card()}
        if args.profile:
            rec["kernels_ms_count"] = profile(lambda: step(src, limit))
        print(json.dumps(rec), flush=True)
        torch.cuda.empty_cache()
    if failed:
        print(json.dumps({"failed": failed}), flush=True)
        sys.exit(1)


if __name__ == "__main__":
    main()
