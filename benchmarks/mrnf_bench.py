"""Groupby min_row_number_filter (QUALIFY ROW_NUMBER() OVER (PARTITION BY k ORDER BY o DESC) = 1), 1 x H100.

    python benchmarks/mrnf_bench.py [--rows 268435456] [--batch 16777216] [--reps 3] [--cases main,window,contention,growth,big]

Data of benchmarks/window_bench.py, resident in HBM: `--rows` rows of an int64 key k in [0, 10^6), a float64 order key o
(synth.device_fill's uniform doubles in [0, 1)) and an int64 row id r, fed in `--batch`-row batches.  Cases:
  main        MRNF ORDER BY o DESC keeping (k, o, r); alternates in the same process with a plain groupby step (SUM(r) by k, the
              same batches: groupby_ms) so its cost above an aggregation is a measured difference
  window      the same query as window row_number OVER (PARTITION BY k ORDER BY o DESC) plus the filter rn == 1 (torch), which
              stores and sorts every row
  contention  k in [0, 30): every row of a batch lands on one of 30 slots
  growth      k = (r * odd) mod 2^27: exactly 2^27 groups of two rows, the table grows from its default 2^21 slots
  big         2^31 + 2^24 rows (more than the window's 2^31), generated batch by batch with b200_synth_fill (k in [0, 10^6),
              o uniform) into two reused buffers; the generation is inside the timed step and is reported (gen_ms) from a
              separate timing of the generator alone
One step = init -> consume every batch (is_last on the last) -> produce -> delete, timed with CUDA events on the operator's
stream; the median of `--reps` steps after one warm-up (big: one step, no warm-up).  Every case is checked against an independent
torch computation (stable sort by o descending, then a stable sort by k, the first row per k; big: the same per batch, merged
with the winners so far); the process exits non-zero on a mismatch.  Printed per case: ms_per_step, rows_per_s, groups, table
rebuilds, the card's name and power limit.
"""

from __future__ import annotations

import argparse
import json
import os
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
    ap.add_argument("--cases", type=str, default="main,window,contention,growth,big")
    ap.add_argument("--big-rows", type=int, default=(1 << 31) + (1 << 24))
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

    def batches(k, o, r, total, batch):
        for r0 in range(0, total, batch):
            r1 = min(total, r0 + batch)
            yield Table([Column(k[r0:r1]), Column(o[r0:r1]), Column(r[r0:r1])], names), r1 == total

    def mrnf_state(**kw):
        return G.init_groupby_state(-1, (0,), MRNF, (0, 0), (), mrnf_sort_col_inds=(1,), mrnf_sort_col_asc=(False,), mrnf_sort_col_na=(True,),
                                    mrnf_col_inds_keep=(0, 1, 2), output_batch_size=1 << 30, device=0, stream=sp, **kw)

    def mrnf_step(source, keep=False):
        st = mrnf_state()
        for t, last in source():
            G.groupby_build_consume_batch(st, t, last, True)
        out, _ = G.groupby_produce_output_batch(st, True)
        res = [torch.as_tensor(c.data, device=dev).clone() for c in out.columns] if keep else None
        m = (G.get_metric(st, 0), G.get_metric(st, 3))
        G.delete_groupby_state(st)
        return res, m

    def groupby_step(source):
        st = G.init_groupby_state(-1, (0,), ("sum",), (0, 1), (2,), output_batch_size=1 << 30, device=0, stream=sp)
        for t, last in source():
            G.groupby_build_consume_batch(st, t, last, True)
        G.groupby_produce_output_batch(st, True)
        G.delete_groupby_state(st)

    def window_step(source, keep=False):
        st = W.init_window_state(-1, ["k"], ["o"], False, "last", [("rn", "row_number")], names, output_batch_size=1 << 30, device=0, stream=sp)
        for t, last in source():
            W.window_build_consume_batch(st, t, last)
        out, _ = W.window_produce_output_batch(st)
        sel = torch.as_tensor(out.columns[3].data, device=dev) == 1
        res = [torch.as_tensor(c.data, device=dev)[sel].clone() for c in out.columns[:3]]
        W.delete_window_state(st)
        return (res if keep else None), (int(sel.sum()), 0)

    def timed(fn):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(stream)
        r = fn()
        e1.record(stream)
        torch.cuda.synchronize(dev)
        return e0.elapsed_time(e1), r

    def first_per_key(k, o, r):
        """torch: stable sort by o descending, then stably by k; the first row of each k, as (k, o, r) sorted by k."""
        p = torch.sort(o, descending=True, stable=True).indices
        p = p[torch.sort(k[p], stable=True).indices]
        first = torch.ones(p.numel(), dtype=torch.bool, device=dev)
        first[1:] = k[p][1:] != k[p][:-1]
        w = p[first]
        return k[w], o[w], r[w]

    def same(res, exp):
        order = torch.sort(res[0]).indices
        return all(bool(torch.equal(a[order], b)) for a, b in zip(res, exp))

    def report(case, ms, m, check_ok, rows, **extra):
        if not check_ok:
            failed.append(case)
        print(json.dumps({"case": case, "rows": rows, "batch": args.batch, "ms_per_step": round(statistics.median(ms), 2),
                          "all_ms": [round(x, 2) for x in ms], "rows_per_s": round(rows / (statistics.median(ms) / 1e3)), "groups": m[0],
                          "rebuilds": m[1], "result_check": "pass" if check_ok else "FAIL", "card": card(), **extra}), flush=True)

    cases = args.cases.split(",")
    resident = lambda k: (lambda: batches(k, ok, rid, n, args.batch))  # noqa: E731
    for case in cases:
        if case in ("main", "contention", "growth"):
            k = pk if case == "main" else (pk % 30 if case == "contention" else (rid * 0x9E3779B1) & ((1 << 27) - 1))
            src = resident(k)
            res, m = mrnf_step(src, keep=True)
            check_ok = same(res, first_per_key(k, ok, rid))
            del res
            ms, gb = [], []
            for _ in range(args.reps):
                if case == "main":
                    gb.append(timed(lambda: groupby_step(src))[0])
                t, (_, m) = timed(lambda: mrnf_step(src))
                ms.append(t)
            extra = {"groupby_ms": round(statistics.median(gb), 2)} if gb else {}
            report(case, ms, m, check_ok, n, **extra)
            del k
        elif case == "window":
            src = resident(pk)
            res, m = window_step(src, keep=True)
            check_ok = same(res, first_per_key(pk, ok, rid))
            del res
            ms = [timed(lambda: window_step(src))[0] for _ in range(args.reps)]
            report(case, ms, m, check_ok, n)
        elif case == "big":
            total, b = args.big_rows, args.batch
            bufs = [(torch.empty(b, dtype=torch.int64, device=dev), torch.empty(b, dtype=torch.float64, device=dev),
                     torch.empty(b, dtype=torch.int64, device=dev)) for _ in range(2)]

            def gen(i, r0, rows):
                kb, ob, rb = (x[:rows] for x in bufs[i % 2])
                synth.device_fill(kb, None, r0, 10**6, 71, sp)
                synth.device_fill(None, ob, r0, 1, 72, sp)
                torch.arange(r0, r0 + rows, out=rb)
                return kb, ob, rb

            def source():
                for i, r0 in enumerate(range(0, total, b)):
                    rows = min(b, total - r0)
                    kb, ob, rb = gen(i, r0, rows)
                    yield Table([Column(kb), Column(ob), Column(rb)], names), r0 + rows == total

            t, (res, m) = timed(lambda: mrnf_step(source, keep=True))
            gen_ms = timed(lambda: [gen(i, r0, min(b, total - r0)) for i, r0 in enumerate(range(0, total, b))])[0]
            win = None
            for i, r0 in enumerate(range(0, total, b)):
                kb, ob, rb = gen(i, r0, min(b, total - r0))
                bk, bo, br = first_per_key(kb, ob, rb)
                if win is not None:  # the winners so far come first: on a tie the earlier row stays
                    bk, bo, br = first_per_key(torch.cat([win[0], bk]), torch.cat([win[1], bo]), torch.cat([win[2], br]))
                win = (bk, bo, br)
            report(case, [t], m, same(res, win), total, gen_ms=round(gen_ms, 2))
            del res, bufs
        else:
            raise SystemExit(f"unknown case {case}")
        torch.cuda.empty_cache()
    if failed:
        print(json.dumps({"failed": failed}), flush=True)
        sys.exit(1)


if __name__ == "__main__":
    main()
