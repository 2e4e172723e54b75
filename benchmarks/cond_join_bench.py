"""Equi-join key plus a range condition: the conditional join against join-then-filter_project, 1 x H100.

    python benchmarks/cond_join_bench.py [--keys 1048576] [--k 1,8] [--probe-rows 0] [--alone-rows 268435456] [--reps 3]

Shape (events into validity windows): the build side has `--keys` accounts x k non-overlapping windows [start, end) of width
W = 1000 (columns acct, start, end, wid = the build row id); probe rows have a uniform account and a timestamp uniform in
[0, k W), so exactly one of a probe row's k candidate windows passes `start <= ts < end`.  Columns are int64 and device
resident.  Arms, alternated in one process (one warm-up step per arm):
  cond_inner    init_join_state(..., non_equi_condition=(ts >= start) & (ts < end)), inner; keeps wid and eid
  filter_inner  the join on acct alone (k output rows per probe row: start, end, wid, ts, eid), then PhysicalFilterProject with
                the same predicate keeping wid and eid (for k = 1 the unconditioned join takes the unique-key Slot32 path)
  cond_left / filter_left   the same with how="left".  Every probe row has exactly one passing window here, so filtering the
                left join's output gives the left join's result; with a probe row without one it would not (the row would vanish).
The probe size of these arms is the largest power of two (at most 2^28) whose unconditioned output, inputs and scratch fit in
60 % of the free HBM (`--probe-rows` overrides it).  Then the conditional inner join alone runs at `--alone-rows` probe rows.
  ms          median over `--reps` of one probe call (+ the filter call for the filter arms), CUDA events on the stream
  build_ms    median of the build call
  check       output rows, and the sums mod 2^64 of wid, eid and wid * eid, equal between the arms of one k
The card's name and power limit are printed with the numbers.
"""

from __future__ import annotations

import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from benchmarks.float_join_bench import card  # noqa: E402

W = 1000
M64 = (1 << 64) - 1


def checksum(wid, eid):
    import torch

    w, e = wid.view(torch.int64), eid.view(torch.int64)
    return [int(w.sum().item()) & M64, int(e.sum().item()) & M64, int((w * e).sum().item()) & M64]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--keys", type=int, default=1 << 20)
    ap.add_argument("--k", default="1,8")
    ap.add_argument("--probe-rows", type=int, default=0)
    ap.add_argument("--alone-rows", type=int, default=1 << 28)
    ap.add_argument("--reps", type=int, default=3)
    args = ap.parse_args()

    import torch

    from bodo_b200 import _lib
    from bodo_b200.expr import build_col, col, probe_col
    from bodo_b200.physical import OperatorResult, PhysicalFilterProject
    from bodo_b200.streaming import join as J
    from bodo_b200.table import Column, Table

    _lib.require_gpu()
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    stream = torch.cuda.current_stream(dev)
    sp = stream.cuda_stream
    print(json.dumps({"card": card(), "torch_device": torch.cuda.get_device_name(dev)}), flush=True)
    gen = torch.Generator(device=dev).manual_seed(5)
    cond = (probe_col("ts") >= build_col("start")) & (probe_col("ts") < build_col("end"))
    pred = (col("ts") >= col("start")) & (col("ts") < col("end"))

    def build_side(k):
        nb = args.keys * k
        acct = torch.arange(args.keys, device=dev, dtype=torch.int64).repeat_interleave(k)
        start = (torch.arange(nb, device=dev, dtype=torch.int64) % k) * W
        perm = torch.randperm(nb, device=dev, generator=gen)  # build rows in no particular order
        acct, start = acct[perm], start[perm]
        return Table([Column(acct), Column(start), Column(start + W), Column(torch.arange(nb, device=dev, dtype=torch.int64))],
                     ["acct", "start", "end", "wid"])

    def probe_side(k, n):
        acct = torch.randint(0, args.keys, (n,), device=dev, dtype=torch.int64, generator=gen)
        ts = torch.randint(0, k * W, (n,), device=dev, dtype=torch.int64, generator=gen)
        return Table([Column(acct), Column(ts), Column(torch.arange(n, device=dev, dtype=torch.int64))], ["acct", "ts", "eid"])

    def step(arm, bt, pt):
        conditional, left = arm.startswith("cond"), arm.endswith("left")
        st = J.init_join_state(-1, (0,), (0,), tuple(bt.names), tuple(pt.names), False, left, device=0, stream=sp,
                               expected_build_rows=bt.n_rows, non_equi_condition=cond if conditional else None)
        e = [torch.cuda.Event(enable_timing=True) for _ in range(4)]
        e[0].record(stream)
        J.join_build_consume_batch(st, bt, True)
        e[1].record(stream)
        e[2].record(stream)
        if conditional:
            out, _, _ = J.join_probe_consume_batch(st, pt, True, True, ([3], [2]))
            wid, eid = out.columns[0].data, out.columns[1].data
        else:
            out, _, _ = J.join_probe_consume_batch(st, pt, True, True, ([1, 2, 3], [1, 2]))
            fp = PhysicalFilterProject(pred, [("wid", col("wid")), ("eid", col("eid"))], device=0, stream=sp)
            out, _ = fp.ProcessBatch(out, OperatorResult.NEED_MORE_INPUT)
            wid, eid = out.columns[0].data, out.columns[1].data
        e[3].record(stream)
        torch.cuda.synchronize(dev)
        n = out.n_rows
        res = {"build_ms": e[0].elapsed_time(e[1]), "ms": e[2].elapsed_time(e[3]), "rows": n,
               "check": checksum(torch.as_tensor(wid, device=dev)[:n], torch.as_tensor(eid, device=dev)[:n]),
               "path": [J.get_metric(st, m) for m in (5, 6, 7, 8, 9)]}
        J.delete_join_state(st)
        return res

    def median(xs):
        return sorted(xs)[len(xs) // 2]

    for k in [int(x) for x in args.k.split(",")]:
        bt = build_side(k)
        free = torch.cuda.mem_get_info(dev)[0]
        per_row = 24 + 16 + k * (45 + 8) + 16  # probe input, join scratch, unconditioned output (+ validity), filtered copy
        n = args.probe_rows or min(1 << 28, 1 << int((0.6 * free / per_row)).bit_length() - 1)
        pt = probe_side(k, n)
        arms = ["cond_inner", "filter_inner", "cond_left", "filter_left"]
        runs = {a: [] for a in arms}
        for a in arms:
            step(a, bt, pt)  # warm-up
        for _ in range(args.reps):
            for a in arms:
                runs[a].append(step(a, bt, pt))
        res = {a: {"ms": median([r["ms"] for r in runs[a]]), "build_ms": median([r["build_ms"] for r in runs[a]]), "rows": runs[a][-1]["rows"],
                   "check": runs[a][-1]["check"], "path": runs[a][-1]["path"]} for a in arms}
        ok = len({(r["rows"], tuple(r["check"])) for rs in runs.values() for r in rs}) == 1 and res["cond_inner"]["rows"] == n
        print(json.dumps({"k": k, "build_rows": bt.n_rows, "probe_rows": n, "arms": res, "check_ok": ok}), flush=True)
        del pt
        torch.cuda.empty_cache()
        pt = probe_side(k, args.alone_rows)
        step("cond_inner", bt, pt)
        alone = [step("cond_inner", bt, pt) for _ in range(args.reps)]
        ok = all(r["rows"] == args.alone_rows and r["path"][4] == args.alone_rows and r["path"][3] == k * args.alone_rows for r in alone)
        print(json.dumps({"k": k, "build_rows": bt.n_rows, "probe_rows": args.alone_rows, "cond_inner_alone_ms": median([r["ms"] for r in alone]),
                          "rows_per_s": args.alone_rows / (median([r["ms"] for r in alone]) / 1e3), "check_ok": ok}), flush=True)
        del pt, bt
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
