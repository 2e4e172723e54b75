"""Streaming top-k (ORDER BY key DESC LIMIT K), 1 x H100.

    python benchmarks/topk_bench.py [--rows 1000000000] [--batch 16777216] [--reps 3] [--small-rows 134217728] [--small-batch 32768]

Data, resident in HBM: `--rows` rows of a float64 key (synth.device_fill's uniform doubles in [0, 1)), p = row id (int64) and one
float64 payload, fed in `--batch`-row batches.  Cases:
  random         K in {10, 1000, 100000}, descending, the synthetic keys in row order: after the first cutoff almost every row is
                 dropped by the filter kernel;
  adversarial    the same K with key = p (rising keys, sorted descending): every batch beats the cutoff, the candidate store fills
                 and overflows, and reduces run all the time;
  per_call       K = 1000 on the first `--small-rows` random rows in `--small-batch`-row batches: the cost of one consume call.
Reported per case:
  ms_per_step    one step = init -> consume every batch (is_last on the last) -> produce -> delete; median of `--reps` after one
                 warm-up step, CUDA events on the operator's stream
  rows_per_s     rows / step time
  gbps           bytes the algorithm must move / step time: rows x 8 key bytes, plus per admitted candidate its 24 input bytes and
                 the 41 bytes of its store row (key word, NA class, arrival index, 3 columns); the data-sheet bound is 3.35 TB/s
                 (8 GB of keys alone take >= 2.39 ms)
  metrics        the operator's metrics 0-6 (rows consumed, admitted, reduce steps, count reads, filter launches, admitted while a
                 cutoff existed, store capacity)
  torch_topk_ms  torch.topk over the whole key column plus a gather of p and the payload, same process (a reference point only:
                 it sees one resident column, not a stream of batches)
  check          the output keys equal torch.topk's sorted values, key[p] == out_key on every row, and p rises inside runs of
                 equal keys; the process exits non-zero on a mismatch
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

STORE_ROW_BYTES = 8 + 1 + 8 + 24
INPUT_ROW_BYTES = 24


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30).stdout.strip()
    except Exception as e:
        q = f"nvidia-smi unavailable ({e})"
    return q


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=1_000_000_000)
    ap.add_argument("--batch", type=int, default=1 << 24)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--small-rows", type=int, default=1 << 27)
    ap.add_argument("--small-batch", type=int, default=32768)
    ap.add_argument("--ks", type=str, default="10,1000,100000")
    args = ap.parse_args()

    import torch

    from bodo_b200 import _lib, synth
    from bodo_b200.streaming import sort as S
    from bodo_b200.table import Column, Table

    _lib.require_gpu()
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    stream = torch.cuda.current_stream(dev)
    sp = stream.cuda_stream
    n = args.rows
    print(json.dumps({"card": card(), "torch_device": torch.cuda.get_device_name(dev)}), flush=True)

    key = torch.empty(n, dtype=torch.float64, device=dev)
    pay = torch.empty(n, dtype=torch.float64, device=dev)
    synth.device_fill(None, key, 0, 1, 51, sp)
    synth.device_fill(None, pay, 0, 1, 52, sp)
    p = torch.arange(n, dtype=torch.int64, device=dev)
    adv = p.to(torch.float64)
    torch.cuda.synchronize(dev)
    names = ["k", "p", "v"]

    def step(k_col, rows, batch, K):
        st = S.init_stream_sort_state(-1, K, 0, ["k"], [False], ["last"], names, output_batch_size=1 << 30, device=0, stream=sp)
        for r0 in range(0, rows, batch):
            r1 = min(rows, r0 + batch)
            S.sort_build_consume_batch(st, Table([Column(k_col[r0:r1]), Column(p[r0:r1]), Column(pay[r0:r1])], names), r1 == rows)
        out, _ = S.produce_output_batch(st)
        res = [torch.as_tensor(c.data, device=dev).clone() for c in out.columns]
        metrics = [S.get_metric(st, w) for w in range(7)]
        S.delete_stream_sort_state(st)
        return res, metrics

    def timed(fn):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(stream)
        r = fn()
        e1.record(stream)
        torch.cuda.synchronize(dev)
        return e0.elapsed_time(e1), r

    def verify(k_col, rows, K, res):
        ok_k, ok_p, ok_v = res
        ref = torch.topk(k_col[:rows], min(K, rows)).values
        if not torch.equal(ok_k, ref):
            return "MISMATCH: keys differ from torch.topk"
        if not torch.equal(k_col[ok_p], ok_k) or not torch.equal(pay[ok_p], ok_v):
            return "MISMATCH: key[p] or payload[p] differs from the output row"
        same = ok_k[1:] == ok_k[:-1]
        if bool((same & (ok_p[1:] <= ok_p[:-1])).any()):
            return "MISMATCH: p does not rise inside a run of equal keys"
        return "ok"

    def case(name, k_col, rows, batch, K):
        step(k_col, rows, batch, K)  # warm-up
        times = []
        for _ in range(args.reps):
            ms, (res, metrics) = timed(lambda: step(k_col, rows, batch, K))
            times.append(ms)
        ms = sorted(times)[len(times) // 2]
        tt = []
        for _ in range(args.reps):
            t_ms, _ = timed(lambda: (lambda r: (p[r.indices], pay[r.indices]))(torch.topk(k_col[:rows], min(K, rows))))
            tt.append(t_ms)
        moved = rows * 8 + metrics[1] * (INPUT_ROW_BYTES + STORE_ROW_BYTES)
        chk = verify(k_col, rows, K, res)
        out = {"case": name, "K": K, "rows": rows, "batch": batch, "ms_per_step": round(ms, 3), "runs_ms": [round(x, 3) for x in times],
               "rows_per_s": round(rows / (ms * 1e-3), 1), "gbps": round(moved / (ms * 1e-3) / 1e9, 1),
               "share_of_3350_gbps": round(moved / (ms * 1e-3) / 3.35e12, 4), "ms_per_call": round(ms / -(-rows // batch), 4),
               "metrics": metrics, "torch_topk_ms": round(sorted(tt)[len(tt) // 2], 3), "check": chk, "card": card()}
        print(json.dumps(out), flush=True)
        return chk == "ok"

    ok = True
    ks = [int(x) for x in args.ks.split(",")]
    for K in ks:
        ok &= case("random", key, n, args.batch, K)
    for K in ks:
        ok &= case("adversarial", adv, n, args.batch, K)
    ok &= case("per_call", key, min(args.small_rows, n), args.small_batch, 1000)
    if not ok:
        sys.exit(3)


if __name__ == "__main__":
    main()
