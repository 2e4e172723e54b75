"""Full streaming sort (ORDER BY without LIMIT), 1 x H100.

    python benchmarks/sort_bench.py [--rows 536870912] [--batch 16777216] [--reps 3] [--profile DIR]

Data, resident in HBM: `--rows` rows of a float64 key (synth.device_fill's uniform doubles in [0, 1)), p = row id (int64) and
one float64 payload, fed in `--batch`-row batches.  Cases:
  random_asc     the float64 key, ascending;
  random_desc    the same key, descending;
  int_1e6        an int64 key in [0, 10^6) instead: the five upper bytes are constant, so five of its eight passes are skipped;
  two_keys       a nullable int32 key in [0, 10^6) with 10 % NA (ascending, NA last), then the float64 key descending (4 columns:
                 at 2^29 rows it does not fit next to this benchmark's inputs on an 80 GB card; run it with --rows 268435456).
Reported per case:
  ms_per_step    one step = init -> consume every batch (is_last on the last) -> produce -> delete; median of `--reps` after one
                 warm-up step, CUDA events on the operator's stream
  rows_per_s     rows / step time
  passes         metrics 7 (digit passes run) and 8 (skipped), and the plan the benchmark predicts from the data
  bytes, gbps    bytes the algorithm moves, from the shapes and the passes run (see moved_bytes), over the step time; the share
                 of the data sheet's 3350 GB/s
  torch_ms       torch.sort(stable=True) of the key (two_keys: of both keys, least significant first) plus gathers of the
                 other columns, same process: a reference point only
  peak_gb        device memory the step needs at its peak, computed from the shapes: the inputs, plus during the last consume
                 call the chunk store, the pair buffers, the look-back words and the output store with its validity bytes;
                 used_gb is cudaMemGetInfo's used bytes right after the last consume call (pooled blocks included)
  check          single key: output keys equal torch's sorted keys, key[p] == out_key, p rises within ties.  two_keys: adjacent
                 output rows are ordered by (NA class, int key, -float key), p rises within ties, every column equals the input
                 at p.  The process exits non-zero on a mismatch.
With --profile DIR, one more step of each case runs under torch.profiler and the per-kernel CUDA times go to DIR/kernels.json.
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

TILE = 4096
PEAK_GBPS = 3350.0


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30).stdout.strip()
    except Exception as e:
        q = f"nvidia-smi unavailable ({e})"
    return q


def plan(torch, words, widths, can_na, nas):
    """Per key (least significant first as given): (width, byte passes run, byte passes skipped, class pass run, skipped)."""
    out = []
    for w, b, cn, na in zip(words, widths, can_na, nas):
        run = sum(1 for i in range(b) if int(((w >> (8 * i)) & 255).min()) != int(((w >> (8 * i)) & 255).max()))
        n = w.numel()
        cls_run = int(cn and 0 < na < n)
        out.append((b, run, b - run, cls_run, int(cn) - cls_run))
    return out


def moved_bytes(n, row_bytes, n_nullable, key_bytes, key_plan):
    """append: read the batch, write the chunk (row bytes + one validity byte per nullable column); histogram: read the keys;
    passes: the first pass of a key reads its column (through the permutation after the first key: + 4 B of row id) and writes
    (word, id) pairs, every further pass reads and writes pairs; gather: read ids, read and write every column and validity byte;
    pack: read the validity bytes, write the bitmaps."""
    chunk = row_bytes + n_nullable
    total = n * row_bytes + n * chunk + n * key_bytes
    first_key = True
    for b, run, _, cls_run, _ in key_plan:
        passes = run + cls_run
        if passes == 0:
            continue
        pair = (4 if b <= 4 else 8) + 4
        total += n * ((b + (0 if first_key else 4)) + pair) + (passes - 1) * n * 2 * pair
        first_key = False
    total += n * 4 + 2 * n * chunk + n * n_nullable + n * n_nullable / 8
    return int(total)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=1 << 29)
    ap.add_argument("--batch", type=int, default=1 << 24)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--cases", type=str, default="random_asc,random_desc,int_1e6,two_keys")
    ap.add_argument("--profile", type=str, default="")
    args = ap.parse_args()

    import torch

    from bodo_b200 import _lib, synth
    from bodo_b200.streaming import sort as S
    from bodo_b200.table import ArrTypes, Column, CTypes, Table

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
    g = torch.Generator(device=dev).manual_seed(53)
    ikey = torch.randint(0, 10**6, (n,), generator=g, device=dev, dtype=torch.int64)
    ikey32 = ikey.to(torch.int32)
    valid = torch.rand(n, generator=g, device=dev) >= 0.1
    vpad = torch.zeros((n + 7) // 8 * 8, dtype=torch.uint8, device=dev)
    vpad[:n] = valid.to(torch.uint8)
    vbits = (vpad.view(-1, 8).to(torch.int32) << torch.arange(8, device=dev, dtype=torch.int32)).sum(1).to(torch.uint8)
    torch.cuda.synchronize(dev)

    def f64_word(x, desc=False):
        b = torch.where(x == 0, torch.zeros_like(x), x).view(torch.int64)
        w = torch.where(b < 0, b ^ 0x7FFFFFFFFFFFFFFF, b)
        return ~w if desc else w

    cases = {
        "random_asc": dict(cols=[key, p, pay], names=["k", "p", "v"], by=["k"], asc=[True], nap=["last"]),
        "random_desc": dict(cols=[key, p, pay], names=["k", "p", "v"], by=["k"], asc=[False], nap=["last"]),
        "int_1e6": dict(cols=[ikey, p, pay], names=["k", "p", "v"], by=["k"], asc=[True], nap=["last"]),
        "two_keys": dict(cols=[ikey32, key, p, pay], names=["i", "k", "p", "v"], by=["i", "k"], asc=[True, False], nap=["last", "last"]),
    }

    def make_batch(c, r0, r1):
        cols = []
        for name, t in zip(c["names"], c["cols"]):
            if name == "i":
                assert r0 % 8 == 0
                cols.append(Column(t[r0:r1], vbits[r0 // 8:(r1 + 7) // 8], CTypes.INT32, ArrTypes.NULLABLE_INT_BOOL, r1 - r0))
            else:
                cols.append(Column(t[r0:r1]))
        return Table(cols, c["names"])

    def step(c, keep=False):
        st = S.init_stream_sort_state(-1, None, 0, c["by"], c["asc"], c["nap"], c["names"], output_batch_size=1 << 30, device=0,
                                      stream=sp, full=True)
        for r0 in range(0, n, args.batch):
            r1 = min(n, r0 + args.batch)
            S.sort_build_consume_batch(st, make_batch(c, r0, r1), r1 == n)
        free, total = torch.cuda.mem_get_info(dev)
        step.used_gb = (total - free) / 1e9
        out, _ = S.produce_output_batch(st)
        res = None
        if keep:
            res = [torch.as_tensor(col.data, device=dev).clone() for col in out.columns]
            if out.columns[0].validity is not None:
                vb = torch.as_tensor(out.columns[0].validity, device=dev)
                res.append(((vb.repeat_interleave(8).view(-1)[: n].to(torch.int32) >> torch.arange(n, device=dev).remainder(8).to(torch.int32)) & 1).bool())
        metrics = [S.get_metric(st, w) for w in range(9)]
        S.delete_stream_sort_state(st)
        return res, metrics

    def timed(fn):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(stream)
        r = fn()
        e1.record(stream)
        torch.cuda.synchronize(dev)
        return e0.elapsed_time(e1), r

    def verify(name, res):
        if name != "two_keys":
            k_col = cases[name]["cols"][0]
            ok_k, ok_p, ok_v = res
            ref = torch.sort(k_col, descending=not cases[name]["asc"][0], stable=True).values
            if not torch.equal(ok_k, ref):
                return "MISMATCH: keys differ from torch.sort"
            if not torch.equal(k_col[ok_p], ok_k) or not torch.equal(pay[ok_p], ok_v):
                return "MISMATCH: key[p] or payload[p] differs from the output row"
            same = ok_k[1:] == ok_k[:-1]
            if bool((same & (ok_p[1:] <= ok_p[:-1])).any()):
                return "MISMATCH: p does not rise within a run of equal keys"
            return "ok"
        oi, ok_k, ok_p, ok_v, ovalid = res
        if not (torch.equal(ovalid, valid[ok_p]) and torch.equal(ok_k, key[ok_p]) and torch.equal(ok_v, pay[ok_p])
                and torch.equal(oi[ovalid], ikey32[ok_p][ovalid])):
            return "MISMATCH: a column differs from the input row at p"
        cls = (~ovalid).to(torch.int64)
        a = torch.where(ovalid, oi.to(torch.int64), 0)
        b = -ok_k
        lt = (cls[:-1] < cls[1:]) | ((cls[:-1] == cls[1:]) & ((a[:-1] < a[1:]) | ((a[:-1] == a[1:]) & (b[:-1] < b[1:]))))
        eq = (cls[:-1] == cls[1:]) & (a[:-1] == a[1:]) & (b[:-1] == b[1:])
        if not bool((lt | eq).all()):
            return "MISMATCH: adjacent rows out of (NA class, int key, -float key) order"
        if bool((eq & (ok_p[1:] <= ok_p[:-1])).any()):
            return "MISMATCH: p does not rise within ties"
        return "ok"

    def torch_ref(name):
        c = cases[name]
        if name == "two_keys":
            idx = torch.sort(key, descending=True, stable=True).indices
            k2 = torch.where(valid, ikey32, torch.iinfo(torch.int32).max).to(torch.int64) + (~valid).to(torch.int64)  # NA last
            idx = idx[torch.sort(k2[idx], stable=True).indices]
        else:
            idx = torch.sort(c["cols"][0], descending=not c["asc"][0], stable=True).indices
        return [t[idx] for t in c["cols"]]

    ok = True
    prof_rows = {}
    for name in args.cases.split(","):
        c = cases[name]
        if name == "two_keys":
            words = [f64_word(key, True), torch.where(valid, ikey32.to(torch.int64) ^ 0x80000000, 0)]
            kp = plan(torch, words, [8, 4], [True, True], [0, int((~valid).sum())])
            row_bytes, n_nullable, key_bytes = 4 + 24, 1, 12 + 1
        else:
            w = f64_word(c["cols"][0]) if c["cols"][0].dtype == torch.float64 else c["cols"][0] ^ (-(2 ** 63))
            kp = plan(torch, [w], [8], [c["cols"][0].dtype == torch.float64], [0])
            row_bytes, n_nullable, key_bytes = 24, 0, 8
        step.used_gb = 0.0
        step(c)  # warm-up
        times = []
        for _ in range(args.reps):
            ms, (_, metrics) = timed(lambda: step(c))
            times.append(ms)
        used_gb = step.used_gb
        ms = sorted(times)[len(times) // 2]
        res, metrics = step(c, keep=True)
        chk = verify(name, res)
        del res
        tt = []
        for _ in range(args.reps):
            t_ms, r = timed(lambda: torch_ref(name))
            del r
            tt.append(t_ms)
        torch.cuda.empty_cache()  # the reference's buffers and the library's pooled blocks go back to the driver
        _lib.lib().b200_pool_trim(0, 0)
        predicted = (sum(x[1] + x[3] for x in kp), sum(x[2] + x[4] for x in kp))
        if predicted != (metrics[7], metrics[8]):
            chk = f"MISMATCH: passes run/skipped {metrics[7:9]} differ from the plan {predicted}" if chk == "ok" else chk
        moved = moved_bytes(n, row_bytes, n_nullable, key_bytes, kp)
        chunk_row = row_bytes + n_nullable
        wmax = max([4 if b <= 4 else 8 for b, run, _, cls_run, _ in kp if run + cls_run] or [0])
        lib_bytes = (-(-n // (1 << 24)) * (1 << 24) * chunk_row + (2 * n * (wmax + 4) + -(-n // TILE) * 2048 if wmax else 0)
                     + n * chunk_row)
        input_bytes = sum(t.numel() * t.element_size() for t in c["cols"]) + (vbits.numel() if name == "two_keys" else 0)
        out = {"case": name, "rows": n, "batch": args.batch, "ms_per_step": round(ms, 3), "runs_ms": [round(x, 3) for x in times],
               "rows_per_s": round(n / (ms * 1e-3), 1), "passes_run": metrics[7], "passes_skipped": metrics[8],
               "bytes": moved, "gbps": round(moved / (ms * 1e-3) / 1e9, 1), "share_of_3350_gbps": round(moved / (ms * 1e-3) / 1e9 / PEAK_GBPS, 4),
               "torch_ms": round(sorted(tt)[len(tt) // 2], 3), "peak_gb": round((lib_bytes + input_bytes) / 1e9, 2), "used_gb": round(used_gb, 2), "metrics": metrics, "check": chk, "card": card()}
        print(json.dumps(out), flush=True)
        ok &= chk == "ok"
        if args.profile:
            from torch.profiler import ProfilerActivity, profile

            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                step(c)
                torch.cuda.synchronize(dev)
            rows = {}
            for e in prof.key_averages():
                if e.device_type.name == "CUDA" or "kernel" in e.key:
                    rows[e.key] = {"count": e.count, "cuda_ms": round(getattr(e, "device_time_total", getattr(e, "cuda_time_total", 0)) / 1e3, 3)}
            prof_rows[name] = rows
            print(json.dumps({"case": name, "profile": {k: v for k, v in rows.items() if "fsort" in k or "pack_bitmap" in k or "Memset" in k}}), flush=True)
    if args.profile:
        os.makedirs(args.profile, exist_ok=True)
        with open(os.path.join(args.profile, "kernels.json"), "w") as f:
            json.dump(prof_rows, f, indent=1)
    if not ok:
        sys.exit(3)


if __name__ == "__main__":
    main()
