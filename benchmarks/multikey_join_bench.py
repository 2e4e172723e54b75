"""Two-column join key against the same join on one int64 key, 1 x H100.

    python benchmarks/multikey_join_bench.py [--build-rows 100000000] [--probe-rows 1000000000] [--probe-batch 250000000] [--reps 3]

Shape: the join of bench.py --workload join (`--probe-rows` probe rows against `--build-rows` unique build keys k = randperm, probe
keys uniform over the build keys so every probe row matches, 2 payload columns per side), with the key either the int64 k or the
two columns k1 = k >> 10 (int64) and k2 = k & 1023 (int32) on both sides.  All inputs are resident in HBM.  One step = init state ->
build (one batch) -> probe in `--probe-batch`-row batches, every batch materialising its rows (kept columns: the build key
column(s) and payloads, the probe payloads).  Four arms, alternated in one process:
  multi_inner   two-column key, inner join (the general CSR path: multi-column keys never take the unique-key tables)
  single_inner  int64 key, inner join (the default path: the inline Slot32 table)
  multi_left    two-column key, how="left"
  single_left   int64 key, how="left" (an outer probe side takes the general path for one key too)
Every probe row matches, so the left joins produce the inner result through the general path for both key shapes: multi_left
against single_left isolates the cost of the tuple hash and the column compare; multi_inner against single_inner is what a user
pays for the second key column.
  ms_per_step   median of `--reps` steps per arm (CUDA events, one warm-up step per arm)
  probe_ms      per probe call, CUDA events on the operator's stream, median over the calls of one step, median over the reps
  path          join metrics 5 (unique-key probe launches), 6 (inline-payload probe launches), 7 (inline builds)
  check         row count, and the sum mod 2^64 of every output column against torch gathers through the inverse permutation
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


def u64sum(t):
    import torch

    t = t.contiguous()
    t = t.view(torch.int64) if t.element_size() == 8 else t.to(torch.int64)
    return int(t.sum().item()) & ((1 << 64) - 1)


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
    split = lambda k: (k >> 10, (k & 1023).to(torch.int32))
    bk1, bk2 = split(bk)
    pk1 = torch.empty(npr, dtype=torch.int64, device=dev)
    pk2 = torch.empty(npr, dtype=torch.int32, device=dev)
    for r0 in range(0, npr, batch):
        pk1[r0:r0 + batch], pk2[r0:r0 + batch] = split(pk[r0:r0 + batch])
    torch.cuda.synchronize(dev)

    def tables(multi, r0=None, r1=None):
        if r0 is None:  # build side
            if multi:
                return Table([Column(bk1), Column(bk2), Column(b1), Column(b2)], ["k1", "k2", "b1", "b2"])
            return Table([Column(bk), Column(b1), Column(b2)], ["k", "b1", "b2"])
        if multi:
            return Table([Column(pk1[r0:r1]), Column(pk2[r0:r1]), Column(p1[r0:r1]), Column(p2[r0:r1])], ["k1", "k2", "p1", "p2"])
        return Table([Column(pk[r0:r1]), Column(p1[r0:r1]), Column(p2[r0:r1])], ["k", "p1", "p2"])

    arms = {"multi_inner": (True, False), "single_inner": (False, False), "multi_left": (True, True), "single_left": (False, True)}

    def step(arm, collect=False):
        multi, left = arms[arm]
        keys = (0, 1) if multi else (0,)
        bt = tables(multi)
        st = J.init_join_state(-1, keys, keys, tuple(bt.names), tuple(tables(multi, 0, 1).names), False, left, expected_build_rows=nb,
                               device=0, stream=sp)
        J.join_build_consume_batch(st, bt, True)
        kept = (list(range(bt.n_cols)), [len(keys), len(keys) + 1])
        rows, sums, evs = 0, [0] * (bt.n_cols + 2), []
        for r0 in range(0, npr, batch):
            r1 = min(npr, r0 + batch)
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(stream)
            out, _, _ = J.join_probe_consume_batch(st, tables(multi, r0, r1), r1 == npr, True, kept)
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

    def timed(arm):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(stream)
        r = step(arm)
        e1.record(stream)
        torch.cuda.synchronize(dev)
        return e0.elapsed_time(e1), r

    for arm in arms:  # warm-up
        step(arm)
    times = {a: [] for a in arms}
    probe_ms = {a: [] for a in arms}
    for _ in range(args.reps):
        for arm in arms:
            ms, r = timed(arm)
            times[arm].append(ms)
            probe_ms[arm].append(r["probe_ms"][len(r["probe_ms"]) // 2])
    info = {arm: step(arm, collect=True) for arm in arms}

    # independent recomputation: inverse permutation + torch gathers over k
    inv = torch.empty(nb, dtype=torch.int64, device=dev)
    inv[bk] = torch.arange(nb, dtype=torch.int64, device=dev)
    exp = {"single": [0] * 5, "multi": [0] * 6}
    for r0 in range(0, npr, batch):
        kk = pk[r0:r0 + batch]
        bi = inv[kk]
        tail = [b1[bi], b2[bi], p1[r0:r0 + batch], p2[r0:r0 + batch]]
        for shape, head in (("single", [bk[bi]]), ("multi", [bk1[bi], bk2[bi]])):
            for j, c in enumerate(head + tail):
                exp[shape][j] = (exp[shape][j] + u64sum(c)) & ((1 << 64) - 1)
        del bi, tail
    shape_of = lambda arm: "multi" if arms[arm][0] else "single"
    check = {a: info[a]["rows"] == npr and info[a]["sums"] == exp[shape_of(a)] for a in arms}

    med = {a: sorted(v)[len(v) // 2] for a, v in times.items()}
    pmed = {a: sorted(v)[len(v) // 2] for a, v in probe_ms.items()}
    print(json.dumps({
        "build_rows": nb, "probe_rows": npr, "probe_batch": batch, "card": card(),
        "ms_per_step": {a: round(v, 3) for a, v in med.items()}, "runs_ms": {a: [round(x, 3) for x in v] for a, v in times.items()},
        "multi_over_single": {"inner": round(med["multi_inner"] / med["single_inner"], 4), "left": round(med["multi_left"] / med["single_left"], 4)},
        "probe_ms": {a: round(v, 3) for a, v in pmed.items()}, "probe_runs_ms": {a: [round(x, 3) for x in v] for a, v in probe_ms.items()},
        "path_metrics_5_6_7": {a: info[a]["path"] for a in arms},
        "check": {a: (f"ok: row count and sum mod 2^64 of all {len(exp[shape_of(a)])} output columns" if check[a]
                      else f"MISMATCH {info[a]['rows']} {info[a]['sums']} {exp[shape_of(a)]}") for a in arms},
    }), flush=True)
    if not all(check.values()):
        sys.exit(3)


if __name__ == "__main__":
    main()
