"""Nested-loop join (no equi-join key) against the constant-key workaround, 1 x H100.

    python benchmarks/nested_loop_join_bench.py [--reps 3] [--configs band,small,cross]

The workaround appends one constant INT8 key column to both sides and runs the equi-join (with the same condition, if any): every
build row is then in one CSR group, one thread per probe row walks all of them twice, and each thread writes its own output rows.
Columns are int64 and device resident.  Configurations:
  band   2^16 build bands [lo, lo + 1049) with lo uniform in [0, 2^20), probe rows x uniform in [0, 2^20): (x >= lo) & (x < hi)
         passes about one pair in 1000.  Probe calls of 2^18 rows, inner and left.  Keeps bid and eid.
  small  the same condition, 64 probe rows against 2^22 build bands: one probe tile, so the nested-loop join's build chunks are
         what spreads the work over the GPU.  A step is --small-calls probe calls of the nested-loop join and the first of them
         for the workaround (whose 64 threads take seconds per call).
  cross  2^10 build rows x 2^18 probe rows per call, 2 columns per side (an id and a value), no condition: nlj_cross_kernel
         against the constant-key equi-join.  A timed step is --cross-calls probe calls.  Output: 2^28 rows x 32 bytes per call.
Both arms of a configuration live in one process, alternated, after one warm-up step each.
  ms        median over --reps steps of the mean probe-call time (CUDA events around each call)
  rate      pairs evaluated per second (band, small), output bytes per second and its share of 3.35 TB/s (cross)
  check     per probe call: output rows and the sums mod 2^64 of the kept columns (the row ids bid and eid; id and value for
            cross), equal between the arms for every call both ran (check_ok)
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

M64 = (1 << 64) - 1
HBM_BYTES_PER_S = 3.35e12
DOMAIN, WIDTH = 1 << 20, 1049


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--configs", default="band,small,cross")
    ap.add_argument("--small-calls", type=int, default=16)
    ap.add_argument("--cross-calls", type=int, default=32)
    args = ap.parse_args()

    import torch

    from bodo_b200 import _lib
    from bodo_b200.expr import build_col, probe_col
    from bodo_b200.streaming import join as J
    from bodo_b200.table import Column, CTypes, Table

    _lib.require_gpu()
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    stream = torch.cuda.current_stream(dev)
    sp = stream.cuda_stream
    print(json.dumps({"card": card(), "torch_device": torch.cuda.get_device_name(dev)}), flush=True)
    gen = torch.Generator(device=dev).manual_seed(7)
    band = (probe_col("x") >= build_col("lo")) & (probe_col("x") < build_col("hi"))

    def i64(t):
        return Column(t.contiguous(), None, CTypes.INT64)

    def with_key(t: Table) -> Table:
        k = torch.zeros(max(t.n_rows, 1), dtype=torch.int8, device=dev)
        return Table(list(t.columns) + [Column(k, None, CTypes.INT8, length=t.n_rows)], list(t.names) + ["k"])

    def bands(n):
        lo = torch.randint(0, DOMAIN, (n,), device=dev, dtype=torch.int64, generator=gen)
        return Table([i64(lo), i64(lo + WIDTH), i64(torch.arange(n, device=dev, dtype=torch.int64))], ["lo", "hi", "bid"])

    def events(n, first_id):
        x = torch.randint(0, DOMAIN, (n,), device=dev, dtype=torch.int64, generator=gen)
        return Table([i64(x), i64(torch.arange(first_id, first_id + n, device=dev, dtype=torch.int64))], ["x", "eid"])

    def two_cols(n, first_id):
        ids = torch.arange(first_id, first_id + n, device=dev, dtype=torch.int64)
        return Table([i64(ids), i64(ids * 0x9E3779B97F4A7C15 % (1 << 62))], ["id", "v"])

    def make_state(arm, bt, pt, cond, left):
        """(state, probe-table transform) of an arm, its build side fed: "nlj" or "const_key"."""
        if arm == "nlj":
            st = J.init_nested_loop_join_state(-1, tuple(bt.names), tuple(pt.names), False, left, cond, device=0, stream=sp,
                                               expected_build_rows=bt.n_rows)
            J.join_build_consume_batch(st, bt, True)
            return st, (lambda t: t)
        nb, npc = bt.n_cols, pt.n_cols
        st = J.init_join_state(-1, (nb,), (npc,), tuple(bt.names) + ("k",), tuple(pt.names) + ("k",), False, left, device=0, stream=sp,
                               expected_build_rows=bt.n_rows, non_equi_condition=cond)
        J.join_build_consume_batch(st, with_key(bt), True)
        return st, with_key

    def step(st, feed, batches, used):
        """One step: a probe call per batch, each timed alone by CUDA events; [(ms, rows, [sums mod 2^64 of the kept columns])]."""
        res = []
        for b in [feed(b) for b in batches]:
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            torch.cuda.synchronize(dev)
            e0.record(stream)
            out, _, _ = J.join_probe_consume_batch(st, b, False, True, used)
            e1.record(stream)
            torch.cuda.synchronize(dev)
            n = out.n_rows  # the output columns are reused by the next call: fold them now
            res.append((e0.elapsed_time(e1), n, [int(torch.as_tensor(c.data, device=dev)[:n].view(torch.int64).sum().item()) & M64 for c in out.columns]))
        return res

    def median(xs):
        return sorted(xs)[len(xs) // 2]

    def compare(name, bt, probe_calls, cond, left, used, rate, const_key_calls=None):
        """Alternate the two arms over the steps of probe_calls (each a list of probe batches); the constant-key arm runs the first
        const_key_calls batches of each step (all by default).  ms: the median over steps of a step's mean probe-call time."""
        arms = {a: make_state(a, bt, probe_calls[0][0], cond, left) for a in ("nlj", "const_key")}
        take = {"nlj": None, "const_key": const_key_calls}
        for a, (st, feed) in arms.items():
            step(st, feed, probe_calls[0][:1], used)  # warm-up
        runs = {a: [] for a in arms}
        for r in range(args.reps):
            for a, (st, feed) in arms.items():
                runs[a].append(step(st, feed, probe_calls[r % len(probe_calls)][: take[a]], used))
        res = {}
        for a, rs in runs.items():
            ms = median([sum(x[0] for x in calls) / len(calls) for calls in rs])
            res[a] = {"ms": ms, "calls_per_step": len(rs[0]), **rate(ms, rs[-1][-1][1]), "rows": [[x[1] for x in calls] for calls in rs],
                      "pairs_evaluated": J.get_metric(arms[a][0], 8), "pairs_passed": J.get_metric(arms[a][0], 9)}
            J.delete_join_state(arms[a][0])
        # the same probe call gives the same rows and row-id sums in both arms
        ok = all(x[1:] == y[1:] for n_, k_ in zip(runs["nlj"], runs["const_key"]) for x, y in zip(n_, k_))
        check = [[x[1], x[2]] for x in runs["nlj"][0]][:4]
        print(json.dumps({"config": name, "left": left, "build_rows": bt.n_rows, "probe_rows_per_call": probe_calls[0][0].n_rows,
                          "arms": res, "speedup": res["const_key"]["ms"] / res["nlj"]["ms"], "check": check, "check_ok": ok}), flush=True)
        torch.cuda.empty_cache()

    configs = args.configs.split(",")
    if "band" in configs:
        bt, n = bands(1 << 16), 1 << 18
        calls = [[events(n, i * n)] for i in range(3)]
        pairs = lambda ms, rows: {"pairs_per_s": n * bt.n_rows / (ms / 1e3)}
        for left in (False, True):
            compare("band", bt, calls, band, left, ([2], [1]), pairs)
        del bt, calls
    if "small" in configs:
        bt, n = bands(1 << 22), 64
        calls = [[events(n, (i * args.small_calls + j) * n) for j in range(args.small_calls)] for i in range(3)]
        pairs = lambda ms, rows: {"pairs_per_s": n * bt.n_rows / (ms / 1e3)}
        compare("small", bt, calls, band, False, ([2], [1]), pairs, const_key_calls=1)
        del bt, calls
    if "cross" in configs:
        bt, n = two_cols(1 << 10, 0), 1 << 18
        calls = [[two_cols(n, (i * args.cross_calls + j) * n) for j in range(args.cross_calls)] for i in range(2)]

        def out_bytes(ms, rows):
            bps = rows * 32 / (ms / 1e3)
            return {"out_bytes_per_s": bps, "share_of_3.35TB/s": bps / HBM_BYTES_PER_S}

        compare("cross", bt, calls, None, False, ([0, 1], [0, 1]), out_bytes)


if __name__ == "__main__":
    main()
