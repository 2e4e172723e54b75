"""As-of join (trades -> latest quote per symbol) against the window workaround, 1 x H100.

    python benchmarks/asof_join_bench.py [--quotes 67108864] [--trades 268435456] [--symbols 65536] [--reps 3]

Workload: quotes (the build side) have `--quotes` rows over `--symbols` symbols: sym (int64), ts (DATETIME, ns), bid and ask
(float64, whole numbers below 2^20 so sums of them are exact); trades (the probe side) have `--trades` rows with a uniform
symbol and a uniform ts over the same range.  Every column is device resident.  Arms, alternated in one process, one warm-up
step each:
  left_backward    init_join_state(..., asof_on=("ts", "ts")), probe_outer: every trade with the latest quote at or before it
  nearest_tol      the same with asof_direction="nearest", asof_tolerance = 1 ms
  inner_backward   left_backward without probe_outer: only trades that have a quote at or before them
  window           the workaround: the union of both sides (quotes first, a bid column that is NULL on trade rows), one window
                   operator LAST_VALUE(bid IGNORE NULLS) OVER (PARTITION BY sym ORDER BY ts ROWS UNBOUNDED PRECEDING), then the
                   trade rows kept (a PhysicalFilterProject on the row kind)
Reported per arm, as the median over `--reps`:
  probe_ms     the probe call (the window arm: the union's sort + window + filter), CUDA events on the stream
  build_ms     the as-of build call, beside equijoin_build_ms, the build of a plain equi-join on sym over the same quotes: the
               difference is the sort of the build side by (slot, ts)
  rows_per_s   trades / probe_ms
  check        matched rows and the sums of bid and ask over them; left_backward's must equal window's
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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--quotes", type=int, default=1 << 26)
    ap.add_argument("--trades", type=int, default=1 << 28)
    ap.add_argument("--symbols", type=int, default=1 << 16)
    ap.add_argument("--reps", type=int, default=3)
    args = ap.parse_args()

    import torch

    from bodo_b200 import _lib
    from bodo_b200.expr import col
    from bodo_b200.physical import OperatorResult, PhysicalFilterProject
    from bodo_b200.streaming import join as J
    from bodo_b200.streaming import window as W
    from bodo_b200.table import ArrTypes, Column, CTypes, Table

    _lib.require_gpu()
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    stream = torch.cuda.current_stream(dev)
    sp = stream.cuda_stream
    print(json.dumps({"card": card(), "torch_device": torch.cuda.get_device_name(dev)}), flush=True)
    gen = torch.Generator(device=dev).manual_seed(7)
    span = 6 * 3600 * 10**9  # one trading day of ns
    i64 = dict(device=dev, dtype=torch.int64, generator=gen)

    def dt(x):
        return Column(x, None, CTypes.DATETIME)

    qsym = torch.randint(0, args.symbols, (args.quotes,), **i64)
    qts = torch.randint(0, span, (args.quotes,), **i64)
    bid = torch.randint(0, 1 << 20, (args.quotes,), **i64).double()
    ask = bid + torch.randint(1, 100, (args.quotes,), **i64).double()
    quotes = Table([Column(qsym), dt(qts), Column(bid), Column(ask)], ["sym", "ts", "bid", "ask"])
    tsym = torch.randint(0, args.symbols, (args.trades,), **i64)
    tts = torch.randint(0, span, (args.trades,), **i64)
    trades = Table([Column(tsym), dt(tts)], ["sym", "ts"])

    def timed(f):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(stream)
        r = f()
        e1.record(stream)
        torch.cuda.synchronize(dev)
        return e0.elapsed_time(e1), r

    def check(n, b, a, valid):
        b, a = b[:n], a[:n]
        if valid is not None:
            b, a = b[valid], a[valid]
        return [int(b.numel()), float(b.sum().item()), float(a.sum().item())]

    def asof_arm(direction, left, tol=None):
        st = J.init_join_state(-1, (0,), (0,), quotes.names, trades.names, False, left, device=0, stream=sp, output_batch_size=1 << 30,
                               expected_build_rows=args.quotes, asof_on=("ts", "ts"), asof_direction=direction, asof_tolerance=tol)
        build_ms, _ = timed(lambda: J.join_build_consume_batch(st, quotes, True))
        probe_ms, (out, _, _) = timed(lambda: J.join_probe_consume_batch(st, trades, True, True, ([2, 3], [1])))
        n = out.n_rows
        valid = None
        if out.columns[0].validity is not None:
            bits = torch.as_tensor(out.columns[0].validity, device=dev)[: (n + 7) // 8]
            valid = ((bits.unsqueeze(1) >> torch.arange(8, device=dev, dtype=torch.uint8)) & 1).flatten()[:n].bool()
        chk = check(n, torch.as_tensor(out.columns[0].data, device=dev), torch.as_tensor(out.columns[1].data, device=dev), valid)
        J.delete_join_state(st)
        return {"build_ms": build_ms, "probe_ms": probe_ms, "check": chk}

    def equijoin_build():
        st = J.init_join_state(-1, (0,), (0,), quotes.names, trades.names, False, True, device=0, stream=sp, expected_build_rows=args.quotes)
        ms, _ = timed(lambda: J.join_build_consume_batch(st, quotes, True))
        J.delete_join_state(st)
        return ms

    def window_arm():
        def run():
            nq, nt = args.quotes, args.trades
            kind = torch.cat([torch.zeros(nq, device=dev, dtype=torch.int8), torch.ones(nt, device=dev, dtype=torch.int8)])
            vbits = torch.zeros((nq + nt + 7) // 8 + 8, device=dev, dtype=torch.uint8)
            vbits[: nq // 8] = 0xFF  # quotes are a multiple of 8 rows: their bid and ask are valid, the trades' NULL
            z = torch.zeros(nt, device=dev, dtype=torch.float64)
            union = Table([Column(torch.cat([qsym, tsym])), dt(torch.cat([qts, tts])),
                           Column(torch.cat([bid, z]), vbits, CTypes.FLOAT64, ArrTypes.NULLABLE_INT_BOOL),
                           Column(torch.cat([ask, z]), vbits, CTypes.FLOAT64, ArrTypes.NULLABLE_INT_BOOL), Column(kind)],
                          ["sym", "ts", "bid", "ask", "kind"])
            st = W.init_window_state(-1, ["sym"], ["ts"], True, "last", [("lb", "last_value", "bid", "rows", "ignore_nulls"),
                                                                      ("la", "last_value", "ask", "rows", "ignore_nulls")],
                                     union.names, output_batch_size=1 << 40, device=0, stream=sp)
            W.window_build_consume_batch(st, union, True)
            out, _ = W.window_produce_output_batch(st)
            fp = PhysicalFilterProject(col("kind") == 1, [("lb", col("lb")), ("la", col("la"))], device=0, stream=sp)
            kept, _ = fp.ProcessBatch(out, OperatorResult.NEED_MORE_INPUT)
            return st, kept

        ms, (st, kept) = timed(run)
        n = kept.n_rows
        m = torch.as_tensor(kept.columns[0].validity, device=dev)[: (n + 7) // 8]
        valid = ((m.unsqueeze(1) >> torch.arange(8, device=dev, dtype=torch.uint8)) & 1).flatten()[:n].bool()
        chk = check(n, torch.as_tensor(kept.columns[0].data, device=dev), torch.as_tensor(kept.columns[1].data, device=dev), valid)
        W.delete_window_state(st)
        del kept
        return {"build_ms": 0.0, "probe_ms": ms, "check": chk}

    arms = {
        "left_backward": lambda: asof_arm("backward", True),
        "nearest_tol": lambda: asof_arm("nearest", True, 10**6),
        "inner_backward": lambda: asof_arm("backward", False),
        "window": window_arm,
    }
    runs = {a: [] for a in arms}
    eq = []
    for a, f in arms.items():
        f()
        torch.cuda.empty_cache()
    equijoin_build()
    for _ in range(args.reps):
        for a, f in arms.items():
            runs[a].append(f())
            torch.cuda.empty_cache()
        eq.append(equijoin_build())

    def median(xs):
        return sorted(xs)[len(xs) // 2]

    res = {a: {"probe_ms": median([r["probe_ms"] for r in rs]), "build_ms": median([r["build_ms"] for r in rs]),
               "rows_per_s": args.trades / (median([r["probe_ms"] for r in rs]) / 1e3), "check": rs[-1]["check"]} for a, rs in runs.items()}
    ok = res["left_backward"]["check"] == res["window"]["check"] and all(len({tuple(r["check"]) for r in rs}) == 1 for rs in runs.values())
    print(json.dumps({"quotes": args.quotes, "trades": args.trades, "symbols": args.symbols, "equijoin_build_ms": median(eq), "arms": res,
                      "check_ok": ok}), flush=True)


if __name__ == "__main__":
    main()
