"""Streaming window operator (ranking functions OVER (PARTITION BY p ORDER BY o)), 1 x H100.

    python benchmarks/window_bench.py [--rows 268435456] [--batch 16777216] [--reps 3] [--cases rn_rank_dense,all6,no_partition]

Data, resident in HBM: `--rows` rows of an int64 partition key p in [0, 10^6), a float64 order key o (synth.device_fill's uniform
doubles in [0, 1)) and an int64 row id r, fed in `--batch`-row batches.  Cases:
  rn_rank_dense  row_number, rank, dense_rank OVER (PARTITION BY p ORDER BY o)
  all6           all six functions (ntile(4)) over the same window
  no_partition   row_number, rank, dense_rank OVER (ORDER BY o): one partition
  running        SUM(r) ROWS, MAX(r) RANGE and COUNT(*) over the partition, OVER (PARTITION BY p ORDER BY o)
  partition_aggs SUM / MEAN / MIN / MAX(o) over the whole partition
  lag_lead       LAG(r, 1) and LEAD(o, 1, 0.0)
  moving         AVG(o) and MAX(o) ROWS BETWEEN 6 PRECEDING AND CURRENT ROW, SUM(r) ROWS BETWEEN 3 PRECEDING AND 3 FOLLOWING
                 and NTH_VALUE(r, 2), OVER (PARTITION BY p ORDER BY o)
  moving_wide    SUM(r) and MIN(o) ROWS BETWEEN 65535 PRECEDING AND CURRENT ROW OVER (ORDER BY o): one partition, a deep tree
  moments        STDDEV(o) ROWS BETWEEN 19 PRECEDING AND CURRENT ROW (a Bollinger band's width), VAR(o) ROWS (running) and
                 STDDEV_POP(o) over the partition, OVER (PARTITION BY p ORDER BY o)
  bivariate      CORR(o, r) ROWS BETWEEN 19 PRECEDING AND CURRENT ROW (a rolling correlation), COVAR_SAMP(o, r) ROWS (running)
                 and REGR_SLOPE(o, r) over the partition (a beta), OVER (PARTITION BY p ORDER BY o)
  range_moving   AVG(o) and MAX(o) RANGE BETWEEN 2^35 ns PRECEDING AND CURRENT ROW, SUM(r) and COUNT(*) RANGE BETWEEN 2^34 ns
                 PRECEDING AND 2^34 ns FOLLOWING, OVER (PARTITION BY p ORDER BY t): about 8 rows per frame, as in moving
  range_wide     SUM(r) and MIN(o) RANGE BETWEEN 2^28 ns PRECEDING AND CURRENT ROW OVER (ORDER BY t): one partition, about 65 536
                 rows per frame, as in moving_wide
  ignore_nulls   a per-group ffill and bfill and a LAG that skips missing readings: LAST_VALUE(x IGNORE NULLS) ROWS, FIRST_VALUE(x
                 IGNORE NULLS) ROWS BETWEEN CURRENT ROW AND UNBOUNDED FOLLOWING and LAG(x, 1) IGNORE NULLS, OVER (PARTITION BY p
                 ORDER BY o)
The range cases add a fourth column t, an int64 DATETIME key uniform in [0, 2^40) ns, and order by it; ignore_nulls adds a
fourth column x, float64 normal values with about 30 % NaN placed by a hash of the row id; the other cases keep their three
columns.  ignore_nulls alternates with lag_lead (lag_lead_ms), so its cost above RESPECT NULLS navigation is measured too.  `--profile` runs one more step per case under torch.profiler (separately from the timed steps) and
reports the window kernels' device times; with it, nothing is timed (run it separately from the timed run).
The value cases (running to bivariate, and the range cases) also alternate with rn_rank_dense (rn_rank_dense_ms), so their cost above the ranking kernels
is measured too; their result check covers the validity of the nullable columns.  bivariate also alternates with moments
(moments_ms): its scan value is twice the moments' and it reads a second column.
One step = init -> consume every batch (is_last on the last) -> produce -> delete, timed with CUDA events on the operator's stream;
the median of `--reps` steps after one warm-up.  Every window step alternates with a full sort of the same keys and columns in
the same process (sort_ms), so the window's cost above the sort is a measured difference (extra_ms).
Reported per case: ms_per_step, rows_per_s, bytes (the sort's design bytes from benchmarks/sort_bench.py plus the window
kernels' bytes, see window_bytes) and gbps as a share of the data sheet's 3350 GB/s, metric 9 (partitions), the card's name and
power limit, and result_check: the output equals a torch recomputation (two stable torch.sorts, then diff, cummax and cumsum).
The process exits non-zero on a mismatch.
"""

from __future__ import annotations

import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from benchmarks.sort_bench import PEAK_GBPS, card, moved_bytes, plan  # noqa: E402

FUNCS3 = [("rn", "row_number"), ("rk", "rank"), ("dr", "dense_rank")]
FUNCS6 = FUNCS3 + [("pr", "percent_rank"), ("cd", "cume_dist"), ("nt", "ntile", 4)]
RUNNING = [("sr", "sum", "r", "rows"), ("mr", "max", "r", "range"), ("cz", "count", None, "partition")]
PARTITION_AGGS = [(f"{f}o", f, "o", "partition") for f in ("sum", "mean", "min", "max")]
LAG_LEAD = [("lg", "lag", "r", 1), ("ld", "lead", "o", 1, 0.0)]
MOVING = [("ma", "mean", "o", ("rows", -6, 0)), ("sc", "sum", "r", ("rows", -3, 3)), ("mx", "max", "o", ("rows", -6, 0)),
          ("n2", "nth_value", "r", 2)]
MOVING_WIDE = [("sw", "sum", "r", ("rows", -65535, 0)), ("nw", "min", "o", ("rows", -65535, 0))]
MOMENTS = [("sd20", "std", "o", ("rows", -19, 0)), ("vr", "var", "o", "rows"), ("spp", "std_pop", "o", "partition")]
MOMENT_NAMES = ("var", "std", "var_pop", "std_pop")
BIVARIATE = [("rho20", "corr", "o", "r", ("rows", -19, 0)), ("cv", "covar_samp", "o", "r", "rows"), ("beta", "regr_slope", "o", "r", "partition")]
BIVARIATE_NAMES = ("covar_samp", "covar_pop", "corr", "regr_slope", "regr_intercept")
def _ns(k):
    import numpy as np

    return np.timedelta64(k, "ns")


RANGE_MOVING = [("ra", "mean", "o", ("range_between", -_ns(1 << 35), 0)), ("rx", "max", "o", ("range_between", -_ns(1 << 35), 0)),
                ("rs", "sum", "r", ("range_between", -_ns(1 << 34), _ns(1 << 34))),
                ("rc", "count", None, ("range_between", -_ns(1 << 34), _ns(1 << 34)))]
RANGE_WIDE = [("ws", "sum", "r", ("range_between", -_ns(1 << 28), 0)), ("wn", "min", "o", ("range_between", -_ns(1 << 28), 0))]
RANGE_CASES = ("range_moving", "range_wide")
IGNORE_NULLS = [("ff", "last_value", "x", "rows", "ignore_nulls"), ("bf", "first_value", "x", ("rows", 0, None), "ignore_nulls"),
                ("lgx", "lag", "x", 1, None, "ignore_nulls")]
VALUE_CASES = ("running", "partition_aggs", "lag_lead", "moving", "moving_wide", "moments", "bivariate") + RANGE_CASES


def frame_of(f):
    """A value entry's frame: (out, fname, column[, frame]), (out, fname, y, x[, frame]) for the bivariate functions; lag and
    lead have none (their cost is counted as the "range" frame's)."""
    k = 4 if f[1] in BIVARIATE_NAMES else 3
    return f[k] if len(f) > k and f[1] not in ("lag", "lead") else "range"


def n_cols(f):
    """The 8-byte value columns a function reads: two for the bivariate functions."""
    return 2 if f[1] in BIVARIATE_NAMES else 1


def window_bytes(n, key_bytes, n_funcs, n_parts, n_peers):
    """bounds: read each key column once (the row above is the one-row halo, in cache) and write a flag byte; ends: read the flags,
    write D and the size at each partition start and the end at each peer-group start; eval: read the flags and those three
    words once per partition / peer group, write 8 bytes per function and row."""
    ends = 4 * (2 * n_parts + n_peers)
    return int(n * (key_bytes + 1) + (n + ends) + (n + ends) + 8 * n * n_funcs)


def value_bytes(n, funcs, n_parts, n_peers):
    """The value kernels after bounds / tiles / ends (every value column here is 8 bytes wide, numpy).  A scan function (sum,
    count of a column, mean, min, max, var, std, var_pop, std_pop, and the bivariate functions, which read two columns) reads its
    columns and the flags twice (reduce, then rescan) and writes its 8-byte cell, plus
    a validity byte when nullable, at each frame end (min / max also read the chosen cell there); the eval pass reads the flags
    and the partition / peer-group words once, and per function writes 8 bytes (+1 validity) per row, reading the frame end's
    cell for a scan function whose frame ends elsewhere and the source cell for first / last / lag / lead."""
    ends = {"rows": n, "range": n_peers, "partition": n_parts}
    total, evals = 0, False
    for f in funcs:
        fname, col = f[1], f[2]
        vb = 0 if fname == "count" else 1
        frame = frame_of(f)
        if fname in ("lag", "lead", "first_value", "last_value") or col is None:
            evals = True
            total += n * (8 + vb) + (n * 8 if col is not None else 0)
            continue
        total += 2 * n * (1 + 8 * n_cols(f)) + ends[frame] * (8 + vb) + (ends[frame] * 8 if fname in ("min", "max") else 0)
        if frame != "rows":
            evals = True
            total += n * (8 + vb) + ends[frame] * (8 + vb)
    if evals:
        total += n + 4 * (n_parts + n_peers)
    return int(total)


def range_bytes(n, funcs, n_parts, n_peers):
    """The bounds pass of each distinct RANGE frame with value offsets (design bytes, not measured): the flags byte, the partition
    and peer-group words (4 bytes each per partition / peer group), the 8-byte key once (the searches' probes stay near the row
    and are counted once) and the 8-byte (lo, hi) per row."""
    frames = {f[-1] for f in funcs if len(f) > 3 and isinstance(f[-1], tuple) and f[-1][0] == "range_between"}
    return int(len(frames) * (n * (1 + 8 + 8) + 4 * (n_parts + n_peers)))


def nulls_bytes(n, n_funcs, n_cols, n_valid, n_parts, n_peers):
    """The IGNORE NULLS kernels per distinct value column (8-byte numpy cells, design bytes): the count pass reads the column,
    the compaction pass reads it again and writes c (4 bytes per row) and pos (4 bytes per non-null row); the eval pass reads
    the flags and the partition / peer-group words once, and per function and row two words of c, one of pos, the chosen 8-byte
    cell and writes 8 + 1 bytes (the reads of c and pos that neighbouring rows share are counted once each)."""
    build = n * 8 + n * 8 + 4 * n + 4 * n_valid
    return int(n_cols * (build + n + 4 * (n_parts + n_peers)) + n_funcs * n * (4 + 4 + 8 + 8 + 1))


def in_frame_path(f):
    """Functions over a ("rows", start, end) frame and nth_value run in the frame kernels, not in the scans."""
    return f[1] == "nth_value" or isinstance(frame_of(f), tuple)


def frame_bytes(n, funcs, n_parts, n_peers):
    """The frame kernels (8-byte numpy value columns, as value_bytes).  An aggregate over a bounded frame: the tree build reads
    its column once and writes 4 bytes per row of nodes (16-byte nodes of the levels >= 3; 6 bytes per row of 24-byte nodes for
    var / std / var_pop / std_pop, 12 bytes per row of 48-byte nodes for the bivariate functions, which read both columns at each
    step); the query pass reads the flags and
    the partition / peer-group words, the column once more (edge leaves; the nodes and the leaves that neighbouring frames share
    are counted once) and writes 8 + 1 bytes per row.  The gather pass (count(*), first_value, last_value, nth_value) reads the
    flags and words once per launch, and per function and row the source cell and its 8 + 1 output bytes (count(*): 8).  Every
    RANGE frame with value offsets has its own gather launch, and each of its functions reads the 8-byte (lo, hi) per row."""
    words = n + 4 * (n_parts + n_peers)
    total, gather_launches = 0, set()
    for f in funcs:
        fr = f[-1] if len(f) > 3 and isinstance(f[-1], tuple) and f[-1][0] == "range_between" else None
        if fr is not None:
            total += 8 * n
        if f[1] == "nth_value" or f[2] is None or f[1] in ("first_value", "last_value"):
            gather_launches.add(fr)
            total += n * (8 if f[2] is None else 8 + 8 + 1)
        else:
            nodes = 12 if f[1] in BIVARIATE_NAMES else 6 if f[1] in MOMENT_NAMES else 4
            total += n * (8 * n_cols(f) + nodes) + words + n * (8 * n_cols(f) + 8 + 1)
    return int(total + len(gather_launches) * words)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=1 << 28)
    ap.add_argument("--batch", type=int, default=1 << 24)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--cases", type=str, default="rn_rank_dense,all6,no_partition")
    ap.add_argument("--profile", action="store_true")
    args = ap.parse_args()

    import torch

    from bodo_b200 import _lib, synth
    from bodo_b200.streaming import sort as S
    from bodo_b200.streaming import window as W
    from bodo_b200.table import ArrTypes, Column, CTypes, Table

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
    tk = None  # the range cases' DATETIME key, made on first use
    xk = None  # ignore_nulls' value column, made on first use
    torch.cuda.synchronize(dev)
    cases = {"rn_rank_dense": (["p"], FUNCS3), "all6": (["p"], FUNCS6), "no_partition": ([], FUNCS3), "running": (["p"], RUNNING),
             "partition_aggs": (["p"], PARTITION_AGGS), "lag_lead": (["p"], LAG_LEAD), "moving": (["p"], MOVING),
             "moving_wide": ([], MOVING_WIDE), "moments": (["p"], MOMENTS), "bivariate": (["p"], BIVARIATE), "range_moving": (["p"], RANGE_MOVING),
             "range_wide": ([], RANGE_WIDE), "ignore_nulls": (["p"], IGNORE_NULLS)}
    names, order = ["p", "o", "r"], "o"

    def batches():
        for r0 in range(0, n, args.batch):
            r1 = min(n, r0 + args.batch)
            cols = [Column(pk[r0:r1]), Column(ok[r0:r1]), Column(rid[r0:r1])]
            if names[3:] == ["t"]:
                cols.append(Column(tk[r0:r1], None, CTypes.DATETIME, ArrTypes.NUMPY, r1 - r0))
            elif names[3:] == ["x"]:
                cols.append(Column(xk[r0:r1]))
            yield Table(cols, names), r1 == n

    def window_step(part, funcs, keep=False):
        st = W.init_window_state(-1, part, [order], True, "last", funcs, names, output_batch_size=1 << 30, device=0, stream=sp)
        for t, last in batches():
            W.window_build_consume_batch(st, t, last)
        out, _ = W.window_produce_output_batch(st)
        res = None
        if keep:  # each column's data, and for a nullable function column its validity as one bool per row
            res = [torch.as_tensor(c.data, device=dev).clone() for c in out.columns]
            bit = torch.arange(8, device=dev, dtype=torch.uint8)
            res += [None if c.validity is None else
                    ((torch.as_tensor(c.validity, device=dev).unsqueeze(1) >> bit) & 1).flatten()[:n].bool() for c in out.columns[len(names):]]
        m9 = W.get_metric(st, 9)
        W.delete_window_state(st)
        return res, m9

    def sort_step(part):
        st = S.init_stream_sort_state(-1, None, 0, part + [order], [True] * (len(part) + 1), ["last"] * (len(part) + 1), names,
                                      output_batch_size=1 << 30, device=0, stream=sp, full=True)
        for t, last in batches():
            S.sort_build_consume_batch(st, t, last)
        S.produce_output_batch(st)
        m = [S.get_metric(st, w) for w in range(9)]
        S.delete_stream_sort_state(st)
        return m

    def timed(fn):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(stream)
        r = fn()
        e1.record(stream)
        torch.cuda.synchronize(dev)
        return e0.elapsed_time(e1), r

    def check(part, funcs, res):
        """res: the window's output columns (p, o, r, then one per function).  Expected columns are built one at a time, so the
        recomputation fits next to the inputs and the output on an 80 GB card."""
        idx = torch.sort(ok, stable=True).indices
        if part:
            idx = idx[torch.sort(pk[idx], stable=True).indices]
        if not (torch.equal(res[2], idx) and torch.equal(res[0], pk[idx]) and torch.equal(res[1].view(torch.int64), ok[idx].view(torch.int64))):
            return "MISMATCH: an input column differs from the stable sort", 0, 0
        i = torch.arange(n, device=dev, dtype=torch.int64)
        ps = torch.zeros(n, dtype=torch.bool, device=dev)
        ps[0] = True
        if part:
            ps[1:] = torch.diff(pk[idx]) != 0
        qs = ps.clone()
        qs[1:] |= torch.diff(ok[idx]) != 0
        del idx
        P = torch.cummax(torch.where(ps, i, 0), 0).values
        Q = torch.cummax(torch.where(qs, i, 0), 0).values
        D = torch.cumsum(qs.to(torch.int64), 0)
        pid = torch.cumsum(ps.to(torch.int64), 0) - 1
        s = torch.bincount(pid)[pid]
        del pid
        qid = torch.cumsum(qs.to(torch.int64), 0) - 1
        qend = torch.cat([torch.nonzero(qs).flatten()[1:], torch.tensor([n], device=dev)])[qid]
        del qid

        def expected(f):
            if f == "rn":
                return i - P + 1
            if f == "rk":
                return Q - P + 1
            if f == "dr":
                return D - D[P] + 1
            if f == "pr":
                return torch.where(s == 1, 0.0, (Q - P).to(torch.float64) / torch.clamp(s - 1, min=1).to(torch.float64))
            if f == "cd":
                return (qend - P).to(torch.float64) / s.to(torch.float64)
            pos = i - P
            q, r = s // 4, s % 4
            big = r * (q + 1)
            return torch.where(pos < big, pos // (q + 1) + 1, r + (pos - big) // torch.clamp(q, min=1) + 1)

        sr, so, nf = res[2], res[1], len(funcs)
        pid = torch.cumsum(ps.to(torch.int64), 0) - 1
        n_p = int(pid[-1]) + 1

        def value_ok(j, f):
            """The value cases: integer results exactly; partition sums and means of o (>= 0) within 4 (m + 1) u of the exact value
            for a partition of m rows, which covers the device's and torch's summation orders."""
            got, valid = res[3 + j], res[3 + nf + j]
            if f[1] == "count":
                return torch.equal(got, s)
            if f[1] == "lag":
                return torch.equal(valid, ~ps) and torch.equal(torch.where(ps, 0, got), torch.where(ps, 0, torch.roll(sr, 1)))
            if f[1] == "lead":
                last = torch.roll(ps, -1)
                last[-1] = True
                return bool(valid.all()) and torch.equal(got.view(torch.int64), torch.where(last, 0.0, torch.roll(so, -1)).view(torch.int64))
            if not bool(valid.all()):
                return False
            if f[2] == "r" and f[1] == "sum":  # ROWS frame: a segmented cumsum through the offsets at P
                cs = torch.cumsum(sr, 0)
                return torch.equal(got, cs - torch.where(P > 0, cs[(P - 1).clamp(min=0)], 0))
            if f[2] == "r":  # MAX over RANGE: the running max at the peer group's last row
                return torch.equal(got, (torch.cummax((pid << 32) | sr, 0).values & 0xFFFFFFFF)[qend - 1])
            if f[1] in ("min", "max"):
                init = torch.full((n_p,), float("inf") if f[1] == "min" else float("-inf"), dtype=torch.float64, device=dev)
                red = init.scatter_reduce(0, pid, so, "amin" if f[1] == "min" else "amax", include_self=False)
                return torch.equal(got.view(torch.int64), red[pid].view(torch.int64))
            tot = torch.zeros(n_p, dtype=torch.float64, device=dev).index_add_(0, pid, so)[pid]
            exp = tot if f[1] == "sum" else tot / s.to(torch.float64)
            return bool(((got - exp).abs() <= 4 * (s + 1).to(torch.float64) * 2.0 ** -53 * exp.abs()).all())

        def frame_ok(j, f):
            """Bounded frames and nth_value: sums of r as cumsum differences over [lo, hi] (exact); min / max of o over the
            trailing frame [max(P, i - w + 1), i] from maxima / minima of 2^k rows doubled within the partition (bit for bit);
            means of o (>= 0) from w shifted terms, within 4 (w + 1) u; nth_value(r, n) over "range" as the cell at P + n - 1
            when that row is at most the row's last peer, else NA."""
            got, valid = res[3 + j], res[3 + nf + j]
            pe = P + s
            if f[1] == "nth_value":
                src = P + f[3] - 1
                inside = src <= qend - 1
                return torch.equal(valid, inside) and torch.equal(torch.where(inside, got, 0), torch.where(inside, sr[src.clamp(max=n - 1)], 0))
            _, a, b = f[3]
            if not bool(valid.all()):  # every frame here holds its own row
                return False
            lo, hi = torch.maximum(P, i + a), torch.minimum(pe - 1, i + b)
            if f[1] == "sum":
                cs = torch.cat([torch.zeros(1, dtype=torch.int64, device=dev), torch.cumsum(sr, 0)])
                return torch.equal(got, cs[hi + 1] - cs[lo])
            w = 1 - a  # trailing frames (b == 0) of w rows
            if f[1] == "mean":
                tot = torch.zeros(n, dtype=torch.float64, device=dev)
                for k in range(w):
                    tot += torch.where(i - k >= P, torch.roll(so, k), 0.0)
                exp = tot / (i - lo + 1).to(torch.float64)
                return bool(((got - exp).abs() <= 4 * (w + 1) * 2.0 ** -53 * exp).all())
            op, ident = (torch.maximum, float("-inf")) if f[1] == "max" else (torch.minimum, float("inf"))
            m, K = so.clone(), 0  # m[i]: op over [i - 2^K + 1, i] within the row's partition
            while (2 << K) <= w:
                m = op(m, torch.where(i - (1 << K) >= P, torch.roll(m, 1 << K), ident))
                K += 1
            j2 = i - w + (1 << K)
            exp = op(m, torch.where(j2 >= P, m[j2.clamp(min=0)], ident))
            return torch.equal(got.view(torch.int64), exp.view(torch.int64))

        def moment_ok(j, f):
            """var / std of o against torch float64 two-pass computations (the frame's mean, then the sum of squared deviations
            from it): the partition's std_pop through index_add; the trailing 20-row frame's over its 20 shifted terms; the
            running var over a (partition, position) matrix, one prefix length at a time.  Each within DESIGN §3c's bound for
            the device plus 8 m u (M2 + |mean| sqrt(m M2)) for the recomputation's own rounding; validity exactly."""
            got, valid = res[3 + j], res[3 + nf + j]
            u = 2.0 ** -53
            if f[3] == "partition":
                cnt = s.to(torch.float64)
                mu = torch.zeros(n_p, dtype=torch.float64, device=dev).index_add_(0, pid, so)[pid] / cnt
                M2 = torch.zeros(n_p, dtype=torch.float64, device=dev).index_add_(0, pid, (so - mu) ** 2)[pid]
                h = cnt - 1
            elif f[3] == "rows":
                pos = i - P
                L = int(s.max())
                X = torch.zeros(n_p, L, dtype=torch.float64, device=dev)
                X[pid, pos] = so
                means = torch.cumsum(X, 1) / torch.arange(1, L + 1, device=dev, dtype=torch.float64)
                M2s = torch.empty(n_p, L, dtype=torch.float64, device=dev)
                for k in range(L):  # prefix k + 1 of every partition (longer than the partition: unused)
                    M2s[:, k] = ((X[:, :k + 1] - means[:, k:k + 1]) ** 2).sum(1)
                mu, M2 = means[pid, pos], M2s[pid, pos]
                cnt = (pos + 1).to(torch.float64)
                h = cnt - 1
                del X, means, M2s, pos
            else:
                w = -f[3][1] + 1
                lo = torch.maximum(P, i - w + 1)
                cnt = (i - lo + 1).to(torch.float64)
                tot = torch.zeros(n, dtype=torch.float64, device=dev)
                for k in range(w):
                    tot += torch.where(i - k >= P, torch.roll(so, k), 0.0)
                mu = tot / cnt
                M2 = torch.zeros(n, dtype=torch.float64, device=dev)
                for k in range(w):
                    M2 += torch.where(i - k >= P, (torch.roll(so, k) - mu) ** 2, 0.0)
                h = torch.minimum(cnt - 1, 10 + 3 * torch.floor(torch.log2(cnt)))
                del tot, lo
            pop = f[1] in ("var_pop", "std_pop")
            if not torch.equal(valid, cnt >= (1 if pop else 2)):
                return False
            gam = lambda k: k * u / (1 - k * u)  # noqa: E731
            spread = mu.abs() * torch.sqrt(cnt * M2)
            tol = torch.sqrt(h) * (gam(21 * h) * M2 + gam(8 * h) * spread) + 8 * cnt * u * (M2 + spread)
            div = (cnt - (0 if pop else 1)).clamp(min=1)
            var, tv = M2 / div, tol / div
            tv = tv + 2 * u * var
            exp, t = var, tv
            if f[1] in ("std", "std_pop"):
                exp = torch.sqrt(var)
                t = torch.minimum(torch.sqrt(tv), tv / exp.clamp(min=1e-300)) + 2 * u * exp
            return bool(((got - exp).abs() <= t)[valid].all())

        def frame_sums(f, x, y):
            """Per row over f's frame (the partition, the running prefix or a trailing frame): (count, Sxx, Syy, Sxy, the means of
            x and y), two-pass in torch float64, and h, the merge height of §3c's bound."""
            fr = frame_of(f)
            z = lambda: torch.zeros(n_p, dtype=torch.float64, device=dev)  # noqa: E731
            if fr == "partition":
                cnt = s.to(torch.float64)
                mx, my = z().index_add_(0, pid, x)[pid] / cnt, z().index_add_(0, pid, y)[pid] / cnt
                dx, dy = x - mx, y - my
                sums = [z().index_add_(0, pid, a * b)[pid] for a, b in ((dx, dx), (dy, dy), (dx, dy))]
                return cnt, *sums, mx, my, cnt - 1
            if fr == "rows":  # a (partition, position) matrix; per prefix length k + 1, the rows at position k
                pos = i - P
                L = int(s.max())
                X, Y = torch.zeros(n_p, L, dtype=torch.float64, device=dev), torch.zeros(n_p, L, dtype=torch.float64, device=dev)
                X[pid, pos], Y[pid, pos] = x, y
                ar = torch.arange(1, L + 1, device=dev, dtype=torch.float64)
                mxs, mys = torch.cumsum(X, 1) / ar, torch.cumsum(Y, 1) / ar
                by_pos = torch.argsort(pos)
                ends_k = torch.cumsum(torch.bincount(pos, minlength=L), 0).tolist()
                sums = [torch.empty(n, dtype=torch.float64, device=dev) for _ in range(3)]
                for k in range(L):
                    rows = by_pos[(ends_k[k - 1] if k else 0):ends_k[k]]
                    pr = pid[rows]
                    dx, dy = X[pr, :k + 1] - mxs[pr, k:k + 1], Y[pr, :k + 1] - mys[pr, k:k + 1]
                    for out_, a, b in zip(sums, (dx, dy, dx), (dx, dy, dy)):
                        out_[rows] = (a * b).sum(1)
                cnt = (pos + 1).to(torch.float64)
                mx, my = mxs[pid, pos], mys[pid, pos]
                del X, Y, mxs, mys, by_pos, pos
                return cnt, *sums, mx, my, cnt - 1
            w = -fr[1] + 1
            cnt = (i - torch.maximum(P, i - w + 1) + 1).to(torch.float64)
            sx, sy = torch.zeros(n, dtype=torch.float64, device=dev), torch.zeros(n, dtype=torch.float64, device=dev)
            for k in range(w):
                inside = i - k >= P
                sx += torch.where(inside, torch.roll(x, k), 0.0)
                sy += torch.where(inside, torch.roll(y, k), 0.0)
            mx, my = sx / cnt, sy / cnt
            del sx, sy
            sums = [torch.zeros(n, dtype=torch.float64, device=dev) for _ in range(3)]
            for k in range(w):
                inside = i - k >= P
                dx, dy = torch.where(inside, torch.roll(x, k) - mx, 0.0), torch.where(inside, torch.roll(y, k) - my, 0.0)
                for out_, a, b in zip(sums, (dx, dy, dx), (dx, dy, dy)):
                    out_ += a * b
            return cnt, *sums, mx, my, torch.minimum(cnt - 1, 10 + 3 * torch.floor(torch.log2(cnt)))

        def bivariate_ok(j, f):
            """covar_samp / corr / regr_slope(y, x) against torch float64 two-pass co-moments (as moment_ok): each of Sxx, Syy
            and Sxy within DESIGN §3c's bound for the device plus 8 m u times the same terms for the recomputation's own rounding,
            then corr and slope within what those bounds give them (first order, doubled); validity exactly."""
            got, valid = res[3 + j], res[3 + nf + j]
            u = 2.0 ** -53
            y, x = (so if c == "o" else sr.to(torch.float64) for c in (f[2], f[3]))
            cnt, sxx, syy, sxy, mx, my, h = frame_sums(f, x, y)
            gam = lambda k: k * u / (1 - k * u)  # noqa: E731
            sq = lambda v: torch.sqrt(v.clamp(min=0))  # noqa: E731

            def tol(a, b, ma, mb):  # |S_ab - S_ab*| (§3c), with a = b giving S_aa's
                t = sq(a * b) + ma.abs() * sq(cnt * b) + mb.abs() * sq(cnt * a)
                return torch.sqrt(h) * (gam(21 * h) * sq(a * b) + gam(8 * h) * (t - sq(a * b))) + 8 * cnt * u * t

            exy, exx, eyy = tol(sxx, syy, mx, my), tol(sxx, sxx, mx, mx), tol(syy, syy, my, my)
            if f[1] == "covar_samp":
                want, div = cnt >= 2, (cnt - 1).clamp(min=1)
                exp, t = sxy / div, exy / div + 2 * u * (sxy / div).abs()
            elif f[1] == "corr":
                want = (cnt >= 2) & (sxx > 0) & (syy > 0)
                d = sq(sxx * syy).clamp(min=1e-300)
                exp = (sxy / d).clamp(-1, 1)
                t = 2 * (exy / d + exp.abs() * 0.5 * (exx / sxx.clamp(min=1e-300) + eyy / syy.clamp(min=1e-300))) + 4 * u
            else:
                want = sxx > 0
                sl = sxy / sxx.clamp(min=1e-300)
                exp, t = sl, 2 * (exy + sl.abs() * exx) / (sxx - exx).clamp(min=1e-300) + 2 * u * sl.abs()
            if not torch.equal(valid, want):
                return False
            return bool(((got - exp).abs() <= t)[valid].all())

        for j, f in enumerate(funcs):
            if f[1] in BIVARIATE_NAMES:
                if not bivariate_ok(j, f):
                    return f"MISMATCH: {f[0]}", 0, 0
                continue
            if f[1] in MOMENT_NAMES:
                if not moment_ok(j, f):
                    return f"MISMATCH: {f[0]}", 0, 0
                continue
            good = frame_ok(j, f) if in_frame_path(f) else value_ok(j, f) if f[1] in W.VALUE_FUNCS else torch.equal(res[3 + j].view(torch.int64), expected(f[0]).view(torch.int64))
            if not good:
                return f"MISMATCH: {f[0]}", 0, 0
        return "ok", int(ps.sum()), int(qs.sum())

    def range_check(part, funcs, res):
        """The range cases: every row's [lo, hi] from torch.searchsorted over the exact composite (p << 40) | t of the sorted
        rows (CURRENT ROW ends at the row's last peer); sums of r as int64 cumsum differences and COUNT(*) as hi - lo + 1, bit
        for bit; AVG(o) (o >= 0) from the frame's shifted terms within 4 (m + 1) u; MIN / MAX(o) from minima / maxima of 2^k
        rows doubled, bit for bit."""
        idx = torch.sort(tk, stable=True).indices
        if part:
            idx = idx[torch.sort(pk[idx], stable=True).indices]
        if not (torch.equal(res[2], idx) and torch.equal(res[3], tk[idx])):
            return "MISMATCH: an input column differs from the stable sort", 0, 0
        del idx
        sp_ = res[0] if part else torch.zeros(n, dtype=torch.int64, device=dev)
        so, sr, st_k = res[1], res[2], res[3]
        comp = (sp_ << 40) | st_k
        base = sp_ << 40
        ps = torch.ones(n, dtype=torch.bool, device=dev)
        ps[1:] = torch.diff(sp_) != 0
        qs = ps.clone()
        qs[1:] |= torch.diff(st_k) != 0
        n_parts, n_peers = int(ps.sum()), int(qs.sum())
        del ps, qs
        i = torch.arange(n, device=dev, dtype=torch.int64)
        nf = len(funcs)
        for j, f in enumerate(funcs):
            got, valid = res[4 + j], res[4 + nf + j]
            a, b = (int(x) for x in f[3][1:])  # ns
            lo = torch.searchsorted(comp, base + (st_k + a).clamp(min=0))
            hi = torch.searchsorted(comp, comp if b == 0 else base + (st_k + b).clamp(max=(1 << 40) - 1), right=True) - 1
            if valid is not None and not bool(valid.all()):  # every frame here holds its own row
                return f"MISMATCH: {f[0]} validity", 0, 0
            if f[1] == "count":
                good = torch.equal(got, hi - lo + 1)
            elif f[1] == "sum":
                cs = torch.cat([torch.zeros(1, dtype=torch.int64, device=dev), torch.cumsum(sr, 0)])
                good = torch.equal(got, cs[hi + 1] - cs[lo])
                del cs
            elif f[1] == "mean":
                cnt = hi - lo + 1
                tot = torch.zeros(n, dtype=torch.float64, device=dev)
                for k in range(int(cnt.max())):
                    tot += torch.where(lo + k <= hi, so[(lo + k).clamp(max=n - 1)], 0.0)
                exp = tot / cnt.to(torch.float64)
                good = bool(((got - exp).abs() <= 4 * (cnt + 1).to(torch.float64) * 2.0 ** -53 * exp).all())
                del tot, exp, cnt
            else:
                op = torch.maximum if f[1] == "max" else torch.minimum
                w = hi - lo + 1
                K = torch.frexp(w.to(torch.float64))[1].to(torch.int64) - 1
                m, exp, k = so.clone(), torch.empty_like(so), 0
                while True:  # m[x] = op over [x, x + 2^k) (clipped at n)
                    s_ = K == k
                    if bool(s_.any()):
                        exp[s_] = op(m[lo[s_]], m[hi[s_] - (1 << k) + 1])
                    if (2 << k) > int(w.max()):
                        break
                    m = op(m, torch.cat([m[1 << k:], m[-(1 << k):]]))
                    k += 1
                good = torch.equal(got.view(torch.int64), exp.view(torch.int64))
                del m, exp, K, w
            del lo, hi
            if not good:
                return f"MISMATCH: {f[0]}", 0, 0
        return "ok", n_parts, n_peers

    def nulls_check(part, funcs, res):
        """ignore_nulls: the sorted columns against two stable torch.sorts, then per row the last non-null row at or before it
        (a cummax of the non-null positions), the first at or after it (a reversed cummin) and the last before it, each valid when
        it lies in the row's partition; the chosen cells bit for bit."""
        idx = torch.sort(ok, stable=True).indices
        idx = idx[torch.sort(pk[idx], stable=True).indices]
        if not (torch.equal(res[2], idx) and torch.equal(res[3].view(torch.int64), xk[idx].view(torch.int64))):
            return "MISMATCH: an input column differs from the stable sort", 0, 0
        del idx
        sp_, sx = res[0], res[3]
        i = torch.arange(n, device=dev, dtype=torch.int64)
        ps = torch.ones(n, dtype=torch.bool, device=dev)
        ps[1:] = torch.diff(sp_) != 0
        qs = ps.clone()
        qs[1:] |= torch.diff(res[1]) != 0
        P = torch.cummax(torch.where(ps, i, 0), 0).values
        last = torch.roll(ps, -1)
        last[-1] = True
        pe = torch.flip(torch.cummin(torch.flip(torch.where(last, i + 1, n), [0]), 0).values, [0])
        nn = ~torch.isnan(sx)
        prev = torch.cummax(torch.where(nn, i, -1), 0).values
        nxt = torch.flip(torch.cummin(torch.flip(torch.where(nn, i, n), [0]), 0).values, [0])
        before = torch.cat([torch.full((1,), -1, dtype=torch.int64, device=dev), prev[:-1]])
        nf = len(funcs)
        for j, (src, good) in enumerate(((prev, prev >= P), (nxt, nxt < pe), (before, before >= P))):
            got, valid = res[4 + j], res[4 + nf + j]
            exp = sx[src.clamp(0, n - 1)].view(torch.int64)
            if not (torch.equal(valid, good) and torch.equal(torch.where(good, got.view(torch.int64), 0), torch.where(good, exp, 0))):
                return f"MISMATCH: {funcs[j][0]}", 0, 0
        return "ok", int(ps.sum()), int(qs.sum())

    def free():
        torch.cuda.empty_cache()
        _lib.lib().b200_pool_trim(0, 0)

    def profile_case(name, part, funcs):
        """One warm-up step, then one step under torch.profiler: the window kernels' device times (no timing, no check)."""
        from torch.profiler import ProfilerActivity, profile

        window_step(part, funcs)
        torch.cuda.synchronize(dev)
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            window_step(part, funcs)
            torch.cuda.synchronize(dev)
        kern = {}
        for ev in prof.events():
            if str(ev.device_type).endswith("CUDA") and ("window_" in ev.name or "tile_carry_kernel" in ev.name):
                key = ev.name.split("(")[0].replace("void b200::", "")
                kern[key] = kern.get(key, 0.0) + getattr(ev, "device_time", getattr(ev, "cuda_time", 0.0)) / 1e3
        print(json.dumps({"case": name, "profile_kernel_ms": {k: round(v, 3) for k, v in sorted(kern.items())}, "card": card()}), flush=True)
        free()

    ok_all = True
    for name in args.cases.split(","):
        part, funcs = cases[name]
        if name in RANGE_CASES:
            if tk is None:
                tk = torch.randint(0, 1 << 40, (n,), generator=g, device=dev, dtype=torch.int64)
            names, order = ["p", "o", "r", "t"], "t"
        elif name == "ignore_nulls":
            if xk is None:  # NaN where a multiplicative hash of the row id falls in the lowest 30 % of [0, 2^10)
                xk = torch.randn(n, generator=g, device=dev, dtype=torch.float64)
                h = ((rid * -7046029254386353131) >> 54) & 1023
                xk[h < 307] = float("nan")
                del h
            names, order = ["p", "o", "r", "x"], "o"
        else:
            names, order = ["p", "o", "r"], "o"
        if args.profile:
            profile_case(name, part, funcs)
            continue
        window_step(part, funcs)  # warm-up
        sort_step(part)
        value_case = name in VALUE_CASES
        if value_case:
            window_step(part, FUNCS3)
        if name == "bivariate":
            window_step(part, MOMENTS)
        if name == "ignore_nulls":
            window_step(part, LAG_LEAD)
        wt, st_, rt, mt, lt = [], [], [], [], []
        for _ in range(args.reps):
            ms, (_, m9) = timed(lambda: window_step(part, funcs))
            wt.append(ms)
            ms, sm = timed(lambda: sort_step(part))
            st_.append(ms)
            if value_case:  # the value kernels' cost next to the ranking kernels', in the same process
                rt.append(timed(lambda: window_step(part, FUNCS3))[0])
            if name == "bivariate":  # next to the moments, whose scan value is half as wide
                mt.append(timed(lambda: window_step(part, MOMENTS))[0])
            if name == "ignore_nulls":  # next to RESPECT NULLS navigation over the same four columns
                lt.append(timed(lambda: window_step(part, LAG_LEAD))[0])
        w_ms, s_ms = sorted(wt)[len(wt) // 2], sorted(st_)[len(st_) // 2]
        free()
        # check
        res, _ = window_step(part, funcs, keep=True)
        free()
        chk, n_parts, n_peers = (range_check if name in RANGE_CASES else nulls_check if name == "ignore_nulls" else check)(part, funcs, res)
        if chk == "ok" and m9 != n_parts:
            chk = f"MISMATCH: metric 9 = {m9}, partitions = {n_parts}"
        del res
        free()
        # design bytes: the sort of the keys (passes from the data, as sort_bench predicts them), then the window kernels
        f64w = lambda x: torch.where(x < 0, x.view(torch.int64) ^ 0x7FFFFFFFFFFFFFFF, x.view(torch.int64))  # noqa: E731
        words = [tk ^ (-(2 ** 63)) if name in RANGE_CASES else f64w(ok)] + ([pk ^ (-(2 ** 63))] if part else [])
        n_valid = int((~torch.isnan(xk)).sum()) if name == "ignore_nulls" else 0
        kp = plan(torch, words, [8] * len(words), [True] + [False] * len(part), [0] * len(words))
        del words
        free()
        key_bytes = 8 * (1 + len(part))
        sort_bytes = moved_bytes(n, 8 * len(names), 0, key_bytes, kp)
        if value_case:  # bounds and ends as the ranking cases (no ranking eval pass), then the value kernels
            ends4 = 4 * (2 * n_parts + n_peers)
            scans = [f for f in funcs if not in_frame_path(f)]
            total = (sort_bytes + window_bytes(n, key_bytes, 0, n_parts, n_peers) - (n + ends4) + value_bytes(n, scans, n_parts, n_peers)
                     + frame_bytes(n, [f for f in funcs if in_frame_path(f)], n_parts, n_peers) + range_bytes(n, funcs, n_parts, n_peers))
        elif name == "ignore_nulls":  # bounds and ends as the ranking cases, then one (c, pos) build and one eval pass
            total = (sort_bytes + window_bytes(n, key_bytes, 0, n_parts, n_peers) - (n + 4 * (2 * n_parts + n_peers))
                     + nulls_bytes(n, len(funcs), 1, n_valid, n_parts, n_peers))
        else:
            total = sort_bytes + window_bytes(n, key_bytes, len(funcs), n_parts, n_peers)
        out = {"case": name, "rows": n, "batch": args.batch, "funcs": [f[1] for f in funcs], "ms_per_step": round(w_ms, 3),
               "runs_ms": [round(x, 3) for x in wt], "sort_ms": round(s_ms, 3), "sort_runs_ms": [round(x, 3) for x in st_],
               "extra_ms": round(w_ms - s_ms, 3), "extra_share_of_sort": round((w_ms - s_ms) / s_ms, 4),
               "rows_per_s": round(n / (w_ms * 1e-3), 1), "bytes": total, "gbps": round(total / (w_ms * 1e-3) / 1e9, 1),
               "share_of_3350_gbps": round(total / (w_ms * 1e-3) / 1e9 / PEAK_GBPS, 4), "metric9_partitions": m9,
               "sort_passes_run_skipped": sm[7:9], "result_check": chk, "card": card()}
        if value_case:
            r_ms = sorted(rt)[len(rt) // 2]
            out.update(rn_rank_dense_ms=round(r_ms, 3), rn_rank_dense_runs_ms=[round(x, 3) for x in rt], extra_over_rn_rank_dense_ms=round(w_ms - r_ms, 3))
        if lt:
            l_ms = sorted(lt)[len(lt) // 2]
            out.update(lag_lead_ms=round(l_ms, 3), lag_lead_runs_ms=[round(x, 3) for x in lt], extra_over_lag_lead_ms=round(w_ms - l_ms, 3))
        if mt:
            m_ms = sorted(mt)[len(mt) // 2]
            out.update(moments_ms=round(m_ms, 3), moments_runs_ms=[round(x, 3) for x in mt], extra_over_moments_ms=round(w_ms - m_ms, 3))
        print(json.dumps(out), flush=True)
        print(f"result_check: {chk}", flush=True)
        ok_all &= chk == "ok"
    if not ok_all:
        sys.exit(3)


if __name__ == "__main__":
    main()
