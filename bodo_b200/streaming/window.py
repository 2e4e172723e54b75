"""Streaming window operator: ranking, aggregate and navigation functions OVER (PARTITION BY p ... ORDER BY o ...).

    ROW_NUMBER() / RANK() / DENSE_RANK() / PERCENT_RANK() / CUME_DIST() / NTILE(n) OVER (PARTITION BY p ORDER BY o)
    SUM / COUNT / AVG / MIN / MAX / FIRST_VALUE / LAST_VALUE (x) OVER (PARTITION BY p ORDER BY o [frame])
    LAG / LEAD (x, k, default) OVER (PARTITION BY p ORDER BY o)
    NTH_VALUE (x, n) OVER (PARTITION BY p ORDER BY o [frame]), and every frame function over ROWS BETWEEN k PRECEDING AND k FOLLOWING
    VAR_SAMP / STDDEV_SAMP / VAR_POP / STDDEV_POP (x) OVER (PARTITION BY p ORDER BY o [frame])
    every frame function over RANGE BETWEEN x PRECEDING AND y FOLLOWING, an offset measured in the ORDER BY value
    COVAR_SAMP / COVAR_POP / CORR / REGR_SLOPE / REGR_INTERCEPT (y, x) OVER (PARTITION BY p ORDER BY o [frame])
    FIRST_VALUE / LAST_VALUE / NTH_VALUE / LAG / LEAD with IGNORE NULLS (a trailing "ignore_nulls" in the entry)

pandas equivalents: groupby(p).cumcount() + 1, groupby(p)[o].rank(method="min" / "dense" / "max", pct=...),
groupby(p)[x].cumsum() / cummin() / cummax() (the "rows" frame), groupby(p)[x].transform("sum" / "mean" / "min" / "max" /
"count" / "size" / "first" / "last" / "var" / "std") (the "partition" frame), groupby(p)[x].expanding().var() / .std() (the
"rows" frame), groupby(p)[x].rolling(w).var() / .std() (a bounded frame), groupby(p).rolling("1h", on=t) (a RANGE frame),
groupby(p)[y].rolling(w).cov(x) / .corr(x) (a bounded frame), groupby(p)[x].shift(k, fill_value=default) (lag;
lead is shift(-k)) and, ordered by a row id, groupby(p)[x].ffill() / ffill(limit=n) / bfill() / bfill(limit=n) (last_value
IGNORE NULLS over "rows" / ("rows", -n, 0), first_value IGNORE NULLS over ("rows", 0, None) / ("rows", 0, n)).  The state is a third form of the streaming sort (streaming/sort.py's SortState, sort.cu's WindowState): batches are
appended to the full sort's device chunk store, is_last sorts every row by (partition keys ascending NA last, order keys, arrival
index), scans the sorted key columns on the device for partition and peer-group boundaries and then scans or gathers the value
columns.

Semantics:
  - keys: 0..4 PARTITION BY columns and 0..4 ORDER BY columns, 1..4 in all, distinct, of the sort's key types (fixed-width
    numeric, bool and temporal, numpy or nullable).  ascending / na_position apply to the ORDER BY keys (one value or one per key).
  - two cells of a key are equal when both are NA (a float NaN is NA) or both are valid and equal, with -0.0 equal to 0.0: NaN and
    NA are one partition and are peers, as in groupby(..., dropna=False).  Without ORDER BY every row of a partition is a peer of
    every other; without PARTITION BY the whole input is one partition.
  - with s the partition size and k the row's 0-based position in it: row_number = k + 1 (ties in arrival order), rank = 1 + rows
    before the row's first peer, dense_rank = 1 + peer groups before the row's, percent_rank = (rank - 1) / (s - 1) (0.0 when
    s = 1), cume_dist = rows up to and including the row's last peer / s, ntile(n) = the SQL bucket (the first s % n buckets hold
    s // n + 1 rows, the others s // n; buckets 1..s when n > s).
  - row_number, rank, dense_rank and ntile are int64 columns, percent_rank and cume_dist float64 (one IEEE double division of two
    integers, so bit-identical to numpy's).
  - value functions read one input column (any column, keys included); covar_samp, covar_pop, corr, regr_slope and
    regr_intercept read two, (y, x), which may be the same column.  Frames start at the row's partition's first row P and
    end at e: "range" (the default; SQL's default frame RANGE BETWEEN UNBOUNDED PRECEDING AND CURRENT ROW) at the row's last peer,
    which is the partition's last row without ORDER BY; "rows" (ROWS BETWEEN UNBOUNDED PRECEDING AND CURRENT ROW) at the row
    itself, ties in arrival order; "partition" (ROWS BETWEEN UNBOUNDED PRECEDING AND UNBOUNDED FOLLOWING) at the partition's last
    row.  ("rows", start, end) is ROWS BETWEEN start AND end, each None (UNBOUNDED) or an integer row offset in (-2^31, 2^31)
    (negative PRECEDING, 0 CURRENT ROW, positive FOLLOWING; start <= end when both are offsets): for row i of the partition
    [P, pe) the frame is [lo, hi] with lo = P (start None) or max(P, i + start), hi = pe - 1 (end None) or min(pe - 1, i + end),
    empty when lo > hi.  ("rows", None, 0) is "rows" and ("rows", None, None) is "partition".  It takes sum, count, mean, min,
    max, first_value, last_value, nth_value, var, std, var_pop and std_pop, which are then defined as below with [lo, hi] in
    place of [P, e], as are the five functions of two columns below; an empty frame gives NA (count 0).  ("range_between", start, end) is RANGE BETWEEN start AND end with the
    same spelling: None is UNBOUNDED, zero CURRENT ROW (the row's peer group: from its first peer / to its last peer; any ORDER
    BY), a negative offset PRECEDING and a positive one FOLLOWING, measured in the single ORDER BY key x.  With x ascending a
    k PRECEDING start is the first row of the partition's non-NA run with x_j >= x_i - k and a k FOLLOWING end the last row
    with x_j <= x_i + k (a PRECEDING end and a FOLLOWING start mirror these); descending swaps the signs.  Integer and temporal
    keys compare exactly (no wrap), float keys against fl(x_i -+ k) in double.  An integer key takes an integer offset, a float
    key an int or float, DATETIME / TIMEDELTA a numpy.timedelta64, datetime.timedelta or pandas.Timedelta, DATE a timedelta of
    whole days.  A dictionary-encoded string key arrives as its INT32 ids, which the window cannot tell from integers: an
    offset over it measures distances between ids, so range offsets are meant for numeric and temporal keys only.  At an NA
    row an offset bound is the NA peer group's boundary; at a non-NA row it never reaches an NA row, and
    one that no row satisfies leaves the frame empty.  It takes the functions ("rows", start, end) takes;
    ("range_between", None, 0) is "range" and ("range_between", None, None) is "partition".  Over [P, e], with a float NaN counted as NA:
      count(x): non-NA cells, count(None): COUNT(*) = e - P + 1; int64 numpy.
      sum(x): the sum of the non-NA cells, NA when there are none; integers and bool wrap in 64 bits (int64 for signed and bool,
        uint64 for unsigned), floats accumulate in double (float32 narrowed once at the end); nullable.
      mean(x): sum / count in double ((double) of the exact 64-bit sum for integers and bool), NA when count = 0; float64,
        nullable.  sum and mean of a temporal column raise.
      min(x) / max(x): the cell of the earliest row holding the least / greatest non-NA value, compared in the sort's key order
        (so every key type works; -0.0 ties 0.0 and the earlier row's bits are returned); NA when no cell is valid; x's type,
        nullable.
      first_value(x) / last_value(x): the cell at P / e as it is, bits and validity (a NaN stays a valid NaN, SQL RESPECT NULLS);
        x's type, nullable.
      nth_value(x, n): the cell at P + n - 1 as first_value gives it when that row is in the frame, else NA; 1 <= n < 2^31;
        frame "range" by default; x's type, nullable.
      var(x) / std(x) / var_pop(x) / std_pop(x): with m the non-NA cells (integers and bool converted to double, exact up to
        2^53) and M2 = sum (x - mean)^2 over them: var = M2 / (m - 1), NA when m < 2 (SQL VAR_SAMP, pandas ddof=1); var_pop =
        M2 / m, NA when m = 0 and 0.0 when m = 1 (VAR_POP, ddof=0); std / std_pop their IEEE sqrt.  M2 is combined from (count,
        mean, M2) by Chan's pairwise merge, with no sum of squares, so it keeps its digits when |mean| >> the spread (DESIGN
        §3c gives the bound); it is never negative and is exactly 0.0 over equal values.  A frame holding +-inf gives a valid
        NaN, as pandas does.  float64, nullable; a temporal column raises.
      covar_samp(y, x) / covar_pop(y, x) / corr(y, x) / regr_slope(y, x) / regr_intercept(y, x), written (out_name, fname,
        y, x[, frame]) in SQL's argument order: over the m rows where both cells are non-NA (pairwise deletion, as SQL and
        pandas; integers and bool converted to double, exact up to 2^53), with means mx, my and Sxx = sum (x - mx)^2, Syy =
        sum (y - my)^2, Sxy = sum (x - mx)(y - my): covar_samp = Sxy / (m - 1), NA when m < 2; covar_pop = Sxy / m, NA when
        m = 0; corr = Sxy / sqrt(Sxx Syy), clamped to [-1, 1], NA when m < 2, Sxx = 0 or Syy = 0 (SQL NULL where pandas gives
        NaN); regr_slope = Sxy / Sxx and regr_intercept = my - regr_slope mx, NA when Sxx = 0.  (count, mx, my, Sxx, Syy, Sxy)
        is combined by the bivariate form of Chan's merge, with no sum of products (DESIGN §3c gives the bound): covar and
        corr are bit-for-bit symmetric in (y, x), corr(x, x) is exactly 1.0 where Sxx > 0, and equal x values give Sxx = 0
        exactly.  A frame whose counted pairs hold +-inf gives a valid NaN.  float64, nullable; a temporal column in either
        position raises.
      lag(x, k=1, default=None) / lead(...): the cell at i - k / i + k if that row is in the row's partition, else default (NA
        when None); 0 <= k < 2^31, k = 0 is the row itself; no frame; x's type, nullable.  default is converted to x's numpy
        dtype and must round-trip exactly.
    IGNORE NULLS: an entry of first_value, last_value, nth_value, lag or lead may end with "ignore_nulls" or "respect_nulls"
    (the default, the definitions above), recognised only as the last element at index 3 or later (so a column named
    "ignore_nulls" is still a column) and removed before the rest is parsed; on any other function it raises.  A cell is null
    exactly when count(x) does not count it: invalid or a float NaN.  This differs from RESPECT NULLS first_value, which returns
    a NaN as a valid cell: IGNORE NULLS skips it, as pandas' ffill / bfill do, so it works on numpy float columns too.  With row
    i's frame [lo, hi] and partition [P, pe) as the RESPECT NULLS function computes them (every frame, the same empty-frame rule):
      first_value(x) / last_value(x): the first / last non-null cell in [lo, hi], NA if none; nth_value(x, n): the n-th non-null
        cell in [lo, hi], NA if there are fewer than n; lag(x, k, default) / lead(...): the k-th non-null cell before row i in
        [P, i) / after it in (i, pe), default if there are fewer than k (k = 0 is the row itself, as above).
      The result is the chosen cell's bits (-0.0 stays -0.0); x's type, nullable; bit-identical across runs and batch splits.
    These follow SQL where pandas differs: groupby().cumsum() / cummin() / cummax() give NA at NA rows where the "rows" frame
    gives the aggregate so far; transform("sum") of an all-NA partition gives 0 where sum gives NA; float sums are combined in
    the scan's order, not sequentially.  Over ("rows", start, end) the results are pandas' groupby(p)[x].rolling(w,
    min_periods=1) ones (count: min_periods=0), with float sums combined in an order that depends only on the frame's bounds.
    Results depend only on the sorted positions: every row that shares a frame end (a bounded frame: both bounds) gets a
    bit-identical result, and float sums, the moments and the co-moments are bit-identical across runs and across any split of
    the rows into batches.
  - output: every input row once, in the stable sort's order by (partition keys, order keys, arrival); every input column in
    input order, then one column per function under the caller's name.  SQL leaves the order open; fixing it makes every column
    comparable bit for bit.
  - at most MAX_WINDOW_ROWS rows per state and MAX_COLS input plus function columns.  A parallel state of init_window_state
    raises at its first consume call when the process group has more than one rank (with one rank it runs locally): the sharded
    window is init_sharded_window_state.

Sharded window (init_sharded_window_state, one process per GPU of a torch.distributed process group).  Every consume call is
collective.  It partitions the batch by key class on the PARTITION BY keys (shuffle.partition_device(by_class=True): NA and NaN
are one class, -0.0 equals 0.0, every key type), agrees the P x P count matrix in one all_reduce and exchanges the rows
(exchange_table); the rows a rank receives go into its own local window.  Every partition thus lives whole on one rank, and the
local window, which is exact, computes it unchanged.  Without PARTITION BY the whole input is one partition: every row goes to
rank 0, which produces the whole result while the other ranks produce one empty batch (correct, not scalable).
  - arrival order: a rank receives rows in the order (consume call, source rank, source row), the arrival order that breaks
    ties.
  - result: rank r's output is the window of one state over the global input in that order, restricted to the partitions rank r
    owns, in the same output order, bit for bit on every input and function column (every result depends only on sorted
    positions within a partition).
  - protocol: every rank calls consume the same number of times and passes is_last in the same call.  A call after which some
    rank would hold MAX_WINDOW_ROWS rows or more raises the same B200Error on every rank before any row moves.  With one rank, or
    without torch.distributed, the state is the local window.
  - a dictionary-encoded string partition key is placed by its ids, which are only right when every rank uses the same
    dictionary builder.
"""

from __future__ import annotations

import datetime
import struct
import warnings

import numpy as np

from .. import _lib
from .._lib import ffi
from ..table import CTypes, Table, np_dtype_of
from .sort import MAX_FULL_SORT_ROWS, MAX_KEYS, SortState, _current_device, _world, agree_receive_rows

# Function codes of b200_window_func (include/bodo_b200.h): the ranking functions, then the value functions.
FUNCS = {"row_number": 0, "rank": 1, "dense_rank": 2, "percent_rank": 3, "cume_dist": 4, "ntile": 5}
VALUE_FUNCS = {"sum": 6, "count": 7, "mean": 8, "min": 9, "max": 10, "first_value": 11, "last_value": 12, "lag": 13, "lead": 14}
FRAMES = {"range": 1, "rows": 2, "partition": 3}
# nth_value, and frame 4, ROWS BETWEEN start AND end (b200_window_func.rows), with its UNBOUNDED sentinels.
FRAME_FUNCS = {"nth_value": 15}
ROWS_BETWEEN = 4
UNBOUNDED_PRECEDING, UNBOUNDED_FOLLOWING = -(1 << 63), (1 << 63) - 1
# VAR_SAMP, STDDEV_SAMP, VAR_POP and STDDEV_POP.
MOMENT_FUNCS = {"var": 16, "std": 17, "var_pop": 18, "std_pop": 19}
# Frame 5, RANGE BETWEEN start AND end (b200_window_func.range), with the kinds of b200_window_range.
RANGE_BETWEEN = 5
RANGE_KINDS = {"unbounded_preceding": 0, "preceding": 1, "current_row": 2, "following": 3, "unbounded_following": 4}
BOUNDED_FUNCS = ("sum", "count", "mean", "min", "max", "first_value", "last_value", "nth_value", "var", "std", "var_pop", "std_pop")
# Functions of two columns (y, x), x's index in arg.  They take
# every frame BOUNDED_FUNCS take.
BIVARIATE_FUNCS = {"covar_samp": 20, "covar_pop": 21, "corr": 22, "regr_slope": 23, "regr_intercept": 24}
# The navigation functions that take a trailing "ignore_nulls" / "respect_nulls" marker (b200_window_func.ignore_nulls).
NULLS_FUNCS = ("first_value", "last_value", "nth_value", "lag", "lead")
NULLS_MARKERS = ("ignore_nulls", "respect_nulls")
_VALUE_NAMES = {c: f for f, c in {**VALUE_FUNCS, **FRAME_FUNCS, **MOMENT_FUNCS, **BIVARIATE_FUNCS}.items()}
_FRAME_NAMES = {c: f for f, c in FRAMES.items()}
MAX_COLS = 32
MAX_WINDOW_ROWS = MAX_FULL_SORT_ROWS
MAX_LAG = (1 << 31) - 1
MAX_FRAME_OFFSET = MAX_LAG
_TEMPORAL = (CTypes.DATE, CTypes.DATETIME, CTypes.TIMEDELTA)
_INTEGER = (CTypes.INT8, CTypes.INT16, CTypes.INT32, CTypes.INT64, CTypes.UINT8, CTypes.UINT16, CTypes.UINT32, CTypes.UINT64)
_NS_PER_UNIT = {"W": 604_800 * 10**9, "D": 86_400 * 10**9, "h": 3_600 * 10**9, "m": 60 * 10**9, "s": 10**9, "ms": 10**6, "us": 10**3,
                "ns": 1}
_DAY_NS = 86_400 * 10**9
_CT_NAMES = {v: k for k, v in vars(CTypes).items() if k.isupper() and isinstance(v, int)}
_FORMS = (f"ranking: (out_name, fname) with fname in {sorted(FUNCS)}, or (out_name, 'ntile', n); value: (out_name, fname, column"
          f"[, frame]) with fname in {sorted(set(VALUE_FUNCS) - {'lag', 'lead'} | set(MOMENT_FUNCS))}, frame in {sorted(FRAMES)}, ('rows', start, end) or ('range_between', start, end), "
          "column None for count(*) only, or (out_name, 'lag' | 'lead', column[, k[, default]]), or (out_name, 'nth_value', column, "
          f"n[, frame]), or (out_name, fname, column1, column2[, frame]) with fname in {sorted(BIVARIATE_FUNCS)}; an entry of "
          f"{', '.join(NULLS_FUNCS)} may end with 'ignore_nulls' or 'respect_nulls' (the default)")


def _names(x):
    if x is None:
        return []
    return [x] if isinstance(x, str) else list(x)


def _parse_value(f, col_names, entry):
    """(out_name, fname, column[, frame]), (out_name, 'lag' | 'lead', column[, k[, default]]) or (out_name, 'nth_value', column,
    n[, frame]) -> (out_name, code, k, column, frame code, default[, (start, end)]); frame code 0 for lag and lead, k = n for
    nth_value, (start, end) for a ROWS_BETWEEN or RANGE_BETWEEN frame only.  f is the entry without its nulls marker, entry the
    entry as written (named in errors)."""
    name, fname, column = f[0], f[1], f[2]
    if not (column is None and fname == "count") and not (isinstance(column, str) and column in col_names):
        raise _lib.B200Error(f"Streaming Window: {entry!r}: unknown column {column!r} (one of {col_names}; None for count only)")
    if fname in ("lag", "lead"):
        if len(f) > 5:
            raise _lib.B200Error(f"Streaming Window: {entry!r}: {fname} takes (out_name, {fname!r}, column[, k[, default]])")
        k = f[3] if len(f) > 3 else 1
        if isinstance(k, str) and k in FRAMES or isinstance(k, (tuple, list)) and len(k) == 3 and k[0] == "range_between":
            raise _lib.B200Error(f"Streaming Window: {entry!r}: {fname} takes no frame")
        if isinstance(k, (bool, np.bool_)) or not isinstance(k, (int, np.integer)) or not 0 <= k <= MAX_LAG:
            raise _lib.B200Error(f"Streaming Window: {entry!r}: {fname} needs an integer k with 0 <= k < 2^31")
        return (name, VALUE_FUNCS[fname], int(k), column, 0, f[4] if len(f) > 4 else None)
    if fname in BIVARIATE_FUNCS:
        if len(f) < 4 or not (isinstance(f[3], str) and f[3] in col_names):
            raise _lib.B200Error(f"Streaming Window: {entry!r}: unknown second column {f[3] if len(f) > 3 else None!r} (one of {col_names}), as "
                                 f"(out_name, {fname!r}, column1, column2[, frame])")
        if len(f) > 5:
            raise _lib.B200Error(f"Streaming Window: {entry!r}: {fname} takes (out_name, {fname!r}, column1, column2[, frame])")
        return (name, BIVARIATE_FUNCS[fname], f[3], column, *_parse_frame(entry, f[4] if len(f) > 4 else "range"))
    if fname == "nth_value":
        nth = f[3] if len(f) > 3 else None
        if len(f) > 5 or isinstance(nth, (bool, np.bool_)) or not isinstance(nth, (int, np.integer)) or not 1 <= nth <= MAX_LAG:
            raise _lib.B200Error(f"Streaming Window: {entry!r}: nth_value takes (out_name, 'nth_value', column, n[, frame]) with an integer "
                                 "1 <= n < 2^31")
        return (name, FRAME_FUNCS[fname], int(nth), column, *_parse_frame(entry, f[4] if len(f) > 4 else "range"))
    if len(f) > 4:
        raise _lib.B200Error(f"Streaming Window: {entry!r}: bad frame (one of {sorted(FRAMES)}, ('rows', start, end) or ('range_between', start, end), as (out_name, "
                             f"{fname!r}, column[, frame]))")
    return (name, {**VALUE_FUNCS, **MOMENT_FUNCS}[fname], 0, column, *_parse_frame(entry, f[3] if len(f) > 3 else "range"))


def _parse_frame(f, frame):
    """A frame name, or ("rows", start, end) with start / end None (UNBOUNDED) or a row offset (negative PRECEDING, 0 CURRENT ROW,
    positive FOLLOWING) -> (frame code, default None[, (start, end)]).  ("rows", None, 0) is "rows" and ("rows", None, None) is
    "partition", so a frame gives the same results however it is spelled."""
    if isinstance(frame, str) and frame in FRAMES:
        return FRAMES[frame], None
    if isinstance(frame, (tuple, list)) and len(frame) == 3 and frame[0] == "range_between":
        return _parse_range(f, frame[1], frame[2])
    if not (isinstance(frame, (tuple, list)) and len(frame) == 3 and frame[0] == "rows"):
        raise _lib.B200Error(f"Streaming Window: {f!r}: bad frame (one of {sorted(FRAMES)}, ('rows', start, end) or ('range_between', start, end), as (out_name, "
                             f"{f[1]!r}, column[, frame]))")
    start, end = frame[1], frame[2]
    for b in (start, end):
        if b is not None and (isinstance(b, (bool, np.bool_)) or not isinstance(b, (int, np.integer))
                              or not -MAX_FRAME_OFFSET <= b <= MAX_FRAME_OFFSET):
            raise _lib.B200Error(f"Streaming Window: {f!r}: bad frame bound {b!r} (None for UNBOUNDED or an integer row offset in "
                                 "(-2^31, 2^31))")
    if start is not None and end is not None and start > end:
        raise _lib.B200Error(f"Streaming Window: {f!r}: frame start {start} is after frame end {end}")
    if f[1] not in BOUNDED_FUNCS and f[1] not in BIVARIATE_FUNCS:
        raise _lib.B200Error(f"Streaming Window: {f!r}: a ('rows', start, end) frame takes one of {list(BOUNDED_FUNCS)}")
    if start is None and end == 0:
        return FRAMES["rows"], None
    if start is None and end is None:
        return FRAMES["partition"], None
    return (ROWS_BETWEEN, None, (UNBOUNDED_PRECEDING if start is None else int(start), UNBOUNDED_FOLLOWING if end is None else int(end)))


def _offset(b):
    """A RANGE offset -> (family, signed value): ("int", int) for a Python or numpy integer (not bool) with |k| < 2^63,
    ("float", float) for a finite float that a double holds exactly, ("ns", int) for a numpy.timedelta64 (not NaT, exact in ns),
    datetime.timedelta or pandas.Timedelta.  None for anything else."""
    if isinstance(b, (bool, np.bool_)):
        return None
    if hasattr(b, "asm8") and isinstance(b, datetime.timedelta):  # pandas.Timedelta, in its own unit
        b = b.asm8
    if isinstance(b, np.timedelta64):
        unit, count = np.datetime_data(b.dtype)
        if np.isnat(b) or unit not in _NS_PER_UNIT and unit not in ("ps", "fs", "as"):
            return None
        v = int(b.astype(np.int64)) * count
        if unit in _NS_PER_UNIT:
            ns = v * _NS_PER_UNIT[unit]
        else:
            per = {"ps": 10**3, "fs": 10**6, "as": 10**9}[unit]
            if v % per:
                return None
            ns = v // per
        return ("ns", ns) if abs(ns) < 1 << 63 else None
    if isinstance(b, datetime.timedelta):
        ns = ((b.days * 86_400 + b.seconds) * 10**6 + b.microseconds) * 1000
        return ("ns", ns) if abs(ns) < 1 << 63 else None
    if isinstance(b, (int, np.integer)):  # numpy.timedelta64 is a numpy integer: handled above
        return ("int", int(b)) if abs(int(b)) < 1 << 63 else None
    if isinstance(b, (float, np.floating)):
        x = float(b)
        return ("float", x) if np.isfinite(x) and x == b else None
    return None


def _parse_range(f, start, end):
    """("range_between", start, end), each None (UNBOUNDED), zero (CURRENT ROW) or a signed offset (negative PRECEDING, positive
    FOLLOWING) -> (RANGE_BETWEEN, None, (start, end)) with zero offsets made 0; (None, 0) is "range" and (None, None) is
    "partition", so a frame gives the same results however it is spelled.  Offsets are checked against the ORDER BY key's type
    at the first consume call (WindowState.ranges)."""
    bounds = []
    for b in (start, end):
        if b is None:
            bounds.append(None)
            continue
        o = _offset(b)
        if o is None:
            raise _lib.B200Error(f"Streaming Window: {f!r}: bad frame bound {b!r} (None for UNBOUNDED, or an offset: an integer with "
                                 "|k| < 2^63, a finite float, or a numpy.timedelta64 / datetime.timedelta / pandas.Timedelta exact in "
                                 "ns; negative PRECEDING, 0 CURRENT ROW, positive FOLLOWING)")
        bounds.append(0 if o[1] == 0 else b)
    start, end = bounds
    if start is not None and end is not None:
        (fs, s), (fe, e) = _offset(start) or ("int", 0), _offset(end) or ("int", 0)
        if (fs == "ns") == (fe == "ns") or s == 0 or e == 0:
            if s > e:
                raise _lib.B200Error(f"Streaming Window: {f!r}: frame start {start!r} is after frame end {end!r}")
    if f[1] not in BOUNDED_FUNCS and f[1] not in BIVARIATE_FUNCS:
        raise _lib.B200Error(f"Streaming Window: {f!r}: a ('range_between', start, end) frame takes one of {list(BOUNDED_FUNCS)}")
    if start is None and end is None:
        return FRAMES["partition"], None
    if start is None and isinstance(end, int) and end == 0:
        return FRAMES["range"], None
    return RANGE_BETWEEN, None, (start, end)


def _range_kind(b, end):
    if b is None:
        return RANGE_KINDS["unbounded_following" if end else "unbounded_preceding"]
    if isinstance(b, int) and not isinstance(b, bool) and b == 0:
        return RANGE_KINDS["current_row"]
    return RANGE_KINDS["preceding" if _offset(b)[1] < 0 else "following"]


def _entry(f, ignore_nulls=False):
    """A parsed value entry as the caller wrote it, with its frame spelled out and its IGNORE NULLS marker (for error messages)."""
    name, code, arg, column, frame = f[:5]
    mark = ("ignore_nulls",) if ignore_nulls else ()
    fr = _FRAME_NAMES.get(frame)
    if len(f) > 6 and frame == ROWS_BETWEEN:
        fr = ("rows", *[None if b in (UNBOUNDED_PRECEDING, UNBOUNDED_FOLLOWING) else b for b in f[6]])
    elif len(f) > 6:
        fr = ("range_between", *f[6])
    if code in BIVARIATE_FUNCS.values():
        return (name, _VALUE_NAMES[code], column, arg, fr)
    if code in (VALUE_FUNCS["lag"], VALUE_FUNCS["lead"]):
        return (name, _VALUE_NAMES[code], column, arg, f[5], *mark)
    return (name, _VALUE_NAMES[code], column, fr, *mark) if code != FRAME_FUNCS["nth_value"] else (name, "nth_value", column, arg, fr, *mark)


def _default_bits(f, ct, ignore_nulls=False):
    """Bits of lag / lead's default in the column's numpy dtype; raises unless it round-trips exactly."""
    default, dt = f[5], np_dtype_of(ct)
    entry = _entry(f, ignore_nulls)
    try:
        with warnings.catch_warnings(), np.errstate(all="ignore"):
            warnings.simplefilter("ignore")
            y = np.array([default]).astype(dt)
        back = y[0].item()
        ok = back == default or (isinstance(back, float) and back != back and default != default)
    except (TypeError, ValueError, OverflowError):
        ok = False
    if not ok:
        raise _lib.B200Error(f"Streaming Window: {entry!r}: default {default!r} is not exactly representable as {dt}")
    return int(y.view(f"u{dt.itemsize}")[0])


def _parse_funcs(funcs, col_names):
    """Ranking entries -> (out_name, code, n); value entries -> (out_name, code, k, column, frame code, default), with a
    seventh field (start, end) for a ROWS_BETWEEN or RANGE_BETWEEN frame.  Returns those and one IGNORE NULLS flag per entry: a
    trailing "ignore_nulls" / "respect_nulls" (the last element, at index 3 or later) is removed before the entry is parsed."""
    out, nulls = [], []
    for f in funcs:
        f = tuple(f)
        marker = f[-1] if len(f) > 3 and isinstance(f[-1], str) and f[-1] in NULLS_MARKERS else None
        value = isinstance(f[1] if len(f) > 1 else None, str) and (f[1] in VALUE_FUNCS or f[1] in FRAME_FUNCS or f[1] in MOMENT_FUNCS
                                                                   or f[1] in BIVARIATE_FUNCS)
        if (len(f) < 2 or not isinstance(f[0], str) or not isinstance(f[1], str) or f[1] not in FUNCS and not value
                or value and len(f) < 3):
            raise _lib.B200Error(f"Streaming Window: unknown window function {f!r} ({_FORMS})")
        name, fname = f[0], f[1]
        if marker is not None and fname not in NULLS_FUNCS:
            raise _lib.B200Error(f"Streaming Window: {f!r}: {marker!r} takes one of {list(NULLS_FUNCS)}")
        nulls.append(marker == "ignore_nulls")
        if value:
            out.append(_parse_value(f[:-1] if marker is not None else f, col_names, f))
            continue
        if fname == "ntile":
            if len(f) != 3 or isinstance(f[2], bool) or not isinstance(f[2], int) or f[2] < 1:
                raise _lib.B200Error(f"Streaming Window: ntile needs an integer n >= 1, as (out_name, 'ntile', n) (got {f!r})")
            arg = int(f[2])
        else:
            if len(f) != 2:
                raise _lib.B200Error(f"Streaming Window: {fname} takes no argument (got {f!r})")
            arg = 0
        out.append((name, FUNCS[fname], arg))
    if not out:
        raise _lib.B200Error("Streaming Window: at least one window function")
    names = [f[0] for f in out]
    dup = sorted({n for n in names if names.count(n) > 1})
    if dup:
        raise _lib.B200Error(f"Streaming Window: duplicate output names {dup}")
    clash = [n for n in names if n in col_names]
    if clash:
        raise _lib.B200Error(f"Streaming Window: output names {clash} clash with input columns")
    if len(col_names) + len(out) > MAX_COLS:
        raise _lib.B200Error(f"Streaming Window: {len(col_names)} input columns and {len(out)} functions exceed {MAX_COLS} output columns")
    return out, nulls


class WindowState(SortState):
    """Python handle of the C window state (created lazily at the first consume call).  The sort state's keys are the partition
    keys (ascending, NA last) followed by the order keys; the produced columns are the input's, then one per function."""

    def __init__(self, operator_id, partition_by, order_by, ascending, na_position, funcs, col_names, parallel, output_batch_size,
                 device, stream, process_group):
        part, order = _names(partition_by), _names(order_by)
        keys = part + order
        if not 1 <= len(keys) <= MAX_KEYS:
            raise _lib.B200Error(f"Streaming Window: 1 to {MAX_KEYS} keys in PARTITION BY and ORDER BY together (got {len(part)} + "
                                 f"{len(order)})")
        col_names = [str(c) for c in col_names]
        missing = [k for k in keys if k not in col_names]
        if missing or len(set(keys)) != len(keys):
            raise _lib.B200Error(f"Streaming Window: PARTITION BY {part} and ORDER BY {order} must be distinct columns of {col_names}")
        asc = [ascending] * len(order) if isinstance(ascending, bool) else [bool(a) for a in ascending]
        nap = [na_position] * len(order) if isinstance(na_position, str) else list(na_position)
        if len(asc) != len(order) or len(nap) != len(order):
            raise _lib.B200Error("Streaming Window: ascending and na_position need one value or one entry per ORDER BY key")
        if any(p not in ("first", "last") for p in nap):
            raise _lib.B200Error(f"Streaming Window: na_position must be 'first' or 'last' (got {nap})")
        parsed, nulls = _parse_funcs(funcs, col_names)
        for f, ign in zip(parsed, nulls):
            if len(f) > 6 and f[4] == RANGE_BETWEEN and len(order) != 1 and any(b not in (None, 0) for b in f[6]):
                raise _lib.B200Error(f"Streaming Window: {_entry(f, ign)!r}: a range offset (k PRECEDING / FOLLOWING) needs exactly one ORDER "
                                     f"BY key (got {order})")
        super().__init__(operator_id, None, 0, keys, [True] * len(part) + asc, ["last"] * len(part) + nap, col_names, parallel,
                         output_batch_size, device, stream, process_group, full=True)
        self.partition_by, self.order_by = part, order
        self.funcs = parsed
        self.ignore_nulls = nulls  # per function: IGNORE NULLS
        self.out_names += [f[0] for f in parsed]
        self.out_order += list(range(len(self.phys), len(self.phys) + len(parsed)))
        self.descs = None

    def descriptors(self, c_types):
        """The b200_window_func fields (code, col, frame, default_valid, arg, default_bits) of every function, given the c-types
        of the input columns in input order; a bivariate function's arg is its second column's physical index.  Raises B200Error
        for sum, mean, var or std of a temporal column, a bivariate function with a temporal column in either position and a lag /
        lead default that does not round-trip through the column's dtype."""
        out = []
        for f, ign in zip(self.funcs, self.ignore_nulls):
            if len(f) == 3:
                out.append((f[1], -1, 0, 0, f[2], 0))
                continue
            name, code, arg, column, frame, default = f[:6]
            if column is None:
                out.append((code, -1, frame, 0, arg, 0))
                continue
            ct = c_types[self.col_names.index(column)]
            if code in BIVARIATE_FUNCS.values():
                if ct in _TEMPORAL or c_types[self.col_names.index(arg)] in _TEMPORAL:
                    raise _lib.B200Error(f"Streaming Window: {_entry(f)!r}: covar, corr and regr need integer, bool or float columns, "
                                         "not temporal ones")
                out.append((code, self.phys.index(self.col_names.index(column)), frame, 0, self.phys.index(self.col_names.index(arg)), 0))
                continue
            moment = code in MOMENT_FUNCS.values()
            if (code in (VALUE_FUNCS["sum"], VALUE_FUNCS["mean"]) or moment) and ct in _TEMPORAL:
                entry = _entry(f)
                what = "var and std" if moment else "sum and mean"
                raise _lib.B200Error(f"Streaming Window: {entry!r}: {what} need an integer, bool or float column, not a temporal one")
            valid = default is not None
            out.append((code, self.phys.index(self.col_names.index(column)), frame, int(valid), arg, _default_bits(f, ct, ign) if valid else 0))
        return out

    def frames(self):
        """The b200_window_frame (start, end) of every function: its bounds for a ('rows', start, end) frame (code ROWS_BETWEEN),
        else (UNBOUNDED_PRECEDING, UNBOUNDED_FOLLOWING), which the library does not read."""
        return [f[6] if len(f) > 6 and f[4] == ROWS_BETWEEN else (UNBOUNDED_PRECEDING, UNBOUNDED_FOLLOWING) for f in self.funcs]

    def ranges(self, c_types):
        """The b200_window_range (start_kind, end_kind, start_bits, end_bits) of every function, given the c-types of the input
        columns in input order: its kinds and offset magnitudes in the ORDER BY key's arithmetic (integers as they are, DATE in
        days, DATETIME / TIMEDELTA in ns, float keys as the bits of a double) for a ('range_between', start, end) frame (code
        RANGE_BETWEEN), else (0, 4, 0, 0), which the library does not read.  Raises B200Error for an offset whose type does not fit
        the key: integers take an integer, floats an integer or float that a double holds exactly, DATETIME / TIMEDELTA a
        timedelta, DATE a timedelta of whole days; a bool key takes none."""
        out = []
        for f, ign in zip(self.funcs, self.ignore_nulls):
            if not (len(f) > 6 and f[4] == RANGE_BETWEEN):
                out.append((RANGE_KINDS["unbounded_preceding"], RANGE_KINDS["unbounded_following"], 0, 0))
                continue
            kinds, bits = [_range_kind(f[6][0], False), _range_kind(f[6][1], True)], [0, 0]
            for j, b in enumerate(f[6]):
                if kinds[j] not in (RANGE_KINDS["preceding"], RANGE_KINDS["following"]):
                    continue
                key = self.order_by[0]
                ct = c_types[self.col_names.index(key)]
                fam, v = _offset(b)
                k = abs(v)
                if ct in _INTEGER and fam == "int":
                    bits[j] = k
                elif ct in (CTypes.FLOAT32, CTypes.FLOAT64) and fam in ("int", "float") and float(k) == k:
                    bits[j] = struct.unpack("<Q", struct.pack("<d", float(k)))[0]
                elif ct in (CTypes.DATETIME, CTypes.TIMEDELTA) and fam == "ns":
                    bits[j] = k
                elif ct == CTypes.DATE and fam == "ns" and k % _DAY_NS == 0:
                    bits[j] = k // _DAY_NS
                else:
                    want = ("an integer" if ct in _INTEGER else "an int or float exactly representable as a double"
                            if ct in (CTypes.FLOAT32, CTypes.FLOAT64) else "a timedelta" if ct in (CTypes.DATETIME, CTypes.TIMEDELTA)
                            else "a timedelta of whole days" if ct == CTypes.DATE else "no offset (an integer, float or temporal key is needed)")
                    raise _lib.B200Error(f"Streaming Window: {_entry(f, ign)!r}: range offset {b!r} does not fit ORDER BY key {key!r} of "
                                         f"type {_CT_NAMES.get(ct, ct)}: it takes {want}")
            out.append((kinds[0], kinds[1], bits[0], bits[1]))
        return out

    def _ensure(self, table: Table, limit=None, offset=None):
        if self.handle is None and table.n_cols == len(self.col_names):
            self.descs = self.descriptors([c.c_type for c in table.columns])
            self.rdescs = self.ranges([c.c_type for c in table.columns])
        super()._ensure(table, limit, offset)

    def _new_handle(self, L, c_types, a_types, n_cols, asc, nal, limit, offset):
        np_ = len(self.partition_by)
        oasc = ffi.new("int32_t[]", [int(a) for a in self.asc[np_:]] or [0])
        onal = ffi.new("int32_t[]", [int(x) for x in self.na_last[np_:]] or [0])
        funcs = zip(self.descs, self.frames(), self.rdescs, self.ignore_nulls)
        fs = ffi.new("b200_window_func[]", [(*d, rows, rng, int(ign)) for d, rows, rng, ign in funcs])
        h = L.b200_window_state_init(self.operator_id, c_types, a_types, n_cols, np_, len(self.order_by), oasc, onal, fs, len(self.descs),
                                     self.output_batch_size, self.device, ffi.cast("void*", self.stream))
        return _lib.check_ptr(h, "init_window_state")


class ShardedWindowState:
    """Python handle of a sharded window (init_sharded_window_state): every consume call moves each row to the rank that owns its
    partition, and `local` is the window over the rows this rank received."""

    def __init__(self, operator_id, partition_by, order_by, ascending, na_position, funcs, col_names, output_batch_size, device, stream,
                 process_group):
        self.local = WindowState(operator_id, partition_by, order_by, ascending, na_position, funcs, col_names, False, output_batch_size,
                                 device, stream, None)
        self.process_group = process_group
        self.n_ranks = None
        self.received = None  # rows each rank has received so far, known alike on every rank
        self.done = False

    def consume(self, table: Table, is_last: bool):
        loc = self.local
        if self.n_ranks is None:
            self.n_ranks, self.rank = _world(self.process_group)
            self.received = np.zeros(self.n_ranks, dtype=np.int64)
        if self.n_ranks > 1:
            table = self._exchange(table)
        loc._ensure(table)
        req = loc._consume(table, is_last)
        if is_last:
            loc.done = self.done = True
        return req

    def _exchange(self, table: Table) -> Table:
        """This call's rows of every rank that belong to this rank's partitions, in (source rank, source row) order."""
        import torch

        from ..shuffle import exchange_table, partition_device, with_schema_validity
        from ..table import Column, to_device

        loc, P = self.local, self.n_ranks
        if table.n_cols != len(loc.col_names):
            raise _lib.B200Error(f"Streaming Window: the batch has {table.n_cols} columns, the state {len(loc.col_names)}")
        if loc.device is None:
            loc.device = table.device if table.device >= 0 else _current_device()
        dev = torch.device("cuda", loc.device)
        phys = with_schema_validity(to_device(table, loc.device).select(loc.phys))  # the partition keys lead
        n = phys.n_rows
        if self.local.partition_by:
            part, send = partition_device(phys, len(loc.partition_by), P, loc.stream, by_class=True)
        else:  # one partition: every row to rank 0, the batch itself is the send buffer
            part = Table([Column(_as_tensor(c.data, dev, n, c.c_type), None if c.validity is None else _as_tensor(c.validity, dev, (n + 7) // 8),
                                 c.c_type, c.arr_type, n) for c in phys.columns], list(phys.names))
            send = [n] + [0] * (P - 1)
        counts = agree_receive_rows(send, dev, self.process_group, received=self.received, cap=MAX_WINDOW_ROWS,
                                    what="Streaming Window: sharded window", cap_name="the window's cap")
        self.received += counts.sum(axis=0)
        got = exchange_table(part, send, self.process_group)
        torch.cuda.synchronize(dev)
        return got.select(loc.out_order[: len(loc.col_names)])  # back to input column order

    def produce(self, produce_output: bool):
        return self.local._produce(produce_output)


def _as_tensor(x, dev, n, c_type=None):
    """The first n cells of a device buffer (torch tensor or library-owned array) as a torch tensor."""
    import torch

    if n == 0:
        dt = np.uint8 if c_type is None else np_dtype_of(c_type)
        return torch.empty(0, dtype=getattr(torch, str(np.dtype(dt))), device=dev)
    return (x if hasattr(x, "is_cuda") else torch.as_tensor(x, device=dev))[:n]


def init_sharded_window_state(operator_id, partition_by, order_by, ascending, na_position, funcs, col_names, *,
                              output_batch_size=32768, device=None, stream=0, process_group=None) -> ShardedWindowState:
    """A sharded window over a torch.distributed process group (one process per GPU): init_window_state's arguments, validation
    and errors, and the same verbs.  Every consume call is collective (every rank calls it the same number of times and passes
    is_last in the same call) and moves each row to the rank that owns its partition (a hash of its PARTITION BY key class).  Rank
    r's output is the window of one state over the global input in (consume call, source rank, source row) order, restricted to
    the partitions rank r owns, in the same output order, bit for bit.  Without PARTITION BY every row goes to rank 0, which
    produces the whole result while the other ranks produce one empty batch.  A call after which a rank would hold MAX_WINDOW_ROWS
    rows or more raises the same B200Error on every rank before any row moves.  Without torch.distributed, or with one rank, it
    is the local window.  A dictionary-encoded string partition key is placed by its ids: every rank must use the same
    dictionary builder."""
    return ShardedWindowState(operator_id, partition_by, order_by, ascending, na_position, funcs, col_names, output_batch_size, device,
                              stream, process_group)


def init_window_state(operator_id, partition_by, order_by, ascending, na_position, funcs, col_names, parallel=False, *,
                      output_batch_size=32768, device=None, stream=0, process_group=None) -> WindowState:
    """A window state over batches with columns `col_names`.

    partition_by / order_by: a column name or a list of names (either may be empty, 1..4 in all); ascending / na_position: one
    value or one per ORDER BY key; funcs: ranking entries (out_name, fname) with fname in FUNCS, or (out_name, "ntile", n) with
    n >= 1; value entries (out_name, fname, column[, frame]) with fname in VALUE_FUNCS other than lag / lead, frame one of FRAMES
    (default "range") or ("rows", start, end) and column None for count(*) only, (out_name, "lag" | "lead", column[, k[,
    default]]) (k = 1 and default None, NA, by default), (out_name, "nth_value", column, n[, frame]), or (out_name, fname,
    column[, frame]) with fname in MOMENT_FUNCS (var, std, var_pop, std_pop) and any frame sum takes, or (out_name, fname, y, x[,
    frame]) with fname in BIVARIATE_FUNCS (covar_samp, covar_pop, corr, regr_slope, regr_intercept; SQL's argument order) and
    any frame sum takes.  An entry of first_value, last_value, nth_value, lag or lead may end with "ignore_nulls" (IGNORE NULLS)
    or "respect_nulls" (the default).
    Examples, a 7-row moving average: ("ma7", "mean", "x", ("rows", -6, 0)); a one-hour time window over a DATETIME ORDER BY
    key: ("s1h", "sum", "amount", ("range_between", -pd.Timedelta("1h"), 0)); a 20-row rolling standard deviation (a Bollinger
    band's width): ("sd20", "std", "x", ("rows", -19, 0)); the population variance of the partition: ("vp", "var_pop", "x",
    "partition"); a 60-row rolling beta of r on the market return mr and their correlation: ("beta", "regr_slope", "r", "mr",
    ("rows", -59, 0)), ("rho", "corr", "r", "mr", ("rows", -59, 0)); the last known reading per sensor (a per-group ffill, ordered
    by time): ("last", "last_value", "x", "rows", "ignore_nulls"); the previous reading that is not missing: ("prev", "lag", "x",
    1, None, "ignore_nulls").
    Raises B200Error for an unknown function, duplicate output names or names that clash with an input column, keys that are
    missing or not distinct, a key count outside 1..4, a bad na_position, ntile n < 1, an unknown value column, a bad frame or
    frame bound, a frame on lag or lead, k outside [0, 2^31), nth_value n outside [1, 2^31), a range offset without exactly one
    ORDER BY key, a missing or unknown second column of a bivariate function, an "ignore_nulls" / "respect_nulls" marker on
    another function; and at the first consume call for sum, mean, var
    or std of a temporal column, a bivariate function with a temporal column in either position, a lag / lead default that the
    column's dtype cannot hold exactly or a range offset whose type does not fit the ORDER BY key."""
    return WindowState(operator_id, partition_by, order_by, ascending, na_position, funcs, col_names, parallel, output_batch_size,
                       device, stream, process_group)


def window_build_consume_batch(state: WindowState, table: Table, is_last: bool):
    """Appends a batch (host batches are staged to the device); is_last sorts and evaluates.  Returns (is_last, request_input)."""
    if state.done:
        raise _lib.B200Error("window_build_consume_batch called after is_last")
    if isinstance(state, ShardedWindowState):
        return bool(is_last), state.consume(table, is_last)
    if state.parallel:
        import torch.distributed as dist

        if dist.is_initialized() and dist.get_world_size(state.process_group) > 1:
            raise _lib.B200Error("Streaming Window: a sharded window is not supported (process group of more than one rank)")
    state._ensure(table)
    req = state._consume(table, is_last)
    if is_last:
        state.done = True
    return bool(is_last), req


def window_produce_output_batch(state: WindowState, produce_output: bool = True):
    """Returns (table, is_last): the next <= output_batch_size output rows, as library-owned device columns that stay valid until
    the state is deleted.  A sharded window produces the rows of the partitions this rank owns."""
    if isinstance(state, ShardedWindowState):
        state = state.local
    if state.handle is None or not state.done:
        raise _lib.B200Error("window_produce_output_batch called before the last batch was consumed")
    return state._produce(produce_output)


def delete_window_state(state: WindowState) -> None:
    if isinstance(state, ShardedWindowState):
        state = state.local
    if state.handle is not None:
        _lib.lib().b200_delete_sort_state(state.handle)
        state.handle = None


def get_metric(state: WindowState, which: int) -> int:
    """The sort's metrics (streaming/sort.py get_metric; 1-5 read 0) and 9, the number of partitions.  A sharded window reports
    this rank's local window (metric 0 the rows it received, 9 the partitions it owns)."""
    if isinstance(state, ShardedWindowState):
        state = state.local
    return int(_lib.lib().b200_sort_get_metric(state.handle, which))
