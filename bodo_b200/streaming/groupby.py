"""Streaming groupby operator API — the host-side mirror of bodo/libs/streaming/groupby.py.

Same four verbs, same argument meaning and the same calling protocol as the reference
(init_groupby_state :702-715, groupby_build_consume_batch :1295-1395, groupby_produce_output_batch
:1502-1600, delete_groupby_state), so the reference's streaming test loops
(bodo/tests/test_streaming/test_groupby.py:51-81) run unchanged against this module.  The work happens in
libbodo_b200.so (CUDA, sm_90a); there is no CPU implementation behind these calls.

Differences: the reference types the state at Numba compile time; here the build-table schema is taken
from the first consumed batch.  With parallel=True the state is one shard of a torch.distributed process
group (one process per GPU): the last consume call runs the hash-partition exchange that replaces the
reference's MPI shuffle (streaming/_shuffle.cpp:687-804).

min_row_number_filter (MRNF): fnames == ("min_row_number_filter",) with the four mrnf_* arguments keeps one row per group,
QUALIFY ROW_NUMBER() OVER (PARTITION BY keys ORDER BY sort columns) = 1, i.e.
df.sort_values(sort columns, kind="stable").drop_duplicates(keys, keep="first")[kept columns]:
  - keys: 1..4 columns (key_inds) with the groupby's key types and equality (float keys: -0.0 equals 0.0, NaN is the NA key);
    dropna=True drops rows with an NA key, dropna=False puts all NA keys in one group.
  - mrnf_sort_col_inds: 1..4 distinct columns (a key column too) of the sort's key types (fixed-width integer, float, bool,
    DATE, DATETIME, TIMEDELTA; numpy or nullable); mrnf_sort_col_asc[j]: ascending; mrnf_sort_col_na[j]: True puts NA last.  A
    float NaN is NA and -0.0 ties with 0.0, as in the sort.
  - winner: the first row of the stable order by (sort columns, arrival), arrival being batch order, then row order: of rows
    that tie on every sort column the earliest wins, even across batches.  The result is bit-identical across runs, batch
    splits and table growth.
  - mrnf_col_inds_keep: the output columns (logical indices, keys allowed, at most 26), in input order under their input
    names, each holding the winner's own cell (bits and validity: a kept float key shows the winner's -0.0), with the input's
    type and array kind.  One row per group; group order unspecified.
  - f_in_offsets / f_in_cols list the function's input columns: f_in_offsets == (0, len(f_in_cols)), f_in_cols non-key
    columns; the operator reads only the keys, the sort columns and the kept columns.
  - every key, sort and kept column is fixed width (anything else raises, naming the column); a parallel state on a process
    group of more than one rank raises at its first consume call (sharded MRNF is not supported), with one rank it runs locally.
The state streams every batch into the groupby's hash table and keeps one winner record per group (DESIGN.md §3d), so it holds
O(groups) device memory whatever the row count.

Sharded min_row_number_filter (init_sharded_mrnf_state, one process per GPU of a torch.distributed process group): only winners
move between ranks.  Consume calls before is_last are local and run no collective: each rank runs an ordinary MRNF that keeps the
union of the keys, the sort columns and the caller's kept columns (at most 26).  The is_last call is collective: each rank
produces its winners (at most groups x n rows), partitions them by key class on the keys (shuffle.partition_device(by_class=True):
NA and NaN one class, -0.0 equal to 0.0, every key type), agrees the count matrix, exchanges them and consumes the rows it received
in one call into a second MRNF with the same keys, sort and n that keeps the caller's columns.  The rows arrive in source-rank
order and the partition is stable, so within a group each source's rows arrive in its own rank order: ties are broken by (rank,
local arrival), and the top n of the union of every rank's top n is the MRNF of the rank inputs concatenated in rank order.

mrnf_limit=n (keyword-only, an int, 1 <= n < 2^31, default 1; only with min_row_number_filter) keeps the first n rows per group,
QUALIFY ROW_NUMBER() OVER (PARTITION BY keys ORDER BY sort columns) <= n, i.e.
df.sort_values(sort columns, kind="stable").groupby(keys, sort=False, dropna=dropna).head(n)[kept columns] as a multiset of rows:
  - everything above holds; of rows that tie on every sort column the earlier arrival ranks first, even across batches, and a
    group with fewer than n rows keeps all of them.
  - a group's rows are consecutive and in rank order in the output, also when the group spans two output batches (group order
    is unspecified), so a cumulative count numbers them.
  - n > 1 keeps candidate rows in a device store reduced by a radix sort of at most 2^31 rows: a batch whose rows, added to the
    survivors (at most groups x n), would pass that raises.  Its memory is O(groups x n + rows admitted between reduces).

Holistic aggregates: "mode", "percentile_cont" and "percentile_disc" (SQL MODE(x), PERCENTILE_CONT(q) / PERCENTILE_DISC(q) WITHIN
GROUP (ORDER BY x); pandas groupby(...).quantile(q) and agg(lambda s: s.mode()[0])) mix with every other function of a state:
  - each takes exactly one input column.  Per group, V is its values with NA cells (and NaN in a float column) skipped, m = |V| and
    v_0 <= ... <= v_{m-1} is V in the sort's order (-0.0 and 0.0 are one value).  A group with m = 0 gets NA; all outputs are nullable.
  - percentile_cont(q): h = q (m - 1), lo = floor(h), f = h - lo; v_lo when f == 0, else a + (b - a) f with a = v_lo, b = v_{lo+1} as
    float64 (pandas' linear quantile, bit for bit).  Integer and float columns; FLOAT64 output.  MEDIAN(x) is percentile_cont with
    q = 0.5 (the name "median" itself is not accepted).
  - percentile_disc(q): v_i with i = clamp(ceil(q m) - 1, 0, m - 1) (np.quantile(..., method="inverted_cdf")).  Integer, float,
    DATE, DATETIME and TIMEDELTA columns; the input's type.
  - mode: the most frequent value, ties to the least (Series.mode().iloc[0]).  Integer, float, bool and temporal columns; the
    input's type.
  - percentiles= (keyword-only) gives q (0 <= q <= 1) for each percentile_cont / percentile_disc entry of fnames, in order.
  - a result depends only on V (a zero comes back as +0.0): bit-identical across runs, batch splits, table growth and rank counts.
  - the state keeps a 4-byte group id and the value per non-NA value (one store per value column, at most 2^31 values each: a batch
    that could pass that raises and leaves the state usable) and sorts each store once, at the last batch.
  - sharded (parallel=True, more than one rank), such a state hash-partitions every batch by key before it consumes it (the
    raw-row form), so each rank aggregates only the groups it owns and nothing is exchanged at the end.  A state that also computes
    first / last, or has a 1- or 2-byte key column, cannot take that form: its first consume call raises.
"""

from __future__ import annotations

import numbers

from .. import _lib
from .._lib import ffi
from ..table import CTable, Table, np_dtype_of, table_from_ctable

# names must match supported_agg_funcs positions / Bodo_FTypes (groupby/_groupby_ftypes.h:17-110).  28..34 and 38..40 continue the
# enum after skew in the reference's order; they are recalled, not read from a reference checkout (17 and 26 are fixed by their
# neighbours).
FTYPES = {"size": 4, "sum": 6, "count": 7, "nunique": 8, "mean": 14, "min": 15, "max": 16, "prod": 17, "first": 18, "last": 19,
          "var_pop": 22, "std_pop": 23, "var": 24, "std": 25, "kurtosis": 26, "skew": 27, "boolor_agg": 28, "booland_agg": 29,
          "boolxor_agg": 30, "bitor_agg": 31, "bitand_agg": 32, "bitxor_agg": 33, "count_if": 34, "mode": 38, "percentile_cont": 39,
          "percentile_disc": 40}
HOLISTIC = ("mode", "percentile_cont", "percentile_disc")  # need every value of a group: kept per group, sorted at finalize
PERCENTILES = ("percentile_cont", "percentile_disc")       # take one fraction each (init_groupby_state's percentiles=)
MRNF = "min_row_number_filter"
MRNF_MAX_SORT, MRNF_MAX_KEEP = 4, 26
MRNF_MAX_LIMIT = 1 << 31  # mrnf_limit < 2^31 (the candidate store's sort holds at most 2^31 rows)
_FIXED_WIDTH = {0, 1, 2, 3, 4, 5, 6, 7, 8, 9, 11, 13, 15, 16}  # CTypes with a fixed-width cell (integers, floats, bool, temporals)


def _mrnf_spec(key_inds, fnames, f_in_offsets, f_in_cols, sort_inds, asc, na, keep):
    """The validated MRNF arguments as (sort_inds, asc, na, keep), or None for an ordinary aggregation."""
    args = {"mrnf_sort_col_inds": sort_inds, "mrnf_sort_col_asc": asc, "mrnf_sort_col_na": na, "mrnf_col_inds_keep": keep}
    given = [k for k, v in args.items() if v is not None]
    if MRNF not in fnames:
        if given:
            raise _lib.B200Error(f"Streaming Groupby: {', '.join(given)} belong to min_row_number_filter, which must then be the only "
                                 f"function (fnames={tuple(fnames)})")
        return None
    if tuple(fnames) != (MRNF,):
        raise _lib.B200Error(f"Streaming Groupby: min_row_number_filter cannot be combined with other functions (fnames={tuple(fnames)})")
    missing = [k for k, v in args.items() if v is None]
    if missing:
        raise _lib.B200Error(f"Streaming Groupby: min_row_number_filter needs {', '.join(missing)}")

    def indices(name, v, lo, hi):
        v = tuple(v)
        if not lo <= len(v) <= hi:
            raise _lib.B200Error(f"Streaming Groupby: {name} must have {lo} to {hi} entries (got {len(v)})")
        if any(isinstance(x, bool) or int(x) != x or x < 0 for x in v):
            raise _lib.B200Error(f"Streaming Groupby: {name} must hold non-negative column indices (got {v})")
        v = tuple(int(x) for x in v)
        if len(set(v)) != len(v):
            raise _lib.B200Error(f"Streaming Groupby: {name} lists a column twice (got {v})")
        return v

    sort = indices("mrnf_sort_col_inds", sort_inds, 1, MRNF_MAX_SORT)
    flags = []
    for name, v in (("mrnf_sort_col_asc", asc), ("mrnf_sort_col_na", na)):
        v = tuple(v)
        if len(v) != len(sort):
            raise _lib.B200Error(f"Streaming Groupby: {name} must have one entry per sort column ({len(sort)}, got {len(v)})")
        flags.append(tuple(bool(x) for x in v))
    kept = indices("mrnf_col_inds_keep", keep, 1, MRNF_MAX_KEEP)
    f_in_offsets, f_in_cols = tuple(f_in_offsets), tuple(f_in_cols)
    if f_in_offsets != (0, len(f_in_cols)):
        raise _lib.B200Error(f"Streaming Groupby: min_row_number_filter needs f_in_offsets == (0, len(f_in_cols)) (got {f_in_offsets})")
    if any(int(c) in key_inds or c < 0 for c in f_in_cols):
        raise _lib.B200Error(f"Streaming Groupby: min_row_number_filter's f_in_cols must be non-key columns (got {f_in_cols})")
    return sort, flags[0], flags[1], kept


def _percentile_fractions(fnames, f_in_offsets, percentiles):
    """One fraction per function (NaN for the functions that take none) from percentiles=, validated, or None without one."""
    f_in_offsets = tuple(int(x) for x in f_in_offsets)
    for j, f in enumerate(fnames):
        if f in HOLISTIC and len(f_in_offsets) == len(fnames) + 1 and f_in_offsets[j + 1] - f_in_offsets[j] != 1:
            raise _lib.B200Error(f"Streaming Groupby: {f} takes exactly one input column (function {j})")
    n_pct = sum(f in PERCENTILES for f in fnames)
    if percentiles is None:
        if n_pct:
            raise _lib.B200Error(f"Streaming Groupby: percentiles must give one fraction per percentile_cont / percentile_disc "
                                 f"({n_pct} in fnames={tuple(fnames)})")
        return None
    if not n_pct:
        raise _lib.B200Error(f"Streaming Groupby: percentiles needs a percentile_cont or percentile_disc function (fnames={tuple(fnames)})")
    if isinstance(percentiles, (str, bytes)) or not hasattr(percentiles, "__len__") or len(percentiles) != n_pct:
        raise _lib.B200Error(f"Streaming Groupby: percentiles must be a sequence of one fraction per percentile_cont / percentile_disc "
                             f"({n_pct}, got {percentiles!r})")
    qs = []
    for q in percentiles:
        if isinstance(q, bool) or not isinstance(q, numbers.Real) or not 0.0 <= float(q) <= 1.0:  # (NaN fails the range test)
            raise _lib.B200Error(f"Streaming Groupby: percentiles entries must be numbers in [0, 1] (got {q!r})")
        qs.append(float(q))
    it = iter(qs)
    return tuple(next(it) if f in PERCENTILES else float("nan") for f in fnames)


class GroupbyState:
    """Python handle of the C GroupbyState (created lazily at the first consume call)."""

    mrnf = None  # (sort_inds, asc, na_last, keep) of a min_row_number_filter state
    mrnf_limit = 1  # rows kept per group by a min_row_number_filter state
    fractions = None  # one per function (NaN where none applies) when some function is a percentile

    def __init__(self, operator_id, key_inds, fnames, f_in_offsets, f_in_cols, parallel, dropna, output_batch_size,
                 expected_groups, device, stream, process_group):
        self.operator_id = int(operator_id)
        self.key_inds = tuple(int(k) for k in key_inds)
        self.fnames = tuple(fnames)
        for f in self.fnames:
            if f not in FTYPES:
                raise _lib.B200Error(
                    f"Streaming Groupby: unsupported aggregate function '{f}' (supported: {sorted(FTYPES)})")
        self.f_in_offsets = tuple(int(x) for x in f_in_offsets)
        self.f_in_cols = tuple(int(x) for x in f_in_cols)
        if len(self.f_in_offsets) != len(self.fnames) + 1:
            raise _lib.B200Error("Streaming Groupby: f_in_offsets must have len(fnames) + 1 entries")
        self.parallel = bool(parallel)
        self.dropna = bool(dropna)
        self.output_batch_size = int(output_batch_size)
        self.expected_groups = int(expected_groups)
        self.device = device
        self.stream = int(stream)
        self.process_group = process_group
        self.handle = None
        self.build_indices = None  # physical column order: keys first (as the reference's build_indices)
        self.out_names = None
        self._out_cols = None
        self._out_tab = None
        self.exchanged = False

    # -- lazy C state creation once the input schema is known
    def _ensure(self, table: Table):
        if self.handle is not None:
            return
        L = _lib.lib()
        _lib.require_gpu()
        n = table.n_cols
        others = [i for i in range(n) if i not in self.key_inds]
        self.build_indices = list(self.key_inds) + others
        remap = {logical: phys for phys, logical in enumerate(self.build_indices)}
        cols = [table.columns[i] for i in self.build_indices]
        c_types = ffi.new("int8_t[]", [c.c_type for c in cols])
        a_types = ffi.new("int8_t[]", [c.arr_type for c in cols])
        if self.device is None:
            self.device = table.device if table.device >= 0 else _current_device()
        if self.mrnf is not None:
            self._init_mrnf(table, remap, c_types, a_types)
            return
        phys_f_in_cols = [remap[c] for c in self.f_in_cols]
        ftypes = ffi.new("int32_t[]", [FTYPES[f] for f in self.fnames] or [0])
        offs = ffi.new("int32_t[]", list(self.f_in_offsets))
        fcols = ffi.new("int32_t[]", phys_f_in_cols or [0])
        n_pes, rank = 1, 0
        if self.parallel:
            import torch.distributed as dist

            n_pes, rank = dist.get_world_size(self.process_group), dist.get_rank(self.process_group)
        self.n_pes, self.rank = n_pes, rank
        self.stays_partial = "first" in self.fnames or "last" in self.fnames or any(
            np_dtype_of(c.c_type).itemsize < 4 for c in cols[:len(self.key_inds)])
        self.holistic = any(f in HOLISTIC for f in self.fnames)
        if self.holistic and self.parallel and n_pes > 1:
            # mode / percentiles do not combine as partial aggregates: the raw-row form from the first batch on (every rank
            # aggregates only the groups it owns), or nothing
            if self.stays_partial:
                cause = ("first / last in the same state (their row order is the rank-major one of partial aggregates)"
                         if "first" in self.fnames or "last" in self.fnames else "a 1- or 2-byte key column (not hash-partitioned)")
                raise _lib.B200Error(f"Streaming Groupby: a sharded state with mode / percentile_cont / percentile_disc hash-partitions "
                                     f"its rows by key before aggregating them, which {cause} rules out")
            self.shuffle_decided = self.raw_row_mode = True
        fractions = ffi.new("double[]", list(self.fractions)) if self.fractions is not None else ffi.NULL
        h = L.b200_groupby_state_init_percentiles(self.operator_id, c_types, a_types, len(cols), ftypes, offs, fcols,
                                                  len(self.fnames), len(self.key_inds), self.output_batch_size,
                                                  int(self.parallel and n_pes > 1), int(self.dropna), self.device, n_pes, rank,
                                                  self.expected_groups, ffi.cast("void*", self.stream), fractions)
        self.handle = _lib.check_ptr(h, "init_groupby_state")
        key_names = [table.names[i] for i in self.key_inds]
        fn_names = []
        for j, f in enumerate(self.fnames):
            lo, hi = self.f_in_offsets[j], self.f_in_offsets[j + 1]
            fn_names.append(table.names[self.f_in_cols[lo]] if hi > lo else f)
        # output names must be unique: a column aggregated more than once gets a _<func> suffix
        seen = set(key_names)
        uniq = []
        for f, nm in zip(self.fnames, fn_names):
            cand, k = nm, 0
            while cand in seen:
                cand = f"{nm}_{f}" if k == 0 else f"{nm}_{f}{k}"
                k += 1
            seen.add(cand)
            uniq.append(cand)
        self.out_names = key_names + uniq

    def _init_mrnf(self, table: Table, remap, c_types, a_types):
        """Creates the C state of a min_row_number_filter once the schema is known (the sharded case was refused before)."""
        L = _lib.lib()
        sort, asc, na_last, keep = self.mrnf
        n = table.n_cols
        for name, inds in (("key_inds", self.key_inds), ("mrnf_sort_col_inds", sort), ("mrnf_col_inds_keep", keep),
                           ("f_in_cols", self.f_in_cols)):
            bad = [i for i in inds if i >= n]
            if bad:
                raise _lib.B200Error(f"Streaming Groupby: {name} {bad} out of range for a batch of {n} columns")
        for what, inds in (("key", self.key_inds), ("sort", sort), ("kept", keep)):
            for i in inds:
                if table.columns[i].c_type not in _FIXED_WIDTH:
                    raise _lib.B200Error(f"Streaming Groupby: min_row_number_filter {what} column '{table.names[i]}' is not a fixed-width "
                                         f"column (c_type {table.columns[i].c_type})")
        self.n_pes, self.rank = 1, 0
        keep_mask = [0] * n
        for i in keep:
            keep_mask[remap[i]] = 1
        h = L.b200_groupby_state_init_mrnf_limit(self.operator_id, c_types, a_types, n, len(self.key_inds),
                                                 ffi.new("int32_t[]", [remap[i] for i in sort]), ffi.new("int32_t[]", [int(x) for x in asc]),
                                                 ffi.new("int32_t[]", [int(x) for x in na_last]), len(sort), ffi.new("int32_t[]", keep_mask),
                                                 self.output_batch_size, 0, int(self.dropna), self.device, 1, 0, self.expected_groups,
                                                 ffi.cast("void*", self.stream), self.mrnf_limit)
        self.handle = _lib.check_ptr(h, "init_groupby_state (min_row_number_filter)")
        # the library returns the kept columns in physical order (keys first); the output lists them in input order
        phys = sorted(remap[i] for i in keep)
        self._mrnf_order = [phys.index(remap[i]) for i in sorted(keep)]
        self.out_names = [table.names[self.build_indices[p]] for p in phys]

    # ---- reduce-or-shuffle (reference: GroupbyIncrementalShuffleState::ShouldShuffleAfterProcessing,
    # bodo/libs/streaming/_groupby.cpp:1655-1711: an HLL estimate of how many NEW groups the pending rows hold decides whether they are
    # pre-reduced locally or shuffled as they are; threshold agg_reduction_threshold = 0.85, :1556) ----
    # Here every batch is aggregated into the local table first (that is the fast kernel), so the uniqueness is measured, not
    # estimated: groups in the tables / rows consumed, summed over the ranks.  While it stays below the threshold the ranks keep
    # pre-aggregating and exchange PARTIAL AGGREGATES once, at the end.  Above it (groups ~ rows: pre-aggregation buys nothing, the
    # table of every rank would grow towards its share of ALL rows and the one final exchange would move them all at once) the
    # state switches to the raw-row form: every further batch is hash-partitioned (b200_shuffle_partition) and exchanged right away
    # (all-to-all-v), each rank aggregates only rows of groups it owns, and the final exchange only carries what was aggregated
    # before the switch.  Collective: decided once, from the first >= B200_SHUFFLE_DECISION_ROWS rows, identically on every rank.
    # A state that computes first or last never switches: a raw row is numbered by the rank that consumes it (its owner), not by
    # the rank it came from, so after the switch first / last would no longer follow the rank-major order (rows of a lower rank
    # first, then row order) that the partial-aggregate form keeps.  Nor does a state with a 1- or 2-byte key column (int8,
    # uint8, int16, uint16, bool), which shuffle_table does not partition.
    raw_row_mode = False
    shuffle_decided = False
    stays_partial = False
    holistic = False  # some function is mode / percentile_cont / percentile_disc: sharded, the raw-row form from the first batch
    raw_rows_shuffled = 0

    def _decide_reduce_or_shuffle(self):
        import os

        import torch
        import torch.distributed as dist

        if self.stays_partial:  # (the same on every rank: no collective needed)
            self.shuffle_decided = True
            return
        L = _lib.lib()
        dev = torch.device("cuda", self.device)
        t = torch.tensor([int(L.b200_groupby_get_metric(self.handle, 13)), int(L.b200_groupby_get_metric(self.handle, 2))], dtype=torch.int64, device=dev)
        dist.all_reduce(t, group=self.process_group)
        groups, rows = (int(x) for x in t.tolist())
        if rows < int(os.environ.get("B200_SHUFFLE_DECISION_ROWS", 1 << 22)):
            return
        thr = min(1.0, max(0.0, float(os.environ.get("BODO_STREAM_GROUPBY_AGG_REDUCTION_THRESHOLD", os.environ.get("B200_AGG_REDUCTION_THRESHOLD", 0.85)))))
        self.shuffle_decided = True
        self.raw_row_mode = rows > 0 and groups / rows >= thr
        self.local_uniqueness = groups / max(rows, 1)

    def _shuffle_rows(self, phys: Table) -> Table:
        import torch

        from ..shuffle import shuffle_table
        from ..table import to_device

        dev_tab = to_device(phys, self.device)
        stream = torch.cuda.ExternalStream(self.stream) if self.stream else torch.cuda.default_stream(self.device)
        with torch.cuda.stream(stream):
            out = shuffle_table(dev_tab, len(self.key_inds), True, group=self.process_group, stream=self.stream)
        self.raw_rows_shuffled += phys.n_rows
        return out

    def _exchange(self):
        """Hash-partition exchange of the partial aggregates after the last local batch: first every nested nunique state (a
        key's (key, value) pairs are owned where the key is owned), then the outer state, each finalized after its exchange."""
        import os
        import time

        import torch

        from . import exchange as X

        L = _lib.lib()
        h = self.handle
        t0 = time.perf_counter()
        slabs = X.get_slabs(self.process_group, self.device)
        for i in range(int(L.b200_groupby_num_inner_states(h))):
            self._exchange_state(_lib.check_ptr(L.b200_groupby_inner_state(h, i), "groupby nunique"), slabs)
        self.exchange_path, self.shuffle_bytes = self._exchange_state(h, slabs)
        self.exchanged = True
        if os.environ.get("B200_TRACE") and self.rank == 0:
            torch.cuda.synchronize()
            print(f"[b200 exchange ms] {self.exchange_path} exchange + finalize = {(time.perf_counter() - t0) * 1e3:.3f}", flush=True)

    def _exchange_state(self, h, slabs):
        """Exchanges and finalizes one C state; returns (path, bytes sent through NCCL or None).

        Fused form (when symmetric memory is available): ONE kernel packs every partial row another rank owns straight into that
        rank's receive slab over NVLink (streaming/exchange.py), a device-side barrier, one combine kernel — no count exchange, no
        send buffer, no host synchronisation before finalize.  NCCL form (no slabs, or finalize reported -2: a rank's share did
        not fit its slab segment): count all-gather + one all-to-all-v of the packed rows, then the same combine."""
        import torch
        import torch.distributed as dist

        from . import exchange as X

        L = _lib.lib()
        null = ffi.NULL
        row_bytes = int(L.b200_groupby_exchange_row_bytes(h))
        if slabs is not None:
            cap_rows = (slabs.slab_bytes - X.HDR_BYTES) // (self.n_pes * row_bytes)
            peers_dev, my_slab, hdl = slabs.next()
            stream = torch.cuda.ExternalStream(self.stream) if self.stream else torch.cuda.default_stream(self.device)
            with torch.cuda.stream(stream):
                _lib.check(L.b200_groupby_exchange_pack(h, ffi.cast("void* const*", peers_dev), cap_rows, null), "groupby exchange (pack)")
                hdl.barrier(channel=0)
                _lib.check(L.b200_groupby_exchange_combine(h, ffi.cast("void*", my_slab), cap_rows, null), "groupby exchange (combine)")
            rc = int(L.b200_groupby_finalize(h))
            if rc != -2:
                _lib.check(rc, "groupby finalize")
                return "fused", None
            # (the fused pack counted every destination's rows exactly)
        else:
            _lib.check(L.b200_groupby_exchange_pack(h, null, 0, null), "groupby exchange (count)")
        counts = ffi.new("int64_t[]", self.n_pes)
        _lib.check(L.b200_groupby_exchange_counts(h, counts), "groupby exchange (counts)")
        send_counts = list(counts)
        dev = torch.device("cuda", self.device)
        words = row_bytes // 8
        n_send = sum(send_counts)
        # counts travel as one small all-gather of the n_pes x n_pes matrix (mpi_comm_info's MPI_Alltoall,
        # _shuffle.cpp:210-213), issued asynchronously so it overlaps the pack kernel
        allc = torch.empty(self.n_pes * self.n_pes, dtype=torch.int64, device=dev)
        work = dist.all_gather_into_tensor(allc, torch.tensor(send_counts, dtype=torch.int64, device=dev), group=self.process_group, async_op=True)
        send = torch.empty((max(n_send, 1), words), dtype=torch.int64, device=dev)
        _lib.check(L.b200_groupby_exchange_pack(h, null, 0, ffi.cast("void*", send.data_ptr())), "groupby exchange (pack)")
        work.wait()
        recv_counts = allc.view(self.n_pes, self.n_pes)[:, self.rank].tolist()
        n_recv = sum(recv_counts)
        recv = torch.empty((max(n_recv, 1), words), dtype=torch.int64, device=dev)
        dist.all_to_all_single(recv[:n_recv], send[:n_send], output_split_sizes=recv_counts,
                               input_split_sizes=send_counts, group=self.process_group)
        torch.cuda.current_stream(dev).synchronize()
        _lib.check(L.b200_groupby_exchange_combine(h, ffi.cast("void*", recv.data_ptr()), 0, ffi.new("int64_t[]", recv_counts)),
                   "groupby exchange (combine)")
        _lib.check(int(L.b200_groupby_finalize(h)), "groupby finalize")  # (reads `recv`: rows that found the table full)
        return "nccl", n_send * row_bytes


def _current_device() -> int:
    import torch

    return torch.cuda.current_device()


def init_groupby_state(operator_id, key_inds, fnames, f_in_offsets, f_in_cols, mrnf_sort_col_inds=None,
                       mrnf_sort_col_asc=None, mrnf_sort_col_na=None, mrnf_col_inds_keep=None, op_pool_size_bytes=-1,
                       parallel=False, *, dropna=True, output_batch_size=32768, expected_groups=0, device=None,
                       stream=0, process_group=None, mrnf_limit=1, percentiles=None) -> GroupbyState:
    """Mirror of bodo.libs.streaming.groupby.init_groupby_state (groupby.py:702-715).

    key_inds / f_in_cols index the logical input table; fnames are names from supported_agg_funcs, or
    ("min_row_number_filter",) with the four mrnf_* arguments (see the module docstring; a bad length, index, duplicate, an empty
    keep list, MRNF arguments beside other functions or min_row_number_filter without them raise B200Error naming the argument).
    op_pool_size_bytes is ignored (the table is sized in HBM, there is no host operator pool).
    Keyword-only extras: dropna (pandas_drop_na of the C++ ctor), output_batch_size, expected_groups
    (sizing hint), device, stream (cudaStream_t as int), process_group (torch.distributed), mrnf_limit (rows kept per group by
    min_row_number_filter, see the module docstring; a bool, a non-integer, a value < 1 or >= 2^31, or a value other than 1
    without min_row_number_filter raise B200Error naming mrnf_limit), percentiles (one fraction q in [0, 1] per percentile_cont /
    percentile_disc entry of fnames, in order; a missing or wrong-length sequence, a bool, NaN or out-of-range entry, or percentiles
    without such a function raise B200Error naming percentiles; mode and the percentiles take exactly one input column).
    """
    key_inds = getattr(key_inds, "meta", key_inds)
    fnames = tuple(getattr(fnames, "meta", fnames))
    f_in_offsets = getattr(f_in_offsets, "meta", f_in_offsets)
    f_in_cols = getattr(f_in_cols, "meta", f_in_cols)
    mrnf = [getattr(x, "meta", x) for x in (mrnf_sort_col_inds, mrnf_sort_col_asc, mrnf_sort_col_na, mrnf_col_inds_keep)]
    spec = _mrnf_spec(tuple(int(k) for k in key_inds), fnames, f_in_offsets, f_in_cols, *mrnf)
    if isinstance(mrnf_limit, bool) or not isinstance(mrnf_limit, numbers.Integral) or not 1 <= mrnf_limit < MRNF_MAX_LIMIT:
        raise _lib.B200Error(f"Streaming Groupby: mrnf_limit must be an integer in [1, 2^31) (got {mrnf_limit!r})")
    if spec is None and mrnf_limit != 1:
        raise _lib.B200Error(f"Streaming Groupby: mrnf_limit={mrnf_limit} needs min_row_number_filter (fnames={fnames})")
    fractions = _percentile_fractions(fnames, f_in_offsets, getattr(percentiles, "meta", percentiles))
    if spec is None:
        st = GroupbyState(operator_id, key_inds, fnames, f_in_offsets, f_in_cols, parallel, dropna, output_batch_size,
                          expected_groups, device, stream, process_group)
        st.fractions = fractions
        return st
    st = GroupbyState(operator_id, key_inds, (), (0,), (), parallel, dropna, output_batch_size, expected_groups, device, stream,
                      process_group)
    st.mrnf = spec
    st.mrnf_limit = int(mrnf_limit)
    st.f_in_cols = tuple(int(c) for c in f_in_cols)
    return st


MRNF_MAX_RECEIVE_ROWS = 1 << 31  # winners one rank may receive: the candidate store's sort holds at most 2^31 rows


def _mrnf_state(operator_id, key_inds, spec, mrnf_limit, dropna, output_batch_size, device, stream):
    """A local min_row_number_filter state of a validated spec (sort_inds, asc, na_last, keep)."""
    st = GroupbyState(operator_id, key_inds, (), (0,), (), False, dropna, output_batch_size, 0, device, stream, None)
    st.mrnf = spec
    st.mrnf_limit = mrnf_limit
    return st


class ShardedMrnfState:
    """Python handle of a sharded min_row_number_filter (init_sharded_mrnf_state).  `local` keeps this rank's winners over the union
    of the key, sort and kept columns; at is_last the winners are exchanged by key and `final` keeps the winners of the groups this
    rank owns (with one rank, `local` keeps the caller's columns and is the result)."""

    def __init__(self, operator_id, key_inds, sort_inds, sort_asc, sort_na, keep_inds, dropna, mrnf_limit, output_batch_size, device,
                 stream, process_group):
        key_inds = tuple(int(k) for k in getattr(key_inds, "meta", key_inds))
        sort, asc, na_last, keep = _mrnf_spec(key_inds, (MRNF,), (0, 0), (), sort_inds, sort_asc, sort_na, keep_inds)
        if isinstance(mrnf_limit, bool) or not isinstance(mrnf_limit, numbers.Integral) or not 1 <= mrnf_limit < MRNF_MAX_LIMIT:
            raise _lib.B200Error(f"Streaming Groupby: mrnf_limit must be an integer in [1, 2^31) (got {mrnf_limit!r})")
        self.union = sorted(set(key_inds) | set(sort) | set(keep))
        if len(self.union) > MRNF_MAX_KEEP:
            raise _lib.B200Error(f"Streaming Groupby: a sharded min_row_number_filter keeps the union of the keys {list(key_inds)}, the sort "
                                 f"columns {list(sort)} and the kept columns {list(keep)} until its exchange: {len(self.union)} columns "
                                 f"{self.union}, more than {MRNF_MAX_KEEP}")
        self.spec = (sort, asc, na_last, keep)
        self.args = (operator_id, key_inds, int(mrnf_limit), bool(dropna))
        self.output_batch_size = int(output_batch_size)
        self.device, self.stream = device, int(stream)
        self.process_group = process_group
        # the winners leave `local` as one batch (output_batch_size 0)
        self.local = _mrnf_state(operator_id, key_inds, (sort, asc, na_last, tuple(self.union)), int(mrnf_limit), dropna, 0, device, stream)
        self.final = None
        self.n_ranks = None

    def consume(self, table: Table, is_last: bool):
        if self.n_ranks is None:
            from .sort import _world

            self.n_ranks, self.rank = _world(self.process_group)
            if self.n_ranks == 1:
                self.local.mrnf, self.local.output_batch_size = self.spec, self.output_batch_size
        res = groupby_build_consume_batch(self.local, table, is_last)
        if is_last:
            self.final = self.local if self.n_ranks == 1 else self._exchange()
        return res

    def _exchange(self):
        """Partition the local winners by key class, exchange them and keep the winners of the groups this rank owns."""
        import torch

        from ..shuffle import exchange_table, partition_device, with_schema_validity
        from ..table import Column
        from .sort import agree_receive_rows

        loc, union = self.local, self.union
        operator_id, key_inds, limit, dropna = self.args
        dev = torch.device("cuda", loc.device)
        out, _ = groupby_produce_output_batch(loc, True)  # every winner, the union's columns in input order
        n = out.n_rows
        cols = []
        for c in out.columns:  # library-owned device columns: wrapped, not copied (an empty one has no address to wrap)
            data = torch.as_tensor(c.data, device=dev) if n else torch.empty(0, dtype=getattr(torch, str(np_dtype_of(c.c_type))), device=dev)
            v = torch.as_tensor(c.validity, device=dev) if n and c.validity is not None else None
            cols.append(Column(data, v, c.c_type, c.arr_type, n))
        kp = [union.index(k) for k in key_inds]
        order = kp + [j for j in range(len(union)) if j not in kp]  # the keys lead
        part, send = partition_device(with_schema_validity(Table(cols, list(out.names)).select(order)), len(kp), self.n_ranks,
                                      loc.stream, by_class=True)
        agree_receive_rows(send, dev, self.process_group, cap=MRNF_MAX_RECEIVE_ROWS,
                           what="Streaming Groupby: sharded min_row_number_filter", cap_name="the min_row_number_filter's cap")
        got = exchange_table(part, send, self.process_group)
        torch.cuda.synchronize(dev)
        delete_groupby_state(loc)  # the winners have been sent
        got = got.select([order.index(j) for j in range(len(union))])
        sort, asc, na_last, keep = self.spec
        spec = (tuple(union.index(i) for i in sort), asc, na_last, tuple(union.index(i) for i in keep))
        fin = _mrnf_state(operator_id, tuple(kp), spec, limit, dropna, self.output_batch_size, loc.device, self.stream)
        groupby_build_consume_batch(fin, got, True)
        return fin


def init_sharded_mrnf_state(operator_id, key_inds, mrnf_sort_col_inds, mrnf_sort_col_asc, mrnf_sort_col_na, mrnf_col_inds_keep, *,
                            dropna=True, mrnf_limit=1, output_batch_size=32768, device=None, stream=0,
                            process_group=None) -> ShardedMrnfState:
    """A sharded min_row_number_filter over a torch.distributed process group (one process per GPU), driven by the groupby verbs:
    the rows all ranks produce are, as a multiset, the MRNF (init_groupby_state's min_row_number_filter with these arguments) of the
    rank inputs concatenated in rank order, bit for bit; of rows that tie on every sort column the lower rank wins.  Each group's
    rows come out on one rank; with mrnf_limit > 1 they are consecutive and in rank order.  Consume calls before is_last are local;
    the is_last call is collective (every rank passes is_last=True in the same call) and raises the same B200Error on every rank
    when a rank would receive MRNF_MAX_RECEIVE_ROWS winners or more.  Raises B200Error for the arguments init_groupby_state refuses
    and when the union of the key, sort and kept columns, which every rank keeps until the exchange, exceeds 26 columns.  Without
    torch.distributed, or with one rank, it is the local min_row_number_filter."""
    return ShardedMrnfState(operator_id, key_inds, mrnf_sort_col_inds, mrnf_sort_col_asc, mrnf_sort_col_na, mrnf_col_inds_keep, dropna,
                            mrnf_limit, output_batch_size, device, stream, process_group)


def groupby_build_consume_batch(groupby_state: GroupbyState, table: Table, is_last: bool, is_final_pipeline: bool = True):
    """Mirror of groupby_build_consume_batch (groupby.py:1295-1395): returns (is_last, request_input).

    Collective when the state is parallel: every rank must pass is_last=True in the same call (ranks that
    ran out of input keep calling with empty batches, as in the reference's pipeline loop,
    bodo/pandas/_pipeline.cpp:453-457)."""
    st = groupby_state
    if isinstance(st, ShardedMrnfState):
        if st.final is not None:
            raise _lib.B200Error("groupby_build_consume_batch called after is_last")
        return st.consume(table, is_last)
    if st.mrnf is not None and st.parallel and st.handle is None:
        import torch.distributed as dist

        if dist.is_initialized() and dist.get_world_size(st.process_group) > 1:
            raise _lib.B200Error("Streaming Groupby: a sharded min_row_number_filter is not supported (process group of more than one "
                                 "rank)")
    st._ensure(table)
    L = _lib.lib()
    phys = table.select(st.build_indices)
    sharded = st.parallel and st.n_pes > 1
    if sharded and st.raw_row_mode:
        phys = st._shuffle_rows(phys)  # this rank's share of every rank's batch: all of its rows are owned here
    ct = CTable(phys)
    req = ffi.new("int32_t*")
    rc = _lib.check(L.b200_groupby_build_consume_batch(st.handle, ct.ptr, int(bool(is_last)), int(bool(is_final_pipeline)), req),
                    "groupby_build_consume_batch")
    if sharded and not is_last and not st.shuffle_decided:
        st._decide_reduce_or_shuffle()
    if is_last and sharded and not st.exchanged and not st.holistic:  # (a holistic state holds only groups it owns)
        st._exchange()
    return bool(rc), bool(req[0])


def groupby_produce_output_batch(groupby_state: GroupbyState, produce_output: bool = True):
    """Mirror of groupby_produce_output_batch (groupby.py:1502-1600): returns (out_table, is_last).
    The returned Table wraps library-owned device columns that stay valid until the next produce call.  A sharded
    min_row_number_filter produces the winners of the groups this rank owns."""
    st = groupby_state
    if isinstance(st, ShardedMrnfState):
        if st.final is None:
            raise _lib.B200Error("groupby_produce_output_batch called before the last batch was consumed")
        st = st.final
    if st.handle is None:
        raise _lib.B200Error("groupby_produce_output_batch called before any build batch was consumed")
    L = _lib.lib()
    ncols = len(st.out_names)
    st._out_cols = ffi.new("b200_column[]", ncols)
    st._out_tab = ffi.new("b200_table*")
    st._out_tab.cols = st._out_cols
    last = ffi.new("int32_t*")
    _lib.check(L.b200_groupby_produce_output_batch(st.handle, st._out_tab, last, int(bool(produce_output))),
               "groupby_produce_output_batch")
    out = table_from_ctable(st._out_tab, ncols, st.out_names, owner=st)
    if st.mrnf is not None:
        out = out.select(st._mrnf_order)
    return out, bool(last[0])


def delete_groupby_state(groupby_state: GroupbyState) -> None:
    if isinstance(groupby_state, ShardedMrnfState):
        for s in (groupby_state.local, groupby_state.final):
            if s is not None:
                delete_groupby_state(s)
        return
    if groupby_state.handle is not None:
        _lib.lib().b200_delete_groupby_state(groupby_state.handle)
        groupby_state.handle = None


def get_metric(groupby_state: GroupbyState, which: int) -> int:
    """A sharded min_row_number_filter reports its local state before is_last and the state its output comes from after it."""
    if isinstance(groupby_state, ShardedMrnfState):
        groupby_state = groupby_state.final or groupby_state.local
    return int(_lib.lib().b200_groupby_get_metric(groupby_state.handle, which))
