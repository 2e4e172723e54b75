"""Streaming sort operator API (ORDER BY ... LIMIT ... OFFSET, and ORDER BY without LIMIT) — the host-side mirror of
bodo/libs/streaming/sort.py.

Same verbs as the reference's streaming sort (init_stream_sort_state, sort_build_consume_batch, produce_output_batch,
delete_stream_sort_state).  LIMIT form: the result is rows [offset, offset + limit) of the input sorted stably by the `by`
columns, equal to

    df.assign(_seq=range(len(df))).sort_values([*by, "_seq"], ascending=[*asc, True], na_position=...).iloc[offset:offset + limit]

with one na_position per key.  The work happens in libbodo_b200.so (sort.cu): one filter kernel per batch against a
device-resident cutoff, and a device sort of the few surviving candidates.

Full form (full=True, no limit, no offset): every row, equal to df.sort_values(by, kind="stable").reset_index(drop=True).  Each
batch is appended to a device-resident chunk store, and is_last runs an LSD radix sort over it (sort.cu).  It is opt-in rather
than limit=None: the state holds the entire input in device memory, so a query that lost its LIMIT fails instead.

With parallel=True the state is one shard of a torch.distributed process group (one process per GPU): every rank reduces its
own stream to at most limit + offset rows, the ranks all-gather those rows at is_last, every rank runs them (rank-major) through
a fresh state, and rank 0 produces the result while the other ranks produce one empty batch.  The answer is the stable top-k
of the rank inputs concatenated in rank order.  A parallel full-sort state of init_stream_sort_state, whose contract would put the
whole result on rank 0, raises at its first consume call when the process group has more than one rank (with one rank it sorts
locally).

The sharded full sort is init_sharded_sort_state: each rank ends up holding one key range of the result.  Every rank sorts its
own rows (the full sort above) and, at is_last, draws min(SAMPLES_PER_RANK, n_r) samples of its sorted rows in the sort's own
key encoding (b200_sort_sample), tagged with (rank, position); the ranks all-gather them and each runs choose_splitters, a pure
function, so all pick the same P - 1 splitters.  A device binary search (b200_sort_count_below) turns the splitters into send
counts, which are agreed through one all_reduce (so a rank that would receive too many rows fails on every rank before any row
moves), and exchange_table sends each rank its contiguous slice of the sorted rows.  The receiver merges the P sorted runs it
got (b200_sort_state_init_runs) instead of sorting again.  DESIGN.md §3i derives the balance bound.
"""

from __future__ import annotations

import numpy as np

from .. import _lib
from .._lib import ffi
from ..table import Column, CTable, Table, table_from_ctable, to_device

MAX_KEYS = 4
# limit + offset cap: the store addresses rows with uint32 ids and keeps two buffers of max(2 (limit + offset), 4 Mi) rows
MAX_LIMIT_PLUS_OFFSET = 1 << 26
# full sort: rows per state (32-bit row ids whose top bit carries a key's NA class during its class pass)
MAX_FULL_SORT_ROWS = 1 << 31
# sharded full sort: samples each rank draws from its sorted rows, and the rows one rank may receive (the full sort's row ids)
SAMPLES_PER_RANK = 4096
MAX_SHARDED_RECEIVE_ROWS = MAX_FULL_SORT_ROWS


class SortState:
    """Python handle of the C sort state (created lazily at the first consume call)."""

    def __init__(self, operator_id, limit, offset, by, asc, na_position, col_names, parallel, output_batch_size, device, stream,
                 process_group, full=False):
        self.full = bool(full)
        if self.full:
            if limit is not None or offset not in (None, 0):
                raise _lib.B200Error(f"Streaming Sort: a full sort takes no limit or offset (got limit={limit}, offset={offset})")
            limit = offset = 0
        elif limit is None:
            raise _lib.B200Error("Streaming Sort: a limit is required (a full sort without LIMIT is not supported)")
        limit, offset = int(limit), int(offset or 0)
        if limit < 0 or offset < 0:
            raise _lib.B200Error(f"Streaming Sort: limit ({limit}) and offset ({offset}) must be non-negative")
        if limit + offset > MAX_LIMIT_PLUS_OFFSET:
            raise _lib.B200Error(f"Streaming Sort: limit + offset = {limit + offset} exceeds the top-k cap of {MAX_LIMIT_PLUS_OFFSET} rows")
        by = [by] if isinstance(by, str) else list(by)
        if not 1 <= len(by) <= MAX_KEYS:
            raise _lib.B200Error(f"Streaming Sort: 1 to {MAX_KEYS} sort keys (got {len(by)})")
        col_names = [str(c) for c in col_names]
        missing = [k for k in by if k not in col_names]
        if missing or len(set(by)) != len(by):
            raise _lib.B200Error(f"Streaming Sort: sort keys {by} must be distinct columns of {col_names}")
        asc = [asc] * len(by) if isinstance(asc, bool) else [bool(a) for a in asc]
        nap = [na_position] * len(by) if isinstance(na_position, str) else list(na_position)
        if len(asc) != len(by) or len(nap) != len(by):
            raise _lib.B200Error("Streaming Sort: ascending and na_position need one entry per sort key")
        if any(p not in ("first", "last") for p in nap):
            raise _lib.B200Error(f"Streaming Sort: na_position must be 'first' or 'last' (got {nap})")
        self.operator_id = int(operator_id)
        self.limit, self.offset = limit, offset
        self.by, self.asc, self.na_last = by, asc, [p == "last" for p in nap]
        self.col_names = col_names
        # physical column order: keys first (the reference's keys-first convention), then the other columns
        self.key_inds = [col_names.index(k) for k in by]
        self.phys = self.key_inds + [i for i in range(len(col_names)) if i not in self.key_inds]
        self.out_order = [self.phys.index(i) for i in range(len(col_names))]
        self.out_names = [col_names[i] for i in self.phys]  # the produced columns, in physical order
        self.parallel = bool(parallel)
        self.output_batch_size = int(output_batch_size)
        self.device = device
        self.stream = int(stream)
        self.process_group = process_group
        self.handle = None
        self.global_state = None  # parallel: the state the gathered rows go through
        self.runs = None  # the run lengths of a state that merges sorted runs (the sharded full sort's receiver)
        self.done = False

    def _ensure(self, table: Table, limit=None, offset=None):
        if self.handle is not None:
            return
        L = _lib.lib()
        _lib.require_gpu()
        if table.n_cols != len(self.col_names):
            raise _lib.B200Error(f"Streaming Sort: the batch has {table.n_cols} columns, the state {len(self.col_names)}")
        if self.device is None:
            self.device = table.device if table.device >= 0 else _current_device()
        cols = [table.columns[i] for i in self.phys]
        c_types = ffi.new("int8_t[]", [c.c_type for c in cols])
        a_types = ffi.new("int8_t[]", [c.arr_type for c in cols])
        asc = ffi.new("int32_t[]", [int(a) for a in self.asc])
        nal = ffi.new("int32_t[]", [int(x) for x in self.na_last])
        lim = self.limit if limit is None else limit
        off = self.offset if offset is None else offset
        self.handle = self._new_handle(L, c_types, a_types, len(cols), asc, nal, lim, off)

    def _new_handle(self, L, c_types, a_types, n_cols, asc, nal, limit, offset):
        if self.runs is not None:
            runs = ffi.new("int64_t[]", [int(r) for r in self.runs])
            h = L.b200_sort_state_init_runs(self.operator_id, c_types, a_types, n_cols, len(self.by), asc, nal, runs, len(self.runs),
                                            self.output_batch_size, self.device, ffi.cast("void*", self.stream))
        elif self.full:
            h = L.b200_sort_state_init_full(self.operator_id, c_types, a_types, n_cols, len(self.by), asc, nal, self.output_batch_size,
                                            self.device, ffi.cast("void*", self.stream))
        else:
            h = L.b200_sort_state_init(self.operator_id, limit, offset, c_types, a_types, n_cols, len(self.by), asc, nal,
                                       self.output_batch_size, self.device, ffi.cast("void*", self.stream))
        return _lib.check_ptr(h, "init_stream_sort_state")

    def _consume(self, table: Table, is_last: bool):
        L = _lib.lib()
        phys = to_device(table.select(self.phys), self.device)
        ct = CTable(phys)
        req = ffi.new("int32_t*")
        _lib.check(L.b200_sort_build_consume_batch(self.handle, ct.ptr, int(bool(is_last)), req), "sort_build_consume_batch")
        return bool(req[0])

    def _produce_phys(self, produce_output: bool):
        """The next output batch in physical column order (keys first), and whether it is the last."""
        L = _lib.lib()
        ncols = len(self.out_names)
        self._out_cols = ffi.new("b200_column[]", ncols)
        self._out_tab = ffi.new("b200_table*")
        self._out_tab.cols = self._out_cols
        last = ffi.new("int32_t*")
        _lib.check(L.b200_sort_produce_output_batch(self.handle, self._out_tab, last, int(bool(produce_output))), "sort produce_output_batch")
        return table_from_ctable(self._out_tab, ncols, self.out_names, owner=self), bool(last[0])

    def _produce(self, produce_output: bool):
        phys, last = self._produce_phys(produce_output)
        return phys.select(self.out_order), last

    def _gather_and_reduce(self):
        """Sharded is_last: all-gather every rank's <= K rows and run them, rank-major, through a fresh local state."""
        from .dist_join import all_gather_table, concat_device

        parts = []
        while True:
            out, last = self._produce(True)
            parts.append(out)
            if last:
                break
        local = concat_device(parts, self.device) if len(parts) > 1 else parts[0]
        gathered = all_gather_table(local, self.device, self.process_group)
        g = SortState(self.operator_id, self.limit, self.offset, self.by, self.asc, ["last" if x else "first" for x in self.na_last],
                      self.col_names, False, self.output_batch_size, self.device, self.stream, None)
        g._ensure(gathered)
        g._consume(gathered, True)
        self.global_state = g


def _current_device() -> int:
    import torch

    return torch.cuda.current_device()


def _world(group):
    """(ranks, this rank) of the process group; (1, 0) without torch.distributed."""
    import torch.distributed as dist

    if not dist.is_initialized():
        return 1, 0
    return dist.get_world_size(group), dist.get_rank(group)


def choose_splitters(records, weights, n_ranks):
    """The P - 1 = n_ranks - 1 splitters of a sharded full sort, from every rank's sample records (b200_sort_sample: rows of
    uint64 words, compared lexicographically) and their weights (the rows each sample stands for).  Splitter k (1 <= k < P) is
    the first record, in record order, whose exclusive cumulative weight is at least k N / P, N the total weight.  Returns the
    finite splitters as a (m, words) uint64 array, m <= P - 1; splitters m + 1 .. P - 1 are +inf.  A pure function of the set of
    (record, weight) pairs: every rank computes the same splitters."""
    w = np.asarray(weights, dtype=np.int64)
    recs = np.asarray(records, dtype=np.uint64)
    if n_ranks < 1:
        raise _lib.B200Error(f"choose_splitters: at least one rank (got {n_ranks})")
    if recs.ndim != 2 or len(recs) != len(w):
        raise _lib.B200Error(f"choose_splitters: one weight per record row (records {recs.shape}, {len(w)} weights)")
    order = np.lexsort(recs.T[::-1]) if len(w) else np.zeros(0, np.int64)  # the first word is the most significant
    recs, w = recs[order], w[order]
    excl_p = (np.cumsum(w) - w) * n_ranks  # exclusive cumulative weight, times P
    total = int(w.sum())
    idx = np.searchsorted(excl_p, [k * total for k in range(1, n_ranks)], side="left")
    return recs[idx[idx < len(w)]]


def agree_receive_rows(send_counts, device, group=None, *, received=0, cap=None, what="Streaming Sort: sharded full sort",
                       cap_name="the full sort's cap"):
    """Every rank's send counts to every rank, agreed through one all_reduce: returns the (P, P) matrix of rows rank i sends
    rank j.  Raises the same B200Error on every rank when any rank would hold `cap` rows or more (default
    MAX_SHARDED_RECEIVE_ROWS, the full sort's 32-bit row ids), counting `received` (a scalar or one entry per rank) rows it holds
    already, before any row moves.  `what` and `cap_name` name the operator and its cap in the message."""
    import torch
    import torch.distributed as dist

    cap = MAX_SHARDED_RECEIVE_ROWS if cap is None else cap
    n_ranks, rank = _world(group)
    m = torch.zeros((n_ranks, n_ranks), dtype=torch.int64, device=device)
    m[rank] = torch.as_tensor(np.asarray(send_counts, dtype=np.int64), device=device)
    dist.all_reduce(m, group=group)
    counts = m.cpu().numpy()
    recv = counts.sum(axis=0) + np.asarray(received, dtype=np.int64)
    over = np.flatnonzero(recv >= cap)
    if len(over):
        raise _lib.B200Error(f"{what}: rank {int(over[0])} would receive {int(recv[over[0]])} rows, at or above {cap_name} of {cap} "
                             "rows per rank")
    return counts


def _segment_bitmaps(bitmap, n, counts, dev):
    """Rows [0, n) of an Arrow bitmap as consecutive segments of counts[d] rows, each re-packed from its own byte: the
    per-destination bitmaps exchange_table sends."""
    import torch

    vb = torch.as_tensor(bitmap, device=dev) if n else None
    segs, off = [], 0
    weights = 1 << torch.arange(8, device=dev, dtype=torch.uint8)
    for c in counts:
        c = int(c)
        idx = torch.arange(off, off + c, device=dev)
        pad = torch.zeros((c + 7) // 8 * 8, dtype=torch.uint8, device=dev)
        if c:
            pad[:c] = (vb[idx >> 3] >> (idx & 7).to(torch.uint8)) & 1
        segs.append((pad.view(-1, 8) * weights).sum(1).to(torch.uint8))
        off += c
    return torch.cat(segs)


class ShardedSortState:
    """Python handle of a sharded full sort (init_sharded_sort_state).  `local` sorts this rank's rows; at is_last the rows are
    range-partitioned across the ranks and `merged` merges the sorted runs this rank received (with one rank, `local` is the
    result)."""

    def __init__(self, operator_id, by, asc, na_position, col_names, output_batch_size, device, stream, process_group):
        obs = int(output_batch_size)
        if obs <= 0:
            raise _lib.B200Error(f"Streaming Sort: output_batch_size must be positive (got {output_batch_size})")
        self.local = SortState(operator_id, None, 0, by, asc, na_position, col_names, False, obs, device, stream, None, full=True)
        self.output_batch_size = obs
        self.process_group = process_group
        self.merged = None  # the state the output comes from
        self.done = False

    def consume(self, table: Table, is_last: bool):
        loc = self.local
        if loc.handle is None:
            self.n_ranks, self.rank = _world(self.process_group)
            if self.n_ranks > 1:
                loc.output_batch_size = 0  # the sorted rows come out as one batch, sliced per destination
            loc._ensure(table)
        loc._consume(table, is_last)
        if is_last:
            self.merged = loc if self.n_ranks == 1 else self._exchange()
            self.done = True
        return True

    def _exchange(self):
        """Sample, choose splitters, count the rows per destination, exchange the slices and merge the received runs."""
        import torch
        import torch.distributed as dist

        from ..shuffle import exchange_table

        loc, L, group, P = self.local, _lib.lib(), self.process_group, self.n_ranks
        dev = torch.device("cuda", loc.device)
        rows, _ = loc._produce_phys(True)
        n = rows.n_rows
        nk = len(loc.by)
        width = 2 * nk + 2
        # samples at sorted positions q_i = floor(i n / s), each weighing the rows up to the next one
        s = min(SAMPLES_PER_RANK, n)
        rec = np.zeros((s, width), dtype=np.uint64)
        _lib.check(L.b200_sort_sample(loc.handle, s, self.rank, ffi.cast("uint64_t*", rec.ctypes.data)), "sharded sort sample")
        q = np.arange(s + 1, dtype=np.int64) * n // max(s, 1)
        mine = np.concatenate([rec.view(np.int64), np.diff(q)[:, None]], axis=1)
        sizes = torch.empty(P, dtype=torch.int64, device=dev)
        dist.all_gather_into_tensor(sizes, torch.tensor([s], dtype=torch.int64, device=dev), group=group)
        sizes = sizes.cpu().tolist()
        smax = max(sizes + [1])
        buf = torch.zeros((smax, width + 1), dtype=torch.int64, device=dev)
        buf[:s] = torch.as_tensor(mine, device=dev)
        allr = torch.empty((P * smax, width + 1), dtype=torch.int64, device=dev)
        dist.all_gather_into_tensor(allr, buf, group=group)
        allr = allr.cpu().numpy().reshape(P, smax, width + 1)
        allr = np.concatenate([allr[r, : sizes[r]] for r in range(P)])
        spl = np.ascontiguousarray(choose_splitters(allr[:, :width].view(np.uint64), allr[:, width], P))
        below = np.full(P + 1, n, dtype=np.int64)
        below[0] = 0
        if len(spl):
            cnt = np.zeros(len(spl), dtype=np.int64)
            _lib.check(L.b200_sort_count_below(loc.handle, ffi.cast("uint64_t*", spl.ctypes.data), len(spl), self.rank,
                                               ffi.cast("int64_t*", cnt.ctypes.data)), "sharded sort split")
            below[1: 1 + len(spl)] = cnt
        send = np.diff(below)
        runs = agree_receive_rows(send, dev, group)[:, self.rank]
        cols = []
        for c in rows.columns:  # library-owned device columns: wrapped, not copied (an empty one has no address to wrap)
            data = torch.as_tensor(c.data, device=dev) if n else torch.empty(0, dtype=getattr(torch, str(c.data.dtype)), device=dev)
            v = _segment_bitmaps(c.validity, n, send, dev) if c.validity is not None else None
            cols.append(Column(data, v, c.c_type, c.arr_type, n))
        got = exchange_table(Table(cols, list(rows.names)), [int(x) for x in send], group)
        torch.cuda.synchronize(dev)
        _lib.lib().b200_delete_sort_state(loc.handle)  # the local sorted rows have been sent
        loc.handle = None
        by, asc, nap = self.local.by, self.local.asc, ["last" if x else "first" for x in self.local.na_last]
        m = SortState(loc.operator_id, None, 0, by, asc, nap, loc.out_names, False, self.output_batch_size, loc.device, loc.stream, None,
                      full=True)
        m.runs = [int(x) for x in runs]
        m._ensure(got)
        m._consume(got, True)
        return m

    def produce(self, produce_output: bool):
        phys, last = self.merged._produce_phys(produce_output)
        return phys.select(self.local.out_order), last

    def delete(self):
        for s in (self.local, self.merged):
            if s is not None and s.handle is not None:
                _lib.lib().b200_delete_sort_state(s.handle)
                s.handle = None


def init_sharded_sort_state(operator_id, by, asc, na_position, col_names, *, output_batch_size=32768, device=None, stream=0,
                            process_group=None) -> ShardedSortState:
    """A sharded full sort (ORDER BY without LIMIT over a torch.distributed process group, one process per GPU): rank r's output
    batches, concatenated, are rank r's slice of the sorted result, and the slices in rank order are
    pd.concat(rank inputs in rank order).sort_values(by, kind="stable").  The key rules are the full sort's.  Consume calls
    before is_last are local; the is_last call is collective (every rank passes is_last=True in the same call) and raises the
    same B200Error on every rank when a rank would receive MAX_SHARDED_RECEIVE_ROWS rows or more.  A rank receives fewer than
    ceil(N / P) + 2 G rows, N the rows of all P ranks and G = sum over ranks with rows of ceil(n_r / s_r), s_r = min(
    SAMPLES_PER_RANK, n_r) its samples (DESIGN.md).  Without torch.distributed, or with one rank, it is the local full sort."""
    return ShardedSortState(operator_id, by, asc, na_position, col_names, output_batch_size, device, stream, process_group)


def init_stream_sort_state(operator_id, limit, offset, by, asc, na_position, col_names, parallel=False, *, output_batch_size=32768,
                           device=None, stream=0, process_group=None, full=False) -> SortState:
    """Mirror of bodo.libs.streaming.sort.init_stream_sort_state.

    by: sort key column names (1..4); asc / na_position: one value or one per key; col_names: the input columns, in order.
    LIMIT form (full=False): raises B200Error without a limit, for a negative limit or offset, or when limit + offset exceeds
    MAX_LIMIT_PLUS_OFFSET.  Full sort (full=True): every row in sorted order; limit must be None and offset None or 0, and the
    state holds at most MAX_FULL_SORT_ROWS rows."""
    return SortState(operator_id, limit, offset, by, asc, na_position, col_names, parallel, output_batch_size, device, stream,
                     process_group, full)


def sort_build_consume_batch(state: SortState, table: Table, is_last: bool):
    """Mirror of sort_build_consume_batch: returns (is_last, request_input).  Host batches are staged to the device.
    Collective when the state is parallel: every rank passes is_last=True in the same call."""
    if state.done:
        raise _lib.B200Error("sort_build_consume_batch called after is_last")
    if isinstance(state, ShardedSortState):
        return bool(is_last), state.consume(table, is_last)
    if state.parallel:
        import torch.distributed as dist

        sharded = dist.is_initialized() and dist.get_world_size(state.process_group) > 1
    else:
        sharded = False
    if sharded and state.full:
        raise _lib.B200Error("Streaming Sort: a sharded full sort is not supported (process group of more than one rank)")
    # a sharded rank keeps its first limit + offset rows: the offset applies to the gathered result only
    state._ensure(table, *((state.limit + state.offset, 0) if sharded else (None, None)))
    req = state._consume(table, is_last)
    if is_last:
        state.done = True
        if sharded:
            state._gather_and_reduce()
            state.rank = dist.get_rank(state.process_group)
    return bool(is_last), req


def produce_output_batch(state: SortState, produce_output: bool = True):
    """Mirror of produce_output_batch: returns (table, is_last).  The table wraps library-owned device columns (input types,
    bits and validity) that stay valid until the state is deleted.  A sharded rank other than 0 returns one empty batch."""
    if isinstance(state, ShardedSortState):
        if not state.done:
            raise _lib.B200Error("produce_output_batch called before the last batch was consumed")
        return state.produce(produce_output)
    if state.handle is None or not state.done:
        raise _lib.B200Error("produce_output_batch called before the last batch was consumed")
    if state.global_state is not None:
        if getattr(state, "rank", 0) != 0:
            return state.global_state._produce(False)[0], True
        return state.global_state._produce(produce_output)
    return state._produce(produce_output)


def delete_stream_sort_state(state: SortState) -> None:
    if isinstance(state, ShardedSortState):
        return state.delete()
    for s in (state.global_state, state):
        if s is not None and s.handle is not None:
            _lib.lib().b200_delete_sort_state(s.handle)
            s.handle = None


def get_metric(state: SortState, which: int) -> int:
    """0 rows consumed, 1 rows admitted as candidates, 2 reduce steps, 3 host reads of the candidate count, 4 filter launches,
    5 rows admitted while a cutoff existed, 6 store capacity in rows, 7 digit passes run (full sort), 8 digit passes skipped
    because their digit is constant over all rows (full sort), 9 partitions (window, streaming/window.py).  Metrics 1-5 read 0 in
    a full sort, 7-9 in a top-k and 9 in a full sort.  A sharded full sort reports the state its output comes from: with more
    than one rank, the merge of the rows it received (metric 0 the rows received; it runs no digit pass)."""
    if isinstance(state, ShardedSortState):
        state = state.merged
    return int(_lib.lib().b200_sort_get_metric(state.handle, which))
