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
of the rank inputs concatenated in rank order.  A sharded full sort is not supported: such a state raises at its first consume
call when the process group has more than one rank (with one rank it sorts locally).
"""

from __future__ import annotations

from .. import _lib
from .._lib import ffi
from ..table import CTable, Table, table_from_ctable, to_device

MAX_KEYS = 4
# limit + offset cap: the store addresses rows with uint32 ids and keeps two buffers of max(2 (limit + offset), 4 Mi) rows
MAX_LIMIT_PLUS_OFFSET = 1 << 26
# full sort: rows per state (32-bit row ids whose top bit carries a key's NA class during its class pass)
MAX_FULL_SORT_ROWS = 1 << 31


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
        if self.full:
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

    def _produce(self, produce_output: bool):
        L = _lib.lib()
        ncols = len(self.out_names)
        self._out_cols = ffi.new("b200_column[]", ncols)
        self._out_tab = ffi.new("b200_table*")
        self._out_tab.cols = self._out_cols
        last = ffi.new("int32_t*")
        _lib.check(L.b200_sort_produce_output_batch(self.handle, self._out_tab, last, int(bool(produce_output))), "sort produce_output_batch")
        phys = table_from_ctable(self._out_tab, ncols, self.out_names, owner=self)
        return phys.select(self.out_order), bool(last[0])

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
    if state.handle is None or not state.done:
        raise _lib.B200Error("produce_output_batch called before the last batch was consumed")
    if state.global_state is not None:
        if getattr(state, "rank", 0) != 0:
            return state.global_state._produce(False)[0], True
        return state.global_state._produce(produce_output)
    return state._produce(produce_output)


def delete_stream_sort_state(state: SortState) -> None:
    for s in (state.global_state, state):
        if s is not None and s.handle is not None:
            _lib.lib().b200_delete_sort_state(s.handle)
            s.handle = None


def get_metric(state: SortState, which: int) -> int:
    """0 rows consumed, 1 rows admitted as candidates, 2 reduce steps, 3 host reads of the candidate count, 4 filter launches,
    5 rows admitted while a cutoff existed, 6 store capacity in rows, 7 digit passes run (full sort), 8 digit passes skipped
    because their digit is constant over all rows (full sort), 9 partitions (window, streaming/window.py).  Metrics 1-5 read 0 in
    a full sort, 7-9 in a top-k and 9 in a full sort."""
    return int(_lib.lib().b200_sort_get_metric(state.handle, which))
