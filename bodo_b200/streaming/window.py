"""Streaming window operator: ranking functions OVER (PARTITION BY p ... ORDER BY o ...).

    ROW_NUMBER() / RANK() / DENSE_RANK() / PERCENT_RANK() / CUME_DIST() / NTILE(n) OVER (PARTITION BY p ORDER BY o)

pandas equivalents: groupby(p).cumcount() + 1 and groupby(p)[o].rank(method="min" / "dense" / "max", pct=...).  The state is a
third form of the streaming sort (streaming/sort.py's SortState, sort.cu's WindowState): batches are appended to the full sort's
device chunk store, is_last sorts every row by (partition keys ascending NA last, order keys, arrival index) and then scans the
sorted key columns on the device for partition and peer-group boundaries.

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
  - output: every input row once, in the stable sort's order by (partition keys, order keys, arrival); every input column in
    input order, then one column per function under the caller's name.  SQL leaves the order open; fixing it makes every column
    comparable bit for bit.
  - at most MAX_WINDOW_ROWS rows per state and MAX_COLS input plus function columns.  A sharded window is not supported: a
    parallel state raises at its first consume call when the process group has more than one rank (with one rank it runs locally).
"""

from __future__ import annotations

from .. import _lib
from .._lib import ffi
from ..table import Table
from .sort import MAX_FULL_SORT_ROWS, MAX_KEYS, SortState

# Function codes of b200_window_state_init (include/bodo_b200.h).
FUNCS = {"row_number": 0, "rank": 1, "dense_rank": 2, "percent_rank": 3, "cume_dist": 4, "ntile": 5}
MAX_COLS = 32
MAX_WINDOW_ROWS = MAX_FULL_SORT_ROWS


def _names(x):
    if x is None:
        return []
    return [x] if isinstance(x, str) else list(x)


def _parse_funcs(funcs, col_names):
    """[(out_name, fname)] or (out_name, "ntile", n) entries -> [(out_name, code, n)]."""
    out = []
    for f in funcs:
        f = tuple(f)
        if len(f) < 2 or not isinstance(f[0], str) or f[1] not in FUNCS:
            raise _lib.B200Error(f"Streaming Window: unknown window function {f!r} (one of {sorted(FUNCS)}, as (out_name, fname) or "
                                 "(out_name, 'ntile', n))")
        name, fname = f[0], f[1]
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
    names = [n for n, _, _ in out]
    dup = sorted({n for n in names if names.count(n) > 1})
    if dup:
        raise _lib.B200Error(f"Streaming Window: duplicate output names {dup}")
    clash = [n for n in names if n in col_names]
    if clash:
        raise _lib.B200Error(f"Streaming Window: output names {clash} clash with input columns")
    if len(col_names) + len(out) > MAX_COLS:
        raise _lib.B200Error(f"Streaming Window: {len(col_names)} input columns and {len(out)} functions exceed {MAX_COLS} output columns")
    return out


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
        parsed = _parse_funcs(funcs, col_names)
        super().__init__(operator_id, None, 0, keys, [True] * len(part) + asc, ["last"] * len(part) + nap, col_names, parallel,
                         output_batch_size, device, stream, process_group, full=True)
        self.partition_by, self.order_by = part, order
        self.funcs = parsed
        self.out_names += [n for n, _, _ in parsed]
        self.out_order += list(range(len(self.phys), len(self.phys) + len(parsed)))

    def _new_handle(self, L, c_types, a_types, n_cols, asc, nal, limit, offset):
        np_ = len(self.partition_by)
        oasc = ffi.new("int32_t[]", [int(a) for a in self.asc[np_:]] or [0])
        onal = ffi.new("int32_t[]", [int(x) for x in self.na_last[np_:]] or [0])
        codes = ffi.new("int32_t[]", [c for _, c, _ in self.funcs])
        args = ffi.new("int64_t[]", [a for _, _, a in self.funcs])
        h = L.b200_window_state_init(self.operator_id, c_types, a_types, n_cols, np_, len(self.order_by), oasc, onal, codes, args,
                                     len(self.funcs), self.output_batch_size, self.device, ffi.cast("void*", self.stream))
        return _lib.check_ptr(h, "init_window_state")


def init_window_state(operator_id, partition_by, order_by, ascending, na_position, funcs, col_names, parallel=False, *,
                      output_batch_size=32768, device=None, stream=0, process_group=None) -> WindowState:
    """A window state over batches with columns `col_names`.

    partition_by / order_by: a column name or a list of names (either may be empty, 1..4 in all); ascending / na_position: one
    value or one per ORDER BY key; funcs: [(out_name, fname)] with fname in FUNCS, or (out_name, "ntile", n) with n >= 1.
    Raises B200Error for an unknown function, duplicate output names or names that clash with an input column, keys that are
    missing or not distinct, a key count outside 1..4, a bad na_position, or ntile n < 1."""
    return WindowState(operator_id, partition_by, order_by, ascending, na_position, funcs, col_names, parallel, output_batch_size,
                       device, stream, process_group)


def window_build_consume_batch(state: WindowState, table: Table, is_last: bool):
    """Appends a batch (host batches are staged to the device); is_last sorts and evaluates.  Returns (is_last, request_input)."""
    if state.done:
        raise _lib.B200Error("window_build_consume_batch called after is_last")
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
    the state is deleted."""
    if state.handle is None or not state.done:
        raise _lib.B200Error("window_produce_output_batch called before the last batch was consumed")
    return state._produce(produce_output)


def delete_window_state(state: WindowState) -> None:
    if state.handle is not None:
        _lib.lib().b200_delete_sort_state(state.handle)
        state.handle = None


def get_metric(state: WindowState, which: int) -> int:
    """The sort's metrics (streaming/sort.py get_metric; 1-5 read 0) and 9, the number of partitions."""
    return int(_lib.lib().b200_sort_get_metric(state.handle, which))
