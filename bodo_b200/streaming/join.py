"""Streaming hash join operator API — the host-side mirror of bodo/libs/streaming/join.py.

Same verbs and calling protocol as the reference (init_join_state :991-1100, join_build_consume_batch
:1270-1330, join_probe_consume_batch :1838-1950, delete_join_state :1959), so the reference's streaming join
test loops (bodo/tests/test_streaming/test_join.py) carry over.  The work happens in libbodo_b200.so.

Output column order is the reference's: kept build-table columns first, then kept probe-table columns
(both in logical input order, the key column included on each side unless dropped through used/kept cols).
"""

from __future__ import annotations

import math
from datetime import timedelta

import numpy as np

from .. import _lib
from .._lib import ffi
from ..expr import OPS, Expr, compile_program
from ..table import Column, CTable, CTypes, Table, table_from_ctable

ASOF_DIRECTIONS = {"backward": 0, "forward": 1, "nearest": 2}


class JoinState:
    def __init__(self, operator_id, build_key_inds, probe_key_inds, build_colnames, probe_colnames, build_outer, probe_outer,
                 output_batch_size, expected_build_rows, device, stream, is_na_equal=False, build_parallel=False, probe_parallel=False,
                 is_mark_join=False, is_anti_join=False, non_equi_condition=None, asof=None, nested_loop=False):
        self.operator_id = int(operator_id)
        self.nested_loop = bool(nested_loop)  # no equi-join key: every (probe row, build row) pair is a candidate (n_keys 0)
        self.is_mark_join = bool(is_mark_join)
        self.is_anti_join = bool(is_anti_join)
        self.build_key_inds = tuple(int(k) for k in build_key_inds)
        self.probe_key_inds = tuple(int(k) for k in probe_key_inds)
        # as-of join: (build on, probe on, direction, allow_exact_matches, tolerance), `on` as physical columns.  Without equi-join
        # keys both sides get one constant INT8 key column appended (const_key), so every build row is in one group.
        self.asof = None
        self.const_key = False
        if asof is not None:
            on, direction, exact, tolerance = asof
            if not self.build_key_inds and not self.probe_key_inds:
                self.const_key = True
                self.build_key_inds, self.probe_key_inds = (len(build_colnames),), (len(probe_colnames),)
            b_on, p_on = resolve_asof_on(on, self.build_key_inds, self.probe_key_inds, build_colnames, probe_colnames)
            self.asof = (b_on, p_on, ASOF_DIRECTIONS[direction], bool(exact), tolerance)
        if self.nested_loop:
            if self.build_key_inds or self.probe_key_inds:
                raise _lib.B200Error("Streaming Join: a nested-loop join has no equi-join keys")
        elif not 1 <= len(self.build_key_inds) <= 4 or len(self.probe_key_inds) != len(self.build_key_inds):
            raise _lib.B200Error("Streaming Join: 1 to 4 equi-join keys per side, the same number on both sides "
                                 f"(got {len(self.build_key_inds)} build and {len(self.probe_key_inds)} probe keys; a join without keys is "
                                 "init_nested_loop_join_state)")
        self.build_colnames = list(build_colnames) if build_colnames is not None else None
        self.probe_colnames = list(probe_colnames) if probe_colnames is not None else None
        self.build_outer = bool(build_outer)
        self.probe_outer = bool(probe_outer)
        self.is_na_equal = bool(is_na_equal)
        self.build_parallel = bool(build_parallel)
        self.probe_parallel = bool(probe_parallel)
        self.output_batch_size = int(output_batch_size)
        self.expected_build_rows = int(expected_build_rows)
        self.device = device
        self.stream = int(stream)
        self.handle = None
        self.build_schema = None  # (c_types, arr_types) of the physical (keys-first) build table
        self.build_indices = None
        self.probe_indices = None
        self.build_names = None
        self._out = None
        self.condition = None  # [(op, arg)] of the non-equi condition, resolved to physical columns
        if non_equi_condition is not None:
            self.condition = compile_condition(non_equi_condition, self.build_key_inds, self.probe_key_inds, self.build_colnames,
                                               self.probe_colnames)

    def _physical(self, table: Table, key_inds):
        others = [i for i in range(table.n_cols) if i not in key_inds]
        return list(key_inds) + others

    def _init_c(self, build: Table):
        """Create the C state at the first build batch (the probe schema is adopted from the first probe batch, so build
        batches go straight to the device and the build overlaps whatever produces them)."""
        L = _lib.lib()
        _lib.require_gpu()
        bct, bat = self.build_schema
        if self.device is None:
            import torch

            self.device = build.device if build.device >= 0 else torch.cuda.current_device()
        h = L.b200_join_state_init(self.operator_id, ffi.new("int8_t[]", bct), ffi.new("int8_t[]", bat), len(bct),
                                   ffi.NULL, ffi.NULL, 0, len(self.build_key_inds), int(self.build_outer), int(self.probe_outer), int(self.is_na_equal),
                                   self.output_batch_size, self.device, self.expected_build_rows, ffi.cast("void*", self.stream))
        self.handle = _lib.check_ptr(h, "init_join_state")
        if self.is_mark_join or self.is_anti_join:
            _lib.check(L.b200_join_set_kind(self.handle, int(self.is_mark_join), int(self.is_anti_join)), "init_join_state")
        if self.condition is not None:
            prog = ffi.new("b200_expr_instr[]", len(self.condition))
            for i, (op, arg) in enumerate(self.condition):
                prog[i].op = op
                prog[i].arg = arg
            _lib.check(L.b200_join_set_condition(self.handle, prog, len(self.condition)), "init_join_state")
        if self.asof is not None:
            b_on, p_on, direction, exact, tolerance = self.asof
            has, tol_i, tol_f = asof_tolerance_units(tolerance, bct[b_on])
            _lib.check(L.b200_join_set_asof(self.handle, b_on, p_on, direction, int(exact), has, tol_i, tol_f), "init_join_state")

    def _with_const_key(self, table: Table) -> Table:
        """`table` with the constant INT8 key column of an as-of join without equi-join keys appended."""
        if not self.const_key:
            return table
        n = table.n_rows
        if table.device >= 0:
            import torch

            key = torch.zeros(max(n, 1), dtype=torch.int8, device=torch.device("cuda", table.device))
        else:
            key = np.zeros(max(n, 1), dtype=np.int8)
        return Table(list(table.columns) + [Column(key, None, CTypes.INT8, length=n)], list(table.names) + ["__asof_key"])


J_MAX_COLS = 32        # columns per side (join.cu); a probe column c is program column J_MAX_COLS + c
EX_MAX_INSTR = 64      # instructions of one program (expr.cuh)
EX_MAX_STACK = 8       # values live at once while it runs
EX_MAX_OUT = 16        # output columns of one filter-projection call: the widest table runtime_join_filter takes


def compile_condition(cond, build_key_inds, probe_key_inds, build_colnames, probe_colnames):
    """The non-equi condition as the postfix program b200_join_set_condition takes: [(op, arg)] ending in END.  Column references
    are build_col(name) / probe_col(name); a name resolves against that side's colnames to its physical column (keys first, then
    the other columns in input order), a probe column c becoming J_MAX_COLS + c.  Runs on the host only."""
    if not isinstance(cond, Expr):
        raise _lib.B200Error(f"Streaming Join: non_equi_condition must be a bodo_b200.expr.Expr built from build_col / probe_col, not "
                             f"{type(cond).__name__} (string conditions are not supported)")
    sides = {"build": (build_colnames, build_key_inds, 0), "probe": (probe_colnames, probe_key_inds, J_MAX_COLS)}
    col_index = {}
    for ref in cond.columns():
        if not (isinstance(ref, tuple) and len(ref) == 2 and ref[0] in sides):
            raise _lib.B200Error(f"Streaming Join: non_equi_condition column {ref!r} names no join side: use build_col({ref!r}) or "
                                 f"probe_col({ref!r})")
        side, name = ref
        names, keys, base = sides[side]
        if names is None:
            raise _lib.B200Error(f"Streaming Join: non_equi_condition reads {side} column {name!r}, but {side}_colnames is None: the "
                                 "condition's names resolve against the column names given at init")
        hits = [i for i, nm in enumerate(names) if nm == name]
        if len(hits) != 1:
            raise _lib.B200Error(f"Streaming Join: non_equi_condition: the {side} side has {'no' if not hits else 'more than one'} column "
                                 f"{name!r} ({side} columns: {list(names)})")
        physical = list(keys) + [i for i in range(len(names)) if i not in keys]
        col_index[ref] = base + physical.index(hits[0])
    prog, _ = compile_program([cond], col_index)
    if len(prog) > EX_MAX_INSTR:
        raise _lib.B200Error(f"Streaming Join: non_equi_condition compiles to {len(prog)} instructions; the limit is {EX_MAX_INSTR}")
    unary = {OPS[o] for o in ("not", "neg", "to_f64", "to_i64", "is_null")}
    depth = max_depth = 0
    for op, _ in prog:
        depth += 1 if op in (OPS["col"], OPS["const_i64"], OPS["const_f64"]) else 0 if op in unary or op == OPS["end"] else -1
        max_depth = max(max_depth, depth)
    if max_depth > EX_MAX_STACK:
        raise _lib.B200Error(f"Streaming Join: non_equi_condition needs a stack of {max_depth} values while it runs; the limit is "
                             f"{EX_MAX_STACK} (split deep nesting, e.g. ((a + b) + c) rather than a + (b + (c + d)))")
    return prog


def resolve_asof_on(on, build_key_inds, probe_key_inds, build_colnames, probe_colnames):
    """asof_on = (build column name, probe column name) as (build, probe) physical columns (keys first, then the other columns in
    input order), resolved against the colnames as the non-equi condition's names are.  Runs on the host only."""
    if not (isinstance(on, (tuple, list)) and len(on) == 2):
        raise _lib.B200Error(f"Streaming Join: asof_on must be (build column name, probe column name), got {on!r}")
    out = []
    for side, name, names, keys in (("build", on[0], build_colnames, build_key_inds), ("probe", on[1], probe_colnames, probe_key_inds)):
        if names is None:
            raise _lib.B200Error(f"Streaming Join: asof_on names {side} column {name!r}, but {side}_colnames is None: the as-of join's "
                                 "names resolve against the column names given at init")
        hits = [i for i, nm in enumerate(names) if nm == name]
        if len(hits) != 1:
            raise _lib.B200Error(f"Streaming Join: asof_on: the {side} side has {'no' if not hits else 'more than one'} column {name!r} "
                                 f"({side} columns: {list(names)})")
        if hits[0] in keys:
            raise _lib.B200Error(f"Streaming Join: asof_on: {side} column {name!r} is an equi-join key; the `on` column is not a key column")
        physical = list(keys) + [i for i in range(max(len(names), max(keys) + 1)) if i not in keys]  # (+ the constant key)
        out.append(physical.index(hits[0]))
    return tuple(out)


def _is_timedelta(x) -> bool:
    import pandas as pd

    return isinstance(x, (pd.Timedelta, timedelta, np.timedelta64))


def check_asof_tolerance(tolerance):
    """Refuse a tolerance that is not an int, a float or a Timedelta, or that is negative or not finite."""
    if tolerance is None:
        return
    import pandas as pd

    if _is_timedelta(tolerance):
        td = pd.Timedelta(tolerance)
        if td is pd.NaT or td < pd.Timedelta(0):
            raise _lib.B200Error(f"Streaming Join: asof_tolerance must be >= 0 (got {tolerance!r})")
        return
    if isinstance(tolerance, (bool, np.bool_)) or not isinstance(tolerance, (int, float, np.integer, np.floating)):
        raise _lib.B200Error(f"Streaming Join: asof_tolerance must be an int, a float or a pd.Timedelta (got {type(tolerance).__name__})")
    if not math.isfinite(float(tolerance)) or tolerance < 0:
        raise _lib.B200Error(f"Streaming Join: asof_tolerance must be finite and >= 0 (got {tolerance!r})")


def asof_tolerance_units(tolerance, c_type):
    """(has_tolerance, tolerance_i64, tolerance_f64) of b200_join_set_asof for an `on` column of `c_type`: an integer in the
    column's units for integer and temporal columns (a Timedelta becomes ns for DATETIME / TIMEDELTA and whole days for DATE), a
    float for float columns."""
    if tolerance is None:
        return 0, 0, 0.0
    import pandas as pd

    if _is_timedelta(tolerance):
        ns = pd.Timedelta(tolerance).value
        if c_type in (CTypes.DATETIME, CTypes.TIMEDELTA):
            return 1, int(ns), 0.0
        if c_type == CTypes.DATE:
            days, rest = divmod(ns, 86_400 * 10**9)
            if rest:
                raise _lib.B200Error(f"Streaming Join: asof_tolerance {tolerance!r} is not a whole number of days (the `on` column is a date)")
            return 1, int(days), 0.0
        raise _lib.B200Error("Streaming Join: a Timedelta asof_tolerance needs a date, datetime or timedelta `on` column")
    if c_type in (CTypes.FLOAT32, CTypes.FLOAT64):
        return 1, 0, float(tolerance)
    if not isinstance(tolerance, (int, np.integer)) and float(tolerance) != int(tolerance):
        raise _lib.B200Error(f"Streaming Join: asof_tolerance {tolerance!r} is not an integer (the `on` column is an integer or temporal column)")
    return 1, int(tolerance), 0.0


def init_join_state(operator_id, build_key_inds, probe_key_inds, build_colnames, probe_colnames, build_outer, probe_outer,
                    interval_build_columns=None, force_broadcast=False, op_pool_size_bytes=-1, non_equi_condition=None,
                    build_parallel=False, probe_parallel=False, *, output_batch_size=32768, expected_build_rows=0, device=None,
                    stream=0, is_na_equal=False, is_mark_join=False, is_anti_join=False, asof_on=None, asof_direction="backward",
                    asof_allow_exact_matches=True, asof_tolerance=None) -> JoinState:
    """Mirror of bodo.libs.streaming.join.init_join_state (join.py:991-1100).  Interval joins (`interval_build_columns`) are out
    of scope (SURVEY.md §2.1 row 3) and must be left at the default.

    `non_equi_condition` joins on the equi-join keys AND a condition between the two sides.  The reference takes a string
    ("left.`A` < right.`B`") and compiles it to a cond_func; here it is a bodo_b200.expr.Expr whose columns are
    build_col(name) / probe_col(name), resolved against build_colnames / probe_colnames at init, e.g.
    `(probe_col("ts") >= build_col("start")) & (probe_col("ts") < build_col("end"))`.  A pair of rows with equal keys joins when the
    condition is valid and true (b200_filter_project's semantics: NA and NaN cells are NA, arithmetic and comparisons propagate
    NA, `&` / `|` are Kleene, DATE is days and DATETIME nanoseconds); the outer, anti and mark kinds then apply to the pairs that
    pass.  The condition may read any column, also one used_cols drops, and adds no output column.  At least one equi-join key
    is required here: a join on a condition alone is init_nested_loop_join_state.

    `is_na_equal` is HashJoinState's option: False is what this door constructs in the reference (join_state_init_py_entry,
    _join.cpp:4087-4136: NA keys never match); the pandas door (bodo/pandas/physical/join.h:267, here PhysicalJoin / merge)
    passes True.  `build_parallel` / `probe_parallel` say that the side is row-distributed over the ranks of the default
    torch.distributed process group: non-owned rows are shuffled to hash_to_rank(key) before they reach the local join
    (_join.cpp:3243-3300), or — `force_broadcast`, or a build side below the broadcast threshold — the build side is
    all-gathered instead (:3317-3405)  (see bodo_b200/streaming/dist_join.py).

    `is_mark_join` (HashJoinState's ctor argument, _join.h:287) / `is_anti_join` (the probe's template argument, selected by the
    reference's planner for LEFT ANTI joins, bodo/pandas/physical/join.h:151): a mark join emits every probe row once, without
    build columns, plus a trailing boolean column that says whether the row has a match; an anti join emits the probe rows
    that have none.

    `asof_on=(build column name, probe column name)` makes an as-of join, the contract of pandas.merge_asof (SQL: ASOF JOIN ...
    MATCH_CONDITION): each probe row matches at most one build row with equal keys (0 to 4 keys; none puts every build row in one
    group), the one whose `on` value is the latest at or before the probe's (`asof_direction="backward"`), the earliest at or
    after it ("forward") or the nearer of those two ("nearest", a tie going to the backward one); among equal `on` values the
    last build row in arrival order for backward, the first for forward.  `asof_allow_exact_matches=False` makes the bounds
    strict; `asof_tolerance` (an int, a float or a pd.Timedelta, in the column's units) drops a match further away than it.
    NA `on` cells never match.  probe_outer=True is the left as-of join (pandas' form: every probe row once), False the inner
    one.  The `on` columns are one per side, of the same type: an integer, float, date, datetime or timedelta column.  Not with
    build_outer, the mark / anti kinds, a non_equi_condition or a sharded join."""
    if interval_build_columns not in (None, (), []):
        raise _lib.B200Error("Streaming Join: interval joins (interval_build_columns) are not supported by bodo_b200")
    g = lambda x: getattr(x, "meta", x)
    asof = None
    if asof_on is not None:
        if build_parallel or probe_parallel:
            raise _lib.B200Error("Streaming Join: a sharded asof join is not supported (build_parallel / probe_parallel)")
        if build_outer:
            raise _lib.B200Error("Streaming Join: a build-outer asof join is not supported (build_outer must be False)")
        if is_mark_join or is_anti_join or non_equi_condition is not None:
            raise _lib.B200Error("Streaming Join: an asof join is not a mark, anti or non_equi_condition join")
        if asof_direction not in ASOF_DIRECTIONS:
            raise _lib.B200Error(f"Streaming Join: asof_direction must be one of {list(ASOF_DIRECTIONS)} (got {asof_direction!r})")
        check_asof_tolerance(asof_tolerance)
        asof = (g(asof_on), asof_direction, asof_allow_exact_matches, asof_tolerance)
    if non_equi_condition is not None and (len(tuple(g(build_key_inds))) == 0 or len(tuple(g(probe_key_inds))) == 0):
        raise _lib.B200Error("Streaming Join: a non_equi_condition without an equi-join key (a nested-loop join) is not supported by "
                             "init_join_state; use init_nested_loop_join_state")
    if build_parallel or probe_parallel:
        from .dist_join import DistJoinState

        return DistJoinState(operator_id, g(build_key_inds), g(probe_key_inds), g(build_colnames), g(probe_colnames), build_outer,
                             probe_outer, output_batch_size, expected_build_rows, device, stream, is_na_equal=is_na_equal,
                             build_parallel=build_parallel, probe_parallel=probe_parallel, force_broadcast=force_broadcast,
                             is_mark_join=is_mark_join, is_anti_join=is_anti_join, non_equi_condition=non_equi_condition)
    return JoinState(operator_id, g(build_key_inds), g(probe_key_inds), g(build_colnames), g(probe_colnames), build_outer,
                     probe_outer, output_batch_size, expected_build_rows, device, stream, is_na_equal=is_na_equal,
                     is_mark_join=is_mark_join, is_anti_join=is_anti_join, non_equi_condition=non_equi_condition, asof=asof)


def init_nested_loop_join_state(operator_id, build_colnames, probe_colnames, build_outer, probe_outer, non_equi_condition=None,
                                build_parallel=False, probe_parallel=False, *, is_mark_join=False, is_anti_join=False,
                                output_batch_size=32768, expected_build_rows=0, device=None, stream=0, asof_on=None,
                                interval_build_columns=None) -> JoinState:
    """A join without an equi-join key (the reference's NestedLoopJoinState, bodo/libs/streaming/_nested_loop_join.cpp): every
    (probe row, build row) pair is a candidate.  Without `non_equi_condition` every pair joins: a cross join (SQL CROSS JOIN, pandas
    how="cross").  With one (an Expr over build_col(name) / probe_col(name), as in init_join_state) the pairs whose condition is
    valid and true join: band, range and threshold joins, `LEFT JOIN ... ON <inequality>`.  build_outer / probe_outer make the
    right / left / full outer joins; is_anti_join keeps the probe rows without a passing pair (NOT EXISTS), is_mark_join emits
    every probe row with a trailing boolean "has a passing pair" column (EXISTS).

    The returned JoinState is driven by join_build_consume_batch / join_probe_consume_batch / delete_join_state / get_metric like a
    hash join's (used_cols included).  Output order is guaranteed: within a probe call, rows follow the probe rows, and a probe
    row's pairs follow the build arrival order (batch order, then row order); a NULL-extended, anti or mark row sits in its probe
    row's place; the unmatched build rows of a right / full join follow the last probe call, in build order.  A cross join
    therefore equals pandas' left.merge(right, how="cross") row for row (probe = left).  One probe call produces at most 2^31
    rows; a bigger one raises B200Error before anything is allocated for the output: feed smaller probe batches.  Metrics 8 / 9
    count the pairs evaluated and passed (0 without a condition).  Not sharded (build_parallel / probe_parallel), not as-of, not an
    interval join, and mark / anti joins do not emit build rows (build_outer must be False)."""
    if build_parallel or probe_parallel:
        raise _lib.B200Error("Streaming Join: a sharded nested-loop join is not supported (build_parallel / probe_parallel)")
    if asof_on is not None:
        raise _lib.B200Error("Streaming Join: a nested-loop join has no as-of form (asof_on); init_join_state runs an as-of join "
                             "without keys")
    if interval_build_columns not in (None, (), []):
        raise _lib.B200Error("Streaming Join: interval joins (interval_build_columns) are not supported by bodo_b200")
    if is_mark_join and is_anti_join:
        raise _lib.B200Error("Streaming Join: a join is a mark join or an anti join, not both")
    if (is_mark_join or is_anti_join) and build_outer:
        raise _lib.B200Error("Streaming Join: mark / anti joins do not emit build rows (build_outer must be False)")
    g = lambda x: getattr(x, "meta", x)
    return JoinState(operator_id, (), (), g(build_colnames), g(probe_colnames), build_outer, probe_outer, output_batch_size,
                     expected_build_rows, device, stream, is_mark_join=is_mark_join, is_anti_join=is_anti_join,
                     non_equi_condition=non_equi_condition, nested_loop=True)


def join_build_consume_batch(join_state: JoinState, table: Table, is_last: bool):
    """Mirror of join_build_consume_batch (join.py:1270-1330): returns (is_last, request_input)."""
    if hasattr(join_state, "build_consume"):  # sharded state (build_parallel / probe_parallel): dist_join.DistJoinState
        return join_state.build_consume(table, is_last)
    st = join_state
    table = st._with_const_key(table)
    if st.build_indices is None:
        st.build_indices = st._physical(table, st.build_key_inds)
        cols = [table.columns[i] for i in st.build_indices]
        st.build_schema = ([c.c_type for c in cols], [c.arr_type for c in cols])
        st.build_names = [table.names[i] for i in st.build_indices]
    phys = table.select(st.build_indices)
    if st.handle is None:
        st._init_c(phys)
    return _feed_build(st, phys, is_last), True


def _feed_build(st: JoinState, phys: Table, is_last: bool) -> bool:
    L = _lib.lib()
    ct = CTable(phys)
    req = ffi.new("int32_t*")
    rc = _lib.check(L.b200_join_build_consume_batch(st.handle, ct.ptr, int(bool(is_last)), req), "join_build_consume_batch")
    return bool(rc)


def join_probe_consume_batch(join_state: JoinState, table: Table, is_last: bool, produce_output: bool = True, used_cols=None):
    """Mirror of join_probe_consume_batch (join.py:1838-1950): returns (out_table, is_last, request_input).
    used_cols = (kept_build_cols, kept_probe_cols) as logical column indices, or None to keep everything."""
    if hasattr(join_state, "probe_consume"):
        return join_state.probe_consume(table, is_last, produce_output, used_cols)
    st = join_state
    L = _lib.lib()
    if st.build_indices is None or st.handle is None:
        raise _lib.B200Error("join_probe_consume_batch called before any build batch was consumed")
    table = st._with_const_key(table)
    if st.probe_indices is None:
        st.probe_indices = st._physical(table, st.probe_key_inds)
    phys = table.select(st.probe_indices)
    if used_cols is None:  # every column but the constant key of an as-of join without keys
        kb_logical = [i for i in sorted(st.build_indices) if not (st.const_key and i in st.build_key_inds)]
        kp_logical = [i for i in sorted(st.probe_indices) if not (st.const_key and i in st.probe_key_inds)]
    else:
        kb_logical, kp_logical = list(used_cols[0]), list(used_cols[1])
    if st.is_mark_join:
        kb_logical = []  # a mark join does not output build table columns
    kb = [st.build_indices.index(i) for i in kb_logical]
    kp = [st.probe_indices.index(i) for i in kp_logical]
    if not st.is_mark_join and not kb and not kp:  # a batch is a list of columns: without one it could not say how many rows it has
        raise _lib.B200Error(f"join_probe_consume_batch: used_cols={used_cols!r} keeps no column; keep at least one build or probe "
                             "column (a mark join always has its mark column)")
    names = [st.build_names[j] for j in kb] + [phys.names[j] for j in kp]
    # unique output names (a key named the same on both sides appears twice, like pandas' _x/_y without renaming)
    seen, uniq = set(), []
    for nm in names:
        cand, k = nm, 1
        while cand in seen:
            cand = f"{nm}_{k}"; k += 1
        seen.add(cand); uniq.append(cand)
    if st.is_mark_join:
        uniq.append("")  # the mark column is unnamed in the reference too (physical/join.h:317)
    ct = CTable(phys)
    ncols = len(kb) + len(kp) + (1 if st.is_mark_join else 0)
    st._out_cols = ffi.new("b200_column[]", max(ncols, 1))
    st._out = ffi.new("b200_table*")
    st._out.cols = st._out_cols
    total = ffi.new("int64_t*")
    out_last = ffi.new("int32_t*")
    _lib.check(L.b200_join_probe_consume_batch(st.handle, ct.ptr, ffi.new("uint64_t[]", kb or [0]), len(kb),
                                               ffi.new("uint64_t[]", kp or [0]), len(kp), st._out, total, int(bool(is_last)), out_last),
               "join_probe_consume_batch")
    out = table_from_ctable(st._out, ncols, uniq, owner=st)
    return out, bool(out_last[0]), True


def delete_join_state(join_state: JoinState) -> None:
    join_state = getattr(join_state, "local", join_state)
    if join_state.handle is not None:
        _lib.lib().b200_delete_join_state(join_state.handle)
        join_state.handle = None


def build_runtime_filter(join_state, n_bloom_blocks: int = 0):
    """Build the bloom filter + key bounds of a finished build side; returns (bloom words as a device tensor aliasing the
    state's memory, [(min, max) of each key column]).  Sharded joins OR / min / max these across ranks (dist_join.DistJoinState
    does)."""
    import torch

    st = getattr(join_state, "local", join_state)
    L = _lib.lib()
    nk = len(st.build_key_inds)
    ptr = ffi.new("void**")
    nb = ffi.new("int64_t*")
    mm = ffi.new("int64_t[]", 2 * nk)
    _lib.check(L.b200_join_build_filter(st.handle, int(n_bloom_blocks), ptr, nb, mm), "runtime_join_filter")
    from ..table import DeviceArray

    words = torch.as_tensor(DeviceArray(int(ffi.cast("uintptr_t", ptr[0])), int(nb[0]) * 8, "int32", st.device, owner=st), device=torch.device("cuda", st.device))
    return words, [(int(mm[2 * j]), int(mm[2 * j + 1])) for j in range(nk)]


def runtime_join_filter(join_states, table: Table, join_keys_idxs, process_col_bitmasks=None) -> Table:
    """Mirror of bodo.libs.streaming.join.runtime_join_filter (join.py:1392-1415; C++ HashJoinState::RuntimeFilter): drop the
    rows of `table` that cannot find a partner in the (finished) build sides of `join_states`.  join_keys_idxs[k] = (index of the
    column of `table` that corresponds to each join key of state k, in key order), -1 = no such column (no filter for that state
    when every entry is -1); process_col_bitmasks[k] = (apply the column-level min / max filter, per key column).  The bloom
    filter is applied whenever every key column is present, as in the reference.  Device-resident tables only (host batches:
    bodo_b200.table.to_device first)."""
    import torch

    from ..expr import col
    from ..physical import filter_project_table

    if table.device < 0:
        raise _lib.B200Error("runtime_join_filter: the table must be device resident")
    L = _lib.lib()
    dev = torch.device("cuda", table.device)
    keep_all = None
    for k, js in enumerate(join_states):
        st = getattr(js, "local", js)
        kcs = [int(c) for c in join_keys_idxs[k]]
        if all(c < 0 for c in kcs) or st.probe_outer:
            continue
        use_mm = [1] * len(kcs) if process_col_bitmasks is None else [int(bool(b)) for b in process_col_bitmasks[k]]
        if len(use_mm) != len(kcs):
            raise _lib.B200Error("runtime_join_filter: process_col_bitmasks[k] needs one entry per key column")
        keep = torch.empty(table.n_rows + 8, dtype=torch.uint8, device=dev)
        ct = CTable(table)
        _lib.check(L.b200_join_runtime_filter_n(st.handle, ct.ptr, ffi.new("int32_t[]", kcs), len(kcs), ffi.new("int32_t[]", use_mm), 1,
                                                ffi.cast("uint8_t*", keep.data_ptr())), "runtime_join_filter")
        keep_all = keep if keep_all is None else keep_all & keep
    if keep_all is None:
        return table
    return filter_project_table(table, keep_all[: table.n_rows])


def get_metric(join_state: JoinState, which: int) -> int:
    join_state = getattr(join_state, "local", join_state)
    return int(_lib.lib().b200_join_get_metric(join_state.handle, which))
