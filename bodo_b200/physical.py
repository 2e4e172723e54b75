"""Physical-operator layer — the Python mirror of the reference's pipeline protocol ("door 2",
bodo/pandas/physical/operator.h:46-50,247-458; aggregate.h:65-365; join.h:58-744; _pipeline.cpp:389-466).

    OperatorResult.{NEED_MORE_INPUT, HAVE_MORE_OUTPUT, FINISHED}
    PhysicalReadPandas / PhysicalReadArrow / PhysicalReadParquet : sources (batches of host columns)
    PhysicalAggregate : sink of one pipeline (ConsumeBatch) and source of the next (ProduceBatch); with mrnf=... the
                        min_row_number_filter (one row per group, the first by some order)
    PhysicalJoin      : sink for the build side, ProcessBatch for the probe side
    PhysicalSort      : ORDER BY ... LIMIT ... OFFSET, or ORDER BY without LIMIT (full=True); sink of one pipeline and source
                        of the next
    PhysicalWindow    : ranking window functions OVER (PARTITION BY ... ORDER BY ...); sink of one pipeline and source of the next
    Pipeline          : while not finished: batch = source.ProduceBatch(); ... sink.ConsumeBatch(batch)

plus two helpers that run those pipelines over pandas frames the way bodo.pandas does for
`df.groupby(keys)[cols].agg(...)` and `left.merge(right, on=...)` (PhysicalReadPandas slices the frame into
STREAMING_BATCH_SIZE-row Arrow batches, bodo/pandas/physical/read_pandas.h:13-120).  All computation happens in
libbodo_b200.so; this module only moves batches between operators.
"""

from __future__ import annotations

import enum
from typing import Iterable, Sequence

from .streaming import groupby as G
from .streaming import join as J
from .streaming import sort as S
from .streaming import window as W
from .table import Table

STREAMING_BATCH_SIZE = 32768  # bodo/libs/streaming/_shuffle.h:27-31


class OperatorResult(enum.Enum):
    NEED_MORE_INPUT = 0
    HAVE_MORE_OUTPUT = 1
    FINISHED = 2


class PhysicalReadPandas:
    """Source: slices a pandas DataFrame into batch_size-row batches (read_pandas.h:13-120)."""

    def __init__(self, df, batch_size: int = STREAMING_BATCH_SIZE):
        self.table = Table.from_pandas(df)
        self.batch_size = batch_size
        self.cur = 0

    def ProduceBatch(self):
        n = self.table.n_rows
        batch = self.table.slice(self.cur, self.cur + self.batch_size)
        self.cur += self.batch_size
        return batch, (OperatorResult.FINISHED if self.cur >= n else OperatorResult.HAVE_MORE_OUTPUT)


class PhysicalReadArrow:
    """Source over an in-memory pyarrow Table: batch_size-row zero-copy slices (the Arrow half of
    PhysicalReadPandas, read_pandas.h:13-120: the reference converts every pandas slice to Arrow first)."""

    def __init__(self, table, batch_size: int = STREAMING_BATCH_SIZE):
        self.arrow = table.combine_chunks()
        self.batch_size = batch_size
        self.cur = 0

    def ProduceBatch(self):
        n = self.arrow.num_rows
        batch = Table.from_arrow(self.arrow.slice(self.cur, self.batch_size))
        self.cur += self.batch_size
        return batch, (OperatorResult.FINISHED if self.cur >= n else OperatorResult.HAVE_MORE_OUTPUT)


class PhysicalReadParquet:
    """Source over a Parquet file or dataset directory (host side of physical/read_parquet.h:31-210 — the reference
    streams Arrow record batches out of its ParquetReader; here pyarrow's reader produces them).  Only the selected
    columns are decoded; every batch has at most batch_size rows; an empty dataset yields one empty, FINISHED batch."""

    def __init__(self, path: str, columns: Sequence[str] | None = None, batch_size: int = STREAMING_BATCH_SIZE):
        import pyarrow.dataset as ds

        self.dataset = ds.dataset(path, format="parquet")
        self.columns = list(columns) if columns is not None else None
        self.schema = self.dataset.schema
        self._it = iter(self.dataset.to_batches(columns=self.columns, batch_size=batch_size))
        self._next = self._pull()

    def _pull(self):
        for rb in self._it:
            if rb.num_rows:
                return rb
        return None

    def ProduceBatch(self):
        import pyarrow as pa

        cur = self._next
        if cur is None:  # empty dataset
            names = self.columns if self.columns is not None else list(self.schema.names)
            empty = pa.table({n: pa.array([], type=self.schema.field(n).type) for n in names})
            return Table.from_arrow(empty), OperatorResult.FINISHED
        self._next = self._pull()
        return Table.from_arrow(cur), (OperatorResult.FINISHED if self._next is None else OperatorResult.HAVE_MORE_OUTPUT)


def _infer_ctype(e, col_ctypes: dict) -> int:
    """Storage type of an expression's value: a bare column keeps its type, arithmetic is FLOAT64 as soon as a float (or a
    true division) is involved and INT64 otherwise, comparisons / logic are BOOL."""
    from .table import CTypes

    if e.op == "col":
        return col_ctypes[e.value]
    if e.op == "const_i64":
        return CTypes.INT64
    if e.op == "const_f64" or e.op in ("div", "to_f64"):
        return CTypes.FLOAT64
    if e.op in ("lt", "le", "gt", "ge", "eq", "ne", "and", "or", "not", "is_null"):
        return CTypes.BOOL
    if e.op == "to_i64":
        return CTypes.INT64
    kinds = [_infer_ctype(a, col_ctypes) for a in e.args]
    return CTypes.FLOAT64 if any(k in (CTypes.FLOAT64, CTypes.FLOAT32) for k in kinds) else CTypes.INT64


class PhysicalFilterProject:
    """Filter + projection in one device pass (bodo/pandas/physical/filter.h + project.h with their expression trees,
    expression.{h,cpp}): `predicate` (bodo_b200.expr.Expr or None) selects rows, `outputs` = [(name, Expr)] are the columns of
    the result (col("x") passes a column through).  Host batches are staged to the device first; the result is a device batch."""

    def __init__(self, predicate, outputs, device: int | None = None, stream: int = 0):
        self.predicate = predicate
        self.outputs = list(outputs)
        if not self.outputs:  # a batch is a list of columns: without one it could not say how many rows were kept
            raise ValueError("PhysicalFilterProject needs at least one output column")
        self.device = device
        self.stream = stream
        self._compiled = None

    def _compile(self, batch: Table):
        from . import _lib
        from .expr import compile_program

        col_index = {n: i for i, n in enumerate(batch.names)}
        col_ctypes = {n: c.c_type for n, c in zip(batch.names, batch.columns)}
        exprs = ([self.predicate] if self.predicate is not None else []) + [e for _, e in self.outputs]
        prog, starts = compile_program(exprs, col_index)
        ffi = _lib.ffi
        cprog = ffi.new("b200_expr_instr[]", len(prog))
        for i, (op, arg) in enumerate(prog):
            cprog[i].op = op
            cprog[i].arg = arg
        pred_start = starts[0] if self.predicate is not None else -1
        out_starts = starts[1:] if self.predicate is not None else starts
        out_ct = [_infer_ctype(e, col_ctypes) for _, e in self.outputs]
        self._compiled = (cprog, len(prog), pred_start, ffi.new("int32_t[]", out_starts or [0]), out_ct)

    def ProcessBatch(self, batch: Table, prev: OperatorResult):
        import torch

        from . import _lib
        from .table import to_device
        from .table import ArrTypes, Column, CTable, np_dtype_of

        dev_i = self.device if self.device is not None else (batch.device if batch.device >= 0 else torch.cuda.current_device())
        batch = to_device(batch, dev_i)
        if self._compiled is None:
            self._compile(batch)
        cprog, n_instr, pred_start, out_starts, out_ct = self._compiled
        dev = torch.device("cuda", dev_i)
        n = batch.n_rows
        cols = []
        for ct in out_ct:
            dt = getattr(torch, str(np_dtype_of(ct)))
            cols.append(Column(torch.empty(max(n, 1), dtype=dt, device=dev), torch.zeros((n + 31) // 32 * 4 + 8, dtype=torch.uint8, device=dev), ct,
                               ArrTypes.NULLABLE_INT_BOOL, n))
        out = Table(cols, [nm for nm, _ in self.outputs])
        cin, cout = CTable(batch), CTable(out)
        L, ffi = _lib.lib(), _lib.ffi
        kept = _lib.check(int(L.b200_filter_project(cin.ptr, cprog, n_instr, pred_start, out_starts, len(out_ct), cout.ptr, ffi.cast("void*", self.stream))),
                          "filter + projection")
        res = Table([Column(c.data[:kept], c.validity, c.c_type, c.arr_type, kept) for c in cols], list(out.names))
        return res, (OperatorResult.FINISHED if prev == OperatorResult.FINISHED else OperatorResult.NEED_MORE_INPUT)


def filter_project_table(table: Table, keep) -> Table:
    """Rows of a device-resident `table` whose entry in `keep` (uint8 device tensor, one byte per row) is non-zero, through the
    fused filter kernel (used by streaming.join.runtime_join_filter).  The kept rows are the input's: same c-types, array types,
    bitmap presence and bits.  Each column passes through the kernel as the signed integer of its width, so a float NaN stays a
    valid NaN (the kernel reads NaN as NA), and a column without a bitmap comes back without one.  Every column is one output of
    the kernel, so a table of more than 16 columns raises B200Error."""
    import torch

    from .expr import col
    from .table import ArrTypes, Column, CTypes, np_dtype_of

    as_int = {1: CTypes.INT8, 2: CTypes.INT16, 4: CTypes.INT32, 8: CTypes.INT64}
    names = [f"c{j}" for j in range(table.n_cols)]
    ins = [Column(c.data, c.validity, as_int[np_dtype_of(c.c_type).itemsize], c.arr_type, c.length) for c in table.columns]
    ext = Table(ins + [Column(keep, None, CTypes.BOOL, ArrTypes.NUMPY, table.n_rows)], names + ["__keep"])
    op = PhysicalFilterProject(col("__keep"), [(nm, col(nm)) for nm in names], device=table.device)
    out, _ = op.ProcessBatch(ext, OperatorResult.NEED_MORE_INPUT)
    cols = [Column(o.data.view(getattr(torch, str(np_dtype_of(c.c_type)))), o.validity if c.validity is not None else None, c.c_type,
                   c.arr_type, o.length) for c, o in zip(table.columns, out.columns)]
    return Table(cols, list(table.names))


class PhysicalReadArrowDevice:
    """Source over an in-memory pyarrow Table that hands out DEVICE batches; string columns named in `dict_builders`
    ({column: DictionaryBuilder}) travel as dictionary ids unified against the builder (bodo_b200.dictionary), everything else
    as its fixed-width Arrow buffers (the H2D half of the reference's convertTableToGPU, bodo/pandas/physical/operator.cpp:293-380)."""

    def __init__(self, table, batch_size: int = STREAMING_BATCH_SIZE, device: int = 0, dict_builders: dict | None = None):
        self.arrow = table.combine_chunks()
        self.batch_size = batch_size
        self.device = device
        self.dict_builders = dict_builders or {}
        self.cur = 0

    def ProduceBatch(self):
        from .table import to_device

        n = self.arrow.num_rows
        sl = self.arrow.slice(self.cur, self.batch_size)
        self.cur += self.batch_size
        plain = [nm for nm in sl.schema.names if nm not in self.dict_builders]
        t = to_device(Table.from_arrow(sl.select(plain)), self.device) if plain else Table([], [])
        cols, names = [], []
        for nm in sl.schema.names:
            if nm in self.dict_builders:
                cols.append(self.dict_builders[nm].unify(sl.column(nm), self.device))
            else:
                cols.append(t.columns[plain.index(nm)])
            names.append(nm)
        return Table(cols, names), (OperatorResult.FINISHED if self.cur >= n else OperatorResult.HAVE_MORE_OUTPUT)


class PhysicalAggregate:
    """Groupby sink/source (aggregate.h:65-365). `aggs` = [(func_name, input_column_index or None for size)].
    mrnf = (sort_col_inds, ascending, na_last, keep_inds) with no aggs: a min_row_number_filter, one row per group, the first by
    the sort columns (streaming.groupby's mrnf_* arguments); mrnf_limit=n (forwarded to init_groupby_state with the other keywords)
    keeps the first n rows per group.  percentiles=(q, ...) (forwarded the same way) gives the fraction of every percentile_cont /
    percentile_disc entry of aggs, in order.  A min_row_number_filter with parallel=True is the sharded one
    (streaming.groupby.init_sharded_mrnf_state: only each rank's winners are exchanged, at the last batch)."""

    def __init__(self, key_inds: Sequence[int], aggs: Sequence[tuple], dropna: bool = True, parallel: bool = False, mrnf=None, **kw):
        if mrnf is not None and parallel and not aggs:
            self.state = G.init_sharded_mrnf_state(-1, tuple(key_inds), *(tuple(x) for x in mrnf), dropna=dropna, **kw)
            self.finished_build = False
            return
        fnames = tuple(f for f, _ in aggs) + ((G.MRNF,) if mrnf is not None else ())
        f_in_offsets, f_in_cols = [0], []
        for _, c in aggs:
            if c is not None:
                f_in_cols.append(c)
            f_in_offsets.append(len(f_in_cols))
        if mrnf is not None:
            f_in_offsets.append(len(f_in_cols))
            kw.update(zip(("mrnf_sort_col_inds", "mrnf_sort_col_asc", "mrnf_sort_col_na", "mrnf_col_inds_keep"), (tuple(x) for x in mrnf)))
        self.state = G.init_groupby_state(-1, tuple(key_inds), fnames, tuple(f_in_offsets), tuple(f_in_cols), parallel=parallel,
                                          dropna=dropna, **kw)
        self.finished_build = False

    def ConsumeBatch(self, batch: Table, prev: OperatorResult) -> OperatorResult:
        is_last = prev == OperatorResult.FINISHED
        global_last, _ = G.groupby_build_consume_batch(self.state, batch, is_last, True)
        self.finished_build = global_last
        return OperatorResult.FINISHED if global_last else OperatorResult.NEED_MORE_INPUT

    def ProduceBatch(self):
        out, last = G.groupby_produce_output_batch(self.state, True)
        return out, (OperatorResult.FINISHED if last else OperatorResult.HAVE_MORE_OUTPUT)

    def Finalize(self):
        G.delete_groupby_state(self.state)


class PhysicalJoin:
    """Hash join: sink for build batches, ProcessBatch for probe batches (join.h:58-744); a nested-loop join without keys."""

    NESTED_LOOP_HOWS = ("inner", "left", "right", "outer", "anti", "mark", "cross")

    def __init__(self, build_key, probe_key, build_names, probe_names, how: str = "inner", **kw):
        """build_key / probe_key: a column index, or a sequence of 1..4 indices (a multi-column key, in key order).  With asof_on=...
        (an as-of join, see streaming.join.init_join_state) how is "left" or "inner" and the key sequences may be empty.  Empty key
        sequences without asof_on make a nested-loop join (streaming.join.init_nested_loop_join_state) of kind `how`, with or without
        a non_equi_condition; how="cross" is the inner nested-loop join without a condition and takes no keys."""
        keys = lambda k: tuple(k) if isinstance(k, (list, tuple)) else (k,)
        if kw.get("asof_on") is not None and how not in ("left", "inner"):
            raise J._lib.B200Error(f"PhysicalJoin: an as-of join (asof_on) is how='left' or how='inner', not {how!r}")
        if how == "cross":
            if keys(build_key) or keys(probe_key):
                raise J._lib.B200Error("PhysicalJoin: a cross join (how='cross') takes no key columns")
            if kw.get("non_equi_condition") is not None:
                raise J._lib.B200Error("PhysicalJoin: a cross join (how='cross') takes no non_equi_condition; a join on a condition "
                                       "alone is how='inner' with empty keys")
        if how == "cross" or (not keys(build_key) and not keys(probe_key) and kw.get("asof_on") is None):
            if how not in self.NESTED_LOOP_HOWS:
                raise J._lib.B200Error(f"PhysicalJoin: a join without keys is how= one of {list(self.NESTED_LOOP_HOWS)}, not {how!r}")
            kw.pop("is_na_equal", None)  # no key to compare
            self.state = J.init_nested_loop_join_state(-1, tuple(build_names), tuple(probe_names), how in ("right", "outer"),
                                                       how in ("left", "outer"), is_mark_join=how == "mark", is_anti_join=how == "anti", **kw)
            return
        build_outer = how in ("right", "outer")   # the build side is the RIGHT table (reference convention)
        probe_outer = how in ("left", "outer")
        if how == "anti":   # LEFT ANTI: probe rows without a partner (physical/join.h:151: no build columns in the output)
            kw["is_anti_join"] = True
        elif how == "mark":
            kw["is_mark_join"] = True
        kw.setdefault("is_na_equal", True)  # pandas merge semantics: NA joins NA (bodo/pandas/physical/join.h:267)
        self.state = J.init_join_state(-1, keys(build_key), keys(probe_key), tuple(build_names), tuple(probe_names), build_outer, probe_outer, **kw)

    def ConsumeBatch(self, batch: Table, prev: OperatorResult) -> OperatorResult:
        is_last = prev == OperatorResult.FINISHED
        J.join_build_consume_batch(self.state, batch, is_last)
        return OperatorResult.FINISHED if is_last else OperatorResult.NEED_MORE_INPUT

    def ProcessBatch(self, batch: Table, prev: OperatorResult):
        is_last = prev == OperatorResult.FINISHED
        out, out_last, _ = J.join_probe_consume_batch(self.state, batch, is_last, True)
        return out, (OperatorResult.FINISHED if out_last else OperatorResult.NEED_MORE_INPUT)

    def Finalize(self):
        J.delete_join_state(self.state)


class PhysicalSort:
    """Sort sink/source (the reference's PhysicalSort, bodo/pandas/physical/sort.h, which DuckDB's TopN lowers to): rows
    [offset, offset + limit) of the input sorted stably by `by` (column names; ascending / na_position per key or one for all).
    With full=True (no limit, no offset) every row, sorted: an ORDER BY without LIMIT; with parallel=True as well, the sharded
    full sort (streaming.sort.init_sharded_sort_state: each rank produces its key range of the result).  The column names are
    taken from the first batch."""

    def __init__(self, by, ascending=True, na_position="last", limit=None, offset=0, parallel: bool = False, full: bool = False, **kw):
        self.args = (by, ascending, na_position, limit, offset, parallel)
        self.full = bool(full)
        self.kw = kw
        self.state = None
        if self.full:
            if limit is not None or offset not in (None, 0):
                raise S._lib.B200Error(f"PhysicalSort: a full sort takes no limit or offset (got limit={limit}, offset={offset})")
        elif limit is None:
            raise S._lib.B200Error("PhysicalSort: a limit is required (a full sort without LIMIT is not supported)")

    def ConsumeBatch(self, batch: Table, prev: OperatorResult) -> OperatorResult:
        if self.state is None:
            by, asc, nap, limit, offset, parallel = self.args
            if self.full and parallel:
                self.state = S.init_sharded_sort_state(-1, by, asc, nap, batch.names, **self.kw)
            else:
                kw = dict(self.kw, full=True) if self.full else self.kw
                self.state = S.init_stream_sort_state(-1, limit, offset, by, asc, nap, batch.names, parallel, **kw)
        is_last = prev == OperatorResult.FINISHED
        S.sort_build_consume_batch(self.state, batch, is_last)
        return OperatorResult.FINISHED if is_last else OperatorResult.NEED_MORE_INPUT

    def ProduceBatch(self):
        out, last = S.produce_output_batch(self.state, True)
        return out, (OperatorResult.FINISHED if last else OperatorResult.HAVE_MORE_OUTPUT)

    def Finalize(self):
        if self.state is not None:
            S.delete_stream_sort_state(self.state)


class PhysicalWindow:
    """Window sink/source: every input row once, in the stable order by (partition_by ascending NA last, order_by), with one
    column per function after the input columns.  funcs: ranking entries (out_name, fname) or (out_name, "ntile", n), fname one
    of streaming.window.FUNCS; value entries (out_name, fname, column[, frame]), fname one of streaming.window.VALUE_FUNCS or
    MOMENT_FUNCS (var, std, var_pop, std_pop) and frame one of "range" (default), "rows", "partition", ("rows", start, end) (ROWS BETWEEN start AND end, None for UNBOUNDED,
    negative offsets PRECEDING, positive FOLLOWING) or ("range_between", start, end) (RANGE BETWEEN start AND end, the same
    spelling with offsets measured in the single ORDER BY key, e.g. -pd.Timedelta("1h")), (out_name, "lag" | "lead", column[, k[,
    default]]), (out_name,
    "nth_value", column, n[, frame]) or (out_name, fname, y, x[, frame]), fname one of streaming.window.BIVARIATE_FUNCS
    (covar_samp, covar_pop, corr, regr_slope, regr_intercept, over any frame sum takes); an entry of first_value, last_value,
    nth_value, lag or lead may end with "ignore_nulls" (IGNORE NULLS) or "respect_nulls" (the default);
    ascending / na_position: one value or one per ORDER BY key.  The column names are taken from the first batch.  With
    parallel=True the window is sharded (streaming.window.init_sharded_window_state: each rank produces the partitions it owns;
    without PARTITION BY rank 0 produces every row)."""

    def __init__(self, partition_by, order_by, funcs, ascending=True, na_position="last", parallel: bool = False, **kw):
        self.args = (partition_by, order_by, ascending, na_position, list(funcs), parallel)
        self.kw = kw
        self.state = None

    def ConsumeBatch(self, batch: Table, prev: OperatorResult) -> OperatorResult:
        if self.state is None:
            part, order, asc, nap, funcs, parallel = self.args
            if parallel:
                self.state = W.init_sharded_window_state(-1, part, order, asc, nap, funcs, batch.names, **self.kw)
            else:
                self.state = W.init_window_state(-1, part, order, asc, nap, funcs, batch.names, False, **self.kw)
        is_last = prev == OperatorResult.FINISHED
        W.window_build_consume_batch(self.state, batch, is_last)
        return OperatorResult.FINISHED if is_last else OperatorResult.NEED_MORE_INPUT

    def ProduceBatch(self):
        out, last = W.window_produce_output_batch(self.state, True)
        return out, (OperatorResult.FINISHED if last else OperatorResult.HAVE_MORE_OUTPUT)

    def Finalize(self):
        if self.state is not None:
            W.delete_window_state(self.state)


class ResultCollector:
    """PhysicalResultCollector: concatenates output batches into one pandas frame."""

    def __init__(self):
        self.frames = []

    def ConsumeBatch(self, batch: Table, prev: OperatorResult) -> OperatorResult:
        self.frames.append(batch.to_pandas())
        return OperatorResult.FINISHED if prev == OperatorResult.FINISHED else OperatorResult.NEED_MORE_INPUT

    def result(self):
        import pandas as pd

        return pd.concat(self.frames, ignore_index=True) if self.frames else pd.DataFrame()


def run_pipeline(source, between: Iterable, sink) -> None:
    """Pipeline::Execute (bodo/pandas/_pipeline.cpp:389-466): push batches source -> between ops -> sink."""
    finished = False
    while not finished:
        batch, res = source.ProduceBatch()
        for op in between:
            batch, res2 = op.ProcessBatch(batch, res)
            if res == OperatorResult.FINISHED and res2 != OperatorResult.FINISHED:
                res2 = OperatorResult.FINISHED
            res = res2
        sink.ConsumeBatch(batch, res)
        finished = res == OperatorResult.FINISHED


def _percentile_aggs(aggs: Sequence[tuple], kw: dict):
    """groupby_agg's aggs as (out_name, column, func) triples, and kw with percentiles= holding the q of every 4-tuple
    (out_name, column, func, q) in order (forwarded by PhysicalAggregate to init_groupby_state)."""
    triples, qs = [], []
    for a in aggs:
        a = tuple(a)
        if len(a) == 4:
            if a[2] not in G.PERCENTILES:
                raise G._lib.B200Error(f"groupby_agg: only percentile_cont / percentile_disc take a fraction (got {a!r})")
            qs.append(a[3])
        elif len(a) != 3 or a[2] in G.PERCENTILES:
            raise G._lib.B200Error(f"groupby_agg: an aggregate is (out_name, column, func), a percentile (out_name, column, func, q) "
                                   f"(got {a!r})")
        triples.append(a[:3])
    if qs:
        if kw.get("percentiles") is not None:
            raise G._lib.B200Error("groupby_agg: give the fractions in the (out_name, column, func, q) tuples, not as percentiles=")
        kw = dict(kw, percentiles=tuple(qs))
    return triples, kw


def groupby_agg(df, by, aggs: Sequence[tuple], dropna: bool = True, batch_size: int = STREAMING_BATCH_SIZE, **kw):
    """df.groupby(by, as_index=False, dropna=dropna).agg(...) through the streaming operators.

    aggs: [(out_name, column, func)] with func one of streaming.groupby.FTYPES: 'size', 'sum', 'count', 'nunique', 'mean', 'min',
    'max', 'prod', 'first', 'last', 'var', 'std', 'var_pop', 'std_pop', 'skew', 'kurtosis', 'boolor_agg', 'booland_agg',
    'boolxor_agg', 'bitor_agg', 'bitand_agg', 'bitxor_agg', 'count_if', 'mode', 'percentile_cont', 'percentile_disc' (no pandas
    aliases: 'any' / 'all' give False for an all-NA group, where boolor_agg / booland_agg give NA).  A percentile is the 4-tuple
    (out_name, column, 'percentile_cont' or 'percentile_disc', q) with 0 <= q <= 1 (MEDIAN(x) is ('m', 'x', 'percentile_cont', 0.5)).
    Returns a pandas DataFrame (group order unspecified, as in the reference)."""
    by = [by] if isinstance(by, str) else list(by)
    cols = list(df.columns)
    aggs, kw = _percentile_aggs(aggs, kw)
    used = list(by)
    for _, c, _ in aggs:
        if c is not None and c not in used:
            used.append(c)
    sub = df[used]
    key_inds = [used.index(k) for k in by]
    agg_spec = [(f, None if f == "size" or c is None else used.index(c)) for _, c, f in aggs]
    op = PhysicalAggregate(key_inds, agg_spec, dropna=dropna, **kw)
    run_pipeline(PhysicalReadPandas(sub, batch_size), [], op)
    coll = ResultCollector()
    run_pipeline(op, [], coll)
    op.Finalize()
    out = coll.result()
    out.columns = by + [name for name, _, _ in aggs]
    return out


def groupby_agg_parquet(path: str, by, aggs: Sequence[tuple], dropna: bool = True, batch_size: int = STREAMING_BATCH_SIZE, **kw):
    """bodo.pandas.read_parquet(path).groupby(by, as_index=False, dropna=dropna).agg(...): PhysicalReadParquet feeding
    PhysicalAggregate.  Only the key and aggregated columns are decoded (column pruning, as the reference's planner does
    for ReadParquet under an aggregate).  Same `aggs` format and result shape as groupby_agg."""
    by = [by] if isinstance(by, str) else list(by)
    aggs, kw = _percentile_aggs(aggs, kw)
    used = list(by)
    for _, c, _ in aggs:
        if c is not None and c not in used:
            used.append(c)
    key_inds = [used.index(k) for k in by]
    agg_spec = [(f, None if f == "size" or c is None else used.index(c)) for _, c, f in aggs]
    op = PhysicalAggregate(key_inds, agg_spec, dropna=dropna, **kw)
    run_pipeline(PhysicalReadParquet(path, used, batch_size), [], op)
    coll = ResultCollector()
    run_pipeline(op, [], coll)
    op.Finalize()
    out = coll.result()
    out.columns = by + [name for name, _, _ in aggs]
    return out


def min_row_number_filter(df, by, order_by, ascending=True, na_position="last", keep=None, dropna: bool = False,
                          batch_size: int = STREAMING_BATCH_SIZE, n: int = 1, **kw):
    """The first n rows per group of `by` by `order_by` (default one): QUALIFY ROW_NUMBER() OVER (PARTITION BY by ORDER BY order_by)
    <= n, the streaming equivalent of df.sort_values(order_by, ascending=..., na_position=..., kind="stable").groupby(by, sort=False,
    dropna=dropna).head(n)[keep] (for n = 1, .drop_duplicates(by, keep="first")[keep]), through PhysicalAggregate(mrnf=...,
    mrnf_limit=n).  by, order_by: a column name or a list (1..4 each); ascending / na_position: one value or one per order_by
    column; keep: the output columns (default: every column).  dropna=False (pandas' drop_duplicates) makes all NA keys one group,
    dropna=True drops their rows.  Group order is unspecified; a group's rows are consecutive, in rank order."""
    cols = list(df.columns)
    by = [by] if isinstance(by, str) else list(by)
    order_by = [order_by] if isinstance(order_by, str) else list(order_by)
    keep = cols if keep is None else ([keep] if isinstance(keep, str) else list(keep))
    asc = [ascending] * len(order_by) if isinstance(ascending, bool) else list(ascending)
    nap = [na_position] * len(order_by) if isinstance(na_position, str) else list(na_position)
    if any(p not in ("first", "last") for p in nap):
        raise ValueError(f"min_row_number_filter: na_position must be 'first' or 'last' (got {na_position!r})")
    mrnf = ([cols.index(c) for c in order_by], asc, [p == "last" for p in nap], [cols.index(c) for c in keep])
    op = PhysicalAggregate([cols.index(k) for k in by], [], dropna=dropna, mrnf=mrnf, mrnf_limit=n, **kw)
    run_pipeline(PhysicalReadPandas(df, batch_size), [], op)
    coll = ResultCollector()
    run_pipeline(op, [], coll)
    op.Finalize()
    return coll.result()[keep]


def sort_values_head(df, by, ascending=True, na_position="last", n: int = 5, offset: int = 0, batch_size: int = STREAMING_BATCH_SIZE, **kw):
    """df.sort_values(by, ascending=..., na_position=..., kind="stable").iloc[offset:offset + n] through PhysicalSort.  ascending and
    na_position may be one value or one per key.  Returns a pandas DataFrame with a fresh index."""
    op = PhysicalSort(by, ascending, na_position, limit=n, offset=offset, **kw)
    run_pipeline(PhysicalReadPandas(df, batch_size), [], op)
    coll = ResultCollector()
    run_pipeline(op, [], coll)
    op.Finalize()
    return coll.result()


def sort_values(df, by, ascending=True, na_position="last", batch_size: int = STREAMING_BATCH_SIZE, **kw):
    """df.sort_values(by, ascending=..., na_position=..., kind="stable").reset_index(drop=True) through PhysicalSort(full=True).
    ascending and na_position may be one value or one per key.  Returns a pandas DataFrame with a fresh index."""
    op = PhysicalSort(by, ascending, na_position, full=True, **kw)
    run_pipeline(PhysicalReadPandas(df, batch_size), [], op)
    coll = ResultCollector()
    run_pipeline(op, [], coll)
    op.Finalize()
    return coll.result()


def window(df, partition_by, order_by, funcs, ascending=True, na_position="last", batch_size: int = STREAMING_BATCH_SIZE, **kw):
    """Ranking, aggregate and navigation window functions OVER (PARTITION BY partition_by ORDER BY order_by) through
    PhysicalWindow (funcs as PhysicalWindow takes them, e.g. [("run", "sum", "x", "rows"), ("prev", "lag", "x", 1, 0),
    ("ma7", "mean", "x", ("rows", -6, 0)), ("sd20", "std", "x", ("rows", -19, 0)), ("beta", "regr_slope", "y", "x", ("rows", -59,
    0)), ("ffill", "last_value", "x", "rows", "ignore_nulls")]).  Returns a pandas
    DataFrame in the operator's output order (stably sorted by partition keys, then order keys) with a fresh index: df's columns,
    then one column per function."""
    op = PhysicalWindow(partition_by, order_by, funcs, ascending, na_position, **kw)
    run_pipeline(PhysicalReadPandas(df, batch_size), [], op)
    coll = ResultCollector()
    run_pipeline(op, [], coll)
    op.Finalize()
    return coll.result()


def _names(x):
    return [] if x is None else [x] if isinstance(x, str) else list(x)


def asof_output_layout(left_cols, right_cols, on=None, left_on=None, right_on=None, by=None, left_by=None, right_by=None, suffixes=("_x", "_y")):
    """The column layout of pandas.merge_asof(left, right, ...): (left on, right on, left by, right by, right's output columns,
    output names).  The output is left's columns, then right's without each `on` / `by` column that has the same name as its left
    partner (on=, by=); a name left and right both still have gets the suffixes.  Runs on the host only."""
    if (on is None) == (left_on is None or right_on is None) or (on is not None and (left_on is not None or right_on is not None)):
        raise ValueError("merge_asof: give on=, or both left_on= and right_on=")
    lon, ron = (on, on) if on is not None else (left_on, right_on)
    if not (isinstance(lon, str) and isinstance(ron, str)):
        raise ValueError("merge_asof: one `on` column per side")
    if by is not None and (left_by is not None or right_by is not None):
        raise ValueError("merge_asof: give by=, or left_by= and right_by=, not both")
    lby, rby = (_names(by), _names(by)) if by is not None else (_names(left_by), _names(right_by))
    if len(lby) != len(rby) or len(lby) > 4:
        raise ValueError(f"merge_asof: left_by and right_by need the same number of columns, at most 4 (got {lby} and {rby})")
    for side, names, cols in (("left", [lon] + lby, left_cols), ("right", [ron] + rby, right_cols)):
        missing = [c for c in names if c not in cols]
        if missing:
            raise ValueError(f"merge_asof: the {side} frame has no column {missing[0]!r}")
    merged = {r for l, r in zip([lon] + lby, [ron] + rby) if l == r}
    right_keep = [c for c in right_cols if c not in merged]
    clash = set(left_cols) & set(right_keep)
    names = [c + suffixes[0] if c in clash else c for c in left_cols] + [c + suffixes[1] if c in clash else c for c in right_keep]
    return lon, ron, lby, rby, right_keep, names


def merge_asof(left, right, on=None, *, left_on=None, right_on=None, by=None, left_by=None, right_by=None, suffixes=("_x", "_y"),
               tolerance=None, allow_exact_matches=True, direction="backward", batch_size: int = STREAMING_BATCH_SIZE, **kw):
    """pandas.merge_asof(left, right, ...) through the streaming join's as-of form (left = probe side, right = build side, how="left"):
    each left row once, in left's order, with the right row of equal `by` keys whose `on` value is the latest at or before its own
    (direction="backward"), the earliest at or after it ("forward") or the nearer one ("nearest"), NULL right columns without one.
    Neither frame needs to be sorted.  NA `by` keys match each other, as in pandas; NA `on` cells match nothing.  Same column layout
    and names as pandas (asof_output_layout).  how="inner" in kw keeps only the matched left rows."""
    import pandas as pd

    lcols, rcols = list(left.columns), list(right.columns)
    lon, ron, lby, rby, right_keep, names = asof_output_layout(lcols, rcols, on, left_on, right_on, by, left_by, right_by, suffixes)
    how = kw.pop("how", "left")
    op = PhysicalJoin([rcols.index(c) for c in rby], [lcols.index(c) for c in lby], rcols, lcols, how=how, asof_on=(ron, lon),
                      asof_direction=direction, asof_allow_exact_matches=allow_exact_matches, asof_tolerance=tolerance, **kw)
    run_pipeline(PhysicalReadPandas(right, batch_size), [], op)
    coll = ResultCollector()
    run_pipeline(PhysicalReadPandas(left, batch_size), [op], coll)
    op.Finalize()
    res = coll.result()  # right's columns, then left's
    cols = [res.iloc[:, len(rcols) + j] for j in range(len(lcols))] + [res.iloc[:, rcols.index(c)] for c in right_keep]
    return pd.concat(cols, axis=1, keys=range(len(cols))).set_axis(names, axis=1) if cols else res


def merge(left, right, left_on=None, right_on=None, how: str = "inner", batch_size: int = STREAMING_BATCH_SIZE, suffixes=("_x", "_y"), **kw):
    """left.merge(right, left_on=..., right_on=..., how=...) through the streaming join (right = build side).  left_on / right_on:
    a column name, or equal-length lists of 1..4 names (a multi-column key).
    Output columns: right's columns then left's columns (the reference's build-then-probe order), renamed on clashes.
    `non_equi_condition=` joins only the key-equal pairs that also satisfy a condition (an Expr; left is the probe side, right
    the build side), e.g. `merge(events, windows, "acct", "acct", how="left",
    non_equi_condition=(probe_col("ts") >= build_col("start")) & (probe_col("ts") < build_col("end")))`.
    Without keys (left_on = right_on = None) the join is a nested-loop join: how="cross" without a condition returns exactly
    left.merge(right, how="cross", suffixes=suffixes) (left's columns then right's, the same suffixes and row order); a
    non_equi_condition alone joins the pairs it accepts, for any `how` of PhysicalJoin, in the layout above, e.g. a band join
    `merge(events, bands, how="left", non_equi_condition=(probe_col("x") >= build_col("lo")) & (probe_col("x") < build_col("hi")))`.
    Rows then follow left's order, and each left row's partners right's order."""
    import pandas as pd

    rcols, lcols = list(right.columns), list(left.columns)
    if left_on is None and right_on is None:
        if how == "cross":
            if kw.get("non_equi_condition") is not None:
                raise ValueError("merge: how='cross' takes no non_equi_condition (a join on a condition alone is how='inner')")
        elif kw.get("non_equi_condition") is None:
            raise ValueError("merge: no key columns: give left_on and right_on, how='cross', or a non_equi_condition")
        lo, ro = [], []
    elif how == "cross":
        raise ValueError("merge: how='cross' takes no left_on / right_on")
    elif left_on is None or right_on is None:
        raise ValueError("merge: give both left_on and right_on, or neither")
    else:
        lo = [left_on] if isinstance(left_on, str) else list(left_on)
        ro = [right_on] if isinstance(right_on, str) else list(right_on)
    if len(lo) != len(ro):
        raise ValueError(f"merge: len(right_on) ({len(ro)}) must equal len(left_on) ({len(lo)})")
    op = PhysicalJoin([rcols.index(c) for c in ro], [lcols.index(c) for c in lo], rcols, lcols, how=how, **kw)
    run_pipeline(PhysicalReadPandas(right, batch_size), [], op)
    coll = ResultCollector()
    run_pipeline(PhysicalReadPandas(left, batch_size), [op], coll)
    op.Finalize()
    res = coll.result()
    if how != "cross":
        return res
    # pandas' cross layout: left's columns, then right's; a name both sides have gets the suffixes
    clash = set(lcols) & set(rcols)
    names = [c + suffixes[0] if c in clash else c for c in lcols] + [c + suffixes[1] if c in clash else c for c in rcols]
    cols = [res.iloc[:, len(rcols) + j] for j in range(len(lcols))] + [res.iloc[:, j] for j in range(len(rcols))]
    return pd.concat(cols, axis=1, keys=range(len(cols))).set_axis(names, axis=1) if cols else res
