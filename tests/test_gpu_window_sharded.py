"""The sharded window (streaming.window.init_sharded_window_state) on one GPU, with R ranks simulated as lock-step threads of this
process (tests/test_gpu_join_sharded.py's LockstepGroup).

The reference is the window of one state (init_window_state, itself checked against exact oracles in tests/test_gpu_window*.py)
over the global input in (consume call, source rank, source row) order.  Each reference output row belongs to the rank that owns
its partition: the key-class partition of the reference's PARTITION BY columns (tests/test_gpu_shuffle_classes.py checks that
placement against a restatement on the oracle's hash functions).  Rank r's output must be the reference restricted to those rows,
in the same order, bit for bit on every input column and every function column (data bytes and validity), except the functions
that accumulate in floating point (sum and mean of a float column, the moments and the co-moments): their combination tree
follows the partition's position among a state's sorted rows, so they agree to rounding (rtol 1e-9) with equal validity and NaN
cells.  So the ranks' partitions are disjoint and cover the input."""

import os
import socket

import numpy as np
import pytest
import torch

from bodo_b200 import _lib
from bodo_b200._lib import B200Error
from bodo_b200.shuffle import partition_device
from bodo_b200.streaming import window as W
from bodo_b200.table import ArrTypes, Column, CTypes, Table
from tests.helpers import table_to_device
from tests.test_gpu_join_sharded import LockstepGroup
from tests.test_gpu_sort import batches_of, col_mask, make_column
from tests.test_gpu_sort_sharded import concat_host

pytestmark = pytest.mark.gpu
RS = (2, 3, 4, 8)
RANKING = [("rn", "row_number"), ("rk", "rank"), ("dr", "dense_rank"), ("pr", "percent_rank"), ("cd", "cume_dist"), ("nt", "ntile", 3)]
VALUES = [("s", "sum", "x"), ("c", "count", "x", "rows"), ("cs", "count", None, "partition"), ("m", "mean", "y", "partition"),
          ("mn", "min", "y", ("rows", -2, 1)), ("mx", "max", "x", ("rows", None, 3)), ("fv", "first_value", "x"),
          ("lv", "last_value", "y", "rows"), ("nv", "nth_value", "x", 2, ("rows", -3, 3)), ("lg", "lag", "y", 2),
          ("ld", "lead", "x", 1, 0.5)]
NULLS = [("fvi", "first_value", "x", ("rows", 0, None), "ignore_nulls"), ("lvi", "last_value", "y", "rows", "ignore_nulls"),
         ("lgi", "lag", "x", 1, None, "ignore_nulls"), ("ldi", "lead", "y", 2, None, "ignore_nulls")]
MOMENTS = [("v", "var", "x", ("rows", -4, 0)), ("sd", "std", "y"), ("vp", "var_pop", "x", "partition"), ("sp", "std_pop", "y", "rows")]
BIVARIATE = [("cv", "covar_samp", "x", "y", ("rows", -3, 0)), ("cp", "covar_pop", "y", "x"), ("co", "corr", "x", "y", "partition"),
             ("sl", "regr_slope", "y", "x", ("rows", None, 2)), ("ic", "regr_intercept", "x", "y")]
RANGES = [("rs", "sum", "x", ("range_between", -3, 2)), ("rm", "max", "y", ("range_between", 0, 5)),
          ("rc", "count", "x", ("range_between", -2, -1))]
FAMILIES = {"ranking": RANKING, "values": VALUES, "ignore_nulls": NULLS, "moments": MOMENTS, "bivariate": BIVARIATE}
PART_TYPES = [CTypes.INT16, CTypes.FLOAT64, CTypes.BOOL, CTypes.DATETIME]


@pytest.fixture
def lockstep(monkeypatch):
    return lambda n: LockstepGroup(n).install(monkeypatch)


@pytest.fixture(autouse=True)
def _return_device_memory():
    yield
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    _lib.lib().b200_pool_trim(torch.cuda.current_device(), 0)


def make_table(rng, n, n_part, part_types=PART_TYPES, groups=6):
    """n_part partition keys (few distinct values, NA and NaN, -0.0 and 0.0), an int64 order key o, values x (float64) and y
    (nullable int32)."""
    cols, names = [], []
    for j in range(n_part):
        c = make_column(part_types[j % len(part_types)], n, rng, j % 2 == 0, na_frac=0.1)
        v = c.values_numpy().copy()
        if v.dtype.kind in "iu":
            v = (v % groups).astype(v.dtype)
        elif v.dtype.kind == "f":
            v = np.where(rng.random(n) < 0.9, np.round(v) % groups, v)
            v[rng.random(n) < 0.05] = -0.0
        cols.append(Column(v, c.validity, c.c_type, c.arr_type, n))
        names.append(f"p{j}")
    cols.append(Column(rng.integers(0, 40, n).astype(np.int64), None, CTypes.INT64, ArrTypes.NUMPY, n))
    x = rng.standard_normal(n) * 10
    x[rng.random(n) < 0.05] = np.nan
    cols.append(make_column(CTypes.INT32, n, rng, True, na_frac=0.1))
    cols.insert(-1, Column(x, None, CTypes.FLOAT64, ArrTypes.NUMPY, n))
    names += ["o", "x", "y"]
    return Table(cols, names)


def rank_batches(tables, sizes, empty_every=0):
    """Per rank, its batches, padded with empty batches so that every rank makes the same number of calls."""
    bs = [batches_of(t, list(sizes), empty_every) for t in tables]
    n = max(len(b) for b in bs)
    return [b + [t.slice(0, 0)] * (n - len(b)) for b, t in zip(bs, tables)]


def collect(st, ncols, produce):
    outs = []
    while True:
        out, last = produce(st)
        outs.append(out)
        if last:
            break
    return [(np.concatenate([o.columns[c].values_numpy() for o in outs]), np.concatenate([col_mask(o.columns[c]) for o in outs]))
            for c in range(ncols)], [o.n_rows for o in outs], outs[0].names


def reference(batches, part, order, asc, nap, funcs):
    """The one-state window over the global input in (call, rank, row) order; its rows' owner ranks."""
    calls = len(batches[0])
    glob = concat_host([batches[r][i] for i in range(calls) for r in range(len(batches))])
    st = W.init_window_state(-1, part, order, asc, nap, funcs, glob.names)
    W.window_build_consume_batch(st, table_to_device(glob), True)
    cols, _, names = collect(st, glob.n_cols + len(funcs), W.window_produce_output_batch)
    W.delete_window_state(st)
    return glob, cols, names


def owners(cols, names, glob, part, R):
    n = len(cols[0][0])
    if not part:
        return np.zeros(n, np.int64)
    keys = []
    for p in part:
        c = glob.columns[glob.names.index(p)]
        v, m = cols[names.index(p)]
        keys.append(Column(np.ascontiguousarray(v), None if c.validity is None else np.packbits(m, bitorder="little"), c.c_type, c.arr_type, n))
    _, counts, perm = partition_device(table_to_device(Table(keys, list(part))), len(part), R, want_perm=True, by_class=True)
    dest = np.empty(n, np.int64)
    dest[perm.cpu().numpy()] = np.repeat(np.arange(R), counts)
    return dest


def run_sharded(pg, batches, part, order, asc, nap, funcs, output_batch_size=32768):
    names = batches[0][0].names

    def rank_fn(r):
        st = W.init_sharded_window_state(-1, part, order, asc, nap, funcs, names, output_batch_size=output_batch_size)
        for i, b in enumerate(batches[r]):
            W.window_build_consume_batch(st, table_to_device(b) if i % 2 == 0 else b, i == len(batches[r]) - 1)
        res = collect(st, len(names) + len(funcs), W.window_produce_output_batch)
        metrics = (W.get_metric(st, 0), W.get_metric(st, 9))
        W.delete_window_state(st)
        return res, metrics
    return pg.run(rank_fn)


def float_accumulated(funcs, glob):
    """Output names of the functions that accumulate in floating point: sum and mean of a float column, the moments and the
    co-moments.  Their combination tree follows the partition's position among the sorted rows of the state, which differs
    between a rank and the one state, so they agree to rounding; every other column agrees bit for bit."""
    out = set()
    for f in funcs:
        if f[1] in W.MOMENT_FUNCS or f[1] in W.BIVARIATE_FUNCS:
            out.add(f[0])
        elif f[1] in ("sum", "mean") and f[2] is not None and glob.columns[glob.names.index(f[2])].c_type in (CTypes.FLOAT32, CTypes.FLOAT64):
            out.add(f[0])
    return out


def compare(R, batches, part, order, asc, nap, funcs, got, output_batch_size=32768):
    """got[r] = ((columns, output batch sizes, names), rows received) of rank r, against the restricted reference."""
    glob, ref, names = reference(batches, part, order, asc, nap, funcs)
    dest = owners(ref, names, glob, part, R)
    rounded = float_accumulated(funcs, glob)
    for r, ((cols, sizes_out, out_names), rows_in) in enumerate(got):
        assert out_names == names
        mine = dest == r
        assert rows_in == int(mine.sum())
        for (v, m), (ev, em), nm in zip(cols, ref, names):
            np.testing.assert_array_equal(m, em[mine], err_msg=f"rank {r} validity of {nm}")
            if nm in rounded:
                e = ev[mine]
                np.testing.assert_array_equal(np.isnan(v[m]), np.isnan(e[m]), err_msg=f"rank {r} NaN cells of {nm}")
                fin = m & ~np.isnan(e)
                scale = float(np.max(np.abs(e[fin]), initial=0.0)) if fin.any() else 0.0
                np.testing.assert_allclose(v[fin], e[fin], rtol=1e-9, atol=1e-9 * scale, err_msg=f"rank {r} column {nm}")
            else:
                np.testing.assert_array_equal(v.view(np.uint8), ev[mine].view(np.uint8), err_msg=f"rank {r} column {nm}")
        assert sum(sizes_out) == rows_in and (sizes_out == [0] or all(0 < s <= -(-output_batch_size // 32) * 32 for s in sizes_out))
    assert sum(g[1] for g in got) == glob.n_rows


def check(pg, tables, part, order, asc, nap, funcs, sizes=(1 << 30,), empty_every=0, output_batch_size=32768):
    batches = rank_batches(tables, sizes, empty_every)
    got = run_sharded(pg, batches, part, order, asc, nap, funcs, output_batch_size)
    compare(pg.n, batches, part, order, asc, nap, funcs, [(res, m[0]) for res, m in got], output_batch_size)
    return got


@pytest.mark.parametrize("family", list(FAMILIES))
@pytest.mark.parametrize("n_part", [1, 2, 3])
def test_function_families(gpu_lib, lockstep, family, n_part):
    rng = np.random.default_rng(10 * list(FAMILIES).index(family) + n_part)
    R = RS[n_part % len(RS)]
    tables = [make_table(rng, int(m), n_part) for m in rng.integers(300, 1500, R)]
    part = [f"p{j}" for j in range(n_part)]
    funcs = FAMILIES[family] + (RANGES if family == "values" else [])
    check(lockstep(R), tables, part, ["o"], [True], ["last"], funcs, sizes=(256, 700))


@pytest.mark.parametrize("R", RS)
def test_four_partition_keys_and_two_order_keys(gpu_lib, lockstep, R):
    rng = np.random.default_rng(R)
    tables = [make_table(rng, 900, 3, groups=3) for _ in range(R)]
    check(lockstep(R), tables, ["p0", "p1"], ["o", "y"], [False, True], ["first", "last"], RANKING + VALUES[:4], sizes=(333,))
    check(lockstep(R), tables, ["p0", "p1", "p2", "o"], [], True, "last", [("rn", "row_number"), ("s", "sum", "x")], sizes=(500,))


def test_without_order_by(gpu_lib, lockstep):
    rng = np.random.default_rng(7)
    tables = [make_table(rng, 800, 2) for _ in range(3)]
    check(lockstep(3), tables, ["p0", "p1"], [], True, "last", RANKING + MOMENTS + [("s", "sum", "x")])


def test_uneven_and_empty_batches_idle_ranks_and_skew(gpu_lib, lockstep):
    rng = np.random.default_rng(11)
    R = 4
    tables = [make_table(rng, m, 1) for m in (2000, 0, 37, 900)]
    check(lockstep(R), tables, ["p0"], ["o"], [True], ["last"], RANKING + VALUES, sizes=(100, 1, 513), empty_every=2)
    skew = [make_table(rng, 3000, 1, groups=2) for _ in range(R)]
    for t in skew:  # one partition holds most rows
        v = t.columns[0].values_numpy()
        v[rng.random(len(v)) < 0.95] = 1
    check(lockstep(R), skew, ["p0"], ["o"], [True], ["last"], RANKING + BIVARIATE, sizes=(1024,), output_batch_size=100)
    empty = [make_table(rng, 0, 1) for _ in range(R)]
    check(lockstep(R), empty, ["p0"], ["o"], [True], ["last"], RANKING)


def test_no_partition_by_goes_to_rank_zero(gpu_lib, lockstep):
    rng = np.random.default_rng(5)
    R = 3
    tables = [make_table(rng, m, 1) for m in (700, 1200, 0)]
    got = check(lockstep(R), tables, [], ["o", "p0"], [True, False], ["last", "first"], RANKING + VALUES, sizes=(400,),
                output_batch_size=512)
    assert got[0][1][0] == 1900
    for r in range(1, R):
        assert got[r][0][1] == [0]  # one empty batch


def test_window_cap_is_refused_on_every_rank_before_rows_move(gpu_lib, lockstep, monkeypatch):
    monkeypatch.setattr(W, "MAX_WINDOW_ROWS", 1000)
    rng = np.random.default_rng(3)
    tables = [make_table(rng, 600, 1, groups=1) for _ in range(2)]  # one partition: 1200 rows on its owner
    for t in tables:
        t.columns[0].values_numpy()[:] = 1
        t.columns[0] = Column(t.columns[0].values_numpy(), None, t.columns[0].c_type, ArrTypes.NUMPY, 600)
    pg = lockstep(2)

    def rank_fn(r):
        st = W.init_sharded_window_state(-1, "p0", "o", True, "last", RANKING, tables[r].names)
        try:
            W.window_build_consume_batch(st, table_to_device(tables[r].slice(0, 300)), False)  # 600 rows: under the cap
            W.window_build_consume_batch(st, table_to_device(tables[r].slice(300, 600)), True)
            return "no error"
        except B200Error as e:
            return str(e)
        finally:
            W.delete_window_state(st)
    msgs = pg.run(rank_fn)
    assert msgs[0] == msgs[1] and "would receive 1200 rows" in msgs[0] and "the window's cap of 1000 rows" in msgs[0]
    assert pg.calls[-1] == "all_reduce" and pg.calls.count("all_reduce") == 2  # the refused call exchanged nothing


def test_one_rank_is_the_local_window(gpu_lib, lockstep):
    rng = np.random.default_rng(2)
    pg = lockstep(1)
    check(pg, [make_table(rng, 3000, 2)], ["p0", "p1"], ["o"], [True], ["last"], RANKING + VALUES, sizes=(999,))
    assert pg.calls == []


class _Source:
    """A pipeline source over host batches."""

    def __init__(self, batches):
        self.batches, self.i = batches, 0

    def ProduceBatch(self):
        from bodo_b200.physical import OperatorResult

        b = self.batches[self.i]
        self.i += 1
        return b, (OperatorResult.FINISHED if self.i == len(self.batches) else OperatorResult.HAVE_MORE_OUTPUT)


def test_physical_window_parallel(gpu_lib, lockstep):
    from bodo_b200.physical import OperatorResult, PhysicalWindow, run_pipeline

    rng = np.random.default_rng(13)
    R = 3
    batches = rank_batches([make_table(rng, m, 2) for m in (1000, 400, 1300)], (300,))
    funcs = [("rn", "row_number"), ("s", "sum", "x", "partition"), ("lg", "lag", "y")]

    def rank_fn(r):
        op = PhysicalWindow(["p0", "p1"], "o", funcs, parallel=True)
        run_pipeline(_Source(batches[r]), [], op)
        assert isinstance(op.state, W.ShardedWindowState)
        outs = []
        while True:
            out, res = op.ProduceBatch()
            outs.append(out)
            if res == OperatorResult.FINISHED:
                break
        cols = [(np.concatenate([o.columns[c].values_numpy() for o in outs]), np.concatenate([col_mask(o.columns[c]) for o in outs]))
                for c in range(outs[0].n_cols)]
        op.Finalize()
        return (cols, [o.n_rows for o in outs], outs[0].names), len(cols[0][0])
    got = lockstep(R).run(rank_fn)
    compare(R, batches, ["p0", "p1"], ["o"], [True], ["last"], funcs, got)


# ---- NCCL: one process per GPU ----
def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _nccl_worker(rank, world, port, q):
    import torch.distributed as dist

    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", rank))
    try:
        rng = np.random.default_rng(5)
        tables = [make_table(rng, 20_000 + 1000 * r, 2) for r in range(world)]
        t = tables[rank]
        st = W.init_sharded_window_state(-1, ["p0", "p1"], "o", True, "last", RANKING + VALUES, t.names, output_batch_size=5000)
        W.window_build_consume_batch(st, table_to_device(t.slice(0, 10_000), rank), False)
        W.window_build_consume_batch(st, table_to_device(t.slice(10_000, 1 << 30), rank), True)
        cols, _, _ = collect(st, t.n_cols + len(RANKING + VALUES), W.window_produce_output_batch)
        W.delete_window_state(st)
        q.put((rank, cols))
    except BaseException as e:  # noqa: BLE001 (reported to the parent)
        q.put((rank, repr(e)))
    finally:
        dist.destroy_process_group()


@pytest.mark.timeout(600)
def test_nccl_ranks():
    import torch.multiprocessing as mp

    world = min(torch.cuda.device_count(), 4)
    if world < 2:
        pytest.skip("needs 2 or more GPUs")
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_nccl_worker, args=(r, world, port, q)) for r in range(world)]
    for p in procs:
        p.start()
    res = dict(q.get(timeout=500) for _ in range(world))
    for p in procs:
        p.join(timeout=60)
    for r in range(world):
        assert not isinstance(res[r], str), res[r]
    rng = np.random.default_rng(5)
    tables = [make_table(rng, 20_000 + 1000 * r, 2) for r in range(world)]
    batches = [[t.slice(0, 10_000), t.slice(10_000, 1 << 30)] for t in tables]
    glob, ref, names = reference(batches, ["p0", "p1"], ["o"], [True], ["last"], RANKING + VALUES)
    dest = owners(ref, names, glob, ["p0", "p1"], world)
    for r in range(world):
        for (v, m), (ev, em) in zip(res[r], ref):
            np.testing.assert_array_equal(v.view(np.uint8), ev[dest == r].view(np.uint8))
            np.testing.assert_array_equal(m, em[dest == r])
