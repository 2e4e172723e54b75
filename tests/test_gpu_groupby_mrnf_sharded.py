"""The sharded min_row_number_filter (streaming.groupby.init_sharded_mrnf_state) on one GPU, with R ranks simulated as lock-step
threads of this process (tests/test_gpu_join_sharded.py's LockstepGroup).

The reference is tests/test_gpu_groupby_mrnf_limit.py's exact numpy oracle over the rank inputs concatenated in rank order (the
rank-major order): rows lexsorted by (key, class / order word per sort column, arrival), the first n per group kept.  The rows all
ranks produce must equal it bit for bit as a multiset (validity and the bits of every valid cell), every group must come out on
one rank, and with a row id column kept each group's rows must be consecutive and in rank order.

Float keys: a numpy float key holds NaN (the NA key) and a nullable one holds NA, but no nullable key column mixes the two.  The
local min_row_number_filter keeps a valid NaN and an NA of one nullable float key column as two groups, where the oracle makes
them one; that is the single-state operator's behaviour, which the sharded one inherits (its key-class placement sends both to
one rank)."""

import numpy as np
import pytest
import torch

from bodo_b200 import _lib
from bodo_b200.streaming import groupby as G
from bodo_b200.table import Column, CTypes, Table
from tests.helpers import table_to_device
from tests.test_gpu_groupby_mrnf import FLOATS, SORT_TYPES, col, host_cells, random_col, rows_of
from tests.test_gpu_groupby_mrnf_limit import oracle_rows
from tests.test_gpu_join_sharded import LockstepGroup
from tests.test_gpu_sort_sharded import concat_host

pytestmark = pytest.mark.gpu
RS = (2, 3, 4, 8)


@pytest.fixture
def lockstep(monkeypatch):
    return lambda n: LockstepGroup(n).install(monkeypatch)


@pytest.fixture(autouse=True)
def _return_device_memory():
    yield
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    _lib.lib().b200_pool_trim(torch.cuda.current_device(), 0)


def make_table(rng, n, key_ct, nullable, row0, groups=None):
    """k (key of type key_ct), o (float64 sort column with ties, NaN and NA), p (int16 payload), id (global row id from row0)."""
    k = random_col(rng, key_ct, n, nullable)
    if nullable and key_ct in FLOATS:  # (see the module docstring)
        v = k.values_numpy().copy()
        v[np.isnan(v)] = 2.5
        k = Column(v, k.validity, key_ct, k.arr_type, n)
    if groups is not None:
        k = col(rng.integers(0, groups, n), key_ct)
    o = random_col(rng, CTypes.FLOAT64, n, True)
    return Table([k, o, random_col(rng, CTypes.INT16, n, True), col(np.arange(row0, row0 + n), CTypes.INT64)], ["k", "o", "p", "id"])


def split(rng, R, sizes, key_ct, nullable, **kw):
    row0, parts = 0, []
    for m in sizes:
        parts.append(make_table(rng, int(m), key_ct, nullable, row0, **kw))
        row0 += int(m)
    return parts


def run_sharded(pg, parts, key_inds, sort, asc, na, keep, n, dropna, batch=700, output_batch_size=32768):
    calls = max(-(-p.n_rows // batch) for p in parts) or 1

    def rank_fn(r):
        st = G.init_sharded_mrnf_state(-1, key_inds, sort, asc, na, keep, dropna=dropna, mrnf_limit=n, output_batch_size=output_batch_size)
        t = parts[r]
        for i in range(calls):
            b = t.slice(i * batch, (i + 1) * batch)
            G.groupby_build_consume_batch(st, table_to_device(b) if i % 2 else b, i == calls - 1)
        outs = []
        while True:
            out, last = G.groupby_produce_output_batch(st)
            outs.append([host_cells(c) for c in out.columns])
            names = list(out.names)
            if last:
                break
        G.delete_groupby_state(st)
        return [(np.concatenate([o[j][0] for o in outs]), np.concatenate([o[j][1] for o in outs])) for j in range(len(keep))], names
    return pg.run(rank_fn)


def check(pg, parts, key_inds, sort, asc, na, keep, n, dropna, **kw):
    glob = concat_host(parts)
    got = run_sharded(pg, parts, key_inds, sort, asc, na, keep, n, dropna, **kw)
    kept, label, rank = oracle_rows(glob, key_inds, sort, asc, na, dropna, n)
    assert all(names == [glob.names[i] for i in sorted(keep)] for _, names in got)
    allrows = sorted(sum((rows_of(cells) for cells, _ in got), []))
    assert allrows == rows_of([host_cells(glob.columns[i]) for i in sorted(keep)], kept)
    if 3 in keep:  # the id column: groups on one rank, consecutive and in rank order
        lab, rk = np.full(glob.n_rows, -1), np.full(glob.n_rows, -1)
        lab[kept], rk[kept] = label, rank
        seen = {}
        for r, (cells, _) in enumerate(got):
            ids = cells[sorted(keep).index(3)][1].astype(np.int64)
            if not len(ids):
                continue
            out_lab, out_rank = lab[ids], rk[ids]
            for g in np.unique(out_lab):
                assert seen.setdefault(int(g), r) == r, "a group on two ranks"
            start = np.r_[True, out_lab[1:] != out_lab[:-1]]
            assert len(np.unique(out_lab)) == int(start.sum()), "a group's rows are not consecutive"
            run_start = np.maximum.accumulate(np.where(start, np.arange(len(ids)), 0))
            np.testing.assert_array_equal(out_rank, np.arange(len(ids)) - run_start)
    return got


@pytest.mark.parametrize("ct", SORT_TYPES)
@pytest.mark.parametrize("nullable", [False, True])
def test_every_key_type(gpu_lib, lockstep, ct, nullable):
    rng = np.random.default_rng(ct * 2 + nullable)
    R = RS[(ct + nullable) % len(RS)]
    parts = split(rng, R, rng.integers(0, 2500, R), ct, nullable)
    for n in (1, 3):
        for dropna in (False, True):
            check(lockstep(R), parts, [0], [1], [n % 2 == 1], [dropna], [0, 1, 2, 3], n, dropna)
    # kept sets without the key, without the sort column
    check(lockstep(R), parts, [0], [1], [False], [True], [2, 3], 2, False)
    check(lockstep(R), parts, [0], [1, 3], [True, False], [False, True], [0, 2], 1, True)


@pytest.mark.parametrize("R", RS)
def test_two_keys_and_two_sort_columns(gpu_lib, lockstep, R):
    rng = np.random.default_rng(100 + R)
    parts = split(rng, R, rng.integers(500, 3000, R), CTypes.INT8, True)
    # keys (k, p) of 1 and 2 bytes, sort (o descending, id)
    check(lockstep(R), parts, [0, 2], [1, 3], [False, True], [True, False], [3, 1], 4, False, batch=333, output_batch_size=64)


def test_ties_across_ranks_go_to_the_lowest_rank(gpu_lib, lockstep):
    R = 4
    parts = []
    for r in range(R):
        m = 300
        parts.append(Table([col(np.arange(m) % 10, CTypes.INT32), col(np.zeros(m), CTypes.FLOAT64), col(np.full(m, r), CTypes.INT16),
                            col(np.arange(r * m, (r + 1) * m), CTypes.INT64)], ["k", "o", "p", "id"]))
    for n in (1, 5):
        got = check(lockstep(R), parts, [0], [1], [True], [True], [0, 2, 3], n, True)
        srcs = np.concatenate([cells[1][1] for cells, _ in got])
        assert (srcs == 0).all()  # every winner came from rank 0


def test_receiver_table_grows(gpu_lib, lockstep):
    rng = np.random.default_rng(4)
    R = 3
    parts = split(rng, R, [200_000, 150_000, 220_000], CTypes.INT64, False, groups=300_000)
    for n in (1, 2):
        check(lockstep(R), parts, [0], [1], [True], [True], [0, 1, 3], n, True, batch=100_000)


def test_idle_ranks_and_empty_input(gpu_lib, lockstep):
    rng = np.random.default_rng(8)
    parts = split(rng, 4, [0, 3000, 0, 10], CTypes.FLOAT32, True)
    check(lockstep(4), parts, [0], [1], [True], [False], [0, 1, 2, 3], 2, False)
    empty = split(rng, 2, [0, 0], CTypes.INT32, True)
    check(lockstep(2), empty, [0], [1], [True], [False], [0, 3], 1, True)


def test_calls_before_is_last_run_no_collective(gpu_lib, lockstep):
    rng = np.random.default_rng(6)
    R = 3
    parts = split(rng, R, [1000, 1000, 1000], CTypes.INT16, True)
    pg = lockstep(R)

    def rank_fn(r):
        st = G.init_sharded_mrnf_state(-1, [0], [1], [True], [True], [3], mrnf_limit=2)
        for i in range(3):
            G.groupby_build_consume_batch(st, table_to_device(parts[r].slice(300 * i, 300 * (i + 1))), False)
        G.delete_groupby_state(st)
    pg.run(rank_fn)
    assert pg.calls == []
    pg = lockstep(R)
    check(pg, parts, [0], [1], [True], [True], [3], 2, False, batch=300)
    assert pg.calls[0] == "all_reduce" and set(pg.calls[1:]) == {"all_to_all_single"}  # only the is_last exchange


def test_one_rank_is_the_local_filter(gpu_lib, lockstep):
    rng = np.random.default_rng(9)
    pg = lockstep(1)
    check(pg, split(rng, 1, [5000], CTypes.UINT8, True), [0], [1], [True], [True], [0, 2, 3], 3, False)
    assert pg.calls == []


def test_physical_aggregate_mrnf_parallel(gpu_lib, lockstep):
    from bodo_b200.physical import OperatorResult, PhysicalAggregate

    rng = np.random.default_rng(12)
    R = 3
    parts = split(rng, R, [900, 900, 900], CTypes.BOOL, True)
    glob = concat_host(parts)

    def rank_fn(r):
        op = PhysicalAggregate([0], [], dropna=False, parallel=True, mrnf=([1], [False], [True], [3, 0]), mrnf_limit=2)
        assert isinstance(op.state, G.ShardedMrnfState)
        for i in range(3):
            op.ConsumeBatch(table_to_device(parts[r].slice(300 * i, 300 * (i + 1))),
                            OperatorResult.FINISHED if i == 2 else OperatorResult.NEED_MORE_INPUT)
        cells = []
        while True:
            out, res = op.ProduceBatch()
            cells.append([host_cells(c) for c in out.columns])
            if res == OperatorResult.FINISHED:
                break
        op.Finalize()
        return rows_of([(np.concatenate([c[j][0] for c in cells]), np.concatenate([c[j][1] for c in cells])) for j in range(2)])
    got = sorted(sum(lockstep(R).run(rank_fn), []))
    kept, _, _ = oracle_rows(glob, [0], [1], [False], [True], False, 2)
    assert got == rows_of([host_cells(glob.columns[i]) for i in (0, 3)], kept)
