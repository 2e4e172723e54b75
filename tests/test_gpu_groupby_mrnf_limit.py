"""GPU tests of the min_row_number_filter's row limit (mrnf_limit=n: QUALIFY ROW_NUMBER() OVER (PARTITION BY k ORDER BY o) <= n)
against an exact numpy oracle: tests/test_gpu_groupby_mrnf.py's oracle with the first n rows per group kept instead of the first
one (rows lexsorted by (key, class / order word per sort column, arrival), then those whose cumulative count in their group is
below n).  Outputs are compared bit for bit (validity, and the bits of every valid cell) as multisets of rows, since group order is
unspecified.  Where a row id column is kept, the output order is checked too: each group's rows consecutive and in rank order,
across output batches.

The file took 62–70 s on one H100 80GB HBM3 (700 W power limit); its budget is 3 minutes."""

import numpy as np
import pandas as pd
import pytest

from bodo_b200._lib import B200Error
from bodo_b200.streaming import groupby as G
from bodo_b200.table import ArrTypes, Column, CTypes, Table
from tests.helpers import table_to_device
from tests.test_gpu_groupby_mrnf import FLOATS, MRNF, SORT_TYPES, col, host_cells, key_parts, order_key, random_col, rows_of

pytestmark = pytest.mark.gpu


def oracle_rows(t: Table, key_inds, sort, asc, na, dropna, n):
    """The kept rows in the stable order (index arrays): (row, group label, rank in the group)."""
    kp = [key_parts(t.columns[i]) for i in key_inds]
    rows = np.arange(t.n_rows)
    if dropna:
        rows = rows[np.logical_and.reduce([m for m, _ in kp])]
    if len(rows) == 0:
        return rows, rows, rows
    lex = [rows]
    for j in reversed(range(len(sort))):
        cls, w = order_key(t.columns[sort[j]], asc[j], na[j])
        lex += [w[rows], cls[rows]]
    order = rows[np.lexsort(lex)]
    g = pd.DataFrame({f"{p}{j}": a[order] for j, (m, b) in enumerate(kp) for p, a in (("m", m), ("b", b))}).groupby(
        [f"{p}{j}" for j in range(len(kp)) for p in "mb"], sort=False)
    label, rank = g.ngroup().to_numpy(), g.cumcount().to_numpy()
    k = rank < n
    return order[k], label[k], rank[k]


def run(t: Table, key_inds, sort, asc, na, keep, n, dropna=False, batch=None, device=True, **kw):
    """(output cells per kept column in output order, metrics 0, 3, 18, 19)."""
    st = G.init_groupby_state(-1, key_inds, MRNF, (0, 0), (), mrnf_sort_col_inds=sort, mrnf_sort_col_asc=asc, mrnf_sort_col_na=na,
                              mrnf_col_inds_keep=keep, dropna=dropna, mrnf_limit=n, **kw)
    rows = t.n_rows
    batch = batch or max(rows, 1)
    starts = list(range(0, rows, batch)) or [0]
    for i, s in enumerate(starts):
        b = t.slice(s, min(rows, s + batch))
        G.groupby_build_consume_batch(st, table_to_device(b) if device else b, i == len(starts) - 1, True)
    outs = []
    while True:
        out, last = G.groupby_produce_output_batch(st, True)
        outs.append([host_cells(c) for c in out.columns])
        names = list(out.names)
        if last:
            break
    metrics = {m: G.get_metric(st, m) for m in (0, 3, 18, 19)}
    G.delete_groupby_state(st)
    assert names == [t.names[i] for i in sorted(keep)]
    cells = [(np.concatenate([o[j][0] for o in outs]), np.concatenate([o[j][1] for o in outs])) for j in range(len(keep))]
    return cells, metrics


def check(t, key_inds, sort, asc, na, keep, n, dropna=False, id_col=None, **kw):
    """Runs the state and compares with the oracle; id_col: a kept column holding the row number, to check the output order."""
    cells, metrics = run(t, key_inds, sort, asc, na, keep, n, dropna, **kw)
    kept, label, rank = oracle_rows(t, key_inds, sort, asc, na, dropna, n)
    got = rows_of(cells)
    assert len(got) == len(kept) == metrics[0]
    assert got == rows_of([host_cells(t.columns[i]) for i in sorted(keep)], kept)
    if id_col is not None and len(kept):
        ids = cells[sorted(keep).index(id_col)][1].astype(np.int64)
        lab, rk = np.full(t.n_rows, -1), np.full(t.n_rows, -1)
        lab[kept], rk[kept] = label, rank
        out_lab, out_rank = lab[ids], rk[ids]
        start = np.r_[True, out_lab[1:] != out_lab[:-1]]
        assert len(np.unique(out_lab)) == int(start.sum()), "a group's rows are not consecutive"
        run_start = np.maximum.accumulate(np.where(start, np.arange(len(ids)), 0))
        np.testing.assert_array_equal(out_rank, np.arange(len(ids)) - run_start)
    return got, metrics


@pytest.mark.parametrize("n", [2, 7])
@pytest.mark.parametrize("ct", SORT_TYPES)
@pytest.mark.parametrize("nullable", [False, True])
def test_every_sort_type_both_directions_and_na_placements(ct, nullable, n):
    rng = np.random.default_rng(ct * 4 + nullable * 2 + n)
    rows = 3000
    t = Table([col(rng.integers(0, 40, rows), CTypes.INT64), random_col(rng, ct, rows, nullable), col(np.arange(rows), CTypes.INT64)],
              ["k", "o", "id"])
    for asc in (True, False):
        for na_last in (True, False):
            check(t, (0,), (1,), (asc,), (na_last,), (0, 1, 2), n, id_col=2, batch=700, output_batch_size=256)


@pytest.mark.parametrize("n_sort", [1, 2, 3, 4])
@pytest.mark.parametrize("n_keys", [1, 2, 3, 4])
def test_sort_columns_and_keys(n_sort, n_keys):
    rng = np.random.default_rng(200 + 4 * n_sort + n_keys)
    rows = 20_000
    key_types = [CTypes.FLOAT64, CTypes.INT32, CTypes.FLOAT32, CTypes.INT64][:n_keys]
    cols, names = [], []
    for j, ct in enumerate(key_types):
        v = rng.choice(np.array([0.0, -0.0, np.nan, 1.5, -2.0, np.inf]), rows) if ct in FLOATS else rng.integers(0, 6 if n_keys > 1 else 300, rows)
        cols.append(col(v, ct, rng.random(rows) > 0.1 if j % 2 == 1 else None))
        names.append(f"k{j}")
    # four 8-byte sort columns: 4 x 65 + 48 bits = five digits, the chained sort
    order_types = ([CTypes.FLOAT64, CTypes.INT64, CTypes.DATETIME, CTypes.UINT64] if n_sort == 4 else [CTypes.FLOAT64, CTypes.INT8, CTypes.UINT16])[:n_sort]
    for j, ct in enumerate(order_types):
        cols.append(random_col(rng, ct, rows, nullable=j % 2 == 0))
        names.append(f"o{j}")
    cols.append(col(np.arange(rows), CTypes.INT64))
    names.append("id")
    t = Table(cols, names)
    sort = tuple(range(n_keys, n_keys + n_sort))
    asc = tuple(bool(j % 2) for j in range(n_sort))
    na = tuple(j % 3 != 1 for j in range(n_sort))
    for dropna in (False, True):
        check(t, tuple(range(n_keys)), sort, asc, na, tuple(range(len(cols))), 3, dropna, id_col=len(cols) - 1, batch=6_000)
    check(t, (0,), (0, n_keys), (False, True), (True, False), (len(cols) - 1, n_keys), 5, id_col=len(cols) - 1, batch=4_096)


def test_ties_keep_the_earliest_arrivals_and_batch_splits_agree():
    rng = np.random.default_rng(7)
    rows = 100_003
    t = Table([col(rng.integers(0, 5000, rows), CTypes.INT64), col(rng.integers(0, 3, rows), CTypes.INT16), col(np.arange(rows), CTypes.INT64)],
              ["k", "o", "id"])
    results = [check(t, (0,), (1,), (True,), (True,), (0, 1, 2), 4, id_col=2, batch=b)[0] for b in (7, 1000, None)]
    assert results[0] == results[1] == results[2]
    small = t.slice(0, 2_000)
    one_row = check(small, (0,), (1,), (False,), (True,), (0, 1, 2), 3, id_col=2, batch=1)[0]
    assert one_row == check(small, (0,), (1,), (False,), (True,), (0, 1, 2), 3, id_col=2)[0]
    # every row ties: the first n arrivals of each group
    same = Table([col(np.arange(rows) % 10, CTypes.INT64), col(np.zeros(rows), CTypes.FLOAT64), col(np.arange(rows), CTypes.INT64)], ["k", "o", "id"])
    got = check(same, (0,), (1,), (False,), (True,), (2,), 6, batch=777)[0]
    assert sorted(r[1] for r in got) == list(range(60))


def test_growth_with_live_candidates_one_million_groups():
    rng = np.random.default_rng(11)
    rows = 1 << 22
    k = rng.permutation(rows) % 1_000_000
    t = Table([col(k, CTypes.INT64), col(rng.random(rows), CTypes.FLOAT64), col(np.arange(rows), CTypes.INT64)], ["k", "o", "id"])
    # 2^18-row batches: the groups arrive over several batches, so the table grows while earlier survivors are in the store
    got, metrics = check(t, (0,), (1,), (False,), (True,), (0, 1, 2), 3, id_col=2, batch=1 << 18, expected_groups=1)
    assert metrics[3] >= 2 and len(got) == np.minimum(np.bincount(k), 3).sum()
    t2 = Table([col(k // 1000, CTypes.INT32), col(k % 1000, CTypes.INT64), col(rng.random(rows), CTypes.FLOAT32), col(np.arange(rows), CTypes.INT64)],
               ["a", "b", "o", "id"])
    _, metrics2 = check(t2, (0, 1), (2,), (True,), (False,), (3,), 3, id_col=3, batch=1 << 18, expected_groups=1)
    assert metrics2[3] >= 2


def test_small_groups_empty_input_and_all_na_keys():
    rng = np.random.default_rng(9)
    rows = 5000
    t = Table([col(rng.integers(0, 2000, rows), CTypes.INT64), col(rng.random(rows), CTypes.FLOAT64), col(np.arange(rows), CTypes.INT64)],
              ["k", "o", "id"])
    got = check(t, (0,), (1,), (True,), (True,), (0, 1, 2), 4, id_col=2, batch=999)[0]
    assert len(got) == np.minimum(np.bincount(t.columns[0].values_numpy()), 4).sum()
    everything = check(t, (0,), (1,), (True,), (True,), (0, 1, 2), 1000, id_col=2, batch=999)[0]
    assert len(everything) == rows
    empty = Table([col([], CTypes.INT64), col([], CTypes.FLOAT64)], ["k", "o"])
    assert rows_of(run(empty, (0,), (1,), (True,), (True,), (0, 1), 3)[0]) == []
    na_keys = Table([col(rng.integers(0, 9, 1000), CTypes.INT64, np.zeros(1000, dtype=bool)), col(rng.random(1000), CTypes.FLOAT64),
                     col(np.arange(1000), CTypes.INT64)], ["k", "o", "id"])
    got = check(na_keys, (0,), (1,), (True,), (True,), (0, 1, 2), 5, dropna=False, id_col=2, batch=300)[0]
    assert len(got) == 5 and all(r[0] is False for r in got)
    assert check(na_keys, (0,), (1,), (True,), (True,), (0, 1, 2), 5, dropna=True, batch=300)[0] == []


def test_na_nan_and_negative_zero_keys_and_sort_values():
    """NaN keys (numpy float columns) and NA keys (a nullable int column), -0.0 meeting 0.0 in keys and in the sort column."""
    rng = np.random.default_rng(13)
    rows = 30_000
    f = rng.choice(np.array([0.0, -0.0, np.nan, 1.0, -1.0]), rows)
    o = rng.choice(np.array([0.0, -0.0, np.nan, 2.0, -2.0]), rows)
    t = Table([col(f, CTypes.FLOAT64), col(rng.integers(0, 50, rows), CTypes.INT32, rng.random(rows) > 0.2),
               col(o, CTypes.FLOAT64), col(np.arange(rows), CTypes.INT64)], ["f", "i", "o", "id"])
    for dropna in (False, True):
        check(t, (0,), (2,), (True,), (False,), (0, 2, 3), 6, dropna, id_col=3, batch=4000)
        check(t, (0, 1), (2,), (False,), (True,), (0, 1, 2, 3), 2, dropna, id_col=3, batch=4000)
        f32 = Table([col(f, CTypes.FLOAT32), col(o, CTypes.FLOAT32), col(np.arange(rows), CTypes.INT64)], ["f", "o", "id"])
        check(f32, (0,), (1,), (True,), (True,), (0, 1, 2), 3, dropna, id_col=2, batch=5000)


def _arrival_case(adversarial, rows=1 << 23, groups=1000, n=3):
    import torch

    g = torch.Generator(device="cuda").manual_seed(17)
    k = torch.randint(0, groups, (rows,), device="cuda", generator=g, dtype=torch.int64)
    o = torch.arange(rows, device="cuda", dtype=torch.float64) if adversarial else torch.rand(rows, device="cuda", generator=g, dtype=torch.float64)
    rid = torch.arange(rows, device="cuda", dtype=torch.int64)
    st = G.init_groupby_state(-1, (0,), MRNF, (0, 0), (), mrnf_sort_col_inds=(1,), mrnf_sort_col_asc=(False,), mrnf_sort_col_na=(True,),
                              mrnf_col_inds_keep=(0, 1, 2), mrnf_limit=n, output_batch_size=1 << 30)
    batch = 1 << 20
    for s in range(0, rows, batch):
        e = min(rows, s + batch)
        t = Table([Column(c[s:e], None, ct, ArrTypes.NUMPY, e - s) for c, ct in ((k, CTypes.INT64), (o, CTypes.FLOAT64), (rid, CTypes.INT64))],
                  ["k", "o", "id"])
        G.groupby_build_consume_batch(st, t, e == rows, True)
    out, last = G.groupby_produce_output_batch(st, True)
    assert last
    got_ids = torch.as_tensor(out.columns[2].values_numpy()).to("cuda")
    metrics = {m: G.get_metric(st, m) for m in (0, 18, 19)}
    G.delete_groupby_state(st)
    # torch: stable sort by o descending, then stable by k; the first n rows of each k
    p = torch.sort(o, descending=True, stable=True).indices
    p = p[torch.sort(k[p], stable=True).indices]
    ks = k[p]
    start = torch.ones(rows, dtype=torch.bool, device="cuda")
    start[1:] = ks[1:] != ks[:-1]
    pos = torch.arange(rows, device="cuda")
    first = torch.cummax(torch.where(start, pos, torch.zeros_like(pos)), 0).values
    exp = p[(pos - first) < n]
    assert torch.equal(torch.sort(got_ids).values, torch.sort(exp).values)
    # order: the output lists each group's rows consecutively and by descending o (o is distinct)
    ko, oo = k[got_ids], o[got_ids]
    same = ko[1:] == ko[:-1]
    assert bool((oo[1:][same] < oo[:-1][same]).all())
    assert int(same.logical_not().sum()) + 1 == int(torch.unique(ko).numel())
    return metrics


def test_adversarial_arrival_admits_every_row_and_the_reduce_is_amortised():
    rows = 1 << 23
    m = _arrival_case(True, rows)
    assert m[18] == rows and m[0] == 3000
    # survivors stay at 3000 << 4 Mi: a reduce per 4 Mi admitted rows, plus the last one
    assert 2 <= m[19] <= rows // (1 << 22) + 1


def test_random_arrival_admits_few_rows():
    """Every row is a candidate until the first reduce (4 Mi admitted rows: the survivors, 3000, are fewer); after it the cutoffs
    reject nearly every row."""
    rows = 1 << 23
    m = _arrival_case(False, rows)
    assert m[0] == 3000 and m[19] >= 2
    assert (1 << 22) <= m[18] < (1 << 22) + rows // 100


def test_heavy_groups_against_torch():
    import torch

    rows = (1 << 22) + 5
    g = torch.Generator(device="cuda").manual_seed(5)
    k = torch.randint(0, 30, (rows,), device="cuda", generator=g, dtype=torch.int64)
    o = torch.randint(-1000, 1000, (rows,), device="cuda", generator=g, dtype=torch.int64).to(torch.float64) / 8
    rid = torch.arange(rows, device="cuda", dtype=torch.int64)
    t = Table([Column(k, None, CTypes.INT64, ArrTypes.NUMPY, rows), Column(o, None, CTypes.FLOAT64, ArrTypes.NUMPY, rows),
               Column(rid, None, CTypes.INT64, ArrTypes.NUMPY, rows)], ["k", "o", "id"])
    st = G.init_groupby_state(-1, (0,), MRNF, (0, 0), (), mrnf_sort_col_inds=(1,), mrnf_sort_col_asc=(False,), mrnf_sort_col_na=(True,),
                              mrnf_col_inds_keep=(0, 1, 2), mrnf_limit=1000, output_batch_size=4096)
    G.groupby_build_consume_batch(st, t, True, True)
    ids = []
    while True:
        out, last = G.groupby_produce_output_batch(st, True)
        ids.append(out.columns[2].values_numpy().copy())
        if last:
            break
    G.delete_groupby_state(st)
    got = torch.as_tensor(np.concatenate(ids)).to("cuda")
    p = torch.sort(o, descending=True, stable=True).indices
    p = p[torch.sort(k[p], stable=True).indices]
    ks = k[p]
    start = torch.ones(rows, dtype=torch.bool, device="cuda")
    start[1:] = ks[1:] != ks[:-1]
    pos = torch.arange(rows, device="cuda")
    first = torch.cummax(torch.where(start, pos, torch.zeros_like(pos)), 0).values
    exp = p[(pos - first) < 1000]
    assert len(got) == 30_000
    # groups are consecutive and each is in rank order, across the 4096-row output batches
    kg = k[got]
    starts = torch.nonzero(torch.cat([torch.ones(1, dtype=torch.bool, device="cuda"), kg[1:] != kg[:-1]])).flatten().tolist() + [len(got)]
    assert len(starts) == 31
    exp_by_key = {int(k[exp[i]]): exp[i:i + 1000] for i in range(0, 30_000, 1000)}
    for a, b in zip(starts[:-1], starts[1:]):
        assert torch.equal(got[a:b], exp_by_key[int(kg[a])])


def test_every_payload_type_and_a_kept_float_key_holding_negative_zero():
    rng = np.random.default_rng(3)
    rows = 5000
    cols = [col(rng.choice(np.array([0.0, -0.0, 1.0, np.nan]), rows), CTypes.FLOAT64), col(rng.integers(0, 1000, rows), CTypes.INT32)]
    for j, ct in enumerate(SORT_TYPES):
        cols.append(random_col(rng, ct, rows, nullable=j % 2 == 1))
    cols.append(col(np.arange(rows), CTypes.INT64))
    t = Table(cols, [f"c{j}" for j in range(len(cols))])
    for dropna in (False, True):
        check(t, (0,), (1,), (True,), (True,), tuple(range(len(cols))), 40, dropna, id_col=len(cols) - 1, batch=999, output_batch_size=40)
        check(t, (0,), (1,), (True,), (True,), tuple(range(len(cols))), 3, dropna, id_col=len(cols) - 1, batch=999, output_batch_size=7,
              device=False)
    t2 = Table([col([-0.0, 0.0, 0.0, -0.0], CTypes.FLOAT64), col([1, 2, 0, 3], CTypes.INT64)], ["f", "o"])
    got, _ = run(t2, (0,), (1,), (True,), (True,), (0, 1), 2)
    zero, neg = 0, int(np.float64(-0.0).view(np.uint64))
    assert rows_of(got) == sorted([(True, zero, True, 0), (True, neg, True, 1)])


def test_limit_one_is_the_default_filter():
    rng = np.random.default_rng(4)
    rows = 50_000
    t = Table([col(rng.integers(0, 3000, rows), CTypes.INT64, rng.random(rows) > 0.05), col(rng.integers(0, 7, rows), CTypes.INT8),
               col(np.arange(rows), CTypes.INT64)], ["k", "o", "id"])
    one, m1 = run(t, (0,), (1,), (False,), (True,), (0, 1, 2), 1, batch=4096)
    st = G.init_groupby_state(-1, (0,), MRNF, (0, 0), (), mrnf_sort_col_inds=(1,), mrnf_sort_col_asc=(False,), mrnf_sort_col_na=(True,),
                              mrnf_col_inds_keep=(0, 1, 2), dropna=False)
    for s in range(0, rows, 4096):
        G.groupby_build_consume_batch(st, table_to_device(t.slice(s, min(rows, s + 4096))), s + 4096 >= rows, True)
    out, _ = G.groupby_produce_output_batch(st, True)
    default = rows_of([host_cells(c) for c in out.columns])
    G.delete_groupby_state(st)
    assert rows_of(one) == default and m1[18] == 0 and m1[19] == 0 and m1[0] == len(default)


def test_agrees_with_window_row_number_and_pandas():
    from bodo_b200.physical import min_row_number_filter, window

    rng = np.random.default_rng(21)
    rows = 30_000
    df = pd.DataFrame({"k": pd.array(rng.integers(0, 800, rows), dtype="Int64"), "o": rng.random(rows).round(2), "v": rng.integers(0, 10, rows),
                       "id": np.arange(rows)})
    df.loc[rng.random(rows) < 0.02, "k"] = pd.NA
    for dropna in (False, True):
        got = min_row_number_filter(df, "k", ["o", "v"], ascending=[False, True], keep=["id", "k", "o"], dropna=dropna, n=3, batch_size=4096)
        assert list(got.columns) == ["id", "k", "o"]
        exp = df.sort_values(["o", "v"], ascending=[False, True], kind="stable").groupby("k", sort=False, dropna=dropna).head(3)
        assert sorted(got["id"].tolist()) == sorted(exp["id"].tolist())
    w = window(df, ["k"], ["o", "v"], [("rn", "row_number")], ascending=[False, True], batch_size=4096)
    got = min_row_number_filter(df, "k", ["o", "v"], ascending=[False, True], keep="id", n=3)
    assert sorted(w.loc[w["rn"] <= 3, "id"].tolist()) == sorted(got["id"].tolist())


def test_parallel_state_with_one_rank_runs_locally():
    import socket

    import torch.distributed as dist

    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    dist.init_process_group("gloo", init_method=f"tcp://127.0.0.1:{port}", rank=0, world_size=1)
    try:
        rng = np.random.default_rng(2)
        rows = 10_000
        t = Table([col(rng.integers(0, 100, rows), CTypes.INT64), col(rng.random(rows), CTypes.FLOAT64), col(np.arange(rows), CTypes.INT64)],
                  ["k", "o", "id"])
        check(t, (0,), (1,), (True,), (True,), (0, 1, 2), 4, id_col=2, parallel=True, batch=3000)
    finally:
        dist.destroy_process_group()


def test_the_candidate_limit_is_refused_before_reading_the_batch():
    """A batch whose rows, added to the survivors, pass the store's 2^31-row sort raises B200Error naming the limit.  The batch is a
    descriptor of 2^31 rows whose columns have no data: the refusal comes before any check or kernel would read them."""
    from bodo_b200 import _lib

    ffi, L = _lib.ffi, _lib.lib()
    rng = np.random.default_rng(1)
    t = Table([col(rng.integers(0, 10, 100), CTypes.INT64), col(rng.random(100), CTypes.FLOAT64)], ["k", "o"])
    st = G.init_groupby_state(-1, (0,), MRNF, (0, 0), (), mrnf_sort_col_inds=(1,), mrnf_sort_col_asc=(True,), mrnf_sort_col_na=(True,),
                              mrnf_col_inds_keep=(0, 1), mrnf_limit=5)
    G.groupby_build_consume_batch(st, table_to_device(t), False, True)
    cols = ffi.new("b200_column[]", 2)
    for c, ct in zip(cols, (CTypes.INT64, CTypes.FLOAT64)):
        c.data, c.validity, c.c_type, c.arr_type, c.length = ffi.NULL, ffi.NULL, ct, ArrTypes.NUMPY, 1 << 31
    big = ffi.new("b200_table*")
    big.n_rows, big.n_cols, big.cols, big.device = 1 << 31, 2, cols, st.device
    req = ffi.new("int32_t*")
    assert L.b200_groupby_build_consume_batch(st.handle, big, 0, 1, req) < 0
    msg = ffi.string(L.b200_last_error()).decode()
    assert "2^31" in msg and "groups x rows_per_group" in msg and "survivors" in msg, msg
    # the state is intact: the last batch and the output still come through
    G.groupby_build_consume_batch(st, table_to_device(t), True, True)
    out, _ = G.groupby_produce_output_batch(st, True)
    both = Table([col(np.r_[t.columns[0].values_numpy(), t.columns[0].values_numpy()], CTypes.INT64),
                  col(np.r_[t.columns[1].values_numpy(), t.columns[1].values_numpy()], CTypes.FLOAT64)], ["k", "o"])
    kept, _, _ = oracle_rows(both, (0,), (1,), (True,), (True,), False, 5)
    assert rows_of([host_cells(c) for c in out.columns]) == rows_of([host_cells(c) for c in both.columns], kept)
    G.delete_groupby_state(st)
    with pytest.raises(B200Error, match="mrnf_limit"):
        G.init_groupby_state(-1, (0,), MRNF, (0, 0), (), mrnf_sort_col_inds=(1,), mrnf_sort_col_asc=(True,), mrnf_sort_col_na=(True,),
                             mrnf_col_inds_keep=(0, 1), mrnf_limit=1 << 31)
