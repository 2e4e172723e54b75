"""GPU tests of the groupby's min_row_number_filter (QUALIFY ROW_NUMBER() OVER (PARTITION BY k ORDER BY o) = 1) against an exact
numpy oracle: keys canonicalised (float -0.0 is 0.0, NaN is NA), rows lexsorted by (key, class / order word per sort column,
arrival), the first row per group kept.  Outputs are compared bit for bit (validity, and the bits of every valid cell) as
multisets of rows, since group order is unspecified."""

import numpy as np
import pandas as pd
import pytest

from bodo_b200.streaming import groupby as G
from bodo_b200.table import ArrTypes, Column, CTypes, Table
from tests.helpers import table_to_device

pytestmark = pytest.mark.gpu

MRNF = ("min_row_number_filter",)
NP = {CTypes.INT8: np.int8, CTypes.UINT8: np.uint8, CTypes.INT16: np.int16, CTypes.UINT16: np.uint16, CTypes.INT32: np.int32,
      CTypes.UINT32: np.uint32, CTypes.INT64: np.int64, CTypes.UINT64: np.uint64, CTypes.FLOAT32: np.float32,
      CTypes.FLOAT64: np.float64, CTypes.BOOL: np.bool_, CTypes.DATE: np.int32, CTypes.DATETIME: np.int64, CTypes.TIMEDELTA: np.int64}
SIGNED = {CTypes.INT8, CTypes.INT16, CTypes.INT32, CTypes.INT64, CTypes.DATE, CTypes.DATETIME, CTypes.TIMEDELTA}
FLOATS = {CTypes.FLOAT32, CTypes.FLOAT64}


def col(values, ct, valid=None):
    values = np.ascontiguousarray(np.asarray(values).astype(NP[ct]))
    bm = None if valid is None else np.packbits(np.asarray(valid, dtype=bool), bitorder="little")
    return Column(values, bm, ct, ArrTypes.NUMPY if valid is None else ArrTypes.NULLABLE_INT_BOOL, len(values))


def random_col(rng, ct, n, nullable):
    """n cells of type ct with the type's extremes, ties, and (floats) NaN, +-0.0 and +-inf; 15 % NA when nullable."""
    if ct in FLOATS:
        v = rng.choice(np.array([np.nan, 0.0, -0.0, np.inf, -np.inf, 1.5, -1.5, 7.0, 1e300 if ct == CTypes.FLOAT64 else 3e38]), n)
        v = np.where(rng.random(n) < 0.5, v, rng.integers(-5, 5, n).astype(np.float64))
    elif ct == CTypes.BOOL:
        v = rng.random(n) < 0.5
    else:
        info = np.iinfo(NP[ct])
        v = rng.choice(np.array([info.min, info.max, 0, 1, info.max - 1], dtype=NP[ct]), n)
        v = np.where(rng.random(n) < 0.6, v, rng.integers(max(info.min, -5), 6, n).astype(NP[ct]))
    return col(v, ct, rng.random(n) > 0.15 if nullable else None)


def host_cells(c: Column):
    """(valid, bits) of a column: bits as uint64, 0 where the cell is NA."""
    v = c.values_numpy()
    u = v.view({1: np.uint8, 2: np.uint16, 4: np.uint32, 8: np.uint64}[v.dtype.itemsize]).astype(np.uint64)
    m = c.valid_mask_numpy()
    m = np.ones(len(v), dtype=bool) if m is None else m
    return m, np.where(m, u, 0)


def order_key(c: Column, asc: bool, na_last: bool):
    """(class, value) arrays whose lexicographic order is the sort's order of the column's cells."""
    v = c.values_numpy()
    m = c.valid_mask_numpy()
    na = np.zeros(len(v), dtype=bool) if m is None else ~m
    if c.c_type in FLOATS:
        f = v.astype(np.float64)
        na = na | np.isnan(f)
        w = np.where(na, 0.0, f) + 0.0  # -0.0 ties with 0.0
        w = w if asc else -w
    else:
        u = v.astype(np.int64).view(np.uint64) ^ np.uint64(1 << 63) if c.c_type in SIGNED else v.astype(np.uint64)
        w = np.where(na, np.uint64(0), u if asc else ~u)
    cls = np.where(na, 1 if na_last else 0, 0 if na_last else 1)
    return cls, w


def key_parts(c: Column):
    """Canonical key cells: (valid, bits) with float -0.0 as 0.0 and NaN as NA."""
    m, bits = host_cells(c)
    if c.c_type in FLOATS:
        f = c.values_numpy().astype(np.float64)
        m = m & ~np.isnan(f)
        bits = np.where(m, (f + 0.0).view(np.uint64), 0)
    return m, bits


def oracle(t: Table, key_inds, sort, asc, na, keep, dropna):
    n = t.n_rows
    kp = [key_parts(t.columns[i]) for i in key_inds]
    rows = np.arange(n)
    if dropna:
        ok = np.logical_and.reduce([m for m, _ in kp])
        rows = rows[ok]
    lex = [rows]
    for j in reversed(range(len(sort))):
        cls, w = order_key(t.columns[sort[j]], asc[j], na[j])
        lex += [w[rows], cls[rows]]
    order = rows[np.lexsort(lex)]
    g = pd.DataFrame({f"{p}{j}": a[order] for j, (m, b) in enumerate(kp) for p, a in (("m", m), ("b", b))})
    win = order[~g.duplicated(keep="first").to_numpy()] if len(order) else order
    return rows_of([host_cells(t.columns[i]) for i in sorted(keep)], win)


def rows_of(cells, idx=None):
    """The rows as a sorted list of tuples (valid_0, bits_0, valid_1, ...)."""
    parts = []
    for m, b in cells:
        parts += [m if idx is None else m[idx], b if idx is None else b[idx]]
    if not parts or len(parts[0]) == 0:
        return []
    return sorted(zip(*[p.tolist() for p in parts]))


def run(t: Table, key_inds, sort, asc, na, keep, dropna=False, batch=None, device=True, **kw):
    st = G.init_groupby_state(-1, key_inds, MRNF, (0, 0), (), mrnf_sort_col_inds=sort, mrnf_sort_col_asc=asc, mrnf_sort_col_na=na,
                              mrnf_col_inds_keep=keep, dropna=dropna, **kw)
    n = t.n_rows
    batch = batch or max(n, 1)
    starts = list(range(0, n, batch)) or [0]
    for i, s in enumerate(starts):
        b = t.slice(s, min(n, s + batch))
        G.groupby_build_consume_batch(st, table_to_device(b) if device else b, i == len(starts) - 1, True)
    outs = []
    while True:
        out, last = G.groupby_produce_output_batch(st, True)
        outs.append([host_cells(c) for c in out.columns])
        names = list(out.names)
        if last:
            break
    metrics = {m: G.get_metric(st, m) for m in (0, 3)}
    G.delete_groupby_state(st)
    assert names == [t.names[i] for i in sorted(keep)]
    cells = [(np.concatenate([o[j][0] for o in outs]), np.concatenate([o[j][1] for o in outs])) for j in range(len(keep))]
    return rows_of(cells), metrics


def check(t, key_inds, sort, asc, na, keep, dropna=False, **kw):
    got, metrics = run(t, key_inds, sort, asc, na, keep, dropna, **kw)
    exp = oracle(t, key_inds, sort, asc, na, keep, dropna)
    assert len(got) == len(exp)
    assert got == exp
    return got, metrics


SORT_TYPES = [CTypes.INT8, CTypes.UINT8, CTypes.INT16, CTypes.UINT16, CTypes.INT32, CTypes.UINT32, CTypes.INT64, CTypes.UINT64,
              CTypes.FLOAT32, CTypes.FLOAT64, CTypes.BOOL, CTypes.DATE, CTypes.DATETIME, CTypes.TIMEDELTA]


@pytest.mark.parametrize("ct", SORT_TYPES)
@pytest.mark.parametrize("nullable", [False, True])
def test_every_sort_type_both_directions_and_na_placements(ct, nullable):
    rng = np.random.default_rng(ct * 2 + nullable)
    n = 3000
    t = Table([col(rng.integers(0, 40, n), CTypes.INT64), random_col(rng, ct, n, nullable), col(np.arange(n), CTypes.INT64)],
              ["k", "o", "id"])
    for asc in (True, False):
        for na_last in (True, False):
            check(t, (0,), (1,), (asc,), (na_last,), (0, 1, 2), batch=700)


@pytest.mark.parametrize("n_sort", [1, 2, 3, 4])
@pytest.mark.parametrize("n_keys", [1, 2, 3, 4])
def test_sort_columns_and_keys(n_sort, n_keys):
    rng = np.random.default_rng(100 + 4 * n_sort + n_keys)
    n = 20_000
    key_types = [CTypes.FLOAT64, CTypes.INT32, CTypes.FLOAT32, CTypes.INT64][:n_keys]
    cols, names = [], []
    for j, ct in enumerate(key_types):
        if ct in FLOATS:
            v = rng.choice(np.array([0.0, -0.0, np.nan, 1.5, -2.0, np.inf]), n)
        else:
            v = rng.integers(0, 6 if n_keys > 1 else 300, n)
        cols.append(col(v, ct, rng.random(n) > 0.1 if j % 2 == 1 else None))
        names.append(f"k{j}")
    order_types = [CTypes.FLOAT64, CTypes.INT8, CTypes.DATETIME, CTypes.UINT16][:n_sort]
    for j, ct in enumerate(order_types):
        cols.append(random_col(rng, ct, n, nullable=j % 2 == 0))
        names.append(f"o{j}")
    cols.append(col(np.arange(n), CTypes.INT64))
    names.append("id")
    t = Table(cols, names)
    sort = tuple(range(n_keys, n_keys + n_sort))
    asc = tuple(bool(j % 2) for j in range(n_sort))
    na = tuple(j % 3 != 1 for j in range(n_sort))
    for dropna in (False, True):
        check(t, tuple(range(n_keys)), sort, asc, na, tuple(range(len(cols))), dropna, batch=6_000)
    # a sort column that is also the key, and keys that are not kept
    check(t, (0,), (0, n_keys), (False, True), (True, False), (len(cols) - 1, n_keys), batch=4_096)


def test_ties_across_batches_keep_the_earliest_row_and_batch_splits_agree():
    rng = np.random.default_rng(7)
    n = 100_003
    t = Table([col(rng.integers(0, 5000, n), CTypes.INT64), col(rng.integers(0, 3, n), CTypes.INT16), col(np.arange(n), CTypes.INT64)],
              ["k", "o", "id"])
    results = [check(t, (0,), (1,), (True,), (True,), (0, 1, 2), batch=b)[0] for b in (7, 32768, None)]
    assert results[0] == results[1] == results[2]
    assert len(results[0]) == len(np.unique(t.columns[0].values_numpy()))
    small = t.slice(0, 2_000)
    one_row = check(small, (0,), (1,), (False,), (True,), (0, 1, 2), batch=1)[0]
    assert one_row == check(small, (0,), (1,), (False,), (True,), (0, 1, 2))[0]


def test_growth_mid_batch_one_million_groups():
    rng = np.random.default_rng(11)
    n = 1 << 22
    k = rng.permutation(n)[:n] % 1_000_000
    t = Table([col(k, CTypes.INT64), col(rng.random(n), CTypes.FLOAT64), col(np.arange(n), CTypes.INT64)], ["k", "o", "id"])
    got, metrics = check(t, (0,), (1,), (False,), (True,), (0, 1, 2), batch=1 << 21, expected_groups=1)
    assert metrics[3] >= 1 and len(got) == 1_000_000
    # a multi-column key grows the tag table too
    t2 = Table([col(k // 1000, CTypes.INT32), col(k % 1000, CTypes.INT64), col(rng.random(n), CTypes.FLOAT32), col(np.arange(n), CTypes.INT64)],
               ["a", "b", "o", "id"])
    got2, metrics2 = check(t2, (0, 1), (2,), (True,), (False,), (3,), batch=1 << 21, expected_groups=1)
    assert metrics2[3] >= 1 and len(got2) == 1_000_000


def test_many_rows_few_groups_against_torch():
    import torch

    n = (1 << 24) + 3
    g = torch.Generator(device="cuda").manual_seed(5)
    k = torch.randint(0, 30, (n,), device="cuda", generator=g, dtype=torch.int64)
    o = torch.randint(-1000, 1000, (n,), device="cuda", generator=g, dtype=torch.int64).to(torch.float64) / 8
    rid = torch.arange(n, device="cuda", dtype=torch.int64)
    t = Table([Column(k, None, CTypes.INT64, ArrTypes.NUMPY, n), Column(o, None, CTypes.FLOAT64, ArrTypes.NUMPY, n),
               Column(rid, None, CTypes.INT64, ArrTypes.NUMPY, n)], ["k", "o", "id"])
    st = G.init_groupby_state(-1, (0,), MRNF, (0, 0), (), mrnf_sort_col_inds=(1,), mrnf_sort_col_asc=(False,), mrnf_sort_col_na=(True,),
                              mrnf_col_inds_keep=(0, 1, 2))
    G.groupby_build_consume_batch(st, t, True, True)
    out, last = G.groupby_produce_output_batch(st, True)
    assert last
    got = sorted(zip(*[c.values_numpy().tolist() for c in out.columns]))
    G.delete_groupby_state(st)
    # torch: stable sort by o descending, then stable by k; the first row of each k
    p = torch.sort(o, descending=True, stable=True).indices
    p = p[torch.sort(k[p], stable=True).indices]
    first = torch.ones(n, dtype=torch.bool, device="cuda")
    first[1:] = k[p][1:] != k[p][:-1]
    w = p[first]
    exp = sorted(zip(k[w].tolist(), o[w].tolist(), rid[w].tolist()))
    assert got == exp and len(got) == 30


def test_every_payload_type_and_a_kept_float_key_holding_negative_zero():
    rng = np.random.default_rng(3)
    n = 5000
    cols = [col(rng.choice(np.array([0.0, -0.0, 1.0, np.nan]), n), CTypes.FLOAT64), col(rng.integers(0, 1000, n), CTypes.INT32)]
    for j, ct in enumerate(SORT_TYPES):
        cols.append(random_col(rng, ct, n, nullable=j % 2 == 1))
    t = Table(cols, [f"c{j}" for j in range(len(cols))])
    for dropna in (False, True):
        got, _ = check(t, (0,), (1,), (True,), (True,), tuple(range(len(cols))), dropna, batch=999)
        keys = {(r[0], r[1]) for r in got}
        assert len(keys) == len(got)
    # the winner's own -0.0 comes back, not the canonical key
    t2 = Table([col([-0.0, 0.0, 0.0], CTypes.FLOAT64), col([1, 2, 0], CTypes.INT64)], ["f", "o"])
    got2, _ = run(t2, (0,), (1,), (True,), (True,), (0, 1))
    assert got2 == [(True, 0, True, 0)]
    got3, _ = run(t2, (0,), (1,), (False,), (True,), (0,), batch=1)  # o DESC: row 1 (0.0) wins
    assert got3 == [(True, 0)]
    t3 = Table([col([0.0, -0.0, 0.0], CTypes.FLOAT64), col([1, 0, 2], CTypes.INT64)], ["f", "o"])
    got4, _ = run(t3, (0,), (1,), (True,), (True,), (0,), batch=2)  # o ASC: row 1 (-0.0) wins
    assert got4 == [(True, int(np.float64(-0.0).view(np.uint64)))]


def test_empty_input_all_na_keys_and_small_output_batches():
    empty = Table([col([], CTypes.INT64), col([], CTypes.FLOAT64)], ["k", "o"])
    assert run(empty, (0,), (1,), (True,), (True,), (0, 1))[0] == []
    n = 1000
    rng = np.random.default_rng(9)
    na_keys = Table([col(rng.integers(0, 9, n), CTypes.INT64, np.zeros(n, dtype=bool)), col(rng.random(n), CTypes.FLOAT64),
                     col(np.arange(n), CTypes.INT64)], ["k", "o", "id"])
    got, _ = check(na_keys, (0,), (1,), (True,), (True,), (0, 1, 2), dropna=False, batch=300)
    assert len(got) == 1 and got[0][0] is False
    assert check(na_keys, (0,), (1,), (True,), (True,), (0, 1, 2), dropna=True, batch=300)[0] == []
    t = Table([col(rng.integers(0, 500, 20_000), CTypes.INT64, rng.random(20_000) > 0.05), col(rng.random(20_000), CTypes.FLOAT32),
               col(np.arange(20_000), CTypes.INT64, rng.random(20_000) > 0.5)], ["k", "o", "id"])
    check(t, (0,), (1,), (True,), (False,), (2, 0), output_batch_size=40)
    check(t, (0,), (1,), (True,), (False,), (2,), output_batch_size=7, device=False)


def test_agrees_with_window_row_number_and_pandas():
    from bodo_b200.physical import min_row_number_filter, window

    rng = np.random.default_rng(21)
    n = 30_000
    df = pd.DataFrame({"k": pd.array(rng.integers(0, 800, n), dtype="Int64"), "o": rng.random(n).round(2), "v": rng.integers(0, 10, n),
                       "id": np.arange(n)})
    df.loc[rng.random(n) < 0.02, "k"] = pd.NA
    got = min_row_number_filter(df, "k", ["o", "v"], ascending=[False, True], keep=["id", "k", "o"], batch_size=4096)
    assert list(got.columns) == ["id", "k", "o"]
    exp = df.sort_values(["o", "v"], ascending=[False, True], kind="stable").drop_duplicates("k", keep="first")[["id", "k", "o"]]
    assert sorted(got["id"].tolist()) == sorted(exp["id"].tolist())
    w = window(df, ["k"], ["o", "v"], [("rn", "row_number")], ascending=[False, True], batch_size=4096)
    assert sorted(w.loc[w["rn"] == 1, "id"].tolist()) == sorted(got["id"].tolist())
    # dropna=True drops the NA key's row
    got_d = min_row_number_filter(df, "k", "o", keep="id", dropna=True)
    assert len(got_d) == df["k"].nunique()


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
        n = 10_000
        t = Table([col(rng.integers(0, 100, n), CTypes.INT64), col(rng.random(n), CTypes.FLOAT64), col(np.arange(n), CTypes.INT64)],
                  ["k", "o", "id"])
        check(t, (0,), (1,), (True,), (True,), (0, 1, 2), parallel=True, batch=3000)
    finally:
        dist.destroy_process_group()
