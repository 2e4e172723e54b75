"""Ranking window functions (ROW_NUMBER, RANK, DENSE_RANK, PERCENT_RANK, CUME_DIST, NTILE) on the GPU, bit for bit.

The oracle is numpy / pandas, independent of the device's radix words: the stable permutation is tests/test_gpu_sort.py's
oracle_perm over (partition keys ascending NA last, order keys); partition and peer boundaries come from adjacent equality of
(isna_j, key_j) in that order (NaN is NA, -0.0 == 0.0); the functions follow their SQL definitions from the boundaries.  Every
input column is compared byte for byte with the input rows at the oracle's permutation, and every function column exactly."""

import numpy as np
import pandas as pd
import pyarrow as pa
import pytest
import torch

from bodo_b200 import _lib
from bodo_b200._lib import B200Error
from bodo_b200.streaming import window as W
from bodo_b200.table import ArrTypes, Column, CTypes, Table, np_dtype_of
from tests.helpers import table_to_device
from tests.test_gpu_sort import KEY_TYPES, batches_of, col_mask, make_column, oracle_perm

pytestmark = pytest.mark.gpu

TILE = 2048  # rows per window-kernel tile
CHUNK = 1 << 24  # rows per store chunk
ALL = [("rn", "row_number"), ("rk", "rank"), ("dr", "dense_rank"), ("pr", "percent_rank"), ("cd", "cume_dist"), ("nt3", "ntile", 3)]


@pytest.fixture(autouse=True)
def _return_device_memory():
    yield
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    _lib.lib().b200_pool_trim(torch.cuda.current_device(), 0)


def oracle(table, part, order, asc, nap, funcs):
    """(permutation, {out_name: expected column}, number of partitions)."""
    keys = part + order
    perm = oracle_perm(table, keys, [True] * len(part) + list(asc), ["last"] * len(part) + list(nap))
    n = len(perm)
    idx = np.arange(n, dtype=np.int64)

    def adjacent_equal(name):
        c = table.columns[table.names.index(name)]
        v = c.values_numpy()[perm]
        na = ~col_mask(c)[perm]
        if v.dtype.kind == "f":
            na |= np.isnan(v)
        v = np.where(na, 0, v)
        return (na[1:] == na[:-1]) & (v[1:] == v[:-1])

    pstart = np.ones(n, bool)
    qstart = np.ones(n, bool)
    if n:
        peq = np.ones(n - 1, bool)
        for k in part:
            peq &= adjacent_equal(k)
        oeq = peq.copy()
        for k in order:
            oeq &= adjacent_equal(k)
        pstart[1:] = ~peq
        qstart[1:] = ~oeq
    P = np.maximum.accumulate(np.where(pstart, idx, 0)) if n else idx
    Q = np.maximum.accumulate(np.where(qstart, idx, 0)) if n else idx
    D = np.cumsum(qstart)
    pid = np.cumsum(pstart) - 1
    s = np.bincount(pid, minlength=1)[pid].astype(np.int64)
    starts = np.flatnonzero(qstart)
    qend = np.append(starts[1:], n)[np.cumsum(qstart) - 1] if n else idx
    pos = idx - P
    rank = Q - P + 1
    exp = {}
    for f in funcs:
        name, fn = f[0], f[1]
        if fn == "row_number":
            exp[name] = pos + 1
        elif fn == "rank":
            exp[name] = rank
        elif fn == "dense_rank":
            exp[name] = (D - D[P] + 1).astype(np.int64)
        elif fn == "percent_rank":
            exp[name] = np.where(s == 1, 0.0, (rank - 1).astype(np.float64) / np.maximum(s - 1, 1).astype(np.float64))
        elif fn == "cume_dist":
            exp[name] = (qend - P).astype(np.float64) / s.astype(np.float64)
        else:
            nb = f[2]
            q, r = s // nb, s % nb
            big = r * (q + 1)
            exp[name] = np.where(pos < big, pos // (q + 1) + 1, r + (pos - big) // np.maximum(q, 1) + 1).astype(np.int64)
    return perm, exp, int(pstart.sum()) if n else 0


def run_window(table, part, order, asc, nap, funcs, sizes=(1 << 30,), device=True, empty_every=0, output_batch_size=32768):
    st = W.init_window_state(-1, part, order, asc, nap, funcs, table.names, output_batch_size=output_batch_size)
    bs = batches_of(table, list(sizes), empty_every)
    for i, b in enumerate(bs):
        W.window_build_consume_batch(st, table_to_device(b) if device else b, i == len(bs) - 1)
    outs = []
    while True:
        out, last = W.window_produce_output_batch(st)
        outs.append(out)
        if last:
            break
    metrics = [W.get_metric(st, w) for w in range(10)]
    ncols = table.n_cols + len(funcs)
    assert all(o.n_cols == ncols for o in outs)
    assert outs[0].names == list(table.names) + [f[0] for f in funcs]
    res = [(np.concatenate([o.columns[c].values_numpy() for o in outs]),
            np.concatenate([col_mask(o.columns[c]) for o in outs]),
            outs[0].columns[c]) for c in range(ncols)]
    W.delete_window_state(st)
    return res, metrics, [o.n_rows for o in outs]


def check(table, part, order, asc, nap, funcs=ALL, **kw):
    part, order = list(part), list(order)
    perm, exp, n_parts = oracle(table, part, order, asc, nap, funcs)
    got, metrics, sizes = run_window(table, part, order, asc, nap, funcs, **kw)
    for c, (vals, mask, oc) in zip(table.columns, got):
        assert oc.c_type == c.c_type and oc.arr_type == c.arr_type
        e = c.values_numpy()[perm]
        assert vals.dtype == np_dtype_of(c.c_type) and len(vals) == len(perm)
        np.testing.assert_array_equal(vals.view(np.uint8), e.view(np.uint8))
        np.testing.assert_array_equal(mask, col_mask(c)[perm])
    for f, (vals, mask, oc) in zip(funcs, got[table.n_cols:]):
        real = f[1] in ("percent_rank", "cume_dist")
        assert oc.c_type == (CTypes.FLOAT64 if real else CTypes.INT64) and oc.arr_type == ArrTypes.NUMPY and oc.validity is None
        assert mask.all() and vals.dtype == (np.float64 if real else np.int64)
        np.testing.assert_array_equal(vals.view(np.uint64), exp[f[0]].view(np.uint64), err_msg=f[0])
    assert metrics[0] == table.n_rows and metrics[1:6] == [0] * 5 and metrics[9] == n_parts
    return metrics, sizes


def _i64(v):
    return Column(np.ascontiguousarray(v, dtype=np.int64), None, CTypes.INT64, ArrTypes.NUMPY, len(v))


# ---- every key type as a PARTITION BY and as an ORDER BY key ----
@pytest.mark.parametrize("ct", KEY_TYPES)
@pytest.mark.parametrize("nullable", [False, True])
def test_key_types(gpu_lib, ct, nullable):
    rng = np.random.default_rng(100 + ct * 2 + nullable)
    n = 5000
    k = make_column(ct, n, rng, nullable)  # many ties, the type's edge values (+-0.0, NaN next to NA, +-inf, subnormals)
    o = make_column(CTypes.INT16, n, rng, True, na_frac=0.1)
    g = make_column(CTypes.INT8, n, rng, False)
    p = make_column(CTypes.FLOAT64, n, rng, True, small=False)
    t = Table([p, k, o, g], ["p", "k", "o", "g"])
    check(t, ["k"], ["o"], [True], ["last"], sizes=(1000,), empty_every=2)
    for asc in (True, False):
        for nap in ("first", "last"):
            check(t, ["g"], ["k"], [asc], [nap], sizes=(1777,))


@pytest.mark.parametrize("n_keys", [1, 2, 3, 4])
def test_every_split_of_the_keys(gpu_lib, n_keys):
    rng = np.random.default_rng(200 + n_keys)
    n = 20_000
    types = [CTypes.INT32, CTypes.FLOAT64, CTypes.DATETIME, CTypes.UINT16][:n_keys]
    cols = [make_column(ct, n, rng, True, na_frac=0.1) for ct in types] + [make_column(CTypes.FLOAT32, n, rng, True, small=False)]
    names = [f"k{j}" for j in range(n_keys)] + ["x"]
    t = Table(cols, names)
    for n_part in range(n_keys + 1):
        part, order = names[:n_part], names[n_part:n_keys]
        asc = [j % 2 == 0 for j in range(len(order))]
        nap = ["first" if j % 3 == 1 else "last" for j in range(len(order))]
        check(t, part, order, asc, nap, sizes=(4096, 1000))
    # keys need not be the leading columns, and may come in any column order
    check(Table(cols[::-1], names[::-1]), names[:n_keys][::-1][:1], names[:n_keys][::-1][1:], [False] * (n_keys - 1),
          ["first"] * (n_keys - 1), sizes=(32768,))


def test_degenerate_partitions(gpu_lib):
    rng = np.random.default_rng(3)
    n = 3 * TILE + 17
    t = Table([_i64(rng.integers(0, 40, n)), _i64(np.full(n, 5)), _i64(rng.permutation(n)), _i64(rng.integers(0, 7, n))],
              ["g", "c", "u", "o"])
    check(t, [], ["o"], [True], ["last"])        # no PARTITION BY: one partition
    check(t, ["g"], [], [], [])                  # no ORDER BY: every row of a partition is a peer
    check(t, ["c"], ["o"], [False], ["last"])    # a single partition
    check(t, ["u"], ["o"], [True], ["last"])     # every row its own partition
    check(t, ["g"], ["c"], [True], ["last"])     # a constant order key
    check(t, ["u"], [], [], [])


def test_ntile_and_percent_rank_edges(gpu_lib):
    sizes = [1, 2, 3, 4, 5, 6, 7, 10, 16, 33, 100, 1000, 2049]
    g = np.repeat(np.arange(len(sizes)), sizes)
    rng = np.random.default_rng(4)
    perm = rng.permutation(len(g))
    t = Table([_i64(g[perm]), _i64(rng.integers(0, 5, len(g)))], ["g", "o"])
    funcs = [("pr", "percent_rank"), ("cd", "cume_dist")] + [(f"nt{m}", "ntile", m) for m in (1, 2, 3, 4, 7, 10, 33, 1000, 2049, 1 << 40)]
    check(t, ["g"], ["o"], [True], ["last"], funcs=funcs, sizes=(999,))
    got, _, _ = run_window(t, ["g"], ["o"], [True], ["last"], funcs)
    gs = got[0][0]
    pos = np.concatenate([np.arange(s) for s in sizes])
    s_of = np.asarray(sizes)[gs]
    np.testing.assert_array_equal(got[2 + 2][0], np.ones(len(g), np.int64))                 # ntile(1)
    np.testing.assert_array_equal(got[2 + 11][0], pos + 1)                                    # ntile(n > s)
    np.testing.assert_array_equal(got[2][0][s_of == 1], 0.0)                                  # percent_rank with s = 1


@pytest.mark.parametrize("n", [1, 2, TILE - 1, TILE, TILE + 1, 3 * TILE + 17, 40_000])
def test_tile_edges_and_batches(gpu_lib, n):
    """Partitions and peer groups straddle the window kernels' tile edges; batch sizes around the tile; empty batches."""
    rng = np.random.default_rng(n)
    i = np.arange(n)
    t = Table([_i64(i // 1500), _i64(i // 7 % 5), make_column(CTypes.INT32, n, rng, True, small=False)], ["g", "o", "x"])
    check(t, ["g"], ["o"], [True], ["last"], sizes=(TILE - 1, TILE, TILE + 1), empty_every=3)
    check(t, [], ["g"], [False], ["first"], sizes=(1000,), device=False)  # host batches are staged; peer groups of 1500 rows
    check(t, ["o"], ["g"], [True], ["last"], output_batch_size=1000)


def test_output_batch_slicing(gpu_lib):
    rng = np.random.default_rng(5)
    n = 10_000
    t = Table([make_column(CTypes.INT32, n, rng, True), make_column(CTypes.BOOL, n, rng, True)], ["k", "b"])
    _, sizes = check(t, ["b"], ["k"], [True], ["last"], output_batch_size=1000)
    assert sizes == [1024] * 9 + [n - 9 * 1024]  # validity bitmaps are sliced at 32-row words


def test_zero_rows(gpu_lib):
    t = Table([Column(np.empty(0, np.float32), None, CTypes.FLOAT32, ArrTypes.NUMPY, 0),
               Column(np.empty(0, np.int8), np.empty(0, np.uint8), CTypes.INT8, ArrTypes.NULLABLE_INT_BOOL, 0)], ["k", "p"])
    got, m, sizes = run_window(t, ["k"], ["p"], [True], ["last"], ALL)
    assert sizes == [0] and [len(v) for v, _, _ in got] == [0] * 8
    assert [c.c_type for _, _, c in got] == [CTypes.FLOAT32, CTypes.INT8] + [CTypes.INT64] * 3 + [CTypes.FLOAT64] * 2 + [CTypes.INT64]
    assert m[0] == 0 and m[9] == 0


def test_large_input_against_torch(gpu_lib):
    """2^24 + a few tiles of device rows, so that partitions cross the first chunk's edge; checked against a torch recomputation
    (two stable sorts, then diff, cummax and cumsum on the device)."""
    n = CHUNK + 3 * TILE + 5
    dev = torch.device("cuda", 0)
    g = torch.Generator(device=dev).manual_seed(7)
    pk = torch.randint(0, 1000, (n,), generator=g, device=dev, dtype=torch.int64)
    ok = torch.round(torch.randn(n, generator=g, device=dev, dtype=torch.float64) * 64) / 4
    rid = torch.arange(n, device=dev, dtype=torch.int64)
    funcs = ALL + [("nt7", "ntile", 7)]
    st = W.init_window_state(-1, ["p"], ["o"], [False], ["last"], funcs, ["p", "o", "r"], output_batch_size=1 << 30)
    b = 3_000_000
    for r0 in range(0, n, b):
        t = Table([Column(pk[r0:r0 + b], None, CTypes.INT64), Column(ok[r0:r0 + b], None, CTypes.FLOAT64),
                   Column(rid[r0:r0 + b], None, CTypes.INT64)], ["p", "o", "r"])
        W.window_build_consume_batch(st, t, r0 + b >= n)
    out, last = W.window_produce_output_batch(st)
    assert last and out.n_rows == n
    got = [torch.as_tensor(c.data, device=dev) for c in out.columns]
    idx = torch.sort(ok, descending=True, stable=True).indices
    idx = idx[torch.sort(pk[idx], stable=True).indices]
    assert torch.equal(got[2], idx) and torch.equal(got[0], pk[idx]) and torch.equal(got[1].view(torch.int64), ok[idx].view(torch.int64))
    sp, so = pk[idx], ok[idx]
    i = torch.arange(n, device=dev, dtype=torch.int64)
    ps = torch.ones(n, dtype=torch.bool, device=dev)
    ps[1:] = torch.diff(sp) != 0
    qs = ps.clone()
    qs[1:] |= torch.diff(so) != 0
    P = torch.cummax(torch.where(ps, i, 0), 0).values
    Q = torch.cummax(torch.where(qs, i, 0), 0).values
    D = torch.cumsum(qs.to(torch.int64), 0)
    pid = torch.cumsum(ps.to(torch.int64), 0) - 1
    s = torch.bincount(pid)[pid]
    qid = torch.cumsum(qs.to(torch.int64), 0) - 1
    qend = torch.cat([torch.nonzero(qs).flatten()[1:], torch.tensor([n], device=dev)])[qid]
    rank = Q - P + 1
    pos = i - P
    exp = {"rn": pos + 1, "rk": rank, "dr": D - D[P] + 1,
           "pr": torch.where(s == 1, 0.0, (rank - 1).to(torch.float64) / torch.clamp(s - 1, min=1).to(torch.float64)),
           "cd": (qend - P).to(torch.float64) / s.to(torch.float64)}
    for m in (3, 7):
        q, r = s // m, s % m
        big = r * (q + 1)
        exp[f"nt{m}"] = torch.where(pos < big, pos // (q + 1) + 1, r + (pos - big) // torch.clamp(q, min=1) + 1)
    for j, f in enumerate(funcs):
        gv, ev = got[3 + j], exp[f[0]]
        assert torch.equal(gv.view(torch.int64), ev.view(torch.int64)), f[0]
    assert W.get_metric(st, 9) == int(ps.sum()) == 1000
    W.delete_window_state(st)


# ---- pandas and pipelines ----
def test_cross_check_with_pandas(gpu_lib):
    from bodo_b200.physical import window

    rng = np.random.default_rng(8)
    n = 50_000
    df = pd.DataFrame({"p": rng.integers(0, 300, n), "o": rng.integers(0, 50, n).astype(np.float64), "v": rng.random(n)})
    got = window(df, "p", "o", [("rn", "row_number"), ("rk", "rank"), ("dr", "dense_rank"), ("cd", "cume_dist")], batch_size=7000)
    srt = df.sort_values(["p", "o"], kind="stable").reset_index(drop=True)
    pd.testing.assert_frame_equal(got[["p", "o", "v"]], srt)
    gb = srt.groupby("p", sort=False)
    np.testing.assert_array_equal(got["rn"].to_numpy(), gb.cumcount().to_numpy() + 1)
    np.testing.assert_array_equal(got["rk"].to_numpy(), gb["o"].rank(method="min").to_numpy().astype(np.int64))
    np.testing.assert_array_equal(got["dr"].to_numpy(), gb["o"].rank(method="dense").to_numpy().astype(np.int64))
    np.testing.assert_array_equal(got["cd"].to_numpy(), gb["o"].rank(method="max", pct=True).to_numpy())


def test_qualify_row_number_dedup(gpu_lib):
    """SELECT * FROM t QUALIFY ROW_NUMBER() OVER (PARTITION BY cust ORDER BY ts DESC) = 1."""
    from bodo_b200.expr import col, lit
    from bodo_b200.physical import PhysicalFilterProject, PhysicalReadPandas, PhysicalWindow, ResultCollector, run_pipeline

    rng = np.random.default_rng(9)
    n = 30_000
    df = pd.DataFrame({"cust": rng.integers(0, 2000, n), "ts": rng.integers(0, 100, n), "amt": rng.random(n)})
    op = PhysicalWindow("cust", "ts", [("rn", "row_number")], ascending=False)
    run_pipeline(PhysicalReadPandas(df, 4096), [], op)
    coll = ResultCollector()
    run_pipeline(op, [PhysicalFilterProject(col("rn") == lit(1), [(c, col(c)) for c in df.columns])], coll)
    op.Finalize()
    got = coll.result().sort_values("cust").reset_index(drop=True)
    exp = df.sort_values("ts", ascending=False, kind="stable").drop_duplicates("cust", keep="first").sort_values("cust").reset_index(drop=True)
    np.testing.assert_array_equal(got["cust"].to_numpy(dtype=np.int64), exp["cust"].to_numpy())
    np.testing.assert_array_equal(got["ts"].to_numpy(dtype=np.int64), exp["ts"].to_numpy())
    np.testing.assert_array_equal(got["amt"].to_numpy(dtype=np.float64), exp["amt"].to_numpy())


def test_partition_by_a_dictionary_encoded_string(gpu_lib):
    from bodo_b200.dictionary import DictionaryBuilder
    from bodo_b200.physical import PhysicalReadArrowDevice, PhysicalWindow, ResultCollector, run_pipeline

    rng = np.random.default_rng(10)
    n = 20_000
    words = np.array(["ant", "bee", "cat", "dog", "eel", "fox", None], dtype=object)
    s = words[rng.integers(0, len(words), n)]
    o = rng.integers(0, 30, n)
    at = pa.table({"s": pa.array(s, type=pa.string()), "o": pa.array(o, type=pa.int64())})
    b = DictionaryBuilder()
    op = PhysicalWindow("s", "o", [("rk", "rank"), ("rn", "row_number")])
    run_pipeline(PhysicalReadArrowDevice(at, 3000, 0, {"s": b}), [], op)
    coll = ResultCollector()
    run_pipeline(op, [], coll)
    op.Finalize()
    got = coll.result()
    big = 1 << 40  # NA ids sort last
    ids = np.array([b.index[x] if x is not None else big for x in s], dtype=np.int64)
    srt = pd.DataFrame({"id": ids, "o": o, "seq": np.arange(n)}).sort_values(["id", "o", "seq"]).reset_index(drop=True)
    gb = srt.groupby("id", sort=False)
    np.testing.assert_array_equal(got["s"].fillna(-1).to_numpy(dtype=np.int64), np.where(srt["id"] == big, -1, srt["id"]))
    np.testing.assert_array_equal(got["o"].to_numpy(dtype=np.int64), srt["o"].to_numpy())
    np.testing.assert_array_equal(got["rn"].to_numpy(), gb.cumcount().to_numpy() + 1)
    np.testing.assert_array_equal(got["rk"].to_numpy(), gb["o"].rank(method="min").to_numpy().astype(np.int64))
    assert sorted(b.values) == [w for w in words if w is not None] and got["s"].isna().sum() == (s == None).sum()  # noqa: E711


def test_device_errors(gpu_lib):
    n = 10
    good = Table([_i64(np.zeros(n)), _i64(np.arange(n))], ["k", "o"])
    other = Table([Column(np.zeros(n, np.int32), None, CTypes.INT32, ArrTypes.NUMPY, n), _i64(np.arange(n))], ["k", "o"])
    st = W.init_window_state(-1, ["k"], ["o"], True, "last", [("rn", "row_number")], ["k", "o"])
    W.window_build_consume_batch(st, good, False)
    with pytest.raises(B200Error, match="before the last batch"):
        W.window_produce_output_batch(st)
    with pytest.raises(B200Error, match="column types differ"):
        W.window_build_consume_batch(st, other, True)
    W.delete_window_state(st)
