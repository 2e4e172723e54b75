"""Streaming top-k (ORDER BY ... LIMIT ... OFFSET) on the GPU against pandas.

The oracle is pandas' sort over explicit columns, independent of the device key encoding: for every key an `_na_j` column
(isna of the key; sorted ascending for NA-last, descending for NA-first) goes right before the key (its NA entries set to one
constant), `_seq` (the arrival index) is the last key, and the result is `.iloc[offset:offset + limit]` of the sorted rows.  The
device output is compared bit for bit with the input rows at those positions: data bytes, validity and dtypes."""

import datetime
import os
import socket

import numpy as np
import pandas as pd
import pyarrow as pa
import pytest
import torch

from bodo_b200._lib import B200Error
from bodo_b200.streaming import sort as S
from bodo_b200.table import ArrTypes, Column, CTypes, Table, np_dtype_of
from tests.helpers import table_to_device

pytestmark = pytest.mark.gpu

NP = {CTypes.INT8: "int8", CTypes.INT16: "int16", CTypes.INT32: "int32", CTypes.INT64: "int64", CTypes.UINT8: "uint8",
      CTypes.UINT16: "uint16", CTypes.UINT32: "uint32", CTypes.UINT64: "uint64", CTypes.FLOAT32: "float32", CTypes.FLOAT64: "float64",
      CTypes.BOOL: "bool", CTypes.DATE: "int32", CTypes.DATETIME: "int64", CTypes.TIMEDELTA: "int64"}
KEY_TYPES = list(NP)


def gen_values(ct, n, rng, small=True):
    """n values of Bodo type ct with many ties (small=True) and the type's edge values mixed in."""
    dt = np.dtype(NP[ct])
    if ct == CTypes.BOOL:
        return rng.integers(0, 2, n).astype(bool)
    if dt.kind == "f":
        v = rng.integers(-20, 20, n).astype(dt) / 4 if small else rng.standard_normal(n).astype(dt)
        fi = np.finfo(dt)
        edge = np.array([0.0, -0.0, np.inf, -np.inf, np.nan, fi.tiny, -fi.tiny, fi.smallest_subnormal, -fi.smallest_subnormal, fi.max,
                         -fi.max, 1.0, np.nextafter(dt.type(1.0), dt.type(2.0)), np.nextafter(dt.type(1.0), dt.type(0.0))], dtype=dt)
    else:
        ii = np.iinfo(dt)
        lo, hi = (max(ii.min, -20), min(ii.max, 20)) if small else (ii.min, ii.max)
        v = rng.integers(lo, hi, n, dtype=dt, endpoint=True)
        edge = np.array([ii.min, ii.max, 0, 1, ii.max - 1, ii.min + 1 if ii.min < 0 else 2], dtype=dt)
    pos = rng.integers(0, n, min(n, 4 * len(edge))) if n else np.empty(0, np.int64)
    v[pos] = np.resize(edge, len(pos))
    return v


def make_column(ct, n, rng, nullable, na_frac=0.15, small=True):
    data = gen_values(ct, n, rng, small)
    if ct == CTypes.BOOL:
        data = data.astype(np.uint8)
    if not nullable:
        return Column(np.ascontiguousarray(data), None, ct, ArrTypes.NUMPY, n)
    valid = rng.random(n) >= na_frac
    return Column(np.ascontiguousarray(data), np.packbits(valid, bitorder="little"), ct, ArrTypes.NULLABLE_INT_BOOL, n)


def col_mask(c):
    return c.valid_mask_numpy() if c.validity is not None else np.ones(c.length, bool)


def oracle_perm(table, by, asc, nap):
    """Row positions of the stable sort, from pandas over (_na_j, key_j, ..., _seq)."""
    d, keys, ascs = {}, [], []
    for j, name in enumerate(by):
        c = table.columns[table.names.index(name)]
        v = c.values_numpy().copy()
        na = ~col_mask(c)
        if v.dtype.kind == "f":
            na |= np.isnan(v)
        v[na] = 0
        d[f"_na{j}"], d[f"_k{j}"] = na, v
        keys += [f"_na{j}", f"_k{j}"]
        ascs += [nap[j] == "last", asc[j]]
    d["_seq"] = np.arange(table.n_rows)
    df = pd.DataFrame(d)
    return df.sort_values(keys + ["_seq"], ascending=ascs + [True])["_seq"].to_numpy()


def batches_of(table, sizes, empty_every=0):
    """Host slices of `table` cycling through `sizes`, with an empty batch after every `empty_every`-th one (and first)."""
    out, pos, i = [], 0, 0
    if empty_every:
        out.append(table.slice(0, 0))
    while pos < table.n_rows:
        s = sizes[i % len(sizes)]
        out.append(table.slice(pos, pos + s))
        pos += s
        i += 1
        if empty_every and i % empty_every == 0:
            out.append(table.slice(pos, pos))
    if not out:
        out.append(table.slice(0, 0))
    return out


def run_topk(table, by, asc, nap, limit, offset, sizes=(1 << 30,), device=True, empty_every=0, output_batch_size=32768):
    st = S.init_stream_sort_state(-1, limit, offset, by, asc, nap, table.names, output_batch_size=output_batch_size)
    bs = batches_of(table, list(sizes), empty_every)
    for i, b in enumerate(bs):
        S.sort_build_consume_batch(st, table_to_device(b) if device else b, i == len(bs) - 1)
    outs = []
    while True:
        out, last = S.produce_output_batch(st)
        outs.append(out)
        if last:
            break
    metrics = [S.get_metric(st, w) for w in range(7)]
    res = [(np.concatenate([o.columns[c].values_numpy() for o in outs]),
            np.concatenate([col_mask(o.columns[c]) for o in outs]),
            outs[0].columns[c]) for c in range(table.n_cols)]
    S.delete_stream_sort_state(st)
    return res, metrics


def check(table, by, asc, nap, limit, offset, **kw):
    perm = oracle_perm(table, by, asc, nap)[offset:offset + limit]
    got, metrics = run_topk(table, by, asc, nap, limit, offset, **kw)
    for c, (vals, mask, oc) in zip(table.columns, got):
        assert oc.c_type == c.c_type and oc.arr_type == c.arr_type
        assert (oc.validity is None) == (c.arr_type == ArrTypes.NUMPY)
        exp = c.values_numpy()[perm]
        assert vals.dtype == np_dtype_of(c.c_type) and vals.itemsize == exp.itemsize and len(vals) == len(perm)
        np.testing.assert_array_equal(vals.view(np.uint8), exp.view(np.uint8))
        np.testing.assert_array_equal(mask, col_mask(c)[perm])
    return metrics


# ---- key matrix: every key type, numpy and nullable, both directions, both NA placements ----
@pytest.mark.parametrize("ct", KEY_TYPES)
@pytest.mark.parametrize("nullable", [False, True])
def test_key_types(gpu_lib, ct, nullable):
    rng = np.random.default_rng(ct * 2 + nullable)
    n = 5000
    t = Table([make_column(ct, n, rng, nullable), make_column(CTypes.INT64, n, rng, True, small=False)], ["k", "p"])
    for asc in (True, False):
        for nap in ("first", "last"):
            check(t, ["k"], [asc], [nap], 100, 7, sizes=(1000,), empty_every=2)
    check(t, ["k"], [True], ["last"], n + 5, 0, sizes=(777,))  # K > rows: the whole input, sorted


@pytest.mark.parametrize("n_keys", [1, 2, 3, 4])
def test_multi_key_mixed_directions(gpu_lib, n_keys):
    rng = np.random.default_rng(40 + n_keys)
    n = 20_000
    types = [CTypes.INT32, CTypes.FLOAT64, CTypes.DATETIME, CTypes.UINT16][:n_keys]
    cols = [make_column(ct, n, rng, True, na_frac=0.1) for ct in types] + [make_column(CTypes.FLOAT32, n, rng, True, small=False)]
    names = [f"k{j}" for j in range(n_keys)] + ["p"]
    t = Table(cols, names)
    asc = [j % 2 == 0 for j in range(n_keys)]
    nap = ["first" if j % 3 == 1 else "last" for j in range(n_keys)]
    check(t, names[:n_keys], asc, nap, 1000, 7, sizes=(4096, 1000))
    # keys need not be the leading columns: the state moves them first and restores the input order on output
    t2 = Table(cols[::-1], names[::-1])
    check(t2, names[:n_keys][::-1], asc[::-1], nap[::-1], 300, 0, sizes=(32768,))


def test_ties_are_stable(gpu_lib):
    rng = np.random.default_rng(7)
    n = 50_000
    p = Column(np.arange(n, dtype=np.int64), None, CTypes.INT64, ArrTypes.NUMPY, n)
    same = Column(np.full(n, 3, np.int64), None, CTypes.INT64, ArrTypes.NUMPY, n)
    all_na = Column(rng.integers(0, 9, n).astype(np.float64), np.zeros((n + 7) // 8, np.uint8), CTypes.FLOAT64, ArrTypes.NULLABLE_INT_BOOL, n)
    nans = Column(np.full(n, np.nan), None, CTypes.FLOAT64, ArrTypes.NUMPY, n)
    zeros = Column(np.where(rng.random(n) < 0.5, 0.0, -0.0), None, CTypes.FLOAT64, ArrTypes.NUMPY, n)
    for key in (same, all_na, nans, zeros):
        t = Table([key, p], ["k", "p"])
        for asc, nap in ((True, "last"), (False, "first")):
            check(t, ["k"], [asc], [nap], 1000, 0, sizes=(1000,))
            check(t, ["k"], [asc], [nap], 10, 7, sizes=(32768,))


@pytest.mark.parametrize("limit", [0, 1, 10, 1000, 100_000, 300_000])
@pytest.mark.parametrize("offset", [0, 7, 250_000])
def test_limit_offset_sizes(gpu_lib, limit, offset):
    rng = np.random.default_rng(limit + offset)
    n = 250_000
    t = Table([make_column(CTypes.FLOAT64, n, rng, True, small=False), make_column(CTypes.INT32, n, rng, True)], ["k", "p"])
    check(t, ["k"], [False], ["last"], limit, offset, sizes=(32768, 1000), empty_every=3)


@pytest.mark.parametrize("sizes", [(1,), (1000,), (32768,), (1 << 30,)])
def test_batch_sizes_and_host_batches(gpu_lib, sizes):
    rng = np.random.default_rng(sizes[0] % 1000)
    n = 3000 if sizes == (1,) else 100_000
    t = Table([make_column(CTypes.INT16, n, rng, True), make_column(CTypes.UINT64, n, rng, False, small=False)], ["k", "p"])
    check(t, ["k", "p"], [True, False], ["first", "last"], 500, 7, sizes=sizes, empty_every=5)
    check(t, ["k", "p"], [False, True], ["last", "first"], 500, 0, sizes=sizes, device=False)  # host batches are staged


def test_empty_input_keeps_the_schema(gpu_lib):
    t = Table([Column(np.empty(0, np.float32), None, CTypes.FLOAT32, ArrTypes.NUMPY, 0),
               Column(np.empty(0, np.int8), np.empty(0, np.uint8), CTypes.INT8, ArrTypes.NULLABLE_INT_BOOL, 0)], ["k", "p"])
    got, m = run_topk(t, ["k"], [True], ["last"], 10, 0, empty_every=1)
    assert [len(v) for v, _, _ in got] == [0, 0] and [c.c_type for _, _, c in got] == [CTypes.FLOAT32, CTypes.INT8]
    assert m[0] == 0


def test_payload_fidelity(gpu_lib):
    """Every payload type, numpy and nullable, with -0.0 and NaN payload bits (a signalling-style NaN pattern included)."""
    rng = np.random.default_rng(11)
    n = 40_000
    cols, names = [make_column(CTypes.INT64, n, rng, False)], ["k"]
    for ct in KEY_TYPES:
        for nullable in (False, True):
            cols.append(make_column(ct, n, rng, nullable, small=False))
            names.append(f"p{ct}_{int(nullable)}")
    f = cols[names.index(f"p{CTypes.FLOAT64}_0")].data
    f[::5] = -0.0
    f[1::7] = np.array([0x7FF4000000000001], dtype=np.int64).view(np.float64)[0]
    f32 = cols[names.index(f"p{CTypes.FLOAT32}_1")].data
    f32[::3] = -0.0
    f32[1::11] = np.array([0x7FC12345], dtype=np.int32).view(np.float32)[0]
    t = Table(cols, names)
    check(t, ["k"], [True], ["last"], 5000, 3, sizes=(4096,))


def test_adversarial_order_fills_the_store(gpu_lib):
    """Rising keys sorted descending: every batch beats the cutoff, so the store overflows (reduce on overflow) and batches
    larger than its free room are consumed in slices."""
    n = 13 << 20
    key = np.arange(n, dtype=np.int64) // 3  # ties too
    t = Table([Column(key, None, CTypes.INT64, ArrTypes.NUMPY, n), Column(np.arange(n, dtype=np.int32), None, CTypes.INT32, ArrTypes.NUMPY, n)], ["k", "p"])
    m = check(t, ["k"], [False], ["last"], 100_000, 5, sizes=(6 << 20, 1 << 20))
    cap = m[6]
    assert cap == 4 << 20
    assert m[2] >= 3, m  # overflow reduces
    assert m[4] > 4, m   # 3 batches, some of them sliced


def test_the_filter_filters(gpu_lib):
    """Random-order float keys, 2^24 rows in 64 batches, K = 10: after the first cutoff almost every row is dropped on the
    device, and the host reads the candidate count far less often than once per batch."""
    n, nb, K = 1 << 24, 64, 10
    dev = torch.device("cuda", 0)
    g = torch.Generator(device=dev).manual_seed(5)
    key = torch.rand(n, generator=g, device=dev, dtype=torch.float64)
    pid = torch.arange(n, device=dev, dtype=torch.int64)
    st = S.init_stream_sort_state(-1, K, 0, ["k"], [False], ["last"], ["k", "p"])
    b = n // nb
    for i in range(nb):
        t = Table([Column(key[i * b:(i + 1) * b], None, CTypes.FLOAT64), Column(pid[i * b:(i + 1) * b], None, CTypes.INT64)], ["k", "p"])
        S.sort_build_consume_batch(st, t, i == nb - 1)
    out, last = S.produce_output_batch(st)
    assert last
    after_cutoff, reads = S.get_metric(st, 5), S.get_metric(st, 3)
    assert after_cutoff <= 4 * K * nb, after_cutoff
    assert reads <= nb // 8, reads
    ref = torch.topk(key, K)
    got_k = torch.as_tensor(out.columns[0].data, device=dev)
    got_p = torch.as_tensor(out.columns[1].data, device=dev)
    assert torch.equal(got_k, ref.values)
    assert torch.equal(key[got_p], got_k)
    S.delete_stream_sort_state(st)


def test_pipeline_and_helper(gpu_lib):
    from bodo_b200.physical import PhysicalReadPandas, PhysicalSort, ResultCollector, run_pipeline, sort_values_head

    rng = np.random.default_rng(3)
    n = 70_000
    df = pd.DataFrame({"a": rng.integers(0, 50, n), "b": pd.array(rng.standard_normal(n)).astype("Float64"),
                       "c": pd.array(rng.integers(-5, 5, n), dtype="Int32")})
    df.loc[rng.random(n) < 0.1, "b"] = pd.NA
    df.loc[rng.random(n) < 0.1, "c"] = pd.NA
    exp = df.sort_values(["a", "b"], ascending=[False, True], na_position="first", kind="stable").iloc[11:11 + 40].reset_index(drop=True)
    got = sort_values_head(df, ["a", "b"], ascending=[False, True], na_position="first", n=40, offset=11, batch_size=5000)
    pd.testing.assert_frame_equal(got, exp)
    op = PhysicalSort(["c"], True, "last", limit=25)
    run_pipeline(PhysicalReadPandas(df, 8192), [], op)
    coll = ResultCollector()
    run_pipeline(op, [], coll)
    op.Finalize()
    pd.testing.assert_frame_equal(coll.result(), df.sort_values("c", kind="stable").head(25).reset_index(drop=True))


def test_errors(gpu_lib):
    n = 10
    bad = Table([Column(np.zeros(n, np.int64), None, CTypes.DECIMAL, ArrTypes.NUMPY, n)], ["k"])
    st = S.init_stream_sort_state(-1, 5, 0, ["k"], [True], ["last"], ["k"])
    with pytest.raises(B200Error, match="unsupported column dtype"):
        S.sort_build_consume_batch(st, bad, True)
    good = Table([Column(np.zeros(n, np.int64), None, CTypes.INT64, ArrTypes.NUMPY, n)], ["k"])
    other = Table([Column(np.zeros(n, np.int32), None, CTypes.INT32, ArrTypes.NUMPY, n)], ["k"])
    st = S.init_stream_sort_state(-1, 5, 0, ["k"], [True], ["last"], ["k"])
    S.sort_build_consume_batch(st, good, False)
    with pytest.raises(B200Error, match="column types differ"):
        S.sort_build_consume_batch(st, other, True)
    S.delete_stream_sort_state(st)


# ---- TPC-H Q3 shape: filters -> two joins -> REVENUE projection -> 3-key groupby -> top 10 ----
def _q3_tables(rng):
    n_c, n_o, n_l = 3000, 30_000, 120_000
    segs = np.array(["AUTOMOBILE", "BUILDING", "FURNITURE", "HOUSEHOLD", "MACHINERY"])
    d0 = (datetime.date(1992, 1, 1) - datetime.date(1970, 1, 1)).days
    customer = pd.DataFrame({"C_CUSTKEY": np.arange(1, n_c + 1, dtype=np.int64), "C_MKTSEGMENT": segs[rng.integers(0, 5, n_c)]})
    orders = pd.DataFrame({"O_ORDERKEY": rng.permutation(n_o).astype(np.int64) * 4 + 1, "O_CUSTKEY": rng.integers(1, n_c + 1, n_o),
                           "O_ORDERDATE": (d0 + rng.integers(0, 2400, n_o)).astype(np.int32), "O_SHIPPRIORITY": rng.integers(0, 2, n_o).astype(np.int32)})
    lineitem = pd.DataFrame({"L_ORDERKEY": orders["O_ORDERKEY"].to_numpy()[rng.integers(0, n_o, n_l)],
                             "L_EXTENDEDPRICE": rng.integers(900, 105_000, n_l).astype(np.float64),
                             "L_DISCOUNT": rng.integers(0, 2, n_l) / 16.0,  # multiples of 1/16: every product and sum is exact
                             "L_SHIPDATE": (d0 + rng.integers(0, 2500, n_l)).astype(np.int32)})
    return customer, orders, lineitem


def _arrow(df, dates=()):
    return pa.table({c: pa.array(df[c].to_numpy(), type=pa.date32()) if c in dates else pa.array(df[c].to_numpy()) for c in df.columns})


def test_tpch_q3_shape(gpu_lib):
    from bodo_b200.dictionary import DictionaryBuilder
    from bodo_b200.expr import col, lit
    from bodo_b200.physical import (PhysicalAggregate, PhysicalFilterProject, PhysicalJoin, PhysicalReadArrowDevice, PhysicalSort,
                                    ResultCollector, run_pipeline)

    rng = np.random.default_rng(2024)
    customer, orders, lineitem = _q3_tables(rng)
    cut = datetime.date(1995, 3, 15)
    cut_days = (cut - datetime.date(1970, 1, 1)).days
    seg = DictionaryBuilder()
    building = int(seg.unify(pa.array(["BUILDING"]), 0).values_numpy()[0])
    bs = 8192
    src_c = PhysicalReadArrowDevice(_arrow(customer), bs, 0, {"C_MKTSEGMENT": seg})
    fp_c = PhysicalFilterProject(col("C_MKTSEGMENT") == lit(building), [("C_CUSTKEY", col("C_CUSTKEY"))])
    j1 = PhysicalJoin(0, 1, ["C_CUSTKEY"], list(orders.columns))
    run_pipeline(src_c, [fp_c], j1)
    src_o = PhysicalReadArrowDevice(_arrow(orders, ("O_ORDERDATE",)), bs, 0)
    fp_o = PhysicalFilterProject(col("O_ORDERDATE") < lit(cut), [(c, col(c)) for c in orders.columns])
    j1_names = ["C_CUSTKEY"] + list(orders.columns)
    j2 = PhysicalJoin(1, 0, j1_names, ["L_ORDERKEY", "L_EXTENDEDPRICE", "L_DISCOUNT"])
    run_pipeline(src_o, [fp_o, j1], j2)
    src_l = PhysicalReadArrowDevice(_arrow(lineitem, ("L_SHIPDATE",)), bs, 0)
    fp_l = PhysicalFilterProject(col("L_SHIPDATE") > lit(cut), [(c, col(c)) for c in ("L_ORDERKEY", "L_EXTENDEDPRICE", "L_DISCOUNT")])
    rev = PhysicalFilterProject(None, [("L_ORDERKEY", col("L_ORDERKEY")), ("O_ORDERDATE", col("O_ORDERDATE")), ("O_SHIPPRIORITY", col("O_SHIPPRIORITY")),
                                       ("REVENUE", col("L_EXTENDEDPRICE") * (lit(1.0) - col("L_DISCOUNT")))])
    agg = PhysicalAggregate((0, 1, 2), [("sum", 3)])
    run_pipeline(src_l, [fp_l, j2, rev], agg)
    top = PhysicalSort(["REVENUE", "O_ORDERDATE"], [False, True], limit=10)
    run_pipeline(agg, [], top)
    coll = ResultCollector()
    run_pipeline(top, [], coll)
    top.Finalize(); agg.Finalize(); j2.Finalize(); j1.Finalize()
    got = coll.result()
    got.columns = ["L_ORDERKEY", "O_ORDERDATE", "O_SHIPPRIORITY", "REVENUE"]

    # pandas Q3 (benchmarks/tpch dataframe_queries.py tpch_q3), dates as days since the epoch
    c = customer[customer["C_MKTSEGMENT"] == "BUILDING"]
    o = orders[orders["O_ORDERDATE"] < cut_days]
    li = lineitem[lineitem["L_SHIPDATE"] > cut_days]
    jn = c.merge(o, left_on="C_CUSTKEY", right_on="O_CUSTKEY").merge(li, left_on="O_ORDERKEY", right_on="L_ORDERKEY")
    jn["REVENUE"] = jn["L_EXTENDEDPRICE"] * (1.0 - jn["L_DISCOUNT"])
    gb = jn.groupby(["L_ORDERKEY", "O_ORDERDATE", "O_SHIPPRIORITY"], as_index=False)["REVENUE"].sum()
    exp = gb.sort_values(["REVENUE", "O_ORDERDATE"], ascending=[False, True]).head(10).reset_index(drop=True)
    assert len(got) == 10
    got_dates = got["O_ORDERDATE"].to_numpy().astype("datetime64[D]").astype(np.int64)
    np.testing.assert_array_equal(got["REVENUE"].to_numpy(), exp["REVENUE"].to_numpy())
    np.testing.assert_array_equal(got_dates, exp["O_ORDERDATE"].to_numpy())
    pairs = list(zip(exp["REVENUE"], exp["O_ORDERDATE"]))
    for i in range(10):
        if pairs.count(pairs[i]) == 1:
            assert got["L_ORDERKEY"][i] == exp["L_ORDERKEY"][i] and got["O_SHIPPRIORITY"][i] == exp["O_SHIPPRIORITY"][i]


# ---- sharded: 2 GPUs, one process each ----
def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _sharded_data(rank):
    rng = np.random.default_rng(100 + rank)
    n = 200_000 + 1000 * rank
    return Table([make_column(CTypes.INT32, n, rng, True), make_column(CTypes.FLOAT64, n, rng, True, small=False),
                  make_column(CTypes.INT64, n, rng, False, small=False)], ["k", "f", "p"])


def _sharded_worker(rank, world, port, q):
    import torch.distributed as dist

    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", rank))
    try:
        t = _sharded_data(rank)
        st = S.init_stream_sort_state(-1, 500, 9, ["k", "f"], [False, True], ["first", "last"], t.names, parallel=True, device=rank)
        bs = batches_of(t, [30_000], 2)
        for i, b in enumerate(bs):
            S.sort_build_consume_batch(st, table_to_device(b, rank), i == len(bs) - 1)
        rows = []
        while True:
            out, last = S.produce_output_batch(st)
            rows.append([(c.values_numpy(), col_mask(c)) for c in out.columns])
            if last:
                break
        S.delete_stream_sort_state(st)
        q.put((rank, [(np.concatenate([r[c][0] for r in rows]), np.concatenate([r[c][1] for r in rows])) for c in range(3)]))
    except Exception:
        import traceback
        q.put((rank, traceback.format_exc()))
    finally:
        dist.destroy_process_group()


@pytest.mark.timeout(600)
def test_sharded_topk(gpu_lib):
    import torch.multiprocessing as mp

    world = min(torch.cuda.device_count(), 4)
    if world < 2:
        pytest.skip("needs at least 2 GPUs")
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_sharded_worker, args=(r, world, port, q)) for r in range(world)]
    for p in procs:
        p.start()
    res = dict(q.get(timeout=500) for _ in range(world))
    for p in procs:
        p.join(timeout=60)
    for r in range(world):
        assert not isinstance(res[r], str), res[r]
    parts = [_sharded_data(r) for r in range(world)]
    cols = []
    for c in range(3):
        cs = [p.columns[c] for p in parts]
        n = sum(x.length for x in cs)
        v = np.concatenate([x.values_numpy() for x in cs])
        m = np.concatenate([col_mask(x) for x in cs])
        cols.append(Column(v, np.packbits(m, bitorder="little") if cs[0].validity is not None else None, cs[0].c_type, cs[0].arr_type, n))
    full = Table(cols, ["k", "f", "p"])
    perm = oracle_perm(full, ["k", "f"], [False, True], ["first", "last"])[9:509]
    for c in range(3):
        vals, mask = res[0][c]
        np.testing.assert_array_equal(vals.view(np.uint8), full.columns[c].values_numpy()[perm].view(np.uint8))
        np.testing.assert_array_equal(mask, col_mask(full.columns[c])[perm])
    for r in range(1, world):
        assert all(len(v) == 0 for v, _ in res[r])
