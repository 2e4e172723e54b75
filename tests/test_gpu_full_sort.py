"""Full streaming sort (ORDER BY without LIMIT, `sort_values`) on the GPU against pandas' stable sort.

The oracle is the same as the top-k tests' (tests/test_gpu_sort.py): pandas' sort over explicit (_na_j, key_j, ..., _seq)
columns, independent of the device's radix words.  Every output column is compared bit for bit with the input rows at the
oracle's permutation: data bytes, validity and dtypes.  The pass-skipping cases also pin metrics 7 (digit passes run) and 8
(digit passes skipped); a key has one pass per byte of its width, plus one NA-class pass when it is nullable or a float."""

import datetime
import os

import numpy as np
import pandas as pd
import pyarrow.parquet as pq
import pytest
import torch

from bodo_b200 import _lib
from bodo_b200._lib import B200Error
from bodo_b200.streaming import sort as S
from bodo_b200.table import ArrTypes, Column, CTypes, Table, np_dtype_of
from tests.helpers import table_to_device
from tests.test_gpu_sort import KEY_TYPES, NP, batches_of, col_mask, make_column, oracle_perm

pytestmark = pytest.mark.gpu

TILE = 4096  # rows per fsort_pass_kernel tile
CHUNK = 1 << 24  # rows per store chunk


@pytest.fixture(autouse=True)
def _return_device_memory():
    """These tests allocate gigabytes (chunk stores, pair buffers, torch references).  After each one, the library pool's freed
    blocks and torch's cached blocks go back to the driver, so they do not take device memory from the tests that follow."""
    yield
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    _lib.lib().b200_pool_trim(torch.cuda.current_device(), 0)


def run_full(table, by, asc, nap, sizes=(1 << 30,), device=True, empty_every=0, output_batch_size=32768):
    st = S.init_stream_sort_state(-1, None, 0, by, asc, nap, table.names, output_batch_size=output_batch_size, full=True)
    bs = batches_of(table, list(sizes), empty_every)
    for i, b in enumerate(bs):
        S.sort_build_consume_batch(st, table_to_device(b) if device else b, i == len(bs) - 1)
    outs = []
    while True:
        out, last = S.produce_output_batch(st)
        outs.append(out)
        if last:
            break
    metrics = [S.get_metric(st, w) for w in range(9)]
    res = [(np.concatenate([o.columns[c].values_numpy() for o in outs]),
            np.concatenate([col_mask(o.columns[c]) for o in outs]),
            outs[0].columns[c]) for c in range(table.n_cols)]
    S.delete_stream_sort_state(st)
    return res, metrics, [o.n_rows for o in outs]


def check(table, by, asc, nap, perm=None, **kw):
    if perm is None:
        perm = oracle_perm(table, by, asc, nap)
    got, metrics, sizes = run_full(table, by, asc, nap, **kw)
    for c, (vals, mask, oc) in zip(table.columns, got):
        assert oc.c_type == c.c_type and oc.arr_type == c.arr_type
        assert (oc.validity is None) == (c.arr_type == ArrTypes.NUMPY)
        exp = c.values_numpy()[perm]
        assert vals.dtype == np_dtype_of(c.c_type) and vals.itemsize == exp.itemsize and len(vals) == len(perm)
        np.testing.assert_array_equal(vals.view(np.uint8), exp.view(np.uint8))
        np.testing.assert_array_equal(mask, col_mask(c)[perm])
    assert metrics[0] == table.n_rows and metrics[1:6] == [0] * 5
    assert metrics[6] == -(-table.n_rows // CHUNK) * CHUNK
    return metrics, sizes


def n_candidate_passes(table, by):
    n = 0
    for k in by:
        c = table.columns[table.names.index(k)]
        n += np.dtype(NP[c.c_type]).itemsize + (c.arr_type != ArrTypes.NUMPY or c.c_type in (CTypes.FLOAT32, CTypes.FLOAT64))
    return n


# ---- key matrix: every key type, numpy and nullable, both directions, both NA placements ----
@pytest.mark.parametrize("ct", KEY_TYPES)
@pytest.mark.parametrize("nullable", [False, True])
def test_key_types(gpu_lib, ct, nullable):
    rng = np.random.default_rng(ct * 2 + nullable)
    n = 5000
    t = Table([make_column(ct, n, rng, nullable), make_column(CTypes.INT64, n, rng, True, small=False)], ["k", "p"])
    for asc in (True, False):
        for nap in ("first", "last"):
            m, _ = check(t, ["k"], [asc], [nap], sizes=(1000,), empty_every=2)
            assert m[7] + m[8] == n_candidate_passes(t, ["k"]), m
    # wide values: every byte digit varies
    t = Table([make_column(ct, n, rng, nullable, small=False), make_column(CTypes.INT64, n, rng, True, small=False)], ["k", "p"])
    check(t, ["k"], [False], ["first"], sizes=(777,))


@pytest.mark.parametrize("n_keys", [1, 2, 3, 4])
def test_multi_key_mixed_directions(gpu_lib, n_keys):
    """Heavy ties on every key (small value ranges, 10 % NA): stability decides most of the order."""
    rng = np.random.default_rng(40 + n_keys)
    n = 20_000
    types = [CTypes.INT32, CTypes.FLOAT64, CTypes.DATETIME, CTypes.UINT16][:n_keys]
    cols = [make_column(ct, n, rng, True, na_frac=0.1) for ct in types] + [make_column(CTypes.FLOAT32, n, rng, True, small=False)]
    names = [f"k{j}" for j in range(n_keys)] + ["p"]
    t = Table(cols, names)
    asc = [j % 2 == 0 for j in range(n_keys)]
    nap = ["first" if j % 3 == 1 else "last" for j in range(n_keys)]
    m, _ = check(t, names[:n_keys], asc, nap, sizes=(4096, 1000))
    assert m[7] + m[8] == n_candidate_passes(t, names[:n_keys])
    # keys need not be the leading columns
    t2 = Table(cols[::-1], names[::-1])
    check(t2, names[:n_keys][::-1], asc[::-1], nap[::-1], sizes=(32768,))


# ---- pass skipping: metrics 7 (run) and 8 (skipped) ----
def _i64(v):
    return Column(np.ascontiguousarray(v, dtype=np.int64), None, CTypes.INT64, ArrTypes.NUMPY, len(v))


def test_pass_skipping(gpu_lib):
    rng = np.random.default_rng(9)
    n = 30_000
    p = _i64(np.arange(n))
    # a constant key: every pass skipped, the output is the input order
    m, _ = check(Table([_i64(np.full(n, -7)), p], ["k", "p"]), ["k"], [True], ["last"], perm=np.arange(n), sizes=(7000,))
    assert (m[7], m[8]) == (0, 8), m
    m, _ = check(Table([_i64(np.full(n, -7)), p], ["k", "p"]), ["k"], [False], ["first"], perm=np.arange(n))
    assert (m[7], m[8]) == (0, 8), m
    # an int64 key in [0, 255]: exactly one digit pass, both directions
    small = Table([_i64(rng.integers(0, 256, n)), p], ["k", "p"])
    for asc in (True, False):
        m, _ = check(small, ["k"], [asc], ["last"], sizes=(5000,))
        assert (m[7], m[8]) == (1, 7), m
    # values that differ in one middle byte only (byte 3)
    mid = Table([_i64(0x0102030400000005 + (rng.integers(0, 256, n) << 24)), p], ["k", "p"])
    m, _ = check(mid, ["k"], [False], ["last"])
    assert (m[7], m[8]) == (1, 7), m
    # an all-NA key: every pass skipped (words are 0, one NA class), input order
    all_na = Column(rng.integers(-9, 9, n).astype(np.int32), np.zeros((n + 7) // 8, np.uint8), CTypes.INT32, ArrTypes.NULLABLE_INT_BOOL, n)
    m, _ = check(Table([all_na, p], ["k", "p"]), ["k"], [True], ["first"], perm=np.arange(n))
    assert (m[7], m[8]) == (0, 5), m
    # a nullable column without NAs: its byte passes run, its class pass does not
    no_na = Column(rng.integers(-30000, 30000, n).astype(np.int16), np.full((n + 7) // 8, 0xFF, np.uint8), CTypes.INT16,
                   ArrTypes.NULLABLE_INT_BOOL, n)
    m, _ = check(Table([no_na, p], ["k", "p"]), ["k"], [True], ["last"])
    assert (m[7], m[8]) == (2, 1), m
    # doubles in [0.5, 1): the top byte is constant, and without NaN so is the class
    f = Column(0.5 + rng.random(n) / 2, None, CTypes.FLOAT64, ArrTypes.NUMPY, n)
    m, _ = check(Table([f, p], ["k", "p"]), ["k"], [True], ["last"])
    assert (m[7], m[8]) == (7, 2), m
    # two keys: a constant one (8 skipped) and a small one (1 run, 7 skipped)
    m, _ = check(Table([_i64(np.full(n, 3)), small.columns[0], p], ["a", "k", "p"]), ["a", "k"], [True, False], ["last", "last"])
    assert (m[7], m[8]) == (1, 15), m


# ---- sizes ----
def test_empty_input_keeps_the_schema(gpu_lib):
    t = Table([Column(np.empty(0, np.float32), None, CTypes.FLOAT32, ArrTypes.NUMPY, 0),
               Column(np.empty(0, np.int8), np.empty(0, np.uint8), CTypes.INT8, ArrTypes.NULLABLE_INT_BOOL, 0)], ["k", "p"])
    got, m, sizes = run_full(t, ["k"], [True], ["last"], empty_every=1)
    assert [len(v) for v, _, _ in got] == [0, 0] and [c.c_type for _, _, c in got] == [CTypes.FLOAT32, CTypes.INT8]
    assert [c.arr_type for _, _, c in got] == [ArrTypes.NUMPY, ArrTypes.NULLABLE_INT_BOOL]
    assert m[0] == 0 and m[6:9] == [0, 0, 0] and sizes == [0]


@pytest.mark.parametrize("n", [1, 2, TILE - 1, TILE, TILE + 1, 3 * TILE + 17])
def test_small_sizes_and_tile_edges(gpu_lib, n):
    rng = np.random.default_rng(n)
    t = Table([make_column(CTypes.INT32, n, rng, True, small=False), make_column(CTypes.FLOAT64, n, rng, True),
               make_column(CTypes.UINT8, n, rng, False)], ["k", "f", "p"])
    check(t, ["k"], [True], ["last"], sizes=(1000,), empty_every=3)
    check(t, ["f", "k"], [False, True], ["first", "last"])


@pytest.mark.parametrize("n", [CHUNK - 1, CHUNK + 1])
def test_chunk_boundary(gpu_lib, n):
    """2^24 +- 1 rows in 3 M-row batches, so one batch straddles the chunk boundary.  The oracle here is numpy's lexsort over
    (NA class, key, arrival index): pandas is slow at this size."""
    rng = np.random.default_rng(n % 1000)
    k = make_column(CTypes.INT32, n, rng, True, na_frac=0.05, small=False)
    k.data[:] = rng.integers(-5000, 5000, n)  # many ties
    p = make_column(CTypes.FLOAT64, n, rng, True, small=False)
    t = Table([k, p], ["k", "p"])
    na = ~col_mask(k)
    kv = np.where(na, 0, k.data.astype(np.int64))
    perm = np.lexsort((np.arange(n), -kv, ~na))  # descending, NA first
    m, _ = check(t, ["k"], [False], ["first"], perm=perm, sizes=(3_000_000,))
    assert m[6] == (2 * CHUNK if n > CHUNK else CHUNK)


@pytest.mark.parametrize("sizes", [(1,), (1000,), (32768,), (1 << 30,)])
def test_batch_sizes_and_host_batches(gpu_lib, sizes):
    rng = np.random.default_rng(sizes[0] % 1000)
    n = 3000 if sizes == (1,) else 100_000
    t = Table([make_column(CTypes.INT16, n, rng, True), make_column(CTypes.UINT64, n, rng, False, small=False)], ["k", "p"])
    check(t, ["k", "p"], [True, False], ["first", "last"], sizes=sizes, empty_every=5)
    check(t, ["k", "p"], [False, True], ["last", "first"], sizes=sizes, device=False)  # host batches are staged


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
    check(t, ["k"], [True], ["last"], sizes=(4096,))


def test_output_batch_size_not_a_multiple_of_32(gpu_lib):
    rng = np.random.default_rng(12)
    n = 10_000
    t = Table([make_column(CTypes.INT32, n, rng, True), make_column(CTypes.BOOL, n, rng, True)], ["k", "p"])
    _, sizes = check(t, ["k"], [True], ["last"], output_batch_size=1000)
    assert sizes == [1024] * 9 + [n - 9 * 1024]  # validity bitmaps are sliced at 32-row words


@pytest.mark.parametrize("descending", [False, True])
def test_large_float_key_against_torch_sort(gpu_lib, descending):
    """2^27 device rows of a float64 key with many ties and -0.0 / 0.0 mixed in (no NaN): the permutation equals
    torch.sort(stable=True)'s."""
    n = 1 << 27
    dev = torch.device("cuda", 0)
    g = torch.Generator(device=dev).manual_seed(21)
    key = torch.round(torch.randn(n, generator=g, device=dev, dtype=torch.float64) * 4096) / 8
    zeros = torch.rand(n, generator=g, device=dev) < 0.01
    key = torch.where(zeros, torch.where(torch.rand(n, generator=g, device=dev) < 0.5, -0.0, 0.0).to(torch.float64), key)
    pid = torch.arange(n, device=dev, dtype=torch.int64)
    st = S.init_stream_sort_state(-1, None, 0, ["k"], [not descending], ["last"], ["k", "p"], output_batch_size=1 << 30, full=True)
    b = 1 << 24
    for r0 in range(0, n, b):
        t = Table([Column(key[r0:r0 + b], None, CTypes.FLOAT64), Column(pid[r0:r0 + b], None, CTypes.INT64)], ["k", "p"])
        S.sort_build_consume_batch(st, t, r0 + b >= n)
    out, last = S.produce_output_batch(st)
    assert last and out.n_rows == n
    got_k = torch.as_tensor(out.columns[0].data, device=dev)
    got_p = torch.as_tensor(out.columns[1].data, device=dev)
    ref = torch.sort(key, descending=descending, stable=True)
    assert torch.equal(got_p, ref.indices)
    assert torch.equal(got_k.view(torch.int64), key[ref.indices].view(torch.int64))  # the input bits, -0.0 included
    assert S.get_metric(st, 7) >= 1
    S.delete_stream_sort_state(st)


# ---- pipelines ----
def test_sort_values_and_physical_sort(gpu_lib):
    from bodo_b200.physical import PhysicalReadPandas, PhysicalSort, ResultCollector, run_pipeline, sort_values

    rng = np.random.default_rng(3)
    n = 70_000
    df = pd.DataFrame({"a": rng.integers(0, 50, n), "b": pd.array(rng.standard_normal(n)).astype("Float64"),
                       "c": pd.array(rng.integers(-5, 5, n), dtype="Int32"), "d": rng.random(n)})
    df.loc[rng.random(n) < 0.1, "b"] = pd.NA
    df.loc[rng.random(n) < 0.1, "c"] = pd.NA
    exp = df.sort_values(["a", "b"], ascending=[False, True], na_position="first", kind="stable").reset_index(drop=True)
    got = sort_values(df, ["a", "b"], ascending=[False, True], na_position="first", batch_size=5000)
    pd.testing.assert_frame_equal(got, exp)
    pd.testing.assert_frame_equal(sort_values(df, "c"), df.sort_values("c", kind="stable").reset_index(drop=True))
    op = PhysicalSort(["c", "a"], [True, False], "last", full=True)
    run_pipeline(PhysicalReadPandas(df, 8192), [], op)
    coll = ResultCollector()
    run_pipeline(op, [], coll)
    op.Finalize()
    pd.testing.assert_frame_equal(coll.result(), df.sort_values(["c", "a"], ascending=[True, False], kind="stable").reset_index(drop=True))


def test_tpch_q1_order_by_on_the_device(gpu_lib):
    """TPC-H Q1 on the reference fixture with its final ORDER BY l_returnflag, l_linestatus done by the full sort.  The
    dictionary ids of the two string keys are assigned in order of first appearance, so the groupby output is re-encoded with
    ids in string order before it is sorted, as a planner would for an ORDER BY on dictionary-encoded strings."""
    from bodo_b200.dictionary import DictionaryBuilder
    from bodo_b200.expr import col, lit
    from bodo_b200.physical import PhysicalAggregate, PhysicalFilterProject, PhysicalReadArrowDevice, ResultCollector, run_pipeline, sort_values
    from tests.test_gpu_pipeline import GOLDEN, _tpch_q1_pandas

    at = pq.read_table(os.path.join(GOLDEN, "tpch_q1_lineitem.parquet"))
    builders = {"L_RETURNFLAG": DictionaryBuilder(), "L_LINESTATUS": DictionaryBuilder()}
    src = PhysicalReadArrowDevice(at, 4096, 0, builders)
    price, disc, tax = col("L_EXTENDEDPRICE"), col("L_DISCOUNT"), col("L_TAX")
    fp = PhysicalFilterProject(col("L_SHIPDATE") <= lit(datetime.date(1998, 9, 2)),
                               [("L_RETURNFLAG", col("L_RETURNFLAG")), ("L_LINESTATUS", col("L_LINESTATUS")), ("L_QUANTITY", col("L_QUANTITY")),
                                ("L_EXTENDEDPRICE", price), ("DISC_PRICE", price * (lit(1.0) - disc)),
                                ("CHARGE", price * (lit(1.0) - disc) * (lit(1.0) + tax)), ("L_DISCOUNT", disc), ("L_ORDERKEY", col("L_ORDERKEY"))])
    aggs = [("sum", 2), ("sum", 3), ("sum", 4), ("sum", 5), ("mean", 2), ("mean", 3), ("mean", 6), ("size", None)]
    agg = PhysicalAggregate((0, 1), aggs)
    run_pipeline(src, [fp], agg)
    coll = ResultCollector()
    run_pipeline(agg, [], coll)
    agg.Finalize()
    grouped = coll.result()
    names = ["L_RETURNFLAG", "L_LINESTATUS", "SUM_QTY", "SUM_BASE_PRICE", "SUM_DISC_PRICE", "SUM_CHARGE", "AVG_QTY", "AVG_PRICE", "AVG_DISC", "COUNT_ORDER"]
    grouped.columns = names
    dec = {nm: builders[nm].decode(grouped[nm].to_numpy(dtype="int64")) for nm in ("L_RETURNFLAG", "L_LINESTATUS")}
    for nm, s in dec.items():
        grouped[nm] = np.searchsorted(np.unique(s), s).astype(np.int64)  # ids in string order
    grouped["_row"] = np.arange(len(grouped), dtype=np.int64)
    got = sort_values(grouped, ["L_RETURNFLAG", "L_LINESTATUS"])
    rows = got.pop("_row").to_numpy()
    for nm, s in dec.items():
        got[nm] = s[rows]
    exp = _tpch_q1_pandas(at.to_pandas())
    assert len(got) == len(exp) > 1
    assert list(got["L_RETURNFLAG"]) == list(exp["L_RETURNFLAG"]) and list(got["L_LINESTATUS"]) == list(exp["L_LINESTATUS"])
    assert (got["COUNT_ORDER"].to_numpy(dtype="int64") == exp["COUNT_ORDER"].to_numpy()).all()
    for c in exp.columns[2:-1]:
        np.testing.assert_allclose(got[c].to_numpy(dtype="float64"), exp[c].to_numpy(dtype="float64"), rtol=1e-9, err_msg=c)


# ---- errors ----
def test_errors(gpu_lib):
    n = 10
    good = Table([Column(np.zeros(n, np.int64), None, CTypes.INT64, ArrTypes.NUMPY, n)], ["k"])
    other = Table([Column(np.zeros(n, np.int32), None, CTypes.INT32, ArrTypes.NUMPY, n)], ["k"])
    st = S.init_stream_sort_state(-1, None, 0, ["k"], [True], ["last"], ["k"], full=True)
    S.sort_build_consume_batch(st, good, False)
    with pytest.raises(B200Error, match="before the last batch"):
        S.produce_output_batch(st)
    with pytest.raises(B200Error, match="column types differ"):
        S.sort_build_consume_batch(st, other, True)
    S.delete_stream_sort_state(st)
    bad = Table([Column(np.zeros(n, np.int64), None, CTypes.DECIMAL, ArrTypes.NUMPY, n)], ["k"])
    st = S.init_stream_sort_state(-1, None, 0, ["k"], [True], ["last"], ["k"], full=True)
    with pytest.raises(B200Error, match="unsupported column dtype"):
        S.sort_build_consume_batch(st, bad, True)
    for kw in (dict(limit=5), dict(offset=1)):
        with pytest.raises(B200Error, match="full sort takes no limit or offset"):
            S.init_stream_sort_state(-1, kw.get("limit"), kw.get("offset", 0), ["k"], [True], ["last"], ["k"], full=True)
