"""Groupby on float64 / float32 key columns (and nunique of float value columns), compared with pandas.

Float keys are held in the int64 tables as canon_float_key (common.cuh): -0.0 and 0.0 are one group, NaN is the marker key
(one group with dropna=False, dropped with dropna=True), every other value is its own key."""

import os
import socket

import numpy as np
import pandas as pd
import pytest
import torch

from tests.helpers import assert_frames_equal, positional, stream_groupby, table_to_device

pytestmark = pytest.mark.gpu

# 0.0 / -0.0, NaN, +-inf, subnormals, the smallest normal, neighbours of 1.0 one ulp apart, huge magnitudes
SPECIAL = np.array([0.0, -0.0, np.nan, np.inf, -np.inf, 5e-324, -5e-324, 1e-310, 2.2250738585072014e-308, 1.0,
                    np.nextafter(1.0, 2.0), np.nextafter(1.0, 0.0), 1e300, -1e300, 0.5, -2.5])


def _float_keys(rng, n, n_other=200):
    pool = np.concatenate([SPECIAL, rng.standard_normal(n_other) * 10.0 ** rng.integers(-5, 5, n_other)])
    return pool[rng.integers(0, len(pool), n)]


def _aggs_spec(aggs):
    """[(func, column index or None)] -> (fnames, f_in_offsets, f_in_cols)."""
    offs, cols = [0], []
    for _, c in aggs:
        if c is not None:
            cols.append(c)
        offs.append(len(cols))
    return tuple(f for f, _ in aggs), tuple(offs), tuple(cols)


def _expect(df, keys, aggs, dropna):
    g = df.groupby(keys, as_index=False, dropna=dropna)
    out = g.size()[keys]
    for j, (f, c) in enumerate(aggs):
        out[f"o{j}"] = (g.size()["size"] if f == "size" else g.agg(x=(df.columns[c], f))["x"]).values
    return out


def _assert_keys_exact(got, exp, col):
    """Float key columns value for value (the frame comparison is within a tolerance): -0.0 and 0.0 are one key."""
    a = np.sort(got[col].to_numpy(dtype="float64", na_value=np.nan) + 0.0)
    b = np.sort(exp[col].to_numpy(dtype="float64", na_value=np.nan) + 0.0)
    assert np.array_equal(a, b, equal_nan=True), col


def _check(got, df, keys, aggs, dropna):
    exp = _expect(df, keys, aggs, dropna)
    got = got.copy()
    got.columns = list(exp.columns)
    for k in keys:
        _assert_keys_exact(got, exp, k)
    assert_frames_equal(positional(got), positional(exp))


def _run_state(df, key_inds, aggs, dropna=True, batches=1, to_device=True, metrics=(), **kw):
    """One state fed `batches` slices of df (host or device); returns (output frame, {metric: value})."""
    from bodo_b200.streaming.groupby import (delete_groupby_state, get_metric, groupby_build_consume_batch,
                                             groupby_produce_output_batch, init_groupby_state)
    from bodo_b200.table import Table
    fn, offs, cols = _aggs_spec(aggs)
    st = init_groupby_state(-1, key_inds, fn, offs, cols, dropna=dropna, output_batch_size=1 << 30, **kw)
    t = Table.from_pandas(df)
    cuts = np.linspace(0, len(df), batches + 1).astype(np.int64)
    for b in range(batches):
        part = t.slice(int(cuts[b]), int(cuts[b + 1]))
        groupby_build_consume_batch(st, table_to_device(part) if to_device else part, b == batches - 1, True)
    out, last = groupby_produce_output_batch(st, True)
    assert last
    got = out.to_pandas()
    m = {w: get_metric(st, w) for w in metrics}
    delete_groupby_state(st)
    return got, m


ALL_AGGS = [("sum", 1), ("count", 1), ("size", None), ("mean", 2), ("min", 2), ("max", 1), ("first", 1), ("last", 2),
            ("var", 2), ("nunique", 1)]


@pytest.mark.timeout(300)
@pytest.mark.parametrize("dropna", [True, False])
@pytest.mark.parametrize("to_device", [True, False])
def test_float64_keys_every_aggregate(gpu_lib, dropna, to_device):
    rng = np.random.default_rng(1)
    n = 200_003
    df = pd.DataFrame({"k": _float_keys(rng, n), "v": rng.integers(-1000, 1000, n).astype(np.int64), "w": rng.standard_normal(n)})
    fn, offs, cols = _aggs_spec(ALL_AGGS)
    from bodo_b200.table import Table
    got = stream_groupby(Table.from_pandas(df), (0,), fn, offs, cols, batch_size=60_000, to_device=to_device, dropna=dropna,
                         output_batch_size=1 << 30)
    _check(got, df, ["k"], ALL_AGGS, dropna)
    assert len(got) == len(SPECIAL) + 200 - (2 if dropna else 1)  # +-0.0 are one key


@pytest.mark.timeout(300)
@pytest.mark.parametrize("dropna", [True, False])
@pytest.mark.parametrize("to_device", [True, False])
def test_float_keys_coalesced_small_batches(gpu_lib, dropna, to_device):
    """Small batches of the SUM / COUNT signature are buffered (coalesced) as canonical keys, then take the fast kernels."""
    rng = np.random.default_rng(2)
    n = 1_500_000
    df = pd.DataFrame({"k": _float_keys(rng, n, 5000), "v": rng.integers(-(1 << 40), 1 << 40, n).astype(np.int64)})
    aggs = [("sum", 1), ("count", 1)]
    got, m = _run_state(df, (0,), aggs, dropna=dropna, batches=12, to_device=to_device, metrics=(11,))
    assert m[11] >= 1, "the small batches were expected to be coalesced"
    _check(got, df, ["k"], aggs, dropna)


@pytest.mark.timeout(300)
@pytest.mark.parametrize("dropna", [True, False])
def test_float32_keys(gpu_lib, dropna):
    rng = np.random.default_rng(3)
    n = 300_001
    df = pd.DataFrame({"k": _float_keys(rng, n).astype(np.float32), "v": rng.integers(-50, 50, n).astype(np.int64),
                       "w": rng.standard_normal(n).astype(np.float32)})
    aggs = [("sum", 1), ("count", 1), ("mean", 2), ("max", 2), ("first", 1), ("nunique", 1)]
    got, _ = _run_state(df, (0,), aggs, dropna=dropna, batches=3)
    assert got["k"].dtype == np.float32
    _check(got, df, ["k"], aggs, dropna)


@pytest.mark.timeout(300)
@pytest.mark.parametrize("dropna", [True, False])
def test_nullable_float64_keys(gpu_lib, dropna):
    rng = np.random.default_rng(4)
    n = 250_000
    k = _float_keys(rng, n)
    k[np.isnan(k)] = 3.5  # a nullable column's missing values are NA (validity bitmap), not NaN
    ks = pd.array(k, dtype="Float64")
    ks[rng.random(n) < 0.05] = pd.NA
    df = pd.DataFrame({"k": ks, "v": rng.integers(-50, 50, n).astype(np.int64)})
    aggs = [("sum", 1), ("count", 1), ("size", None), ("min", 1)]
    got, _ = _run_state(df, (0,), aggs, dropna=dropna, batches=2)
    assert str(got["k"].dtype) == "Float64"
    assert got["k"].isna().sum() == (0 if dropna else 1)
    _check(got, df, ["k"], aggs, dropna)


def _many_keys(rng, n_distinct, with_nan):
    base = (rng.permutation(n_distinct).astype(np.float64) - n_distinct / 2) * 0.375 + 0.0625
    k = np.concatenate([base, base[rng.permutation(n_distinct)]])
    if with_nan:
        k[rng.random(len(k)) < 0.001] = np.nan
        k[rng.random(len(k)) < 0.001] = -0.0
        k[rng.random(len(k)) < 0.001] = 0.0
    return k


@pytest.mark.timeout(600)
@pytest.mark.parametrize("hint", [0, 3_000_000])
def test_many_float_keys_sm_partitioned_paths(gpu_lib, hint):
    """~3 M distinct float keys in one device batch: the SM-partitioned pair for SUM / COUNT (metric 8), the generic
    SM-partitioned pair for min / max / mean (metric 12); without a hint the table grows."""
    rng = np.random.default_rng(5)
    k = _many_keys(rng, 3_000_000, with_nan=True)
    n = len(k)
    df = pd.DataFrame({"k": k, "v": rng.integers(-(1 << 40), 1 << 40, n).astype(np.int64)})
    aggs = [("sum", 1), ("count", 1)]
    got, m = _run_state(df, (0,), aggs, dropna=False, metrics=(3, 8), expected_groups=hint)
    assert m[8] >= 1, "the SM-partitioned kernels were expected to run on float keys"
    if hint == 0:
        assert m[3] >= 1, "the table was expected to grow"
    _check(got, df, ["k"], aggs, False)
    aggs_g = [("size", None), ("sum", 1), ("min", 1), ("max", 1), ("mean", 1)]
    got, m = _run_state(df, (0,), aggs_g, dropna=True, metrics=(12,), expected_groups=hint)
    assert m[12] >= 1, "the generic SM-partitioned kernels were expected to run on float keys"
    _check(got, df, ["k"], aggs_g, True)


@pytest.mark.timeout(300)
def test_few_float_keys_low_cardinality_path(gpu_lib):
    rng = np.random.default_rng(6)
    n = 1_300_003
    pool = np.concatenate([[0.0, -0.0, np.inf, -np.inf, 5e-324, 1.0, np.nextafter(1.0, 2.0)], rng.standard_normal(24)])
    df = pd.DataFrame({"k": pool[rng.integers(0, len(pool), n)], "v": rng.integers(-(2 ** 62), 2 ** 62, n).astype(np.int64)})
    aggs = [("sum", 1), ("count", 1)]
    got, m = _run_state(df, (0,), aggs, metrics=(10,), expected_groups=30)
    assert m[10] >= 1, "the low-cardinality kernel was expected to run on float keys"
    assert len(got) == 30
    _check(got, df, ["k"], aggs, True)


@pytest.mark.timeout(300)
@pytest.mark.parametrize("dropna", [True, False])
def test_two_column_key_float_and_nullable_int(gpu_lib, dropna):
    rng = np.random.default_rng(7)
    n = 120_000
    a0 = rng.choice(np.array([0.0, -0.0, np.nan, 1.5, -1.5, np.inf, 5e-324, 2.0, 7.25]), n)
    a1 = pd.array(rng.integers(0, 5, n).astype(np.int32), dtype="Int32")
    a1[rng.random(n) < 0.15] = pd.NA
    df = pd.DataFrame({"a0": a0, "a1": a1, "w": rng.integers(-50, 50, n).astype(np.int64)})
    aggs = [("sum", 2), ("count", 2), ("max", 2)]
    got, _ = _run_state(df, (0, 1), aggs, dropna=dropna, batches=2, expected_groups=8)  # (tiny hint: the table grows)
    _check(got, df, ["a0", "a1"], aggs, dropna)


@pytest.mark.timeout(300)
@pytest.mark.parametrize("key_float", [False, True])
def test_nunique_of_float_values(gpu_lib, key_float):
    rng = np.random.default_rng(8)
    n = 200_000
    k = rng.integers(0, 1000, n).astype(np.int64)
    vals = np.array([0.0, -0.0, np.nan, 1.0, np.nextafter(1.0, 2.0), -np.inf, 5e-324, 3.25])
    df = pd.DataFrame({"k": k * 0.5 if key_float else k, "u": vals[rng.integers(0, len(vals), n)]})
    aggs = [("nunique", 1), ("count", 1)]
    got, _ = _run_state(df, (0,), aggs, batches=2)
    _check(got, df, ["k"], aggs, True)
    assert got.iloc[:, 1].max() == 6  # NaN is not a value, 0.0 and -0.0 are one


@pytest.mark.timeout(300)
def test_physical_groupby_agg_float_key(gpu_lib):
    from bodo_b200 import physical
    rng = np.random.default_rng(9)
    n = 100_000
    df = pd.DataFrame({"price": _float_keys(rng, n), "qty": rng.integers(0, 100, n).astype(np.int64)})
    got = physical.groupby_agg(df, "price", [("s", "qty", "sum"), ("c", "qty", "count")], dropna=False)
    exp = df.groupby("price", as_index=False, dropna=False).agg(s=("qty", "sum"), c=("qty", "count"))
    _assert_keys_exact(got, exp, "price")
    assert_frames_equal(positional(got), positional(exp))


# ---- two GPUs: the owner of a float key is the rank shuffle_table sends its rows to ----

def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _worker(rank, world, port, q):
    import ctypes as C

    import torch.distributed as dist
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", rank))
    try:
        from bodo_b200.streaming import exchange as X
        from bodo_b200.streaming.groupby import (delete_groupby_state, groupby_build_consume_batch,
                                                 groupby_produce_output_batch, init_groupby_state)
        from bodo_b200.table import Table
        from oracle import oracle as O
        L = O.lib()

        def owner(x):  # hash_keys of a float column (NaN hashes as 0) % world
            return L.oracle_hash_inner_32_f64(float(x), 0xB0D01289) % world

        results = []
        # (name, rows, environment): fused exchange; NCCL fallback (slab too small); raw-row mode (unique keys)
        rng = np.random.default_rng(17)  # the same global rows on every rank
        few = _float_keys(rng, 240_000, 3000)
        many = np.concatenate([(np.arange(239_000) - 100_000) * 0.125 + 0.0625, SPECIAL[rng.integers(0, len(SPECIAL), 1000)]])
        rng.shuffle(many)
        for name, keys, env in (("fused", few, {}), ("nccl", few, {"B200_XCHG_SLAB_BYTES": "8192"}),
                                ("raw-rows", many, {"B200_SHUFFLE_DECISION_ROWS": "20000", "B200_COALESCE": "0"})):
            os.environ.update(env)
            X._CACHE.clear()
            n = len(keys)
            w = np.random.default_rng(23).integers(-9, 9, n).astype(np.int64)
            c = (n + world - 1) // world
            mine = pd.DataFrame({"k": keys[rank * c:(rank + 1) * c], "w": w[rank * c:(rank + 1) * c]})
            fn = ("sum", "count", "nunique")
            st = init_groupby_state(-1, (0,), fn, tuple(range(len(fn) + 1)), (1,) * len(fn), parallel=True, dropna=False,
                                    device=rank, output_batch_size=1 << 30)
            nb = 6
            for b in range(nb):
                sl = mine.iloc[b * len(mine) // nb:(b + 1) * len(mine) // nb]
                tb = Table.from_pandas(sl)
                groupby_build_consume_batch(st, tb if b % 2 else table_to_device(tb, rank), b == nb - 1, True)
            path = (st.exchange_path, st.raw_row_mode)
            out, _ = groupby_produce_output_batch(st, True)
            g = out.to_pandas()
            delete_groupby_state(st)
            for k in env:
                os.environ.pop(k, None)
            g.columns = ["k", "s", "c", "u"][:len(fn) + 1]
            ok_place = all(owner(x) == rank for x in g.k.to_numpy())
            allg = [None] * world
            dist.all_gather_object(allg, g)
            u = pd.concat(allg, ignore_index=True)
            full = pd.DataFrame({"k": keys, "w": w})
            e = full.groupby("k", as_index=False, dropna=False).agg(s=("w", "sum"), c=("w", "count"), u=("w", "nunique"))[list(g.columns)]
            canon = lambda d: d.assign(k=d.k.to_numpy() + 0.0).sort_values("k", na_position="last").reset_index(drop=True)
            cu, ce = canon(u), canon(e)
            ok = len(cu) == len(ce) and np.array_equal(cu.k.to_numpy(), ce.k.to_numpy(), equal_nan=True) and all(
                (cu[x].to_numpy() == ce[x].to_numpy()).all() for x in g.columns[1:])
            results.append((name, path, bool(ok), bool(ok_place)))
        X._CACHE.clear()
        q.put((rank, results))
    except Exception:
        import traceback
        q.put((rank, traceback.format_exc()))
    finally:
        dist.destroy_process_group()


@pytest.mark.timeout(600)
def test_sharded_float_keys_owner_placement(gpu_lib):
    world = min(torch.cuda.device_count(), 4)
    if world < 2:
        pytest.skip("needs at least 2 GPUs")
    import torch.multiprocessing as mp
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_worker, args=(r, world, port, q)) for r in range(world)]
    for p in procs:
        p.start()
    res = [q.get(timeout=500) for _ in range(world)]
    for p in procs:
        p.join(timeout=60)
    for rank, r in sorted(res, key=lambda x: x[0]):
        assert not isinstance(r, str), r
        paths = {name: path for name, path, _, _ in r}
        assert all(ok and placed for _, _, ok, placed in r), r
        assert paths["nccl"][0] == "nccl" and paths["raw-rows"][1], r
