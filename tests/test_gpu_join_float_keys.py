"""Float64 and float32 join keys.  -0.0 and 0.0 are one key; a NaN key is an NA key (it joins NaN and NA keys under
is_na_equal=True, and nothing under False); ±inf and subnormals are ordinary keys; one-ulp neighbours are different keys.  Outputs
carry the input bits.

Expected rows come from the CPU oracle's hash join over canonical int64 keys computed here (the float's bits, -0.0 as 0.0, NaN
as invalid), and from pandas where pandas defines the result (is_na_equal=True)."""

import numpy as np
import pandas as pd
import pytest

from bodo_b200 import _lib
from bodo_b200.streaming.join import (build_runtime_filter, delete_join_state, get_metric, init_join_state, join_build_consume_batch,
                                      join_probe_consume_batch, runtime_join_filter)
from bodo_b200.table import Table
from tests.helpers import table_to_device
from tests.test_gpu_join import assert_rowset_equal

pytestmark = pytest.mark.gpu

NAN, INF = np.nan, np.inf
NA_BITS = -1  # NaN and NA in bits_sorted: not the pattern of any float64 a test writes


def canon_keys(s):
    """(canonical int64 keys, validity): the float's bits (float32 widened), -0.0 as 0.0, NaN and NA invalid."""
    if hasattr(s.array, "_mask"):
        v = np.asarray(s.array._data, dtype=np.float64)
        valid = ~np.asarray(s.array._mask)
    else:
        v = s.to_numpy().astype(np.float64)
        valid = np.ones(len(v), dtype=bool)
    valid &= ~np.isnan(v)
    k = np.where(v == 0, 0.0, v).view(np.int64).copy()
    k[~valid] = 0
    return k, valid


def oracle_frame(oracle, build, probe, bo=False, po=False, is_na_equal=True, build_key_from_probe=False):
    """The oracle's join rows: build columns then probe columns, NULL where a side is absent.  build_key_from_probe: the build key
    column holds the probe key's value (the unique-key paths write the probe row's key)."""
    bk, bv = canon_keys(build.iloc[:, 0])
    pk, pv = canon_keys(probe.iloc[:, 0])
    bi, pi = oracle.hash_join(bk, bv, pk, pv, bo, po, is_na_equal)
    out = {}
    for pre, df, idx in (("b", build, bi), ("p", probe, pi)):
        for c in df.columns:  # as float64 values (exact for the test data), NULL as NaN: what bits_sorted compares
            v = df[c].to_numpy(dtype="float64", na_value=np.nan)[np.where(idx >= 0, idx, 0)]
            v[idx < 0] = np.nan
            out[f"{pre}_{c}"] = v
    e = pd.DataFrame(out)
    if build_key_from_probe:
        e.iloc[:, 0] = e.iloc[:, build.shape[1]].to_numpy()
    return e


def bits_sorted(df):
    """Every column as float64 bits (NaN and NA: NA_BITS), rows sorted: equality here is equality of the output bits."""
    cols = {}
    for i, c in enumerate(df.columns):
        v = df[c].to_numpy(dtype="float64", na_value=np.nan)
        b = v.view(np.int64).copy()
        b[np.isnan(v)] = NA_BITS
        cols[f"c{i}"] = b
    out = pd.DataFrame(cols)
    return out.sort_values(list(out.columns)).reset_index(drop=True)


def assert_bits_equal(got, exp):
    g, e = bits_sorted(got), bits_sorted(exp)
    assert g.shape == e.shape, (g.shape, e.shape)
    np.testing.assert_array_equal(g.to_numpy(), e.to_numpy())


def run(build, probe, bo=False, po=False, is_na_equal=True, to_device=True, batch=None, used_cols=None, **kind):
    """One join state fed `batch`-row build then probe batches: (output frame, metrics 5..7)."""
    bt, pt = Table.from_pandas(build), Table.from_pandas(probe)
    st = init_join_state(-1, (0,), (0,), tuple(build.columns), tuple(probe.columns), bo, po, is_na_equal=is_na_equal, **kind)
    bs = batch or max(bt.n_rows, pt.n_rows, 1)
    for i0 in range(0, max(bt.n_rows, 1), bs):
        b = bt.slice(i0, i0 + bs)
        join_build_consume_batch(st, table_to_device(b) if to_device else b, i0 + bs >= bt.n_rows)
    outs = []
    for i0 in range(0, max(pt.n_rows, 1), bs):
        p = pt.slice(i0, i0 + bs)
        out, _, _ = join_probe_consume_batch(st, table_to_device(p) if to_device else p, i0 + bs >= pt.n_rows, True, used_cols)
        outs.append(out.to_pandas())
    m = [get_metric(st, j) for j in (5, 6, 7)]
    delete_join_state(st)
    return pd.concat(outs, ignore_index=True), m


def special_pool(dtype, side):
    """Keys for both sides: -0.0 on the build side and 0.0 on the probe side; NaN, ±inf, subnormals, normal values and, on the
    probe side, the one-ulp neighbours of 1.0 (which must not match the build side's 1.0)."""
    f = np.dtype(dtype).type
    tiny = np.finfo(dtype).smallest_subnormal
    common = [NAN, INF, -INF, tiny, -tiny, 3 * tiny, np.finfo(dtype).tiny, 1.0, -2.5, 1e30, 7.75]
    if side == "build":
        extra = [-0.0]
    else:
        extra = [0.0, np.nextafter(f(1.0), f(2.0)), np.nextafter(f(1.0), f(0.0)), np.nextafter(f(7.75), f(0.0)), 123.0]
    return np.array(common + extra + [x * 0.5 for x in range(-20, 20) if x], dtype=dtype)


def float_frames(rng, dtype, nb, npr):
    bk = rng.choice(special_pool(dtype, "build"), nb)
    pk = rng.choice(special_pool(dtype, "probe"), npr)
    build = pd.DataFrame({"k": bk, "b1": rng.integers(-1000, 1000, nb), "b2": rng.random(nb).astype(dtype)})
    probe = pd.DataFrame({"k": pk, "p1": rng.integers(-1000, 1000, npr)})
    return build, probe


HOW = {"inner": (False, False), "left": (False, True), "right": (True, False), "outer": (True, True)}  # probe = left table


@pytest.mark.parametrize("how", list(HOW))
@pytest.mark.parametrize("is_na_equal", [True, False])
@pytest.mark.parametrize("to_device", [False, True])
def test_every_join_kind(gpu_lib, oracle, how, is_na_equal, to_device):
    rng = np.random.default_rng(61)
    build, probe = float_frames(rng, np.float64, 3_000, 5_000)
    bo, po = HOW[how]
    got, m = run(build, probe, bo, po, is_na_equal, to_device, batch=1_700)
    assert m == [0, 0, 0]  # duplicated build keys: the general (CSR) path
    assert_bits_equal(got, oracle_frame(oracle, build, probe, bo, po, is_na_equal))
    if is_na_equal:  # pandas: probe = left table, build = right table
        exp = probe.merge(build.rename(columns={"k": "kb"}), left_on="k", right_on="kb", how=how)
        assert_rowset_equal(got, exp[["kb", "b1", "b2", "k", "p1"]])


@pytest.mark.parametrize("is_na_equal", [True, False])
def test_float32_keys(gpu_lib, oracle, is_na_equal):
    rng = np.random.default_rng(62)
    build, probe = float_frames(rng, np.float32, 2_000, 4_000)
    for bo, po in ((False, False), (True, True)):
        got, _ = run(build, probe, bo, po, is_na_equal, batch=1_500)
        assert_bits_equal(got, oracle_frame(oracle, build, probe, bo, po, is_na_equal))
    # unique float32 build keys: 4-byte keys take the Slot16 table, never the inline one
    ub = pd.DataFrame({"k": np.array([-0.0, NAN, INF, 1e-45, 1.5, -3.0], dtype=np.float32), "b1": np.arange(6, dtype=np.int64)})
    up = pd.DataFrame({"k": np.array([0.0, NAN, INF, 1e-45, 1.5000001, -3.0, 2.0], dtype=np.float32), "p1": np.arange(7, dtype=np.int64)})
    got, m = run(ub, up, is_na_equal=is_na_equal)
    assert m == [1, 0, 0]
    assert_bits_equal(got, oracle_frame(oracle, ub, up, is_na_equal=is_na_equal, build_key_from_probe=True))
    assert len(got) == (5 if is_na_equal else 4)


def unique_build(rng, nb, nan_row=True):
    k = rng.permutation(nb).astype(np.float64) * 0.5 + 0.25
    k[:5] = [-0.0, INF, -INF, 5e-324, 1.0]
    if nan_row:
        k[5] = NAN
    return pd.DataFrame({"k": k, "b1": rng.integers(-(1 << 40), 1 << 40, nb), "b2": rng.random(nb)})


def unique_probe(rng, nb, npr):
    pk = rng.integers(0, 2 * nb, npr).astype(np.float64) * 0.5 + 0.25
    pk[:8] = [0.0, INF, -INF, 5e-324, NAN, np.nextafter(1.0, 2.0), np.nextafter(1.0, 0.0), 1.0]
    pk[8::997] = NAN
    return pd.DataFrame({"k": pk, "p1": rng.integers(0, 1 << 40, npr)})


@pytest.mark.parametrize("schema", ["inline", "slot16_int32", "slot16_nullable"])
@pytest.mark.parametrize("is_na_equal", [True, False])
@pytest.mark.parametrize("inline_env", ["1", "0"])
def test_unique_build_keys(gpu_lib, oracle, monkeypatch, schema, is_na_equal, inline_env):
    """Float64 key with <= 2 eight-byte payloads: the Slot32 (inline) table and probe kernel; a 4-byte or nullable payload: the
    Slot16 table.  One NaN build row; B200_JOIN_INLINE=0 turns the inline build off.  On these paths the build key column holds the
    probe key's bits."""
    monkeypatch.setenv("B200_JOIN_INLINE", inline_env)
    rng = np.random.default_rng(63)
    nb, npr = 30_000, 80_000
    build, probe = unique_build(rng, nb), unique_probe(rng, nb, npr)
    if schema == "slot16_int32":
        build["b2"] = rng.integers(-1000, 1000, nb).astype(np.int32)
    elif schema == "slot16_nullable":
        build["b1"] = build["b1"].astype("Int64").mask(rng.random(nb) < 0.1)
    got, m = run(build, probe, is_na_equal=is_na_equal, batch=50_000)
    inline = schema == "inline" and inline_env == "1"
    assert m == ([2, 2, 1] if inline else [2, 0, 0]), m  # metric 5 counts every unique-key probe batch, inline ones included
    assert_bits_equal(got, oracle_frame(oracle, build, probe, is_na_equal=is_na_equal, build_key_from_probe=True))
    np.testing.assert_array_equal(got.iloc[:, 0].to_numpy().view(np.int64), got.iloc[:, 3].to_numpy().view(np.int64))
    n_nan = int(np.isnan(probe.k).sum())
    assert int(np.isnan(got.iloc[:, 3]).sum()) == (n_nan if is_na_equal else 0)
    assert (np.signbit(got.iloc[:, 0]) & (got.iloc[:, 0] == 0)).sum() == 0  # the probe's 0.0 matched the build's -0.0


@pytest.mark.parametrize("unique", [True, False])
def test_path_parity_with_int64_keys(gpu_lib, unique):
    """A float64-key join takes the table form and per-batch kernels of the int64-key join its keys were made from."""
    rng = np.random.default_rng(64)
    nb, npr = 20_000, 60_000
    ki = rng.permutation(nb).astype(np.int64) if unique else rng.integers(0, nb // 4, nb).astype(np.int64)
    pki = rng.integers(0, 2 * nb, npr).astype(np.int64)
    b1, p1 = rng.integers(0, 1 << 40, nb), rng.integers(0, 1 << 40, npr)
    res = {}
    for kind, f in (("int64", lambda k: k), ("float64", lambda k: k * 0.5 + 0.25)):
        build = pd.DataFrame({"k": f(ki), "b1": b1})
        probe = pd.DataFrame({"k": f(pki), "p1": p1})
        res[kind] = run(build, probe, batch=25_000)
    assert res["int64"][1] == res["float64"][1]
    assert res["int64"][1] == ([3, 3, 1] if unique else [0, 0, 0])
    gi, gf = res["int64"][0], res["float64"][0]
    k_int = lambda s: ((s.to_numpy() - 0.25) * 2).astype(np.int64)
    gf = pd.DataFrame({"bk": k_int(gf.iloc[:, 0]), "b1": gf.iloc[:, 1].to_numpy(), "pk": k_int(gf.iloc[:, 2]), "p1": gf.iloc[:, 3].to_numpy()})
    assert_rowset_equal(gf, gi)


@pytest.mark.parametrize("is_na_equal", [True, False])
def test_nullable_float64_na_against_numpy_nan(gpu_lib, oracle, is_na_equal):
    build = pd.DataFrame({"k": pd.array([1.5, None, -0.0, 2.0, None], dtype="Float64"), "b1": [1, 2, 3, 4, 5]})
    probe = pd.DataFrame({"k": np.array([NAN, 0.0, 1.5, 7.0, NAN]), "p1": [10, 20, 30, 40, 50]})
    got, m = run(build, probe, is_na_equal=is_na_equal, batch=2)
    # is_na_equal=False: the NA build rows join nothing, the other keys are unique, and the Slot16 path writes the probe's key
    # (0.0, not the build's -0.0) into the build key column; is_na_equal=True: two NA rows form one key, the general path
    assert m == ([0, 0, 0] if is_na_equal else [3, 0, 0])
    assert_bits_equal(got, oracle_frame(oracle, build, probe, is_na_equal=is_na_equal, build_key_from_probe=not is_na_equal))
    assert len(got) == (2 + 4 if is_na_equal else 2)  # 1.5, ±0.0, and under is_na_equal 2 NaN probe rows x 2 NA build rows
    if is_na_equal:
        exp = probe.merge(build, on="k", how="inner", suffixes=("_p", "_b"))
        assert len(exp) == len(got)


@pytest.mark.parametrize("is_na_equal", [False, True])
@pytest.mark.parametrize("to_device", [False, True])
def test_anti_and_mark_joins(gpu_lib, is_na_equal, to_device):
    rng = np.random.default_rng(65)
    nb, npr = 4_000, 30_000
    build = pd.DataFrame({"k": rng.choice(special_pool(np.float64, "build"), nb), "b1": rng.integers(0, 100, nb)})
    probe = pd.DataFrame({"k": rng.choice(special_pool(np.float64, "probe"), npr), "p1": rng.random(npr), "p2": rng.integers(0, 1 << 40, npr)})
    bk, bv = canon_keys(build.k)
    pk, pv = canon_keys(probe.k)
    has = np.where(~pv, is_na_equal and bool((~bv).any()), np.isin(pk, bk[bv]))
    anti, _ = run(build, probe, is_na_equal=is_na_equal, to_device=to_device, batch=12_000, used_cols=([], [0, 1, 2]), is_anti_join=True)
    assert_bits_equal(anti, probe[~has].reset_index(drop=True))
    mark, _ = run(build, probe, is_na_equal=is_na_equal, to_device=to_device, batch=12_000, used_cols=([], [0, 1, 2]), is_mark_join=True)
    assert mark.shape == (npr, 4)
    np.testing.assert_array_equal(mark.iloc[:, 3].to_numpy(dtype=bool), has)
    np.testing.assert_array_equal(mark.iloc[:, 0].to_numpy().view(np.int64), probe.k.to_numpy().view(np.int64))


def decode_bound(e):
    """The runtime filter's order-preserving int64 bound -> float64 (bits 0..62 flipped when the sign bit is set)."""
    e = int(e)
    k = e ^ 0x7FFFFFFFFFFFFFFF if e < 0 else e
    return float(np.array([k], dtype=np.int64).view(np.float64)[0])


def test_runtime_filter(gpu_lib):
    rng = np.random.default_rng(66)
    nb, npr = 50_000, 400_000
    bk = rng.choice(np.arange(-100_000, 100_000), nb, replace=False).astype(np.float64) * 0.25
    bk[:4] = [-0.0, NAN, -INF, 5e-324]
    build = pd.DataFrame({"k": bk, "b1": rng.integers(0, 100, nb)})
    pk = rng.integers(-150_000, 150_000, npr).astype(np.float64) * 0.25
    pk[:6] = [0.0, NAN, -INF, INF, 5e-324, -5e-324]
    probe = pd.DataFrame({"p0": rng.random(npr), "k": pk})
    st = init_join_state(-1, (0,), (1,), tuple(build.columns), tuple(probe.columns), False, False)
    join_build_consume_batch(st, table_to_device(Table.from_pandas(build)), True)
    _, [(mn, mx)] = build_runtime_filter(st)
    assert decode_bound(mn) == np.nanmin(bk) == -INF and decode_bound(mx) == np.nanmax(bk)
    kept = runtime_join_filter((st,), table_to_device(Table.from_pandas(probe)), ((1,),)).to_pandas()
    bck, bcv = canon_keys(build.k)
    pck, pcv = canon_keys(probe.k)
    partner = pcv & np.isin(pck, bck[bcv])
    kk, kv = canon_keys(kept.k)
    assert np.isin(pck[partner], kk[kv]).all() and kv.all()  # no row with a partner dropped; no NaN row kept
    assert len(kept) < 0.7 * npr  # the bounds and the bloom filter dropped rows
    out, _, _ = join_probe_consume_batch(st, runtime_join_filter((st,), table_to_device(Table.from_pandas(probe)), ((1,),)), True, True)
    delete_join_state(st)
    u, cnt = np.unique(bck[bcv], return_counts=True)  # (0.0 may be drawn besides -0.0: one key, two build rows)
    assert out.n_rows == cnt[np.searchsorted(u, pck[partner])].sum()


@pytest.mark.parametrize("bk_dtype,pk_dtype", [(np.int64, np.float64), (np.float64, np.int64), (np.float32, np.float64), (np.float64, np.float32)])
def test_key_type_rules(gpu_lib, bk_dtype, pk_dtype):
    build = pd.DataFrame({"k": np.arange(10).astype(bk_dtype), "b1": np.arange(10)})
    probe = pd.DataFrame({"k": np.arange(10).astype(pk_dtype), "p1": np.arange(10)})
    names = {np.dtype(bk_dtype).name, np.dtype(pk_dtype).name}
    st = init_join_state(-1, (0,), (0,), ("k", "b1"), ("k", "p1"), False, False)
    join_build_consume_batch(st, table_to_device(Table.from_pandas(build)), True)
    pt = table_to_device(Table.from_pandas(probe))
    try:
        with pytest.raises(_lib.B200Error) as e:
            join_probe_consume_batch(st, pt, True)
        assert all(n in str(e.value) for n in names), str(e.value)
        # the runtime filter's key column follows the same rule
        with pytest.raises(_lib.B200Error) as e:
            runtime_join_filter((st,), pt, ((0,),))
        assert all(n in str(e.value) for n in names), str(e.value)
    finally:
        delete_join_state(st)


@pytest.mark.parametrize("how", ["inner", "left", "right", "outer"])
def test_physical_merge_equals_pandas(gpu_lib, how):
    from bodo_b200.physical import merge
    rng = np.random.default_rng(67)
    left = pd.DataFrame({"price": rng.choice(special_pool(np.float64, "probe"), 3_000), "x": rng.integers(0, 1000, 3_000)})
    right = pd.DataFrame({"px": rng.choice(special_pool(np.float64, "build"), 800), "y": rng.random(800)})
    got = merge(left, right, left_on="price", right_on="px", how=how, batch_size=1_000)
    exp = right.merge(left, left_on="px", right_on="price", how={"left": "right", "right": "left"}.get(how, how))
    assert_rowset_equal(got, exp)


def _sharded_worker(rank, world, port, q):
    import os

    import torch
    import torch.distributed as dist
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", rank))
    try:
        from oracle import oracle as O
        rng = np.random.default_rng(68)  # the same global tables on every rank; each rank feeds its own row slice
        nb, npr = 20_000, 60_000
        bk = rng.integers(0, 8_000, nb).astype(np.float64) * 0.5 - 1_000.0
        bk[:50] = -0.0  # in rank 0's slice
        bk[50:60] = NAN
        pk = rng.integers(0, 12_000, npr).astype(np.float64) * 0.5 - 1_000.0
        pk[-50:] = 0.0  # in the last rank's slice
        pk[-60:-50] = NAN
        build = pd.DataFrame({"k": bk, "b1": rng.integers(0, 1 << 40, nb)})
        probe = pd.DataFrame({"k": pk, "p1": rng.random(npr)})
        results = {}
        for name, kw, bo, po, na_eq in (("shuffle", {}, False, False, False), ("shuffle-outer", {}, True, True, True),
                                        ("broadcast", {"force_broadcast": True}, False, True, True)):
            os.environ["BODO_BCAST_JOIN_THRESHOLD"] = "0" if name != "broadcast" else str(10 << 20)
            st = init_join_state(-1, (0,), (0,), tuple(build.columns), tuple(probe.columns), bo, po, build_parallel=True,
                                 probe_parallel=True, device=rank, is_na_equal=na_eq, **kw)
            bchunk, pchunk = (nb + world - 1) // world, (npr + world - 1) // world
            join_build_consume_batch(st, Table.from_pandas(build.iloc[rank * bchunk:(rank + 1) * bchunk]), True)
            out, _, _ = join_probe_consume_batch(st, Table.from_pandas(probe.iloc[rank * pchunk:(rank + 1) * pchunk]), True, True)
            delete_join_state(st)
            allg = [None] * world
            dist.all_gather_object(allg, out.to_pandas())
            if rank == 0:
                got = pd.concat(allg, ignore_index=True)
                g, e = bits_sorted(got), bits_sorted(oracle_frame(O, build, probe, bo, po, na_eq))
                results[name] = bool(g.shape == e.shape and np.array_equal(g.to_numpy(), e.to_numpy()))
        q.put((rank, results))
    except Exception:
        import traceback
        q.put((rank, traceback.format_exc()))
    finally:
        dist.destroy_process_group()


@pytest.mark.timeout(600)
def test_sharded_join_two_gpus(gpu_lib):
    """Shuffle, shuffle-outer and broadcast joins over the ranks: -0.0 build rows on rank 0 meet 0.0 probe rows on the last rank
    (both hash to one rank), and the union of the ranks' outputs equals the oracle's join of the global tables.  The inner case
    runs with is_na_equal=False, so its NaN probe rows match nothing and the runtime filter drops them before the shuffle; the
    filter's handling of NA keys under is_na_equal=True is checked on one GPU (test_gpu_join_multi_keys.py,
    test_runtime_filter_has_no_false_negatives)."""
    import socket

    import torch
    import torch.multiprocessing as mp
    world = min(torch.cuda.device_count(), 4)
    if world < 2:
        pytest.skip("needs at least 2 GPUs")
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=_sharded_worker, args=(r, world, port, q)) for r in range(world)]
    for p in procs:
        p.start()
    res = [q.get(timeout=500) for _ in range(world)]
    for p in procs:
        p.join(timeout=60)
    for r in res:
        assert isinstance(r[1], dict), r
    r0 = [r for r in res if r[0] == 0][0][1]
    assert r0 == {"shuffle": True, "shuffle-outer": True, "broadcast": True}, r0
