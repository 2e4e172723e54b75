"""The K1 tile loop shared by every SM-partitioned partition kernel (spg_partition_tiles in groupby.cu) at the edges of its tiles.

Each form runs on 2^20 + e rows for e in {0, 1, 511, 2047, 2049, 4095, 4097}: whole tiles only, then a trailing partial tile of
one row, of just under and just over half a 4096-row tile, and of one row under and over a whole tile (K1 and K1g take 2048-row
tiles, K1n 4096).  The state is given the true group count, so the first launch takes every row and the tiles start at row 0.
The metrics confirm which form ran: the 16-byte pair (metric 15) with and without its heavy-hitter table (metric 16), the
narrow-row pair's hash form (metric 14, with the dense form off: metric 17 stays 0), its dense form (metric 17), and the
generic pair (metric 12) with 4- and 8-byte keys and a nullable value column.  Every group is checked bit for bit against a
torch recomputation: SIZE, COUNT (rows with a valid value), SUM (wrapping mod 2^64 like the kernels), MIN and MAX."""
import numpy as np
import pandas as pd
import pytest

pytestmark = pytest.mark.gpu

WIDE = 1 << 40
EXTRA = [0, 1, 511, 2047, 2049, 4095, 4097]
INT64_MIN, INT64_MAX = -(1 << 63), (1 << 63) - 1


def _rows(e):
    return (1 << 20) + e


def _reference(k, v, vvalid):
    """Per ascending key: size, count, sum, min and max over the rows whose value is valid (torch, on the device)."""
    import torch
    uniq, inv = torch.unique(k, return_inverse=True)
    ng = len(uniq)
    z = lambda: torch.zeros(ng, dtype=torch.int64, device=k.device)  # noqa: E731
    vz = torch.where(vvalid, v, 0)
    ref = {"size": torch.bincount(inv, minlength=ng), "count": z().index_add_(0, inv, vvalid.long()), "sum": z().index_add_(0, inv, vz)}
    ref["min"] = torch.full((ng,), INT64_MAX, device=k.device).scatter_reduce_(0, inv[vvalid], v[vvalid], "amin", include_self=False)
    ref["max"] = torch.full((ng,), INT64_MIN, device=k.device).scatter_reduce_(0, inv[vvalid], v[vvalid], "amax", include_self=False)
    return uniq, ref


def _groupby(monkeypatch, table, funcs, hint, env):
    """One groupby over `table` (key column 0, value column 1); returns (device result columns, metrics 12, 14, 15, 16, 17)."""
    import torch

    from bodo_b200.streaming.groupby import (delete_groupby_state, get_metric, groupby_build_consume_batch,
                                             groupby_produce_output_batch, init_groupby_state)
    for name in ("B200_SPG", "B200_SPG_NARROW", "B200_SPG_HOT", "B200_SPG_DENSE", "B200_SPG_GEN"):
        monkeypatch.delenv(name, raising=False)
    for name, val in env.items():
        monkeypatch.setenv(name, val)
    offs = [0]
    for f in funcs:
        offs.append(offs[-1] + (0 if f == "size" else 1))
    st = init_groupby_state(-1, (0,), funcs, tuple(offs), (1,) * offs[-1], expected_groups=hint, output_batch_size=1 << 30)
    try:
        groupby_build_consume_batch(st, table, True, True)
        m = {i: get_metric(st, i) for i in (12, 14, 15, 16, 17)}
        out, last = groupby_produce_output_batch(st, True)
        assert last
        res = [torch.as_tensor(c.data, device="cuda").clone() for c in out.columns]
    finally:
        delete_groupby_state(st)
    return res, m


def _check(res, k, v, vvalid, funcs):
    import torch
    uniq, ref = _reference(k, v, vvalid)
    got_k = res[0].to(torch.int64)
    assert len(got_k) == len(uniq), (len(got_k), len(uniq))
    order = torch.argsort(got_k)
    assert torch.equal(got_k[order], uniq), "group keys differ"
    for j, f in enumerate(funcs):
        got = res[1 + j][order].view(torch.int64)
        bad = int((got != ref[f]).sum())
        assert bad == 0, f"{f}: {bad} of {len(uniq)} groups differ"


def _device_case(monkeypatch, k, v, env):
    """The int64 (key, value) pair through the path that `env` leaves on; returns the metrics."""
    import torch

    from bodo_b200.table import Column, Table
    funcs = ("sum", "count")
    ng = int(torch.unique(k).numel())
    res, m = _groupby(monkeypatch, Table([Column(k), Column(v)], ["k", "v"]), funcs, ng, env)
    _check(res, k, v, torch.ones_like(k, dtype=torch.bool), funcs)
    return m


def _gen(seed):
    import torch
    return torch.Generator(device="cuda").manual_seed(seed)


@pytest.mark.timeout(300)
@pytest.mark.parametrize("e", EXTRA)
def test_tile_edges_16_byte(gpu_lib, monkeypatch, e):
    """K1: keys beyond int32 (the narrow-row pair cannot take them), uniform over 200 k groups: no heavy hitters."""
    import torch
    n, g = _rows(e), _gen(50 + e)
    k = torch.randint(0, 200_000, (n,), device="cuda", generator=g) + WIDE
    v = torch.randint(-(1 << 40), 1 << 40, (n,), device="cuda", generator=g)
    m = _device_case(monkeypatch, k, v, {})
    assert m[15] >= 1 and m[14] == 0 and m[16] == 0, m


@pytest.mark.timeout(300)
@pytest.mark.parametrize("e", EXTRA)
def test_tile_edges_16_byte_hot(gpu_lib, monkeypatch, e):
    """K1 with its heavy-hitter table: a fifth of the rows carry one of three keys, aggregated inside K1."""
    import torch
    n, g = _rows(e), _gen(60 + e)
    k = torch.randint(0, 200_000, (n,), device="cuda", generator=g) + WIDE
    hot = torch.rand(n, device="cuda", generator=g) < 0.2
    k[hot] = WIDE + 3 * torch.randint(0, 3, (int(hot.sum()),), device="cuda", generator=g)
    v = torch.randint(-(1 << 40), 1 << 40, (n,), device="cuda", generator=g)
    m = _device_case(monkeypatch, k, v, {})
    assert m[15] >= 1 and m[16] > 0, m


@pytest.mark.timeout(300)
@pytest.mark.parametrize("e", EXTRA)
def test_tile_edges_narrow_hash(gpu_lib, monkeypatch, e):
    """K1n's hash form (dense form off): int32 keys spread over a range too wide for a dense window anyway."""
    import torch
    n, g = _rows(e), _gen(70 + e)
    k = torch.randint(-(1 << 30), 1 << 30, (200_000,), device="cuda", generator=g)[torch.randint(0, 200_000, (n,), device="cuda", generator=g)]
    v = torch.randint(-(1 << 20), 1 << 20, (n,), device="cuda", generator=g)
    m = _device_case(monkeypatch, k, v, {"B200_SPG_DENSE": "0"})
    assert m[14] > 0 and m[17] == 0, m


@pytest.mark.timeout(300)
@pytest.mark.parametrize("e", EXTRA)
def test_tile_edges_dense(gpu_lib, monkeypatch, e):
    """K1n's dense form: 100 k keys in a small window, small values."""
    import torch
    n, g = _rows(e), _gen(80 + e)
    k = torch.randint(0, 100_000, (n,), device="cuda", generator=g) + 5_000
    v = torch.randint(-500, 500, (n,), device="cuda", generator=g)
    m = _device_case(monkeypatch, k, v, {})
    assert m[17] > 0, m


@pytest.mark.timeout(300)
@pytest.mark.parametrize("e", EXTRA)
@pytest.mark.parametrize("key_dtype", [np.int32, np.int64])
def test_tile_edges_generic(gpu_lib, monkeypatch, e, key_dtype):
    """K1g: 4- or 8-byte keys and a nullable int64 value column (every 7th value NA), so K1g also loads the value bitmap and
    partitions the NA-value rows into the key-only buckets."""
    import torch

    from bodo_b200.table import Table, column_from_pandas
    from tests.helpers import table_to_device
    rng = np.random.default_rng(90 + e)
    n = _rows(e)
    k = rng.integers(-25_000, 25_000, n).astype(key_dtype)  # ~20 rows per group: every group has a valid value
    v = rng.integers(-(1 << 40), 1 << 40, n)
    vvalid = np.arange(n) % 7 != 3
    t = Table([column_from_pandas(pd.Series(k)), column_from_pandas(pd.Series(pd.arrays.IntegerArray(v, ~vvalid)))], ["k", "v"])
    funcs = ("size", "count", "sum", "min", "max")
    res, m = _groupby(monkeypatch, table_to_device(t), funcs, len(np.unique(k)), {})
    assert m[12] >= 1, m
    kt = torch.from_numpy(k.astype(np.int64)).cuda()
    _check(res, kt, torch.from_numpy(v).cuda(), torch.from_numpy(vvalid).cuda(), funcs)
