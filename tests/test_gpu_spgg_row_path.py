"""SPG-G (spgg.cuh: spgg_partition_kernel K1g, spgg_aggregate_kernel K2g, spgg_replay_kernel) against a torch recomputation.

Every case runs the generic SM-partitioned pair (metric 12) and checks each group against torch.unique + bincount (SIZE),
masked index_add_ (COUNT, and SUM, which wraps mod 2^64 like the kernels), scatter_reduce amin / amax (MIN, MAX) and an exact
MEAN, with NA keys and NA values handled by masks.  MEAN's reference is exact: per-group sums of the high (v >> 32) and low
(v & 0xFFFFFFFF) halves in int64 (neither can overflow below 2^31 rows per group), combined in long double and divided by the
count.  The kernels add at most m = 2 * count + 4 doubles per group (a partial per flush of a shared slot, per carry of a high
word, per K1g CTA for the NA-key group), each rounded once when converted; the partials' magnitudes add up to at most
sum|v| + 2^32 * m.  So the stated tolerance is |mean - exact| <= (2 m + 1) * 2^-53 * (sum|v| + 2^32 * m) / count.  A 64-bit
wrap of a partial is off by 2^64 / count, far outside it.

The cases aim at the rare paths: the retry list and its replay (under-hinted), every slot layout near its capacity, both
multi-pass branches of K2g, zero-extended uint32 columns, nullable datetime keys, the marker key, K1g bucket overflow, and
means at the edges of int64."""
import numpy as np
import pandas as pd
import pytest

pytestmark = pytest.mark.gpu

INT64_MIN, INT64_MAX = -(1 << 63), (1 << 63) - 1
GEN_CLS = 448  # spgg.cuh: K1g's counting-sort classes (valued buckets of all passes + NA-value buckets must fit)
LAYOUT_FUNCS = {  # slot layout v = (min / max fields) + 2 * (NA-value counter; needs a nullable value and `size`)
    0: ("sum", "count", "mean"),
    1: ("min", "max", "mean", "count"),
    2: ("sum", "size", "mean"),
    3: ("min", "max", "size", "sum"),
}


def _spgg_group_capacity(layout):
    """GroupbyState::spgg_group_capacity(layout): owners x 70 % of K2g's slots of 16 + 16 * mm + 4 * nn bytes."""
    import torch
    p = torch.cuda.get_device_properties(0)
    sb = 16 + (16 if layout & 1 else 0) + (4 if layout & 2 else 0)
    ns = ((p.shared_memory_per_block_optin - 64) // sb - 1024) & ~1
    return p.multi_processor_count * (ns * 7 // 10)


def _owner(keys, n_owners):
    """spg_owner(spg_hash(key), n_owners) of groupby.cu."""
    x = keys.astype(np.int64).view(np.uint64)
    with np.errstate(over="ignore"):
        h = (x ^ (x >> np.uint64(29))) * np.uint64(0x9E3779B97F4A7C15)
    return ((h >> np.uint64(32)) * np.uint64(n_owners)) >> np.uint64(32)


def _series(x, valid):
    return pd.Series(x) if valid is None else pd.Series(pd.arrays.IntegerArray(x, ~valid))


def _table(k, kvalid, v, vvalid, datetime_keys=False):
    """Host Table: key column (nullable when kvalid is given; datetime64[ns] through Arrow), value column likewise."""
    import pyarrow as pa

    from bodo_b200.table import Table, column_from_arrow, column_from_pandas
    if datetime_keys:
        kc = column_from_arrow(pa.array(k, type=pa.timestamp("ns"), mask=None if kvalid is None else ~kvalid))
    else:
        kc = column_from_pandas(_series(k, kvalid))
    return Table([kc, column_from_pandas(_series(v, vvalid))], ["k", "v"])


def _reference(k, kvalid, v, vvalid, dropna):
    """Per group (ascending key, then the NA-key group): size, count, sum (wrapping), min, max, exact mean, sum|v| (numpy)."""
    import torch
    kt, vt = torch.from_numpy(k.astype(np.int64)).cuda(), torch.from_numpy(v.astype(np.int64)).cuda()
    kv = torch.ones(len(k), dtype=torch.bool, device="cuda") if kvalid is None else torch.from_numpy(kvalid).cuda()
    vv = torch.ones(len(k), dtype=torch.bool, device="cuda") if vvalid is None else torch.from_numpy(vvalid).cuda()
    uniq, inv = torch.unique(kt[kv], return_inverse=True)
    gid = torch.full((len(k),), len(uniq), dtype=torch.int64, device="cuda")
    gid[kv] = inv
    na_group = not dropna and bool((~kv).any())
    ng = len(uniq) + (1 if na_group else 0)
    keep = gid < ng
    gid, vt, vv = gid[keep], vt[keep], vv[keep]
    z = lambda: torch.zeros(ng, dtype=torch.int64, device="cuda")  # noqa: E731
    vz = torch.where(vv, vt, 0)
    r = {"size": torch.bincount(gid, minlength=ng), "count": z().index_add_(0, gid, vv.long()), "sum": z().index_add_(0, gid, vz)}
    r["min"] = torch.full((ng,), INT64_MAX, device="cuda").scatter_reduce_(0, gid[vv], vt[vv], "amin", include_self=False)
    r["max"] = torch.full((ng,), INT64_MIN, device="cuda").scatter_reduce_(0, gid[vv], vt[vv], "amax", include_self=False)
    hi, lo = z().index_add_(0, gid, vz >> 32), z().index_add_(0, gid, vz & 0xFFFFFFFF)
    r["abs"] = torch.zeros(ng, dtype=torch.float64, device="cuda").index_add_(0, gid, vz.double().abs())
    out = {f: x.cpu().numpy() for f, x in r.items()}
    out["exact"] = hi.cpu().numpy().astype(np.longdouble) * np.longdouble(2**32) + lo.cpu().numpy().astype(np.longdouble)
    out["keys"] = uniq.cpu().numpy()
    out["na_group"] = na_group
    return out


def _run(t, funcs, hint, dropna):
    from bodo_b200.streaming.groupby import (delete_groupby_state, get_metric, groupby_build_consume_batch,
                                             groupby_produce_output_batch, init_groupby_state)
    from tests.helpers import table_to_device
    offs = [0]
    for f in funcs:
        offs.append(offs[-1] + (0 if f == "size" else 1))
    st = init_groupby_state(-1, (0,), funcs, tuple(offs), (1,) * offs[-1], expected_groups=hint, output_batch_size=1 << 30, dropna=dropna)
    try:
        groupby_build_consume_batch(st, table_to_device(t), True, True)
        m = {i: get_metric(st, i) for i in (8, 9, 12)}
        out, _ = groupby_produce_output_batch(st, True)
        cols = [(c.values_numpy(), c.valid_mask_numpy()) for c in out.columns]
    finally:
        delete_groupby_state(st)
    return cols, m


def _check(k, kvalid, v, vvalid, funcs, hint, dropna=True, datetime_keys=False):
    """Runs the groupby, checks every group against _reference and that SPG-G ran; returns the metrics."""
    cols, m = _run(_table(k, kvalid, v, vvalid, datetime_keys), funcs, hint, dropna)
    assert m[12] >= 1, f"the generic SM-partitioned kernels were expected to run, metrics {m}"
    ref = _reference(k, kvalid, v, vvalid, dropna)
    gk, gkv = cols[0]
    gk = gk.astype(np.int64)
    gkv = np.ones(len(gk), bool) if gkv is None else gkv
    assert len(gk) == len(ref["keys"]) + ref["na_group"], (len(gk), len(ref["keys"]), ref["na_group"])
    assert (~gkv).sum() == ref["na_group"], "NA-key group"
    order = np.lexsort((gk, ~gkv))  # valid keys ascending, then the NA-key group
    np.testing.assert_array_equal(gk[order][gkv[order]], ref["keys"], err_msg="group keys")
    cnt = ref["count"]
    for j, f in enumerate(funcs):
        vals, valid = cols[1 + j]
        vals = vals[order]
        valid = np.ones(len(vals), bool) if valid is None else valid[order]
        if f in ("size", "count", "sum"):
            np.testing.assert_array_equal(vals.astype(np.int64), ref[f], err_msg=f)
        elif f in ("min", "max"):
            np.testing.assert_array_equal(valid, cnt > 0, err_msg=f"{f} (NA mask)")
            np.testing.assert_array_equal(vals.astype(np.int64)[cnt > 0], ref[f][cnt > 0], err_msg=f)
        else:  # mean: the stated bound of the module docstring
            np.testing.assert_array_equal(valid & ~np.isnan(vals), cnt > 0, err_msg="mean (NA mask)")
            c = cnt[cnt > 0]
            exact = ref["exact"][cnt > 0] / c.astype(np.longdouble)
            err = np.abs(vals[cnt > 0].astype(np.longdouble) - exact).astype(np.float64)
            m_add = 2 * c + 4
            tol = (2 * m_add + 1) * 2.0**-53 * (ref["abs"][cnt > 0] + 2.0**32 * m_add) / c
            bad = np.flatnonzero(err > tol)
            assert len(bad) == 0, f"mean: {len(bad)} groups beyond the bound, e.g. got {vals[cnt > 0][bad[:3]]} exact {exact[bad[:3]]}"
    return m


def _data(seed, n, ng, v_lo=-(1 << 40), v_hi=1 << 40, v_na=0.0, k_na=0.0):
    rng = np.random.default_rng(seed)
    k = rng.integers(0, ng, n).astype(np.int64) * 7 - ng
    v = rng.integers(v_lo, v_hi, n, dtype=np.int64)
    vvalid = rng.random(n) >= v_na if v_na else None
    kvalid = rng.random(n) >= k_na if k_na else None
    return k, kvalid, v, vvalid


@pytest.mark.timeout(300)
@pytest.mark.parametrize("layout", [0, 1, 2, 3])
@pytest.mark.parametrize("shape", ["near_capacity", "under_hinted"])
def test_spgg_layouts_near_capacity_and_through_the_replay(gpu_lib, layout, shape):
    """Each slot layout at 0.95x its group capacity with an accurate hint (second buckets, stash), and at about 1 M groups with a
    hint of 2000: the shared tables overflow into the direct path, the global table fills up and spgg_replay_kernel replays the
    retry list (metric 9)."""
    ng = int(0.95 * _spgg_group_capacity(layout)) if shape == "near_capacity" else 1_000_000
    k, kv, v, vv = _data(50 + layout, 4 * ng, ng, v_na=0.1 if layout & 2 else 0.0)
    if layout == 1:  # nullable values without `size`: an NA-value bucket but no NA-value counter in the slot
        vv = np.random.default_rng(7).random(len(v)) >= 0.1
    m = _check(k, kv, v, vv, LAYOUT_FUNCS[layout], ng if shape == "near_capacity" else 2000)
    if shape == "under_hinted":
        assert m[9] > 0, f"the retry list was expected to be replayed, metrics {m}"


@pytest.mark.timeout(300)
@pytest.mark.parametrize("nullable", [False, True], ids=["virtual_owners", "per_row_pass_test"])
def test_spgg_multi_pass_branches(gpu_lib, nullable):
    """p = GEN_CLS // SMs passes (3 on 132 SMs) with an accurate hint.  Non-null values: the p x SMs valued buckets fit K1g's
    GEN_CLS classes, so K1g partitions into per-pass virtual owners.  Nullable values add SMs NA-value classes, (p + 1) x SMs >
    GEN_CLS, so K2g reads each owner bucket every pass and tests every row's pass."""
    import torch
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    p = GEN_CLS // sms
    if p < 2:
        pytest.skip(f"{sms} SMs leave no room for a multi-pass class table")
    layout = 3 if nullable else 0
    funcs = ("sum", "size", "min", "max") if nullable else ("mean", "count")
    ng = int(_spgg_group_capacity(layout) * (p - 0.5))
    k, kv, v, vv = _data(60, 1 << 24, ng, v_na=0.1 if nullable else 0.0)
    _check(k, kv, v, vv, funcs, ng)


@pytest.mark.timeout(300)
@pytest.mark.parametrize("dtype", ["uint32", "int32"])
def test_spgg_four_byte_columns(gpu_lib, dtype):
    """4-byte keys and values over their whole range: uint32 with the high bit set must be zero-extended, int32 sign-extended."""
    rng = np.random.default_rng(61)
    n, ng = 1 << 22, 400_000
    dt = np.dtype(dtype)
    lo, hi = np.iinfo(dt).min, np.iinfo(dt).max
    pool = np.unique(rng.integers(lo, hi, ng, endpoint=True)).astype(dt)
    k = pool[rng.integers(0, len(pool), n)]
    v = rng.integers(lo, hi, n, endpoint=True).astype(dt)
    vv = rng.random(n) >= 0.05
    _check(k, None, v, vv, ("sum", "count", "mean", "min", "max", "size"), len(pool))


@pytest.mark.timeout(300)
@pytest.mark.parametrize("dropna", [True, False])
def test_spgg_datetime_keys_with_nat(gpu_lib, dropna):
    """Nullable datetime64[ns] keys, 3 % NaT: dropped, or one NA-key group that K1g pre-aggregates per CTA."""
    rng = np.random.default_rng(62)
    n, ng = 1 << 22, 300_000
    k = 1_600_000_000_000_000_000 + rng.integers(0, ng, n).astype(np.int64) * 1_000_000_007
    kv = rng.random(n) >= 0.03
    v = rng.integers(-(1 << 40), 1 << 40, n, dtype=np.int64)
    _check(k, kv, v, None, ("mean", "min", "max", "count"), ng, dropna=dropna, datetime_keys=True)


@pytest.mark.timeout(300)
def test_spgg_marker_key(gpu_lib):
    """The key INT64_MIN (the table's empty marker) on every 997th row of an int64 key column: K1g sends it to the marker slot."""
    k, kv, v, vv = _data(63, 1 << 22, 300_000, v_na=0.1)
    k[::997] = INT64_MIN
    _check(k, kv, v, vv, ("sum", "size", "mean", "max"), 300_000)


@pytest.mark.timeout(300)
def test_spgg_bucket_overflow(gpu_lib):
    """Half the rows on owner 0 through 10^5 keys, nullable values: owner 0's valued and NA-value buckets overflow and K1g sends
    the excess rows the direct way."""
    import torch
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    cand = np.arange(1, 20_000_000, dtype=np.int64)
    owner0 = cand[_owner(cand, sms) == 0][:100_000]
    assert len(owner0) == 100_000
    rng = np.random.default_rng(64)
    n, ng = 1 << 22, 300_000
    k = rng.integers(-ng, ng, n).astype(np.int64)
    skew = rng.random(n) < 0.5
    k[skew] = owner0[rng.integers(0, len(owner0), int(skew.sum()))]
    v = rng.integers(INT64_MIN, INT64_MAX, n, dtype=np.int64, endpoint=True)
    vv = rng.random(n) >= 0.2
    _check(k, None, v, vv, ("sum", "size", "min", "max", "mean"), len(np.unique(k)))


@pytest.mark.timeout(300)
@pytest.mark.parametrize("edge", ["near_int64_max", "int64_min", "na_key_group_near_2_62"])
def test_spgg_mean_at_int64_edges(gpu_lib, edge):
    """MEAN (with MIN and MAX) over values in [2^63 - 2^32, 2^63), where a carry out of the low word makes the high part +2^63;
    over INT64_MIN; and, with dropna=False, over an NA-key group of values near 2^62, whose per-CTA partial sum passes 2^63."""
    rng = np.random.default_rng(65)
    n, ng = 1 << 22, 200_000
    k = rng.integers(0, ng, n).astype(np.int64)
    kv = None
    if edge == "near_int64_max":
        v = INT64_MAX - rng.integers(0, 1 << 32, n, dtype=np.int64)
    elif edge == "int64_min":
        v = np.where(rng.random(n) < 0.5, INT64_MIN, rng.integers(-(1 << 40), 1 << 40, n, dtype=np.int64))
    else:
        v = rng.integers(-(1 << 40), 1 << 40, n, dtype=np.int64)
        kv = rng.random(n) >= 0.1
        v[~kv] = (1 << 62) + rng.integers(0, 1 << 40, int((~kv).sum()), dtype=np.int64)
    _check(k, kv, v, None, ("mean", "min", "max", "count"), ng, dropna=kv is None)
