"""The 16-byte SM-partitioned pair (spg_partition_tma_kernel K1, spg_aggregate_kernel K2 in groupby.cu) against a torch
recomputation.

Each case makes the sampled rows wide (keys beyond int32 or values beyond int32), so the narrow-row pair cannot take them
and K1 / K2 run (metric 15).  Every input runs three times: as it comes, with the narrow-row pair disabled
(B200_SPG_NARROW=0) and with the SM-partitioned path disabled (B200_SPG=0: the direct kernel).  Each result is checked bit for
bit against torch.unique + bincount (COUNT, SIZE) + int64 index_add_ (SUM, which wraps mod 2^64 like the kernels).  The
inputs are generated on the device and wrapped in Column / Table directly.  The cases aim at K2's rare work: the stash and the
direct path near and over its group capacity, multi-pass filtering, keys over all of int64, racing first insertions, the
marker key INT64_MIN, carries into the high word, every function set of the retry wire format, float keys, skew with the
heavy-hitter table off, and retry lists on both in-flight launch slots."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

WIDE = 1 << 40
INT64_MIN, INT64_MAX = -(1 << 63), (1 << 63) - 1
PATHS = {"default": {}, "narrow_off": {"B200_SPG_NARROW": "0"}, "direct": {"B200_SPG": "0"}}


def _spg_ns():
    """(owners = SMs, K2's bucket slots per owner: 16 bytes each, after the 1024 stash slots) as GroupbyState::spg_probe sets them."""
    import torch
    p = torch.cuda.get_device_properties(0)
    return p.multi_processor_count, ((p.shared_memory_per_block_optin - 64) // 16 - 1024) & ~1


def _spg_group_capacity():
    """GroupbyState::spg_group_capacity(): owners x 70 % of the bucket slots."""
    owners, ns = _spg_ns()
    return owners * (ns * 7 // 10)


def _gen(seed):
    import torch
    return torch.Generator(device="cuda").manual_seed(seed)


def _args(funcs):
    nf = len(funcs)
    if funcs == ("size",):
        return (0, 0), ()
    return tuple(range(nf + 1)), (1,) * nf


def _run(monkeypatch, k, v, funcs, hint, env=None, dropna=True):
    """One groupby over device tensors k / v; returns (device columns of the result, metrics 8, 9, 14, 15, 16)."""
    import torch

    from bodo_b200.streaming.groupby import (delete_groupby_state, get_metric, groupby_build_consume_batch,
                                             groupby_produce_output_batch, init_groupby_state)
    from bodo_b200.table import Column, Table
    for name in ("B200_SPG", "B200_SPG_NARROW", "B200_SPG_HOT"):
        monkeypatch.delenv(name, raising=False)
    for name, val in (env or {}).items():
        monkeypatch.setenv(name, val)
    offs, cols = _args(funcs)
    st = init_groupby_state(-1, (0,), funcs, offs, cols, expected_groups=hint, output_batch_size=1 << 30, dropna=dropna)
    try:
        groupby_build_consume_batch(st, Table([Column(k), Column(v)], ["k", "v"]), True, True)
        m = {i: get_metric(st, i) for i in (8, 9, 14, 15, 16)}
        out, last = groupby_produce_output_batch(st, True)
        assert last
        res = [torch.as_tensor(c.data, device="cuda").clone() for c in out.columns]
    finally:
        delete_groupby_state(st)
    return res, m


def _canon(k):
    """Table key of a float64 key (canon_float_key): its bits, with -0.0 -> 0 and NaN -> INT64_MIN."""
    import torch
    b = k.view(torch.int64).clone()
    b[k == 0] = 0
    b[torch.isnan(k)] = INT64_MIN
    return b


def _check(res, k, v, funcs):
    """res against the recomputation over the int64 table keys k (every row) and values v."""
    import torch
    uniq, inv = torch.unique(k, return_inverse=True)
    ref = {"size": torch.bincount(inv, minlength=len(uniq))}
    ref["count"] = ref["size"]
    ref["sum"] = torch.zeros(len(uniq), dtype=torch.int64, device=k.device).index_add_(0, inv, v)  # wraps mod 2^64 like the kernel
    got_k = _canon(res[0]) if res[0].dtype == torch.float64 else res[0]
    assert len(got_k) == len(uniq), (len(got_k), len(uniq))
    order = torch.argsort(got_k)
    assert torch.equal(got_k[order], uniq), "group keys differ"
    for j, f in enumerate(funcs):
        got = res[1 + j][order].view(torch.int64)
        bad = int((got != ref[f]).sum())
        assert bad == 0, f"{f}: {bad} of {len(uniq)} groups differ"


def _all_paths(monkeypatch, k, v, funcs, hint, table_keys=None, dropna=True, paths=PATHS):
    """Runs every configuration of `paths`, checks each result and the pair that ran; returns the metrics by path."""
    import torch
    tk, tv = (k if table_keys is None else table_keys), v
    if dropna and k.dtype == torch.float64:  # dropna drops the NaN group of a float key
        keep = ~torch.isnan(k)
        tk, tv = tk[keep], v[keep]
    ms = {}
    for name, env in paths.items():
        res, m = _run(monkeypatch, k, v, funcs, hint, env, dropna)
        _check(res, tk, tv, funcs)
        if name == "direct":
            assert m[8] == 0, m
        else:
            assert m[15] >= 1 and m[14] == 0, f"{name}: the 16-byte pair was expected to run, metrics {m}"
        ms[name] = m
    return ms


@pytest.mark.timeout(300)
@pytest.mark.parametrize("fill,hint", [(0.95, 1.0), (1.3, 0.5)], ids=["near_capacity", "overfull_one_pass"])
def test_spg_near_and_over_capacity(gpu_lib, monkeypatch, fill, hint):
    """Near spg_group_capacity() many keys live in their second bucket or the stash; 1.3x the capacity with a one-pass hint
    overfills the owners' tables, so keys also take the direct path and the global table fills up (retry list)."""
    import torch
    ng = int(_spg_group_capacity() * fill)
    n = 4 * ng
    g = _gen(31)
    k = torch.randint(0, ng, (n,), device="cuda", generator=g) + WIDE
    v = torch.randint(-500, 500, (n,), device="cuda", generator=g)
    _all_paths(monkeypatch, k, v, ("sum", "count"), int(ng * hint))


@pytest.mark.timeout(300)
@pytest.mark.parametrize("passes", [2, 3])
def test_spg_multi_pass(gpu_lib, monkeypatch, passes):
    """An accurate hint of (passes - 0.5) x the capacity: K2 keeps one hash sub-range of each owner bucket per pass."""
    import torch
    ng = int(_spg_group_capacity() * (passes - 0.5))
    g = _gen(32 + passes)
    k = torch.randint(0, ng, (1 << 24,), device="cuda", generator=g) + WIDE
    v = torch.randint(-(1 << 20), 1 << 20, (1 << 24,), device="cuda", generator=g)
    _all_paths(monkeypatch, k, v, ("sum", "count"), ng)


@pytest.mark.timeout(300)
def test_spg_scrambled_keys(gpu_lib, monkeypatch):
    """1 M keys spread over all of int64, INT64_MAX and INT64_MIN + 1 among them."""
    import torch
    rng = np.random.default_rng(34)
    pool = np.unique(rng.integers(INT64_MIN + 1, INT64_MAX, 1_050_000, endpoint=True))[:1_000_000]
    pool[:2] = [INT64_MAX, INT64_MIN + 1]
    pool_t = torch.from_numpy(np.unique(pool)).cuda()
    g = _gen(34)
    n = 1 << 24
    k = pool_t[torch.randint(0, len(pool_t), (n,), device="cuda", generator=g)]
    v = torch.randint(-(1 << 20), 1 << 20, (n,), device="cuda", generator=g)
    _all_paths(monkeypatch, k, v, ("sum", "count"), len(pool_t))


@pytest.mark.timeout(300)
def test_spg_first_appearances_race(gpu_lib, monkeypatch):
    """1.2 M groups of about two rows each: most rows are a key's first appearance in its owner's table, many at once."""
    import torch
    ng = 1_200_000
    g = _gen(35)
    k = torch.cat([torch.arange(ng, device="cuda"), torch.randint(0, ng, (ng,), device="cuda", generator=g)])
    k = k[torch.randperm(len(k), device="cuda", generator=g)] + WIDE
    v = torch.randint(-1000, 1000, (len(k),), device="cuda", generator=g)
    _all_paths(monkeypatch, k, v, ("sum", "count"), ng)


@pytest.mark.timeout(300)
def test_spg_marker_key_in_every_tile(gpu_lib, monkeypatch):
    """The key INT64_MIN (the table's empty marker) on every 997th row, so every 2048-row tile of K1 has some: those rows take
    the direct path to the marker slot."""
    import torch
    n, ng = 1 << 23, 500_000
    g = _gen(36)
    k = torch.randint(-ng, ng, (n,), device="cuda", generator=g) + WIDE
    k[::997] = INT64_MIN
    v = torch.randint(-(1 << 40), 1 << 40, (n,), device="cuda", generator=g)
    _all_paths(monkeypatch, k, v, ("sum", "count"), ng)


@pytest.mark.timeout(300)
@pytest.mark.parametrize("kind", ["near_int64_limits", "high_word_every_row"])
def test_spg_high_word_carries(gpu_lib, monkeypatch, kind):
    """Values within 2^32 of +-2^63 (low words wrap, high words 0x7FFFFFFF / 0x80000000 take carries), or a non-zero high word on
    every row: K2 adds the high part of almost every row straight to the global table."""
    import torch
    n, ng = 1 << 23, 300_000
    g = _gen(37)
    k = torch.randint(0, ng, (n,), device="cuda", generator=g)
    if kind == "near_int64_limits":
        off = torch.randint(0, 1 << 32, (n,), device="cuda", generator=g)
        v = torch.where(torch.rand(n, device="cuda", generator=g) < 0.5, INT64_MAX - off, INT64_MIN + off)
    else:
        v = torch.randint(1 << 32, 1 << 40, (n,), device="cuda", generator=g)
        v = torch.where(torch.rand(n, device="cuda", generator=g) < 0.5, v, -v)
    _all_paths(monkeypatch, k, v, ("sum", "count"), ng)


@pytest.mark.timeout(300)
@pytest.mark.parametrize("funcs", [("sum",), ("count",), ("size",), ("count", "sum"), ("sum", "count")])
def test_spg_function_sets_through_the_retry_list(gpu_lib, monkeypatch, funcs):
    """Every function set of the fast signature, with a hint of 2000 against 300 k groups: the flushes find the global table at
    its limit and travel the retry list, whose wire order follows the function order (sum_first)."""
    import torch
    n, ng = 1 << 22, 300_000
    g = _gen(38)
    k = torch.randint(0, ng, (n,), device="cuda", generator=g) + WIDE
    v = torch.randint(-(1 << 40), 1 << 40, (n,), device="cuda", generator=g)
    ms = _all_paths(monkeypatch, k, v, funcs, 2000)
    assert ms["default"][9] > 0, "the retry list was expected to be used"


@pytest.mark.timeout(300)
@pytest.mark.parametrize("dropna", [True, False])
def test_spg_float64_keys(gpu_lib, monkeypatch, dropna):
    """About 1 M float64 keys (k * 0.5 + 0.25, whose bits are wide), plus -0.0 / 0.0 (one group) and NaN (dropped, or the group
    of the marker key), compared over the canonical table keys."""
    import torch
    n, ng = 1 << 23, 1_000_000
    g = _gen(39)
    k = torch.randint(0, ng, (n,), device="cuda", generator=g).double() * 0.5 + 0.25
    k[3::101] = -0.0
    k[5::103] = 0.0
    k[7::107] = float("nan")
    v = torch.randint(-(1 << 20), 1 << 20, (n,), device="cuda", generator=g)
    _all_paths(monkeypatch, k, v, ("sum", "count"), ng, table_keys=_canon(k), dropna=dropna)


@pytest.mark.timeout(300)
def test_spg_skew_with_and_without_heavy_hitter_table(gpu_lib, monkeypatch):
    """Zipf(1.2) keys: with the heavy-hitter table off the hottest owners' buckets overflow into K1's direct path; with it on the
    heavy hitters are aggregated in K1.  Both give the recomputed result."""
    import torch
    rng = np.random.default_rng(40)
    n = 1 << 23
    k = torch.from_numpy((rng.zipf(1.2, n) % 1_000_000).astype(np.int64)).cuda() + WIDE
    v = torch.randint(-(1 << 40), 1 << 40, (n,), device="cuda", generator=_gen(40))
    ms = _all_paths(monkeypatch, k, v, ("sum", "count"), 200_000,
                    paths={"hot_on": {}, "hot_off": {"B200_SPG_HOT": "0"}, "direct": {"B200_SPG": "0"}})
    assert ms["hot_on"][16] > 0, "the heavy-hitter table was expected to admit keys"
    assert ms["hot_off"][16] == 0


@pytest.mark.timeout(600)
def test_spg_retry_lists_of_both_launch_slots(gpu_lib, monkeypatch):
    """2^27 + 2^24 rows (two launches, one per in-flight slot), about 2 M groups, a hint of 2000 and a non-zero high word on every
    row: nearly every row and every occupied shared slot of both launches lands in its slot's retry list.  The first spg_finish
    grows the table and merges both lists; the second finds nothing left to do."""
    import torch
    n, ng = (1 << 27) + (1 << 24), 2_000_000
    g = _gen(41)
    k = torch.randint(0, ng, (n,), device="cuda", generator=g)
    v = torch.randint(1 << 32, 1 << 40, (n,), device="cuda", generator=g)
    ms = _all_paths(monkeypatch, k, v, ("sum", "count"), 2000, paths={"default": {}, "direct": {"B200_SPG": "0"}})
    assert ms["default"][15] >= 2, ms
    # the first launch's list holds at most its 2^27 rows plus one entry per shared slot: more means the second one had entries too
    owners, ns = _spg_ns()
    assert ms["default"][9] > (1 << 27) + owners * (ns + 1024), ms
