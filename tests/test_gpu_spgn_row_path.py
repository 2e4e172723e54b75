"""K2n (spgn_aggregate_kernel, bodo_b200/csrc/spgn.cuh), the narrow-row aggregate kernel, against a torch recomputation.

Each case feeds int32-range keys and values in one batch so that the SPG-N pair runs (metric 14), and checks every group's
SUM and COUNT bit for bit against torch.unique + index_add_ / bincount.  The cases aim at the kernel's rare per-row work: keys
that live in their second bucket or in the stash, a table so full that keys take the direct path, low sum words that wrap,
multi-pass filtering, first appearances that race, and rows outside the narrow format mixed in."""
import numpy as np
import pandas as pd
import pytest

from bodo_b200.table import Table

pytestmark = pytest.mark.gpu


def _spgn_group_capacity():
    """GroupbyState::spgn_group_capacity(): owners (one per SM) x 70 % of K2n's bucket slots (the shared memory left after the
    1024 stash slots and the warps' 9 KB of cold-row queues, 12 bytes per slot)."""
    import torch
    p = torch.cuda.get_device_properties(0)
    smem = getattr(p, "shared_memory_per_block_optin", 232448)
    ns = ((smem - 256 - 9216) // 12 - 1024) & ~1
    return p.multi_processor_count * (ns * 7 // 10)


def _unsampled(n):
    """Rows the narrow-format sampler does not read (it reads 32 blocks of 1024 rows at b * n / 32); n is a multiple of 32."""
    return np.arange(n) % (n // 32) >= 1024


def _check(k, v, expected_groups):
    import torch

    from bodo_b200.streaming.groupby import (delete_groupby_state, get_metric, groupby_build_consume_batch,
                                             groupby_produce_output_batch, init_groupby_state)
    from tests.helpers import table_to_device
    t = Table.from_pandas(pd.DataFrame({"k": k, "v": v}))
    st = init_groupby_state(-1, (0,), ("sum", "count"), (0, 1, 2), (1, 1), expected_groups=expected_groups, output_batch_size=1 << 30)
    groupby_build_consume_batch(st, table_to_device(t), True, True)
    used = get_metric(st, 14)
    out, _ = groupby_produce_output_batch(st, True)
    got = out.to_pandas()
    delete_groupby_state(st)
    assert used >= 1, "the narrow-row kernels were expected to run for this shape"

    kt, vt = torch.from_numpy(k).cuda(), torch.from_numpy(v).cuda()
    uniq, inv = torch.unique(kt, return_inverse=True)
    cnt = torch.bincount(inv, minlength=len(uniq))
    s = torch.zeros(len(uniq), dtype=torch.int64, device=kt.device).index_add_(0, inv, vt)  # wraps mod 2^64 like the kernel
    got = got.sort_values(got.columns[0])
    assert len(got) == len(uniq)
    np.testing.assert_array_equal(got.iloc[:, 0].to_numpy(np.int64), uniq.cpu().numpy())
    np.testing.assert_array_equal(got.iloc[:, 1].to_numpy(np.int64), s.cpu().numpy())
    np.testing.assert_array_equal(got.iloc[:, 2].to_numpy(np.int64), cnt.cpu().numpy())


@pytest.mark.timeout(300)
@pytest.mark.parametrize("fill,hint", [(0.95, 1.0), (1.3, 0.5)], ids=["near_capacity", "overfull_one_pass"])
def test_spgn_near_and_over_capacity(gpu_lib, fill, hint):
    """Near spgn_group_capacity() many keys live in their second bucket or the stash; with a low hint (one pass) 1.3x the capacity
    overfills the owners' tables, so keys also take the direct path."""
    rng = np.random.default_rng(21)
    ng = int(_spgn_group_capacity() * fill)
    n = (4 * ng) // 32 * 32
    k = rng.integers(0, ng, n).astype(np.int64) - ng // 2
    v = rng.integers(-500, 500, n).astype(np.int64)
    _check(k, v, int(ng * hint))


@pytest.mark.timeout(300)
def test_spgn_low_word_carries(gpu_lib):
    """Values near +-2^31: almost every add wraps the biased low sum word, so the high word takes carries and borrows."""
    rng = np.random.default_rng(22)
    n, ng = 1 << 23, 300_000
    k = rng.integers(0, ng, n).astype(np.int64)
    big = rng.integers((1 << 31) - 4096, 1 << 31, n).astype(np.int64)
    v = np.where(rng.random(n) < 0.5, big - 1, -big)  # [2^31 - 4097, 2^31 - 2] and [-2^31 + 1, -2^31 + 4096]
    _check(k, v, ng)


@pytest.mark.timeout(300)
def test_spgn_two_passes(gpu_lib):
    """2 M groups: K2n filters each pass's keys (n_pass = 2)."""
    rng = np.random.default_rng(23)
    n, ng = 1 << 24, 2_000_000
    k = rng.integers(0, ng, n).astype(np.int64)
    v = rng.integers(-500, 500, n).astype(np.int64)
    _check(k, v, ng)


@pytest.mark.timeout(300)
def test_spgn_scrambled_keys(gpu_lib):
    """1 M keys spread over all of int32 (no dense range for the bucket hash to spread evenly)."""
    rng = np.random.default_rng(24)
    n = 1 << 24
    pool = np.unique(rng.integers(-(1 << 31) + 1, 1 << 31, 1_050_000))[:1_000_000]
    k = pool[rng.integers(0, len(pool), n)].astype(np.int64)
    v = rng.integers(-(1 << 20), 1 << 20, n).astype(np.int64)
    _check(k, v, len(pool))


@pytest.mark.timeout(300)
def test_spgn_first_appearances_race(gpu_lib):
    """1.2 M groups of about two rows each: most rows are a key's first appearance in its owner's table, many of them at once."""
    rng = np.random.default_rng(25)
    ng = 1_200_000
    k = np.concatenate([np.arange(ng), rng.integers(0, ng, ng)]).astype(np.int64)
    k = k[rng.permutation(len(k))][: len(k) // 32 * 32]
    v = rng.integers(-1000, 1000, len(k)).astype(np.int64)
    _check(k, v, ng)


@pytest.mark.timeout(300)
def test_spgn_wide_stragglers(gpu_lib):
    """A few thousand rows outside the narrow format (key beyond int32, the key INT32_MIN, value beyond int32), none of them where
    the sampler looks, mixed into 1 M narrow groups: they take K1n's direct path and land in the same result."""
    rng = np.random.default_rng(26)
    n, ng = 1 << 23, 1_000_000
    k = rng.integers(0, ng, n).astype(np.int64)
    v = rng.integers(-500, 500, n).astype(np.int64)
    idx = np.arange(n)
    w = (idx % 997 == 5) & _unsampled(n)
    k[w & (idx % 3 == 0)] += 1 << 40
    k[w & (idx % 3 == 1)] = np.iinfo(np.int32).min
    v[w & (idx % 3 == 2)] = (1 << 40) + idx[w & (idx % 3 == 2)]
    _check(k, v, ng)
