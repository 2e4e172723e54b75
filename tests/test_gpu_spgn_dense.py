"""The dense form of the SPG-N pair (spgn_partition_kernel / spgn_aggregate_kernel with DENSE, bodo_b200/csrc/spgn.cuh) against
a torch recomputation.

Each case checks every group's SUM and COUNT (or SIZE) bit for bit against torch.unique + index_add_ / bincount, and which form
ran: metric 17 counts dense launch pairs, metric 14 launch pairs of either SPG-N form.  The cases aim at the dense form's
window (chosen from the sample, with head room), the rows outside it (direct path, and the switch back to the hash form when
they are not rare), wraps of the 32-bit sum word, owner balance under strided keys and a bucket that overflows, every function
set, and the hash form's rare paths with the dense form turned off."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

ENVS = ("B200_SPG", "B200_SPG_NARROW", "B200_SPG_DENSE", "B200_SPG_HOT", "B200_LC")


def _owners():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


def _window(kmin, kmax):
    """GroupbyState::spgd_plan's key window for sampled keys in [kmin, kmax]: (kbase, KB)."""
    pad = (kmax - kmin) // 32
    kbase = 0 if 0 <= kmin <= pad else kmin - pad
    span = kmax - kbase + 1
    need = span + span // 32
    return kbase, max(1, (need - 1).bit_length())


def _unsampled(n):
    """Rows the sampler does not read (32 blocks of 1024 rows at b * n / 32); n is a multiple of 32 * 1024."""
    import torch
    return torch.arange(n, device="cuda") % (n // 32) >= 1024


def _args(funcs):
    if funcs == ("size",):
        return (0, 0), ()
    return tuple(range(len(funcs) + 1)), (1,) * len(funcs)


def _run(monkeypatch, batches, funcs=("sum", "count"), hint=0, env=None):
    """One groupby over the device (key, value) batches; checks the result and returns metrics 14 and 17."""
    import torch

    from bodo_b200.streaming.groupby import (delete_groupby_state, get_metric, groupby_build_consume_batch,
                                             groupby_produce_output_batch, init_groupby_state)
    from bodo_b200.table import Column, Table
    for name in ENVS:
        monkeypatch.delenv(name, raising=False)
    for name, val in (env or {}).items():
        monkeypatch.setenv(name, val)
    offs, cols = _args(funcs)
    st = init_groupby_state(-1, (0,), funcs, offs, cols, expected_groups=hint, output_batch_size=1 << 30)
    try:
        for i, (k, v) in enumerate(batches):
            groupby_build_consume_batch(st, Table([Column(k), Column(v)], ["k", "v"]), i == len(batches) - 1, True)
        m = (get_metric(st, 14), get_metric(st, 17))
        out, last = groupby_produce_output_batch(st, True)
        assert last
        got = [torch.as_tensor(c.data, device="cuda").clone() for c in out.columns]
    finally:
        delete_groupby_state(st)

    k = torch.cat([b[0] for b in batches])
    v = torch.cat([b[1] for b in batches])
    uniq, inv = torch.unique(k, return_inverse=True)
    cnt = torch.bincount(inv, minlength=len(uniq))
    ref = {"size": cnt, "count": cnt,
           "sum": torch.zeros(len(uniq), dtype=torch.int64, device="cuda").index_add_(0, inv, v)}  # wraps mod 2^64 like the kernels
    order = torch.argsort(got[0])
    assert len(got[0]) == len(uniq)
    assert torch.equal(got[0][order], uniq)
    for j, f in enumerate(funcs):
        assert torch.equal(got[1 + j][order].to(torch.int64), ref[f]), f
    return m


def _rand(n, lo, hi, seed):
    import torch
    g = torch.Generator(device="cuda").manual_seed(seed)
    return torch.randint(lo, hi, (n,), device="cuda", generator=g, dtype=torch.int64)


@pytest.mark.timeout(300)
@pytest.mark.parametrize("groups", [5_000, 1_000_000, 2_000_000])
def test_dense_flagship_shapes(gpu_lib, monkeypatch, groups):
    """bench.py's keys (synth: mix64 % groups) and values in [-500, 500); 2 M groups is near the widest window (2^21 keys), 5000
    groups a window of 2^13 keys and 63 slots per owner.  (Below ~2000 groups every key carries 1/1024 of the sample: heavy
    hitters, which the dense form leaves to the 16-byte pair, and below 1024 the low-cardinality kernel takes them.)"""
    import torch

    from bodo_b200 import synth
    n = 1 << 24
    k = torch.empty(n, dtype=torch.int64, device="cuda")
    v = torch.empty(n, dtype=torch.int64, device="cuda")
    synth.device_fill(k, v, 0, groups, 7, torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    assert int(k.min()) >= 0 and int(k.max()) < groups
    m = _run(monkeypatch, [(k, v)], hint=groups)
    assert m[1] >= 1 and m[0] >= m[1]


@pytest.mark.timeout(300)
@pytest.mark.parametrize("base", [-700_000, (1 << 31) - 500_000], ids=["negative", "near_int32_max"])
def test_dense_window_edges(gpu_lib, monkeypatch, base):
    """Keys base + [0, 500 k) in the sample; unsampled rows put keys exactly at the window's first and last key (dense; near
    INT32_MAX the last key of the window is beyond int32) and just outside it (direct path)."""
    import torch
    n = 1 << 23
    k = base + _rand(n, 0, 500_000, 31)
    k[0], k[1] = base, base + 499_999  # (row 0 and 1 are sampled: the sampled range is exactly [base, base + 500 k))
    v = _rand(n, -1000, 1000, 32)
    kbase, kb = _window(base, base + 499_999)
    un = torch.nonzero(_unsampled(n)).flatten()
    edges = torch.tensor([kbase, kbase + (1 << kb) - 1, kbase - 1, kbase + (1 << kb)], device="cuda", dtype=torch.int64)
    k[un[:4000]] = edges.repeat(1000)
    m = _run(monkeypatch, [(k, v)], hint=500_000)
    assert m[1] == 1


@pytest.mark.timeout(300)
def test_dense_wide_rows(gpu_lib, monkeypatch):
    """Rows outside the window (keys beyond it, values beyond the value window), none where the sampler looks.  A few of them in
    the first batch take the direct path and the next launch is dense again; more than 1/64 of the second batch switch the third
    batch back to the hash form."""
    import torch
    n, ng = 1 << 22, 1_000_000
    batches = []
    for b, share in enumerate((997, 16, 997)):
        k = _rand(n, 0, ng, 40 + b)
        v = _rand(n, -500, 500, 50 + b)
        idx = torch.arange(n, device="cuda")
        w = (idx % share == 5) & _unsampled(n)
        k[w & (idx % 3 == 0)] += 1 << 40
        k[w & (idx % 3 == 1)] = -1 - idx[w & (idx % 3 == 1)]
        v[w & (idx % 3 == 2)] = (1 << 40) + idx[w & (idx % 3 == 2)]
        batches.append((k, v))
    m = _run(monkeypatch, batches, hint=ng)
    assert m == (3, 2)


@pytest.mark.timeout(300)
def test_dense_sum_word_wraps(gpu_lib, monkeypatch):
    """5000 keys leave 26 bits of value offset (63 slots per owner); values spread over 2^26 put about 2^35 in each group's sum
    word per launch, so it wraps tens of times and K2d sends the carries to the global table."""
    n = 1 << 23
    k = _rand(n, 0, 5000, 60)
    v = _rand(n, -(1 << 25), 1 << 25, 61)
    m = _run(monkeypatch, [(k, v)], hint=5000)
    assert m[1] == 1


def _owner_of(d, kb, g):
    """Owners of key offsets d (uint64 array) in a window of 2^kb keys over g owners (spgd_scramble, then mod g)."""
    x = (d * np.uint64(0x9E3779B1)) & np.uint64((1 << kb) - 1)
    x ^= x >> np.uint64((kb + 1) // 2)
    return x % np.uint64(g)


@pytest.mark.timeout(300)
@pytest.mark.parametrize("shape", ["stride_owners", "stride_128", "stride_256", "sub_range", "one_owner"])
def test_dense_balance(gpu_lib, monkeypatch, shape):
    """Strided keys and a sub-range of the window spread over the owners; keys that all map to ONE owner overflow its bucket, and
    the rows past its end take the direct path (their key is rebuilt from the bucket word and the owner).  Rows draw from 4000
    or more keys, so that no key carries the 1/1024 of the sample that makes it a heavy hitter."""
    import torch
    g = _owners()
    n = 1 << 23
    if shape == "one_owner":
        kbase, kb = _window(0, 1_500_000)
        assert kbase == 0 and kb == 21
        d = np.arange(1, 1_500_000, dtype=np.uint64)
        pool = np.concatenate([[0], d[_owner_of(d, kb, g) == 0][:4000], [1_500_000]])
    elif shape == "sub_range":
        pool = np.concatenate([[0], np.arange(300_000, 500_000), [666_666]])  # the window is [0, 2^20)
    else:
        stride, count = {"stride_owners": (g, (1 << 20) // g), "stride_128": (128, 8000), "stride_256": (256, 4000)}[shape]
        pool = 1_000 + stride * np.arange(count)
    pool_t = torch.from_numpy(pool.astype(np.int64)).cuda()
    k = pool_t[_rand(n, 0, len(pool), 70)]
    k[1] = pool_t[-1]  # (row 1 is sampled: the sample sees the whole key range)
    v = _rand(n, -500, 500, 71)
    m = _run(monkeypatch, [(k, v)], hint=len(pool))
    assert m[1] == 1


@pytest.mark.timeout(300)
@pytest.mark.parametrize("funcs", [("sum",), ("count",), ("size",), ("count", "sum")])
def test_dense_signatures(gpu_lib, monkeypatch, funcs):
    """Every function set of the fast-path signature, fed as the reference's 32 768-row batches (they go through the coalescing
    buffer before the SM-partitioned pair sees them)."""
    n, ng = 1 << 22, 300_000
    k = _rand(n, 0, ng, 80)
    v = _rand(n, -500, 500, 81)
    step = 32768
    m = _run(monkeypatch, [(k[i:i + step], v[i:i + step]) for i in range(0, n, step)], funcs=funcs, hint=ng)
    assert m[1] >= 1


@pytest.mark.timeout(300)
def test_dense_not_for_nullable_values(gpu_lib, monkeypatch):
    """A value column with a validity bitmap is not the fast-path signature: the dense form does not run."""
    import torch

    from bodo_b200.streaming.groupby import (delete_groupby_state, get_metric, groupby_build_consume_batch,
                                             groupby_produce_output_batch, init_groupby_state)
    from bodo_b200.table import Column, Table
    for name in ENVS:
        monkeypatch.delenv(name, raising=False)
    n, ng = 1 << 22, 100_000
    k = _rand(n, 0, ng, 90)
    v = _rand(n, -500, 500, 91)
    valid = torch.full(((n + 7) // 8,), 0xEF, dtype=torch.uint8, device="cuda")  # every 8th row from 4 on is NA
    st = init_groupby_state(-1, (0,), ("sum", "count"), (0, 1, 2), (1, 1), expected_groups=ng, output_batch_size=1 << 30)
    try:
        groupby_build_consume_batch(st, Table([Column(k), Column(v, valid)], ["k", "v"]), True, True)
        assert get_metric(st, 17) == 0
        out, _ = groupby_produce_output_batch(st, True)
        got = [torch.as_tensor(c.data, device="cuda") for c in out.columns]
    finally:
        delete_groupby_state(st)
    ok = (torch.arange(n, device="cuda") % 8) != 4
    uniq, inv = torch.unique(k, return_inverse=True)
    s = torch.zeros(len(uniq), dtype=torch.int64, device="cuda").index_add_(0, inv[ok], v[ok])
    c = torch.bincount(inv[ok], minlength=len(uniq))
    order = torch.argsort(got[0])
    assert torch.equal(got[0][order], uniq)
    assert torch.equal(got[1][order].to(torch.int64), s)
    assert torch.equal(got[2][order].to(torch.int64), c)


@pytest.mark.timeout(600)
@pytest.mark.parametrize("case", ["near_capacity", "overfull_one_pass", "two_passes", "first_appearances_race", "wide_stragglers"])
def test_hash_form_rare_paths_with_dense_off(gpu_lib, monkeypatch, case):
    """The K2n rare-path cases of test_gpu_spgn_row_path.py, whose shapes now take the dense form, with B200_SPG_DENSE=0: the hash
    form runs them (metric 14, and metric 17 stays 0), so its second-bucket, stash and direct paths stay covered."""
    from bodo_b200.streaming import groupby as G
    from tests import test_gpu_spgn_row_path as rp
    seen = []
    real = G.get_metric

    def get_metric(st, which):
        if which == 14:
            seen.append(real(st, 17))
        return real(st, which)

    for name in ENVS:
        monkeypatch.delenv(name, raising=False)
    monkeypatch.setenv("B200_SPG_DENSE", "0")
    monkeypatch.setattr(G, "get_metric", get_metric)
    if case == "near_capacity":
        rp.test_spgn_near_and_over_capacity(gpu_lib, 0.95, 1.0)
    elif case == "overfull_one_pass":
        rp.test_spgn_near_and_over_capacity(gpu_lib, 1.3, 0.5)
    elif case == "two_passes":
        rp.test_spgn_two_passes(gpu_lib)
    elif case == "first_appearances_race":
        rp.test_spgn_first_appearances_race(gpu_lib)
    else:
        rp.test_spgn_wide_stragglers(gpu_lib)
    assert seen == [0]
