"""The full sort, the top-k and the window at their row caps, against exact references that never hold the input.

sort.cu states its limits as 32-bit row ids and positions: at most MAX_FULL_SORT_ROWS = 2^31 rows in a full sort or a window
(bit 31 of a row id carries a key's NA class; window positions, partition sizes and peer ends are uint32; RANGE bounds are
int2), K = limit + offset <= 2^26 in a top-k (store capacity max(2K, 4 Mi) rows), and 64-bit arrival indices.  The arms here
run each form at those limits on one H100 80GB; tests/test_sort_limits_reference_host.py holds the references and checks them
against brute force on the CPU:
  * every key cell is a hash of its row's arrival index, regenerated batch by batch on the device;
  * full sort and top-k: the payload r is the arrival index; SortChecker proves the output is the stable sort (r a
    permutation, every key cell its row's, adjacent rows strictly increasing in (NA class, key, r));
  * window: key-only inputs over INT16 / UINT8 keys, whose sorted key column and every function are closed forms of the key
    histogram (BinLayout), compared bit for bit.
Each arm trims the library's pool and torch's cache before and after it, and skips only when the device has less free memory
than it needs at its start.  Each prints its wall time and the largest drop in free device memory seen between library calls."""

import time

import pytest
import torch

from bodo_b200 import _lib
from bodo_b200._lib import B200Error
from bodo_b200.streaming import sort as S
from bodo_b200.streaming import window as W
from bodo_b200.table import ArrTypes, Column, CTypes, DeviceArray, Table
from tests.test_sort_limits_reference_host import (BinLayout, SortChecker, gen_float32, gen_int16, gen_int16_nullable, gen_int32_nullable,
                                                   gen_int64, gen_partition_uint8, gen_rising_float64, gen_s3, int16_bins, pack_validity,
                                                   stable_order, unpack_validity)

pytestmark = pytest.mark.gpu

GiB = 1 << 30
N31 = S.MAX_FULL_SORT_ROWS  # 2^31
BATCH = 1 << 28             # rows per consumed and per produced batch
CHECK = 1 << 26             # rows per reference step (its temporaries are a few GiB)


def _trim():
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    _lib.lib().b200_pool_trim(torch.cuda.current_device(), 0)


class _Meter:
    """Wall time and the lowest free device memory sampled between library calls, reported when the arm ends."""

    def __init__(self, name):
        self.name, self.t0 = name, time.perf_counter()
        self.free0 = self.low = torch.cuda.mem_get_info(0)[0]

    def sample(self):
        torch.cuda.synchronize()
        self.low = min(self.low, torch.cuda.mem_get_info(0)[0])

    def report(self):
        name = torch.cuda.get_device_name(0)
        print(f"\n[sort limits] {self.name}: {time.perf_counter() - self.t0:.1f} s, free memory {self.free0 / GiB:.1f} GiB at the start, "
              f"largest drop {(self.free0 - self.low) / GiB:.1f} GiB ({name})")


@pytest.fixture
def meter(request):
    _trim()
    m = _Meter(request.node.name)
    yield m
    _trim()
    m.report()


def _need(gib):
    free = torch.cuda.mem_get_info(0)[0]
    if free < gib * GiB:
        pytest.skip(f"needs {gib} GiB of free device memory (has {free / GiB:.1f} GiB)")


def _arrivals(r0, r1):
    return torch.arange(r0, r1, dtype=torch.int64, device="cuda")


def _nullable(x, valid, ct):
    return Column(x, pack_validity(valid), ct, ArrTypes.NULLABLE_INT_BOOL)


def _cell(c, dtype=None):
    """(values, validity or None) of a produced column as device tensors; dtype reinterprets the values' bits."""
    d = c.data if dtype is None else DeviceArray(c.data.ptr, c.data.length, dtype, c.data.device, c.data.owner)
    x = torch.as_tensor(d, device="cuda")
    v = None if c.validity is None else unpack_validity(torch.as_tensor(c.validity, device="cuda"), c.length)
    return x, v


def _consume(consume, st, batch, r0, r1, last, meter, step=BATCH):
    """Rows [r0, r1) in batches of `step`, the final one with is_last = last (torch's cache is emptied before it, so the sort's
    buffers have the memory)."""
    for b0 in range(r0, r1, step):
        b1 = min(r1, b0 + step)
        t = batch(b0, b1)
        if b1 == r1 and last:
            torch.cuda.empty_cache()
        consume(st, t, b1 == r1 and last)
        del t
        meter.sample()
    if last:
        _lib.lib().b200_pool_trim(0, 0)  # the sort's freed buffers, so the references below have the memory


def _produce(produce, st, meter):
    """Yields (first row, table) of every output batch."""
    r0 = 0
    while True:
        out, last = produce(st)
        meter.sample()
        yield r0, out
        r0 += out.n_rows
        if last:
            break


# ---- full sort ----
def _check_full_sort(st, n, gen, keys, key_dtypes, meter):
    """Every output batch through SortChecker; the payload r is the last output column."""
    ck = SortChecker(n, gen, keys, "cuda")
    for _, out in _produce(S.produce_output_batch, st, meter):
        cells = [_cell(c, dt) for c, dt in zip(out.columns, key_dtypes)]
        r = _cell(out.columns[-1])[0].to(torch.int64)
        for s0 in range(0, out.n_rows, CHECK):
            ck.feed([(x[s0:s0 + CHECK], None if v is None else v[s0:s0 + CHECK]) for x, v in cells], r[s0:s0 + CHECK])
        meter.sample()
    ck.finish()


@pytest.mark.timeout(1800)
def test_s1_full_sort_of_2_31_rows_and_the_refused_row(gpu_lib, meter):
    """n = 2^31 exactly: 128 chunks, row id 0x7FFFFFFF beside the NA-class bit, output positions up to 2^31 - 1.  A nullable
    INT32 key (1/8 NA, mostly [-500, 500) for ties, 1/16 over the full range so all four byte passes run), descending, NA
    first.  A 6-row is_last batch after 2^31 - 5 rows is refused before anything is appended, and the state takes the last
    5 rows afterwards."""
    _need(60)
    n = N31

    def batch(r0, r1):
        i = _arrivals(r0, r1)
        v, ok = gen_int32_nullable(i)
        return Table([_nullable(v, ok, CTypes.INT32), Column(i.to(torch.int32), None, CTypes.INT32)], ["k", "r"])

    st = S.init_stream_sort_state(-1, None, 0, ["k"], [False], ["first"], ["k", "r"], output_batch_size=BATCH, full=True)
    try:
        _consume(S.sort_build_consume_batch, st, batch, 0, n - 5, False, meter)
        six = Table([_nullable(torch.zeros(6, dtype=torch.int32, device="cuda"), torch.ones(6, dtype=torch.bool, device="cuda"), CTypes.INT32),
                     Column(torch.zeros(6, dtype=torch.int32, device="cuda"), None, CTypes.INT32)], ["k", "r"])
        with pytest.raises(B200Error, match=r"at most 2\^31 rows"):
            S.sort_build_consume_batch(st, six, True)
        assert S.get_metric(st, 0) == n - 5
        _consume(S.sort_build_consume_batch, st, batch, n - 5, n, True, meter)
        m = [S.get_metric(st, w) for w in range(9)]
        assert m[0] == m[6] == n and m[1:6] == [0] * 5
        assert (m[7], m[8]) == (5, 0), m  # 4 byte passes and the NA-class pass
        _check_full_sort(st, n, lambda r: [gen_int32_nullable(r)], [(False, False)], [None], meter)
    finally:
        S.delete_stream_sort_state(st)


@pytest.mark.timeout(1800)
def test_s2_full_sort_of_float32_specials_at_2_31_minus_1_rows(gpu_lib, meter):
    """n = 2^31 - 1 of a numpy FLOAT32 key ascending, NaN last: -0.0 ties 0.0 in arrival order, NaNs (both signs, quiet and
    signalling payloads) form the NA class with their bits kept, +-inf and subnormals in place."""
    _need(56)
    n = N31 - 1

    def batch(r0, r1):
        i = _arrivals(r0, r1)
        return Table([Column(gen_float32(i), None, CTypes.FLOAT32), Column(i.to(torch.int32), None, CTypes.INT32)], ["k", "r"])

    st = S.init_stream_sort_state(-1, None, 0, ["k"], [True], ["last"], ["k", "r"], output_batch_size=BATCH, full=True)
    try:
        _consume(S.sort_build_consume_batch, st, batch, 0, n, True, meter)
        assert S.get_metric(st, 0) == n and S.get_metric(st, 6) == N31
        assert (S.get_metric(st, 7), S.get_metric(st, 8)) == (5, 0)
        _check_full_sort(st, n, lambda r: [(gen_float32(r), None)], [(True, True)], [None], meter)
    finally:
        S.delete_stream_sort_state(st)


@pytest.mark.timeout(1800)
def test_s3_two_keys_past_2_30_rows(gpu_lib, meter):
    """n = 2^30 + 4097 by (INT64 descending, UINT16 ascending): the 8-byte word buffers pass 2^33 bytes, and the second key's
    words are read through the permutation (FS_IN_GATHER) at more than 2^30 rows."""
    _need(48)
    n = (1 << 30) + 4097

    def batch(r0, r1):
        i = _arrivals(r0, r1)
        a, b = gen_s3(i)
        return Table([Column(a, None, CTypes.INT64), Column(b, None, CTypes.UINT16), Column(i.to(torch.int32), None, CTypes.INT32)],
                     ["a", "b", "r"])

    def gen(r):  # the UINT16 key as its unsigned value
        a, b = gen_s3(r)
        return [(a, None), (b.to(torch.int64) & 0xFFFF, None)]

    st = S.init_stream_sort_state(-1, None, 0, ["a", "b"], [False, True], ["last", "last"], ["a", "b", "r"], output_batch_size=BATCH,
                                  full=True)
    try:
        _consume(S.sort_build_consume_batch, st, batch, 0, n, True, meter, step=(1 << 28) - 3)
        assert S.get_metric(st, 0) == n and (S.get_metric(st, 7), S.get_metric(st, 8)) == (10, 0)
        ck = SortChecker(n, gen, [(False, True), (True, True)], "cuda")
        for _, out in _produce(S.produce_output_batch, st, meter):
            a = _cell(out.columns[0])[0]
            b = _cell(out.columns[1], "int16")[0].to(torch.int64) & 0xFFFF
            r = _cell(out.columns[2])[0].to(torch.int64)
            for s0 in range(0, out.n_rows, CHECK):
                s1 = s0 + CHECK
                ck.feed([(a[s0:s1], None), (b[s0:s1], None)], r[s0:s1])
        ck.finish()
    finally:
        S.delete_stream_sort_state(st)


# ---- top-k ----
def _run_topk(st, n, batch, meter, step):
    _consume(S.sort_build_consume_batch, st, batch, 0, n, True, meter, step=step)
    outs = [(_cell(out.columns[0]), _cell(out.columns[1])[0]) for _, out in _produce(S.produce_output_batch, st, meter)]
    k = torch.cat([o[0][0] for o in outs])
    v = None if outs[0][0][1] is None else torch.cat([o[0][1] for o in outs])
    r = torch.cat([o[1] for o in outs]).to(torch.int64)
    return k, v, r


@pytest.mark.timeout(1200)
def test_t1_topk_at_the_limit_cap(gpu_lib, meter):
    """limit = 2^26 (the cap), offset 0, over 2^28 + 3 arbitrary INT64 keys in batches that are not tile multiples: the store
    holds cap = 2K = 2^27 rows and its merge passes cut every run at K.  The reference is torch's stable sort of the keys."""
    _need(32)
    n, K = (1 << 28) + 3, S.MAX_LIMIT_PLUS_OFFSET
    keys = gen_int64(_arrivals(0, n))

    def batch(r0, r1):
        return Table([Column(keys[r0:r1], None, CTypes.INT64), Column(_arrivals(r0, r1).to(torch.int32), None, CTypes.INT32)], ["k", "r"])

    st = S.init_stream_sort_state(-1, K, 0, ["k"], [True], ["last"], ["k", "r"], output_batch_size=BATCH)
    try:
        k, _, r = _run_topk(st, n, batch, meter, step=3 * (1 << 24) + 5)
        assert S.get_metric(st, 6) == 2 * K and S.get_metric(st, 0) == n
        idx = torch.sort(keys, stable=True).indices[:K]
        meter.sample()
        assert r.numel() == K and torch.equal(r, idx)
        assert torch.equal(k, keys[idx])
    finally:
        S.delete_stream_sort_state(st)


@pytest.mark.timeout(1200)
def test_t2_topk_every_row_a_candidate(gpu_lib, meter):
    """limit = 2^26 - 12345, offset 12345 over 2^28 rows of a nullable FLOAT64 key that rises with arrival, descending with NA
    first (NaN and NA rows, 2 in 97, form the first class; -0.0 ties 0.0 in the output): every row is a candidate, so the
    store of 2^27 rows overflows and is reduced again and again."""
    _need(32)
    n, off = 1 << 28, 12345
    K = S.MAX_LIMIT_PLUS_OFFSET
    x, ok = gen_rising_float64(_arrivals(0, n), n, K)

    def batch(r0, r1):
        return Table([_nullable(x[r0:r1], ok[r0:r1], CTypes.FLOAT64), Column(_arrivals(r0, r1).to(torch.int32), None, CTypes.INT32)],
                     ["k", "r"])

    st = S.init_stream_sort_state(-1, K - off, off, ["k"], [False], ["first"], ["k", "r"], output_batch_size=BATCH)
    try:
        k, v, r = _run_topk(st, n, batch, meter, step=(1 << 24) + 1)
        assert S.get_metric(st, 2) >= 3 and S.get_metric(st, 1) == n, [S.get_metric(st, w) for w in range(7)]
        idx = stable_order([(x, ok)], [(False, False)])[off:K]
        meter.sample()
        assert r.numel() == K - off and torch.equal(r, idx)
        assert torch.equal(k.view(torch.int64), x[idx].view(torch.int64)) and torch.equal(v, ok[idx])
        assert bool((k.view(torch.int64) == -(1 << 63)).any()) and bool((~v).any()) and bool(torch.isnan(k).any())
    finally:
        S.delete_stream_sort_state(st)


@pytest.mark.timeout(1800)
def test_t3_topk_ties_decided_past_2_32_arrivals(gpu_lib, meter):
    """2^32 + 2^24 rows of an INT8 key that is 1 except for seven 0s, four of them at and after arrival 2^32 - 1; limit 1000,
    offset 3, INT64 payload r = arrival index.  The ties are decided by 64-bit arrival indices: the result is the 0-rows after
    the first three in arrival order, then the earliest 1-rows."""
    _need(16)
    n = (1 << 32) + (1 << 24)
    zeros = [5, 9, (1 << 31) + 3, (1 << 32) - 1, 1 << 32, (1 << 32) + 1, n - 1]

    def batch(r0, r1):
        k = torch.ones(r1 - r0, dtype=torch.int8, device="cuda")
        for z in zeros:
            if r0 <= z < r1:
                k[z - r0] = 0
        return Table([Column(k, None, CTypes.INT8), Column(_arrivals(r0, r1), None, CTypes.INT64)], ["k", "r"])

    st = S.init_stream_sort_state(-1, 1000, 3, ["k"], [True], ["last"], ["k", "r"], output_batch_size=BATCH)
    try:
        k, _, r = _run_topk(st, n, batch, meter, step=BATCH)
        assert S.get_metric(st, 0) == n
        ones = [i for i in range(1100) if i not in zeros][:996]
        assert r.tolist() == zeros[3:] + ones
        assert k.tolist() == [0] * 4 + [1] * 996
    finally:
        S.delete_stream_sort_state(st)


# ---- window ----
def _window_hist(n, flat_of, bins, meter):
    """Histogram of flat bin indices over all n rows, regenerated batch by batch."""
    cnt = torch.zeros(bins, dtype=torch.int64, device="cuda")
    for r0 in range(0, n, BATCH):
        cnt += torch.bincount(flat_of(_arrivals(r0, min(n, r0 + BATCH))), minlength=bins)
    meter.sample()
    return cnt


@pytest.mark.timeout(2400)
@pytest.mark.parametrize("funcs", [[("rn", "row_number"), ("rk", "rank")], [("dr", "dense_rank"), ("pr", "percent_rank")],
                                   [("cd", "cume_dist"), ("nt", "ntile", 7)]], ids=["rn_rank", "dense_pct", "cume_ntile"])
def test_w1_ranking_over_one_partition_of_2_31_rows(gpu_lib, meter, funcs):
    """n = 2^31 rows in one partition (no PARTITION BY), ORDER BY INT16 descending: positions and the partition size reach
    2^31 - 1 and 2^31 in uint32, and the carry scan over 2^20 tiles gives each thread 1,024 of them.  Two functions per state
    (each function column is 16 GiB at this size)."""
    _need(68)
    n = N31

    def batch(r0, r1):
        return Table([Column(gen_int16(_arrivals(r0, r1), 10), None, CTypes.INT16)], ["o"])

    cnt = _window_hist(n, lambda i: gen_int16(i, 10).to(torch.int64) + 32768, 65536, meter)
    lay = BinLayout(*int16_bins(cnt, descending=True), 65536)
    st = W.init_window_state(-1, [], ["o"], [False], ["last"], funcs, ["o"], output_batch_size=BATCH)
    try:
        _consume(W.window_build_consume_batch, st, batch, 0, n, True, meter)
        assert W.get_metric(st, 0) == n and W.get_metric(st, 9) == 1
        for r0, out in _produce(W.window_produce_output_batch, st, meter):
            o = _cell(out.columns[0])[0]
            fs = [_cell(c)[0] for c in out.columns[1:]]
            for s0 in range(0, out.n_rows, CHECK):
                s1 = min(out.n_rows, s0 + CHECK)
                i = _arrivals(r0 + s0, r0 + s1)
                assert torch.equal(o[s0:s1], lay.sorted_values(i).to(torch.int16))
                for f, got in zip(funcs, fs):
                    exp = lay.ranking(i, f[1], f[2] if len(f) > 2 else None)
                    assert torch.equal(got[s0:s1].view(torch.int64), exp.view(torch.int64)), (f, r0 + s0)
    finally:
        W.delete_window_state(st)


@pytest.mark.timeout(1800)
def test_w2_rows_frame_sum_of_2_31_rows_over_a_2_30_row_reach(gpu_lib, meter):
    """n = 2^31, PARTITION BY UINT8 (one partition of ~3/4 of the rows, a single-row one, the rest spread over 1..254), ORDER BY
    INT16: SUM(o) over ROWS BETWEEN 2^30 PRECEDING AND 5 FOLLOWING.  The frame tree takes all three launches (levels up to 31)
    and frames of 2^30 + 6 rows read its top levels; the reference is a prefix sum read off the histogram."""
    _need(66)
    n, single = N31, 1_234_567_891

    def batch(r0, r1):
        i = _arrivals(r0, r1)
        return Table([Column(gen_partition_uint8(i, single), None, CTypes.UINT8), Column(gen_int16(i, 14), None, CTypes.INT16)], ["p", "o"])

    cnt = _window_hist(n, lambda i: gen_partition_uint8(i, single).to(torch.int64) * 65536 + gen_int16(i, 14).to(torch.int64) + 32768,
                       256 * 65536, meter)
    val = torch.arange(-32768, 32768, dtype=torch.int64, device="cuda").repeat(256)
    lay = BinLayout(cnt, val, 65536)
    parts = cnt.view(256, 65536).sum(1)
    assert int(parts[0]) > 1 << 30 and int(parts[255]) == 1
    st = W.init_window_state(-1, ["p"], ["o"], [True], ["last"], [("s", "sum", "o", ("rows", -(1 << 30), 5))], ["p", "o"],
                             output_batch_size=BATCH)
    try:
        _consume(W.window_build_consume_batch, st, batch, 0, n, True, meter)
        assert W.get_metric(st, 9) == int((parts > 0).sum())
        for r0, out in _produce(W.window_produce_output_batch, st, meter):
            p, o = _cell(out.columns[0])[0], _cell(out.columns[1])[0]
            s, sv = _cell(out.columns[2])
            for s0 in range(0, out.n_rows, CHECK):
                s1 = min(out.n_rows, s0 + CHECK)
                i = _arrivals(r0 + s0, r0 + s1)
                b = lay.bin_of(i)
                assert torch.equal(p[s0:s1].to(torch.int64), b // 65536) and torch.equal(o[s0:s1], lay.val[b].to(torch.int16))
                assert torch.equal(s[s0:s1], lay.rows_sum(i, -(1 << 30), 5)), r0 + s0
                assert bool(sv[s0:s1].all())
    finally:
        W.delete_window_state(st)


@pytest.mark.timeout(1800)
def test_w3_range_frame_count_with_empty_frames_at_row_2_31(gpu_lib, meter):
    """n = 2^31, ORDER BY a nullable INT16 ascending NA last: COUNT(*) over RANGE BETWEEN 1 FOLLOWING AND 3 FOLLOWING.  The
    largest non-NA value's frames are empty with their start at the first NA row or at row 2^31 itself (the search for
    o + 1 runs past every non-NA row); a FOLLOWING bound never reaches an NA row, and an NA row's frame is the NA peer group,
    which ends the input."""
    _need(70)
    n = N31

    def batch(r0, r1):
        v, ok = gen_int16_nullable(_arrivals(r0, r1))
        return Table([_nullable(v, ok, CTypes.INT16)], ["o"])

    def flat(i):
        v, ok = gen_int16_nullable(i)
        return torch.where(ok, v.to(torch.int64) + 32768, 65536)

    cnt = _window_hist(n, flat, 65537, meter)
    lay = BinLayout(cnt, torch.arange(-32768, 32769, dtype=torch.int64, device="cuda"), 65537)
    n_na = int(cnt[65536])
    st = W.init_window_state(-1, [], ["o"], [True], ["last"], [("c", "count", None, ("range_between", 1, 3))], ["o"],
                             output_batch_size=BATCH)
    try:
        _consume(W.window_build_consume_batch, st, batch, 0, n, True, meter)
        empty = 0
        for r0, out in _produce(W.window_produce_output_batch, st, meter):
            o, ov = _cell(out.columns[0])
            c = _cell(out.columns[1])[0]
            for s0 in range(0, out.n_rows, CHECK):
                s1 = min(out.n_rows, s0 + CHECK)
                i = _arrivals(r0 + s0, r0 + s1)
                b = lay.bin_of(i)
                assert torch.equal(ov[s0:s1], b != 65536)
                assert torch.equal(o[s0:s1][b != 65536], lay.val[b][b != 65536].to(torch.int16))
                exp = lay.range_count_following(i, 1, 3, 65536)
                assert torch.equal(c[s0:s1], exp), r0 + s0
                empty += int((exp == 0).sum())
        assert empty > 0 and n_na > 0
    finally:
        W.delete_window_state(st)
