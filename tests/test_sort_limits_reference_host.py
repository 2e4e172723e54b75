"""The exact references of tests/test_gpu_sort_limits.py, and their own checks against brute force on the CPU.

The sort operators' caps (2^31 rows for the full sort and the window, K = limit + offset = 2^26 and arrival indices past 2^32
for the top-k) are too large for a reference that keeps the input or sorts it a second time.  So every key cell is a
deterministic integer hash of its row's arrival index, regenerated whenever it is needed, and the result is checked in
batches with O(n) memory:
  * full sort and top-k: the payload r is the arrival index.  A sorted output is exactly the stable sort when r is a
    permutation of [0, n) (SortChecker's seen array), every key cell equals the generator's cell at r (bits and validity), and
    adjacent rows strictly increase in (NA class, key in its direction, ..., r);
  * window over narrow keys (INT16 values, a UINT8 partition key): the sorted key column is fully determined by the key
    histogram, and every function has a closed form in the cumulative histogram (BinLayout).
Every function here is plain torch integer / float64 arithmetic and runs on CPU tensors as well as on the device; the tests
below compare it with numpy's stable sort and direct loops at n <= 10^5."""

import numpy as np
import pytest
import torch

# ---- generators: key cells as a function of the arrival index ----
_M32 = 0xFFFFFFFF


def mix32(x):
    """A 32-bit integer hash (two xorshift-multiply rounds); x: int64 in [0, 2^32).  Products stay below 2^59, so no int64
    arithmetic wraps on any device."""
    x = (((x >> 16) ^ x) * 0x45D9F3B) & _M32
    x = (((x >> 16) ^ x) * 0x45D9F3B) & _M32
    return (x >> 16) ^ x


def hash32(i, salt):
    """int64 in [0, 2^32) from a non-negative int64 arrival index (any size) and a salt."""
    return mix32(mix32((i & _M32) ^ ((salt * 0x9E3779B1) & _M32)) ^ (i >> 32))


def to_int32(u):
    """[0, 2^32) int64 -> the int32 with those bits."""
    return torch.where(u >= 1 << 31, u - (1 << 32), u).to(torch.int32)


def gen_int32_nullable(i):
    """S1's key: ~1/8 NA, ~15/16 of the rest in [-500, 500) (heavy ties), 1/16 over the full int32 range (every byte digit
    varies).  NA cells keep their value bits, which the sort must carry through.  -> (int32 bits, valid)."""
    h = hash32(i, 1)
    wide = ((h >> 3) & 15) == 0
    v = torch.where(wide, hash32(i, 2) - (1 << 31), (h >> 7) % 1000 - 500)
    return v.to(torch.int32), (h & 7) != 0


_F32_SPECIAL = [0x7FC00000, 0xFFC00001, 0x7F800001, 0x80000000, 0x00000000, 0x7F800000, 0xFF800000, 0x00000001, 0x807FFFFF,
                0x00400000]


def gen_float32(i):
    """S2's key: 1/4 of the cells from a list of specials (quiet and signalling NaNs of both signs, -0.0, 0.0, +-inf,
    subnormals of both signs), 1/4 small integers (ties, 0.0 among them), the rest arbitrary 32-bit patterns (more NaNs, infs
    and subnormals included).  -> float32 tensor."""
    h = hash32(i, 3)
    sel = h & 3
    special = torch.tensor(_F32_SPECIAL, dtype=torch.int64, device=i.device)[(h >> 2) % len(_F32_SPECIAL)]
    small = to_int32(((h >> 2) % 64) - 32).to(torch.float32).view(torch.int32).to(torch.int64) & _M32
    bits = torch.where(sel == 0, special, torch.where(sel == 1, small, hash32(i, 4)))
    return to_int32(bits).view(torch.float32)


def gen_s3(i):
    """S3's keys: an INT64 with 4096 distinct values that differ in every byte (heavy ties), and a UINT16 (as int16 bits) that
    breaks most of them.  -> (int64, int16)."""
    h = hash32(i, 5)
    k0 = ((h % 4096) - 2048) * 0x0101010101
    u = hash32(i, 6) & 0xFFFF
    return k0, torch.where(u >= 1 << 15, u - (1 << 16), u).to(torch.int16)


def gen_int64(i):
    """T1's key: arbitrary int64 values."""
    return (hash32(i, 7) - (1 << 31)) * (1 << 32) + hash32(i, 8)


def gen_rising_float64(i, n, K):
    """T2's key: float64 (i // 3) - ((n - K // 2) // 3), so that every row sorts above every earlier one in descending order,
    with 1 row in 97 NA (validity 0) and 1 in 97 a NaN (valid), and the row of each equal triple with i % 3 == 1 a -0.0 where
    the value is 0.  -> (float64, valid)."""
    h = hash32(i, 9) % 97
    v = (i // 3 - (n - K // 2) // 3).to(torch.float64)
    v = torch.where(h == 1, float("nan"), v)
    v = torch.where((v == 0) & (i % 3 == 1), -0.0, v)
    return v, h != 0


def gen_int16(i, salt, wide_every=4):
    """A window ORDER BY key: 1 cell in `wide_every` over the full int16 range, the rest in [-50, 50] (heavy ties).  -> int16."""
    h = hash32(i, salt)
    wide = (h & (wide_every - 1)) == 0
    v = torch.where(wide, (h >> 8) % 65536 - 32768, (h >> 8) % 101 - 50)
    return v.to(torch.int16)


def gen_partition_uint8(i, single=None):
    """W2's PARTITION BY key: 0 for ~3/4 of the rows (one partition of more than 2^30 rows at n = 2^31), else 1..254, and 255
    only at row `single` (a single-row partition).  -> uint8."""
    h = hash32(i, 11)
    p = torch.where((h & 3) != 0, 0, (h >> 2) % 254 + 1)
    if single is not None:
        p = torch.where(i == single, 255, p)
    return p.to(torch.uint8)


def gen_int16_nullable(i):
    """W3's ORDER BY key: gen_int16 with 1 cell in 16 NA.  -> (int16, valid)."""
    return gen_int16(i, 12), (hash32(i, 13) & 15) != 0


# ---- bitmaps ----
def pack_validity(valid):
    """bool tensor -> Arrow validity bitmap (uint8, bit k of byte j is row 8 j + k)."""
    n = valid.numel()
    pad = torch.zeros((n + 7) // 8 * 8, dtype=torch.uint8, device=valid.device)
    pad[:n] = valid.to(torch.uint8)
    w = torch.tensor([1, 2, 4, 8, 16, 32, 64, 128], dtype=torch.uint8, device=valid.device)
    return (pad.view(-1, 8) * w).sum(1, dtype=torch.int64).to(torch.uint8)


def unpack_validity(bitmap, n):
    sh = torch.arange(8, dtype=torch.uint8, device=bitmap.device)
    return ((bitmap[: (n + 7) // 8].unsqueeze(1) >> sh) & 1).flatten()[:n].bool()


# ---- full sort and top-k: order words and the batch checker ----
def order_word(x):
    """An int64 that orders as the sort orders valid key cells: integers as themselves (unsigned ones given as their value),
    floats by value with -0.0 equal to 0.0 (NaN cells are NA and take word 0)."""
    if x.dtype in (torch.float32, torch.float64):
        b = (x.view(torch.int32) if x.dtype == torch.float32 else x.view(torch.int64)).to(torch.int64)
        low = (1 << 31) - 1 if x.dtype == torch.float32 else (1 << 63) - 1
        neg_zero = -(1 << 31) if x.dtype == torch.float32 else -(1 << 63)
        b = torch.where(b == neg_zero, 0, b)
        return torch.where(torch.isnan(x), 0, torch.where(b >= 0, b, b ^ low))
    return x.to(torch.int64)


def na_of(x, valid):
    """NA flags of key cells: invalid, or a float NaN."""
    na = torch.zeros(x.shape, dtype=torch.bool, device=x.device) if valid is None else ~valid
    if x.dtype in (torch.float32, torch.float64):
        na = na | torch.isnan(x)
    return na


def sort_columns(x, valid, asc, na_last):
    """The (NA class, order word) columns of one key, with the word's direction: compared lexicographically with the other
    keys' and the arrival index, they give the stable sort's order.  The NA class is 1 for NA rows with na_last, else 0 (the
    other rows the opposite), and NA rows all take word 0."""
    na = na_of(x, valid)
    cls = (na if na_last else ~na).to(torch.int64)
    return [(cls, True), (torch.where(na, 0, order_word(x)), asc)]


def strictly_increasing(cols):
    """cols: [(int64 tensor, ascending)], all of one length m >= 1.  Whether row j < row j + 1 lexicographically for every j,
    each column compared in its direction."""
    if cols[0][0].numel() < 2:
        return True
    less = torch.zeros(cols[0][0].numel() - 1, dtype=torch.bool, device=cols[0][0].device)
    eq = ~less
    for c, asc in cols:
        a, b = c[:-1], c[1:]
        less |= eq & ((a < b) if asc else (a > b))
        eq &= a == b
    return bool(less.all())


class SortChecker:
    """Checks a sorted output, batch by batch, against the generator: the payload r of the output rows is a permutation of
    [0, n) (every entry of a seen array set exactly once), every key cell equals the generator's at r, and adjacent rows
    (across batch edges too) strictly increase in (NA class_0, key_0, ..., r).

    gen(r) -> [(cells, valid or None)] per key; keys: [(asc, na_last)] per key."""

    def __init__(self, n, gen, keys, device):
        self.n, self.gen, self.keys = n, gen, keys
        self.seen = torch.zeros(n, dtype=torch.bool, device=device)
        self.rows = 0
        self.prev = None  # the last row of the previous batch: ([(cells, valid)], r)

    def feed(self, cells, r):
        """cells: [(cells, valid or None)] per key as produced, r: int64 arrival indices, all of one batch."""
        m = r.numel()
        if m == 0:
            return
        assert int(r.min()) >= 0 and int(r.max()) < self.n
        assert not bool(self.seen[r].any()), "an arrival index is produced twice"
        self.seen[r] = True
        self.rows += m
        exp = self.gen(r)
        for (x, v), (ex, ev) in zip(cells, exp):
            assert x.dtype == ex.dtype and torch.equal(bits_of(x), bits_of(ex)), "a key cell's bits differ from its row's"
            assert (v is None) == (ev is None) and (v is None or torch.equal(v, ev)), "a key cell's validity differs from its row's"
        if self.prev is not None:
            pc, pr = self.prev
            cells = [(torch.cat([a[0][-1:], b[0]]), None if b[1] is None else torch.cat([a[1][-1:], b[1]])) for a, b in zip(pc, cells)]
            r = torch.cat([pr[-1:], r])
        self.prev = ([(x[-1:], None if v is None else v[-1:]) for x, v in cells], r[-1:])
        cols = []
        for (x, v), (asc, na_last) in zip(cells, self.keys):
            cols += sort_columns(x, v, asc, na_last)
        assert strictly_increasing(cols + [(r, True)]), "adjacent output rows are out of order"

    def finish(self):
        assert self.rows == self.n and bool(self.seen.all())


def bits_of(x):
    return x.view({1: torch.uint8, 2: torch.int16, 4: torch.int32, 8: torch.int64}[x.element_size()])


def stable_order(cells, keys):
    """The stable sort's permutation of every row of small inputs (the top-k reference): torch's stable sorts, least
    significant column first."""
    cols = []
    for (x, v), (asc, na_last) in zip(cells, keys):
        cols += sort_columns(x, v, asc, na_last)
    idx = torch.arange(cols[0][0].numel(), device=cols[0][0].device)
    for c, asc in reversed(cols):
        idx = idx[torch.sort(c[idx], descending=not asc, stable=True).indices]
    return idx


# ---- window: closed forms from the key histogram ----
class BinLayout:
    """The sorted rows of a key-only window input as runs of equal keys ("bins", in sorted order): cnt[b] rows of bin b, whose
    ORDER BY value is val[b] (the NA bin's is unused) and whose partition is b // part_bins (part_bins bins per partition, so
    every partition is a contiguous range of bins; empty bins hold no rows).  A bin is one peer group."""

    def __init__(self, cnt, val, part_bins):
        self.cnt, self.val, self.W = cnt.to(torch.int64), val.to(torch.int64), part_bins
        self.incl = torch.cumsum(self.cnt, 0)
        self.excl = self.incl - self.cnt
        self.nz_incl = torch.cumsum((self.cnt > 0).to(torch.int64), 0)
        self.nz_excl = self.nz_incl - (self.cnt > 0).to(torch.int64)
        self.sum_incl = torch.cumsum(self.cnt * self.val, 0)  # exact in int64 for |val| < 2^15, n <= 2^31

    def bin_of(self, i):
        """The bin of sorted positions i (0 <= i < n)."""
        return torch.searchsorted(self.incl, i, right=True)

    def part(self, b):
        """(P, s): first position and size of bin b's partition."""
        f = b // self.W * self.W
        last = f + self.W - 1
        return self.excl[f], self.incl[last] - self.excl[f]

    def prefix_sum(self, x):
        """Sum of the ORDER BY values of sorted positions [0, x), 0 <= x <= n."""
        b = torch.searchsorted(self.incl, x)  # the first bin with incl >= x: excl[b] <= x <= incl[b]
        return self.sum_incl[b] - self.cnt[b] * self.val[b] + (x - self.excl[b]) * self.val[b]

    def sorted_values(self, i):
        return self.val[self.bin_of(i)]

    def ranking(self, i, fname, arg=None):
        """ROW_NUMBER / RANK / DENSE_RANK / PERCENT_RANK / CUME_DIST / NTILE(arg) at sorted positions i: int64 or float64,
        each float one IEEE double division of two integers, as the library computes it."""
        b = self.bin_of(i)
        P, s = self.part(b)
        pos, rank = i - P, self.excl[b] - P + 1
        if fname == "row_number":
            return pos + 1
        if fname == "rank":
            return rank
        if fname == "dense_rank":
            f = b // self.W * self.W
            return self.nz_excl[b] - self.nz_excl[f] + 1
        if fname == "percent_rank":
            return torch.where(s == 1, 0.0, (rank - 1).to(torch.float64) / torch.clamp(s - 1, min=1).to(torch.float64))
        if fname == "cume_dist":
            return (self.incl[b] - P).to(torch.float64) / s.to(torch.float64)
        assert fname == "ntile"
        q, r = s // arg, s % arg
        big = r * (q + 1)
        return torch.where(pos < big, pos // (q + 1) + 1, r + (pos - big) // torch.clamp(q, min=1) + 1)

    def rows_sum(self, i, start, end):
        """SUM(o) OVER (ROWS BETWEEN -start PRECEDING AND end FOLLOWING) at sorted positions i (start <= 0 <= end): the frame
        [max(P, i + start), min(pe - 1, i + end)] always holds row i, so it is never empty."""
        P, s = self.part(self.bin_of(i))
        lo = torch.maximum(P, i + start)
        hi = torch.minimum(P + s - 1, i + end)
        return self.prefix_sum(hi + 1) - self.prefix_sum(lo)

    def range_count_following(self, i, k0, k1, na_bin):
        """COUNT(*) OVER (ORDER BY o ASC NULLS LAST RANGE BETWEEN k0 FOLLOWING AND k1 FOLLOWING) at sorted positions i, one
        partition whose bins are the ascending values (val[b] increasing) and then the NA bin `na_bin`: at a non-NA row the rows
        with o in [o_i + k0, o_i + k1], at an NA row its peer group (every NA row)."""
        b = self.bin_of(i)
        vals = self.val[:na_bin]
        lo_b = torch.searchsorted(vals, self.val[b] + k0)           # first bin with value >= o + k0
        hi_b = torch.searchsorted(vals, self.val[b] + k1, right=True)  # first bin with value > o + k1
        return torch.where(b == na_bin, self.cnt[na_bin], self.excl[hi_b] - self.excl[lo_b])


def int16_bins(counts, descending=False):
    """(cnt, val) of the 65536 INT16 values in sorted order, from counts indexed by value + 32768."""
    val = torch.arange(-32768, 32768, dtype=torch.int64, device=counts.device)
    return (counts.flip(0), val.flip(0)) if descending else (counts, val)


# ================= checks of the references against brute force =================
def _i(n):
    return torch.arange(n, dtype=torch.int64)


def test_hash_is_deterministic_and_spreads():
    i = _i(100_000)
    h = hash32(i, 1)
    assert torch.equal(h, hash32(i, 1)) and not torch.equal(h, hash32(i, 2))
    assert int(h.min()) >= 0 and int(h.max()) < 1 << 32
    assert torch.unique(h).numel() > 99_000
    # indices past 2^32 differ from their low 32 bits
    big = i + (1 << 32)
    assert not torch.equal(hash32(big, 1), h)
    assert torch.equal(hash32(big, 1)[:5], hash32(torch.tensor([1 << 32, (1 << 32) + 1, (1 << 32) + 2, (1 << 32) + 3, (1 << 32) + 4]), 1))


def test_generators_cover_their_edges():
    i = _i(100_000)
    v, ok = gen_int32_nullable(i)
    assert 0.1 < float((~ok).double().mean()) < 0.15
    assert int(v.min()) < -(1 << 30) and int(v.max()) > 1 << 30  # full range
    assert int(((v >= -500) & (v < 500)).sum()) > 80_000  # ties
    f = gen_float32(i)
    b = f.view(torch.int32)
    assert bool(torch.isnan(f).any()) and bool((b == -(1 << 31)).any()) and bool((b == 0).any())
    assert bool(torch.isposinf(f).any()) and bool(torch.isneginf(f).any())
    sub = (f != 0) & (f.abs() < torch.finfo(torch.float32).tiny)
    assert bool((sub & (f > 0)).any()) and bool((sub & (f < 0)).any())
    nan_bits = torch.unique(b[torch.isnan(f)])
    assert nan_bits.numel() > 3  # NaN payloads of both signs
    k0, k1 = gen_s3(i)
    assert torch.unique(k0).numel() == 4096 and k1.dtype == torch.int16 and torch.unique(k1).numel() > 50_000
    w = k0.numpy().view(np.uint8).reshape(-1, 8)
    assert all(len(np.unique(w[:, j])) > 1 for j in range(8))  # every byte digit varies
    n, K = 100_000, 30_000
    x, ok = gen_rising_float64(i, n, K)
    assert bool((x.view(torch.int64) == -(1 << 63)).any()) and bool(torch.isnan(x).any()) and bool((~ok).any())
    fin = ~torch.isnan(x)
    assert bool((torch.diff(x[fin]) >= 0).all())  # rising
    p = gen_partition_uint8(i, single=777)
    assert int((p == 0).sum()) > 70_000 and int((p == 255).sum()) == 1 and p[777] == 255
    o = gen_int16(i, 10)
    assert int(o.min()) < -30000 and int(o.max()) > 30000


def test_validity_bitmap_round_trip():
    for n in (0, 1, 7, 8, 9, 1000):
        v = torch.rand(n) < 0.5
        bm = pack_validity(v)
        assert bm.numel() == (n + 7) // 8
        np.testing.assert_array_equal(bm.numpy(), np.packbits(v.numpy(), bitorder="little"))
        assert torch.equal(unpack_validity(bm, n), v)


def _np_stable_perm(cells, keys):
    """numpy's lexsort over (NA class, key in direction) per key and the arrival index: the brute-force stable sort."""
    cols = []
    for (x, v), (asc, na_last) in zip(cells, keys):
        xn = x.numpy()
        na = (~v.numpy() if v is not None else np.zeros(len(xn), bool))
        if xn.dtype.kind == "f":
            na = na | np.isnan(xn)
        cls = na if na_last else ~na
        if xn.dtype.kind == "f":
            with np.errstate(invalid="ignore"):  # signalling NaNs
                k = np.where(na, 0.0, xn.astype(np.float64) + 0.0)  # -0.0 + 0.0 == 0.0
            k = k if asc else -k
        else:
            k = np.where(na, 0, xn.astype(np.int64))
            k = k if asc else -k
        cols += [cls, k]
    return np.lexsort([np.arange(len(cells[0][0]))] + cols[::-1])


def _run_checker(n, gen, keys, perm, batch):
    ck = SortChecker(n, gen, keys, "cpu")
    r = torch.as_tensor(perm, dtype=torch.int64)
    for r0 in range(0, n, batch):
        rb = r[r0:r0 + batch]
        ck.feed(gen(rb), rb)
    ck.finish()


CASES = {
    "int32_nullable_desc_na_first": (lambda r: [gen_int32_nullable(r)], [(False, False)]),
    "int32_nullable_asc_na_last": (lambda r: [gen_int32_nullable(r)], [(True, True)]),
    "float32_asc_na_last": (lambda r: [(gen_float32(r), None)], [(True, True)]),
    "float32_desc_na_first": (lambda r: [(gen_float32(r), None)], [(False, False)]),
    "int64_desc_uint16_asc": (lambda r: [(gen_s3(r)[0], None), (gen_s3(r)[1], None)], [(False, True), (True, True)]),
}


def _uint16_fix(cells):
    """numpy brute force reads the UINT16 key as unsigned."""
    return [(torch.as_tensor(x.numpy().view(np.uint16).astype(np.int64)) if x.dtype == torch.int16 else x, v) for x, v in cells]


@pytest.mark.parametrize("case", sorted(CASES))
@pytest.mark.parametrize("n", [1, 2, 1000, 100_000])
def test_sort_checker_accepts_the_stable_sort(case, n):
    gen, keys = CASES[case]
    gen_u = (lambda r: [(x.to(torch.int64) & 0xFFFF if x.dtype == torch.int16 else x, v) for x, v in gen(r)])
    perm = _np_stable_perm(_uint16_fix(gen(_i(n))), keys)
    _run_checker(n, gen_u, keys, perm, batch=max(1, n // 3))
    # the torch reference of the top-k agrees
    assert torch.equal(stable_order(gen_u(_i(n)), keys), torch.as_tensor(perm))


def test_sort_checker_rejects_wrong_outputs():
    n = 20_000
    gen, keys = CASES["int32_nullable_desc_na_first"]
    perm = _np_stable_perm(gen(_i(n)), keys)
    # two equal keys in the wrong arrival order (the batch edge between them)
    v, ok = gen(_i(n))[0]
    sv, sok = v[perm], ok[perm]
    j = next(j for j in range(n // 2, n - 1) if sok[j] and sok[j + 1] and sv[j] == sv[j + 1])
    bad = perm.copy()
    bad[[j, j + 1]] = bad[[j + 1, j]]
    with pytest.raises(AssertionError, match="out of order"):
        _run_checker(n, gen, keys, bad, batch=j + 1)
    # a row repeated in place of another
    bad = perm.copy()
    bad[n - 5] = bad[5]
    with pytest.raises(AssertionError, match="twice"):
        _run_checker(n, gen, keys, bad, batch=n // 2)
    # a short output
    with pytest.raises(AssertionError):
        _run_checker(n, gen, keys, perm[:-1], batch=n)

    # a cell whose bits or validity differ from its row's
    def flip(r, what):
        x, v = gen_int32_nullable(r)
        if what == "bits":
            x = x ^ (r == perm[7]).to(torch.int32)
        else:
            v = v ^ (r == perm[7])
        return [(x, v)]

    for what, msg in (("bits", "bits differ"), ("validity", "validity differs")):
        ck = SortChecker(n, gen, keys, "cpu")
        r = torch.as_tensor(perm)
        with pytest.raises(AssertionError, match=msg):
            ck.feed(flip(r, what), r)
    # float keys: -0.0 ties 0.0 (arrival order decides), a NaN is NA
    x = torch.tensor([0.0, -0.0, float("nan"), 1.0, -0.0])
    assert torch.equal(stable_order([(x, None)], [(True, True)]), torch.tensor([0, 1, 4, 3, 2]))
    assert torch.equal(stable_order([(x, None)], [(False, False)]), torch.tensor([2, 3, 0, 1, 4]))


# ---- window closed forms against direct loops ----
def _window_brute(p, o, o_na, n_funcs_kw):
    """Direct per-row loops over the stable sort by (p asc, o asc NA last): the ranking functions, a ROWS frame sum and a RANGE
    FOLLOWING count."""
    n = len(o)
    perm = np.lexsort((np.arange(n), np.where(o_na, 0, o), o_na, p))
    sp, so, sna = p[perm], o[perm], o_na[perm]
    res = {k: np.zeros(n, np.float64 if k in ("percent_rank", "cume_dist") else np.int64) for k in n_funcs_kw}
    start = 0
    while start < n:
        end = start
        while end < n and sp[end] == sp[start]:
            end += 1
        s = end - start
        ps, pna = so[start:end], sna[start:end]
        for i in range(start, end):
            peers = np.nonzero((pna == sna[i]) & (pna | (ps == so[i])))[0]
            first, last = start + peers[0], start + peers[-1]
            rank = first - start + 1
            distinct = len(set(zip(pna[:first - start].tolist(), np.where(pna, 0, ps)[:first - start].tolist())))
            for k, arg in n_funcs_kw.items():
                if k == "row_number":
                    res[k][i] = i - start + 1
                elif k == "rank":
                    res[k][i] = rank
                elif k == "dense_rank":
                    res[k][i] = distinct + 1
                elif k == "percent_rank":
                    res[k][i] = 0.0 if s == 1 else (rank - 1) / (s - 1)
                elif k == "cume_dist":
                    res[k][i] = (last - start + 1) / s
                elif k == "ntile":
                    q, r = divmod(s, arg)
                    bucket, pos = 0, i - start
                    for bk in range(min(arg, s)):
                        size = q + (1 if bk < r else 0)
                        if pos < size:
                            bucket = bk + 1
                            break
                        pos -= size
                    res[k][i] = bucket
                elif k == "rows_sum":
                    a, b = arg
                    res[k][i] = int(so[max(start, i + a):min(end - 1, i + b) + 1].astype(np.int64).sum())
                elif k == "range_count":
                    a, b = arg
                    if sna[i]:
                        res[k][i] = int(pna.sum())
                    else:
                        res[k][i] = int((~pna & (so[i] + a <= ps) & (ps <= so[i] + b)).sum())
        start = end
    return perm, res


def _layout(p, o, o_na, n_part, descending=False):
    """The BinLayout of (p, o) from histograms: per partition 65536 value bins (+ 1 NA bin when o has NAs)."""
    na_bin = o_na is not None
    W = 65536 + na_bin
    cnt = torch.zeros(n_part * W, dtype=torch.int64)
    ok = torch.ones(len(o), dtype=torch.bool) if o_na is None else ~o_na
    flat = p.to(torch.int64) * W + torch.where(ok, o.to(torch.int64) + 32768, 65536)
    cnt += torch.bincount(flat, minlength=n_part * W)
    val = torch.arange(-32768, 32768 + na_bin, dtype=torch.int64).repeat(n_part)
    if descending:
        assert n_part == 1 and not na_bin
        cnt, val = cnt.flip(0), val.flip(0)
    return BinLayout(cnt, val, W)


@pytest.mark.parametrize("n", [1, 2, 3000])
def test_window_closed_forms_one_partition_descending(n):
    i = _i(n)
    o = gen_int16(i, 10)
    lay = _layout(torch.zeros(n, dtype=torch.uint8), o, None, 1, descending=True)
    funcs = {"row_number": None, "rank": None, "dense_rank": None, "percent_rank": None, "cume_dist": None, "ntile": 7}
    # descending order: brute force on -o
    perm, exp = _window_brute(np.zeros(n, np.int64), -o.numpy().astype(np.int64), np.zeros(n, bool), funcs)
    assert torch.equal(lay.sorted_values(i), o[torch.as_tensor(perm)].to(torch.int64))
    for k, arg in funcs.items():
        got = lay.ranking(i, k, arg)
        np.testing.assert_array_equal(got.numpy().view(np.int64), exp[k].view(np.int64), err_msg=k)


@pytest.mark.parametrize("n", [1, 5, 4000])
def test_window_closed_forms_with_partitions(n):
    """UINT8 partitions with a single-row partition and empty partitions (most of 0..255), ORDER BY INT16 ascending: the
    ranking functions and a ROWS frame sum."""
    i = _i(n)
    p = gen_partition_uint8(i, single=n // 2)
    o = gen_int16(i, 10)
    lay = _layout(p, o, None, 256)
    funcs = {"row_number": None, "rank": None, "dense_rank": None, "percent_rank": None, "cume_dist": None, "ntile": 7,
             "rows_sum": (-300, 5)}
    perm, exp = _window_brute(p.numpy().astype(np.int64), o.numpy().astype(np.int64), np.zeros(n, bool), funcs)
    assert torch.equal(lay.sorted_values(i), o[torch.as_tensor(perm)].to(torch.int64))
    assert torch.equal(lay.bin_of(i) // lay.W, p[torch.as_tensor(perm)].to(torch.int64))
    for k, arg in funcs.items():
        got = lay.rows_sum(i, *arg) if k == "rows_sum" else lay.ranking(i, k, arg)
        np.testing.assert_array_equal(got.numpy().view(np.int64), exp[k].view(np.int64), err_msg=k)


@pytest.mark.parametrize("n,all_na", [(1, False), (3000, False), (500, True)])
def test_window_range_count_closed_form(n, all_na):
    """COUNT(*) over RANGE BETWEEN 1 FOLLOWING AND 3 FOLLOWING, ORDER BY a nullable INT16 ascending NA last: empty frames at
    the largest values, the NA rows' frame is their peer group."""
    i = _i(n)
    o, ok = gen_int16_nullable(i)
    o = torch.where(torch.rand(n, generator=torch.Generator().manual_seed(n)) < 0.5, o % 9, o)  # values 1..3 apart
    if all_na:
        ok = torch.zeros(n, dtype=torch.bool)
    lay = _layout(torch.zeros(n, dtype=torch.uint8), o, ~ok, 1)
    perm, exp = _window_brute(np.zeros(n, np.int64), o.numpy().astype(np.int64), ~ok.numpy(), {"range_count": (1, 3)})
    got = lay.range_count_following(i, 1, 3, na_bin=65536)
    np.testing.assert_array_equal(got.numpy(), exp["range_count"])
    assert bool((got == 0).any()) != all_na  # the largest value's frame is empty
