"""The key map of the SPG-N dense form (spgd_scramble / spgd_key in bodo_b200/csrc/spgn.cuh), mirrored in numpy.

For every window size 2^KB (KB <= 21) and owner count G in [2, 256] it checks, over every key offset d < 2^KB, that the scramble
sigma is a bijection whose inverse is the one K2d's flush applies, that umulhi(x, ceil(2^32 / G)) is exactly x div G, and that
(owner, slot) = (x mod G, x div G) is a bijection onto owners [0, G) x slots [0, ceil(2^KB / G))."""
import numpy as np

MUL = 0x9E3779B1  # GroupbyState::SPGD_MUL


def _odd_inverse(m):
    x = m
    for _ in range(4):
        x = (x * (2 - m * x)) & 0xFFFFFFFF
    return x


def _scramble(d, kb):
    x = (d * np.uint64(MUL)) & np.uint64((1 << kb) - 1)
    return x ^ (x >> np.uint64((kb + 1) // 2))


def _unscramble(x, kb, inv):
    x = x ^ (x >> np.uint64((kb + 1) // 2))
    return (x * np.uint64(inv)) & np.uint64((1 << kb) - 1)


def test_odd_inverse():
    assert (MUL * _odd_inverse(MUL)) & 0xFFFFFFFF == 1


def test_scramble_is_a_bijection_with_its_inverse():
    inv = _odd_inverse(MUL)
    for kb in range(1, 22):
        d = np.arange(1 << kb, dtype=np.uint64)
        x = _scramble(d, kb)
        assert np.array_equal(np.sort(x), d), kb
        assert np.array_equal(_unscramble(x, kb, inv), d), kb


def test_owner_slot_split_is_exact_and_bijective():
    for kb in range(1, 22):
        x = np.arange(1 << kb, dtype=np.uint64)
        for g in range(2, 257):
            magic = ((1 << 32) + g - 1) // g  # ceil(2^32 / G), as the host computes it
            assert magic < (1 << 32)
            q = (x * np.uint64(magic)) >> np.uint64(32)  # __umulhi: x < 2^21 and magic < 2^32, so the product fits 64 bits
            assert np.array_equal(q, x // np.uint64(g)), (kb, g)
            owner = x - q * np.uint64(g)
            slots = ((1 << kb) + g - 1) // g
            assert int(q.max()) < slots and int(owner.max()) < g
            # the inverse the flush uses: x = slot * G + owner
            assert np.array_equal(q * np.uint64(g) + owner, x)

