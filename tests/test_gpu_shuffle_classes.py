"""The partition by key class (b200_shuffle_partition_classes, shuffle.partition_device(by_class=True)) against a host
restatement of its policy, row by row through the permutation.

The policy, restated on the oracle's hash functions (the ones its hash_to_rank and hash_keys use): a cell that is NA or a float
NaN hashes as hash_na_val (oracle_hash_inner_32_i64(1)); a float cell as oracle_hash_inner_32_f64 of its value (-0.0 and 0.0
hash alike); a 1-, 2- or 4-byte integer, bool or DATE cell as oracle_hash_inner_32_i32 of its value; an 8-byte cell as
oracle_hash_inner_32_i64; further key columns are folded in with oracle_hash_combine_boost, and the row goes to hash % n_pes.
Beside the restatement, every key class (NA and NaN one class, -0.0 equal to 0.0) must land on exactly one rank, and on 4- and
8-byte keys without NaN the placement must be b200_shuffle_partition's."""

import numpy as np
import pytest

from bodo_b200.shuffle import partition_device
from bodo_b200.table import Column, CTypes, Table
from tests.helpers import table_to_device
from tests.test_gpu_groupby_mrnf import FLOATS, SORT_TYPES, col, host_cells, key_parts, random_col

pytestmark = pytest.mark.gpu
RS = (2, 3, 4, 8)


def _class_hashes(O, c: Column) -> np.ndarray:
    L, seed = O.lib(), O.SEED_HASH_PARTITION
    v = c.values_numpy()
    m = np.ones(len(v), bool) if c.valid_mask_numpy() is None else c.valid_mask_numpy()
    if c.c_type in FLOATS:
        f = v.astype(np.float64)
        m = m & ~np.isnan(f)
        fn, vals = (lambda x: L.oracle_hash_inner_32_f64(float(x), seed)), f
    elif v.dtype.itemsize == 8:
        fn, vals = (lambda x: L.oracle_hash_inner_32_i64(int(x), seed)), v.view(np.int64)
    else:
        fn, vals = (lambda x: L.oracle_hash_inner_32_i32(int(x), seed)), v.astype(np.int64).astype(np.int32)
    uniq, inv = np.unique(vals, return_inverse=True)
    h = np.array([fn(x) for x in uniq], dtype=np.uint32)[inv.reshape(-1)]
    h[~m] = L.oracle_hash_inner_32_i64(1, seed)
    return h


def ref_dest(O, t: Table, n_keys: int, n_pes: int) -> np.ndarray:
    combine = O.lib().oracle_hash_combine_boost
    h = _class_hashes(O, t.columns[0])
    for c in t.columns[1:n_keys]:
        h = np.array([combine(a, b) for a, b in zip(h.tolist(), _class_hashes(O, c).tolist())], dtype=np.uint32)
    return (h.astype(np.int64) % n_pes).astype(np.int64)


def device_dest(t: Table, n_keys: int, n_pes: int, by_class=True):
    """(destination of every input row, send counts, perm) from the device partition."""
    part, counts, perm = partition_device(table_to_device(t), n_keys, n_pes, want_perm=True, by_class=by_class)
    perm = perm.cpu().numpy()
    dest = np.empty(t.n_rows, np.int64)
    dest[perm] = np.repeat(np.arange(n_pes), counts)
    return dest, counts, perm, part


def check(O, t: Table, n_keys: int, n_pes: int):
    dest, counts, perm, part = device_dest(t, n_keys, n_pes)
    exp = ref_dest(O, t, n_keys, n_pes)
    np.testing.assert_array_equal(dest, exp)
    np.testing.assert_array_equal(perm, np.argsort(exp, kind="stable"))  # stable within a destination
    assert counts == np.bincount(exp, minlength=n_pes).tolist()
    for c, oc in zip(t.columns, part.columns):  # every column travels with its row, validity included
        m, b = host_cells(c)
        om, ob = host_cells(Column(oc.data.cpu().numpy(), None if oc.validity is None else _unsegment(oc.validity.cpu().numpy(), counts),
                                   oc.c_type, oc.arr_type, oc.length))
        np.testing.assert_array_equal(om, m[perm])
        np.testing.assert_array_equal(ob, b[perm])
    # every key class on exactly one rank
    cls = np.stack([x for c in t.columns[:n_keys] for x in key_parts(c)], axis=1)
    _, label = np.unique(cls, axis=0, return_inverse=True)
    label = label.reshape(-1)
    lo, hi = np.full(label.max() + 1 if len(label) else 0, n_pes), np.full(label.max() + 1 if len(label) else 0, -1)
    np.minimum.at(lo, label, dest)
    np.maximum.at(hi, label, dest)
    assert (lo == hi).all(), "a key class spans two ranks"
    return dest


def _unsegment(bitmap, counts):
    """The per-destination bitmaps (each from a byte boundary) as one bitmap."""
    bits, byte = [], 0
    for cnt in counts:
        nb = (cnt + 7) // 8
        bits.append(np.unpackbits(bitmap[byte: byte + nb], bitorder="little")[:cnt].astype(bool))
        byte += nb
    return np.packbits(np.concatenate(bits) if bits else np.zeros(0, bool), bitorder="little")


def mixed_key(rng, ct, n, nullable):
    """random_col with NaN, NA, -0.0 and 0.0 all present in a float key."""
    c = random_col(rng, ct, n, nullable)
    if ct in FLOATS:
        v = c.values_numpy().copy()
        v[:4] = [np.nan, -0.0, 0.0, np.nan]
        c = Column(v, c.validity, ct, c.arr_type, n)
    return c


@pytest.mark.parametrize("ct", SORT_TYPES)
@pytest.mark.parametrize("nullable", [False, True])
def test_every_key_type(gpu_lib, oracle, ct, nullable):
    rng = np.random.default_rng(ct * 2 + nullable)
    n = 6000
    t = Table([mixed_key(rng, ct, n, nullable), col(np.arange(n), CTypes.INT64), random_col(rng, CTypes.INT16, n, True)],
              ["k", "id", "p"])
    for R in RS:
        check(oracle, t, 1, R)


@pytest.mark.parametrize("n_keys", [2, 3, 4])
def test_key_tuples(gpu_lib, oracle, n_keys):
    rng = np.random.default_rng(40 + n_keys)
    types = [CTypes.INT8, CTypes.FLOAT64, CTypes.BOOL, CTypes.UINT16, CTypes.FLOAT32, CTypes.DATE][n_keys - 2: n_keys - 2 + n_keys]
    n = 4000
    cols = [mixed_key(rng, ct, n, j % 2 == 0) for j, ct in enumerate(types)]
    t = Table(cols + [col(np.arange(n), CTypes.INT64)], [f"k{j}" for j in range(n_keys)] + ["id"])
    for R in RS + (13, 256):  # the general scatter kernel beyond 8 destinations
        check(oracle, t, n_keys, R)


def test_nan_na_and_zero_share_one_rank(gpu_lib, oracle):
    v = np.array([np.nan, 0.0, -0.0, np.nan, 1.0, 0.0, -0.0, np.nan] * 50)
    valid = np.arange(len(v)) % 3 != 0
    for ct in (CTypes.FLOAT64, CTypes.FLOAT32):
        t = Table([col(v, ct, valid), col(np.arange(len(v)), CTypes.INT64)], ["k", "id"])
        for R in RS:
            dest = check(oracle, t, 1, R)
            na = ~valid | np.isnan(v)
            assert len(set(dest[na])) == 1 and len(set(dest[~na & (v == 0)])) == 1


@pytest.mark.parametrize("ct", [CTypes.INT32, CTypes.UINT32, CTypes.DATE, CTypes.INT64, CTypes.UINT64, CTypes.DATETIME,
                                CTypes.TIMEDELTA, CTypes.FLOAT32, CTypes.FLOAT64])
def test_reference_placement_without_nan(gpu_lib, ct):
    """On 4- and 8-byte keys without a valid NaN the key-class placement is the reference's."""
    rng = np.random.default_rng(ct)
    n = 20_000
    c = random_col(rng, ct, n, True)
    if ct in FLOATS:
        v = c.values_numpy().copy()
        v[np.isnan(v)] = 2.5
        c = Column(v, c.validity, ct, c.arr_type, n)
    t = Table([c, col(np.arange(n), CTypes.INT64)], ["k", "id"])
    for R in RS:
        a = device_dest(t, 1, R)
        b = device_dest(t, 1, R, by_class=False)
        np.testing.assert_array_equal(a[0], b[0])
        np.testing.assert_array_equal(a[2], b[2])


def test_empty_table_and_bad_keys(gpu_lib):
    from bodo_b200._lib import B200Error

    t = Table([col(np.zeros(0), CTypes.INT8), col(np.zeros(0), CTypes.INT64)], ["k", "id"])
    _, counts, _, _ = device_dest(t, 1, 4)
    assert counts == [0, 0, 0, 0]
    one = Table([col(np.arange(5), CTypes.INT16)], ["k"])
    with pytest.raises(B200Error, match="4- or 8-byte"):  # the reference placement still refuses narrow keys
        partition_device(table_to_device(one), 1, 2)
    with pytest.raises(B200Error, match="between 1 and 4 key columns"):
        partition_device(table_to_device(one), 5, 2, by_class=True)
