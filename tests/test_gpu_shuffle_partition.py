"""The row -> rank radix partition (csrc/shuffle.cu: dest_hist / scan_hist / scatter / scatter_small / pack_segment_bitmaps
kernels) against an exact reference, at the tile geometries, column widths, key types and destination counts where the
kernels have separate code.

The reference is independent of the device:
  - destination of a row: hash_to_rank of hash_keys with seed SEED_HASH_PARTITION.  Tables whose keys are all 8-byte
    integers (int64, uint64, DATETIME, TIMEDELTA) go through the oracle's vectorised C (`oracle.hash_keys`); every other
    key table through the oracle's scalar functions (NA -> oracle_hash_inner_32_i64(1); 4-byte integers and DATE ->
    oracle_hash_inner_32_i32 of the raw bits; float32 / float64 -> oracle_hash_inner_32_f64 of the value; further keys
    folded in with oracle_hash_combine_boost), called once per distinct bit pattern of a column;
  - counts = bincount(dest), perm = argsort(dest, stable), every output column = input[perm] compared byte for byte, and
    every destination's bitmap packed LSB-first from a byte boundary, segment d starting at byte sum_{d' < d} ceil(cnt_d' / 8).

What each group reaches in shuffle.cu:
  - tile geometry (`tile_geometry` mirrors :315-318): the per-destination cursor advance across chunks (:139-143 in
    scatter_kernel, :217-221 in scatter_small_kernel), the re-zeroing of wtot (:109) and partial last chunks / tiles
    (the `i < r1` guards, :117, :185);
  - small kernel, every NC, skewed destinations: scatter_small_kernel<1..4> (:168-231), its 16-bit register fields at their
    largest values (256 per warp block, 1792 over the earlier warps, 2048 per chunk) and the second register word
    (destinations 4-7);
  - general kernel, every width: the 8- / 4- / 2- / 1-byte copies (:151-156), validity bytes (:157), 5 to 32 columns,
    9 to 256 destinations (scan_hist_kernel with several destinations per warp, :57-78; dest8 up to 255; wtot rows up to
    256) and empty segments in pack_segment_bitmaps_kernel (:234-251);
  - key types and tuples: hash_keys_row over int32 / uint32 / DATE / int64 / DATETIME / float64 / float32 keys with NAs in
    dest_hist_kernel (:38-53);
  - receive side: partition + merge_segment_bitmaps_kernel (:255-275), as exchange_table assembles it;
  - side stream, the benchmark's own shape (2^26 rows, scatter_small_kernel<2>, ~30 chunks per CTA), hash_to_rank_kernel
    beyond one grid stride (:28-35) and the argument checks of shuffle_partition (:285-306).
"""

import numpy as np
import pytest
import torch

from bodo_b200 import _lib
from bodo_b200._lib import ffi
from bodo_b200.shuffle import hash_keys_table, merge_segment_bitmaps, partition_device, with_schema_validity
from bodo_b200.table import ArrTypes, Column, CTable, CTypes, Table, np_dtype_of
from tests.helpers import table_to_device

gpu = pytest.mark.gpu

PART_THREADS, SC_STEPS = 256, 8
CHUNK = PART_THREADS * SC_STEPS  # rows a CTA of the scatter kernels ranks per chunk
INT64_FAMILY = (CTypes.INT64, CTypes.UINT64, CTypes.DATETIME, CTypes.TIMEDELTA)
SCALAR_REF_MAX_ROWS = 200_000  # the scalar reference makes one Python call per row and key


# ---------------------------------------------------------------------------------------------------------------------
# reference
# ---------------------------------------------------------------------------------------------------------------------

def _column_hashes(O, col: Column) -> np.ndarray:
    """hash_key_column of one host column through the oracle's scalar functions, one call per distinct bit pattern."""
    L, seed = O.lib(), O.SEED_HASH_PARTITION
    data = np.asarray(col.data)
    size = data.dtype.itemsize
    if col.c_type in (CTypes.FLOAT32, CTypes.FLOAT64):
        f = lambda v: L.oracle_hash_inner_32_f64(float(v), seed)  # noqa: E731  (float32 widens exactly)
        as_values = data.dtype
    elif size == 4:
        f = lambda v: L.oracle_hash_inner_32_i32(int(v), seed)  # noqa: E731  (the 4 raw bytes, uint32 included)
        as_values = np.dtype(np.int32)
    elif size == 8:
        f = lambda v: L.oracle_hash_inner_32_i64(int(v), seed)  # noqa: E731
        as_values = np.dtype(np.int64)
    else:
        raise AssertionError(f"no key hash for c_type {col.c_type}")
    bits, inv = np.unique(data.view(f"u{size}"), return_inverse=True)
    table = np.array([f(v) for v in bits.view(as_values)], dtype=np.uint32)
    h = table[inv.reshape(-1)]
    valid = col.valid_mask_numpy()
    if valid is not None:
        h[~valid] = L.oracle_hash_inner_32_i64(1, seed)
    return h


def ref_hashes(O, table: Table, n_keys: int, scalar: bool = False) -> np.ndarray:
    """hash_keys(SEED_HASH_PARTITION) of every row of a host table whose first n_keys columns are the keys (uint32)."""
    keys = table.columns[:n_keys]
    if not scalar and all(c.c_type in INT64_FAMILY for c in keys):
        return O.hash_keys([np.asarray(c.data).view(np.int64) for c in keys], [c.valid_mask_numpy() for c in keys])
    assert table.n_rows <= SCALAR_REF_MAX_ROWS, "the scalar reference is for small tables"
    combine = O.lib().oracle_hash_combine_boost
    h = _column_hashes(O, keys[0])
    for c in keys[1:]:
        h = np.array([combine(a, b) for a, b in zip(h.tolist(), _column_hashes(O, c).tolist())], dtype=np.uint32)
    return h


def ref_dest(O, table: Table, n_keys: int, n_pes: int) -> np.ndarray:
    """hash_to_rank: (uint32) hash % n_pes, as uint8 (n_pes <= 256)."""
    return (ref_hashes(O, table, n_keys).astype(np.int64) % n_pes).astype(np.uint8)


def expected_partition(dest: np.ndarray, n_pes: int):
    """(send counts, source row of every output row): a stable counting sort by destination."""
    return np.bincount(dest, minlength=n_pes), np.argsort(dest, kind="stable")


def _assert_same_bytes(got: np.ndarray, exp: np.ndarray, what: str):
    assert got.dtype == exp.dtype, f"{what}: dtype {got.dtype} != {exp.dtype}"
    g = np.ascontiguousarray(got).view(np.uint8).reshape(len(got), got.dtype.itemsize)
    e = np.ascontiguousarray(exp).view(np.uint8).reshape(len(exp), exp.dtype.itemsize)
    assert g.shape == e.shape, f"{what}: {len(got)} rows != {len(exp)}"
    if not np.array_equal(g, e):
        bad = np.flatnonzero((g != e).any(axis=1))
        raise AssertionError(f"{what}: {len(bad)} of {len(got)} rows differ, first at row {bad[0]}: "
                             f"got bytes {g[bad[0]].tolist()}, expected {e[bad[0]].tolist()}")


def _assert_segment_bitmaps(bitmap: np.ndarray, mask_sorted: np.ndarray, counts, what: str):
    """Destination d's bitmap starts on byte sum_{d' < d} ceil(cnt_d' / 8), LSB first; only its first cnt bits count."""
    row = byte = 0
    for d, cnt in enumerate(counts):
        cnt = int(cnt)
        nbytes = (cnt + 7) // 8
        seg = np.unpackbits(bitmap[byte: byte + nbytes], bitorder="little")[:cnt].astype(bool)
        if not np.array_equal(seg, mask_sorted[row: row + cnt]):
            bad = np.flatnonzero(seg != mask_sorted[row: row + len(seg)]) if len(seg) == cnt else [None]
            raise AssertionError(f"{what}: bitmap of destination {d} ({cnt} rows from byte {byte}) differs, first at bit {bad[0]}")
        row += cnt
        byte += nbytes


def check_partition(O, host: Table, n_keys: int, n_pes: int, dest=None):
    """Partition `host` on the device twice (with and without the permutation) and compare both with the reference:
    counts, perm, every column's bytes, c_type / arr_type and every destination's bitmap.  Returns the first run."""
    dest = ref_dest(O, host, n_keys, n_pes) if dest is None else dest
    counts, perm = expected_partition(dest, n_pes)
    dev = table_to_device(host)
    part, got_counts, got_perm = partition_device(dev, n_keys, n_pes, want_perm=True)
    part_np, counts_np = partition_device(dev, n_keys, n_pes)
    assert got_counts == counts.tolist(), "send counts"
    assert counts_np == counts.tolist(), "send counts (no perm)"
    _assert_same_bytes(got_perm.cpu().numpy(), perm.astype(np.int64), "perm")
    for ci, c in enumerate(host.columns):
        exp = np.asarray(c.data)[perm]
        mask = c.valid_mask_numpy()
        for label, p in (("with perm", part), ("without perm", part_np)):
            oc = p.columns[ci]
            what = f"column {ci} ({host.names[ci]}, c_type {c.c_type}), {label}"
            assert (oc.c_type, oc.arr_type, oc.length) == (c.c_type, c.arr_type, c.length), what
            _assert_same_bytes(oc.data.cpu().numpy(), exp, what)
            if mask is None:
                assert oc.validity is None, what
            else:
                _assert_segment_bitmaps(oc.validity.cpu().numpy(), mask[perm], counts, what)
    return part, got_counts, got_perm


def raw_partition(gpu_lib, table: Table, n_keys: int, n_pes: int):
    """b200_shuffle_partition through the C ABI into output buffers and a b200_table filled with sentinels (0xA5 bytes,
    c_type / arr_type / length / n_rows = -1, send counts = -7), so a test sees exactly what the library wrote."""
    n = table.n_rows
    outs = []
    for c in table.columns:
        size = max(n, 1) * np.dtype(np_dtype_of(c.c_type)).itemsize
        data = torch.full((size,), 0xA5, dtype=torch.uint8, device="cuda")
        v = torch.full(((n + 7) // 8 + max(n_pes, 0) + 8,), 0xA5, dtype=torch.uint8, device="cuda") if c.validity is not None else None
        outs.append(Column(data, v, CTypes.UINT8, ArrTypes.NUMPY, n))
    out = Table(outs)
    cin, cout = CTable(table), CTable(out)
    for i in range(out.n_cols):
        cout.cols[i].c_type, cout.cols[i].arr_type, cout.cols[i].length = -1, -1, -1
    cout.ctab.n_rows = -1
    counts = ffi.new("int64_t[]", [-7] * 260)
    rc = gpu_lib.b200_shuffle_partition(cin.ptr, n_keys, n_pes, cout.ptr, counts, ffi.NULL)
    torch.cuda.synchronize()
    return rc, cout, counts, outs


# ---------------------------------------------------------------------------------------------------------------------
# inputs
# ---------------------------------------------------------------------------------------------------------------------

def tile_geometry(n: int, sms: int):
    """(n_ctas, tile_rows) of the partition kernels for n rows: a mirror of shuffle_partition, csrc/shuffle.cu:315-318 (at
    most 8 CTAs per SM, every tile a whole number of PART_THREADS * SC_STEPS = 2048-row chunks)."""
    n_ctas = min(sms * 8, (n + PART_THREADS - 1) // PART_THREADS)
    tile = ((n + n_ctas - 1) // n_ctas + CHUNK - 1) // CHUNK * CHUNK
    return (n + tile - 1) // tile, tile


def _sms() -> int:
    return torch.cuda.get_device_properties(0).multi_processor_count


GEOMETRIES = ["one_chunk_per_cta", "full_grid_plus_one", "multi_chunk_short_tail"]


def geometry_rows(name: str, sms: int) -> int:
    """A row count with the named tile geometry; asserts that the geometry really occurs, so a change to the tiling
    fails here instead of quietly shrinking the case."""
    full = 8 * sms * CHUNK  # every CTA of the largest grid takes exactly one chunk
    n = {"one_chunk_per_cta": full, "full_grid_plus_one": full + 1, "multi_chunk_short_tail": 3 * full + 777}[name]
    n_ctas, tile = tile_geometry(n, sms)
    last = n - (n_ctas - 1) * tile
    if name == "one_chunk_per_cta":
        assert (n_ctas, tile, last) == (8 * sms, CHUNK, CHUNK)
    elif name == "full_grid_plus_one":
        assert tile == 2 * CHUNK and n_ctas == 4 * sms + 1 and last == 1  # two chunks per CTA, the last tile one row
    else:
        assert tile >= 3 * CHUNK and last < tile and last % CHUNK != 0  # >= 3 chunks per tile, a short partial last tile
    return n


def _float_payload(rng, n: int, dtype) -> np.ndarray:
    """Floats with -0.0, +-inf and NaNs of several bit patterns (quiet, signalling, negative, payload-carrying)."""
    x = (rng.standard_normal(n) * 10.0 ** rng.integers(-5, 6, n)).astype(dtype)
    u = x.view(np.uint64 if dtype == np.float64 else np.uint32)
    if dtype == np.float64:
        special = np.array([0x8000000000000000, 0x7FF8000000000000, 0x7FF8000000000001, 0xFFF0000000000123,
                            0x7FF0000000000001, 0x7FF0000000000000, 0xFFF0000000000000], dtype=np.uint64)
    else:
        special = np.array([0x80000000, 0x7FC00000, 0x7FC00001, 0xFF800123, 0x7F800001, 0x7F800000, 0xFF800000], dtype=np.uint32)
    pos = rng.random(n) < 0.05
    u[pos] = special[rng.integers(0, len(special), int(pos.sum()))]
    return x


def _mask(rng, n, p_na=0.1):
    return np.packbits(rng.random(n) >= p_na, bitorder="little")


def _col(data, c_type, validity=None, nullable=False):
    arr = ArrTypes.NULLABLE_INT_BOOL if (nullable or validity is not None) else ArrTypes.NUMPY
    return Column(np.ascontiguousarray(data), validity, c_type, arr)


def _values(rng, n: int, c_type: int) -> np.ndarray:
    """Random values of a fixed-width type that use every byte of the cell."""
    if c_type in (CTypes.FLOAT32, CTypes.FLOAT64):
        return _float_payload(rng, n, np.float32 if c_type == CTypes.FLOAT32 else np.float64)
    if c_type == CTypes.BOOL:
        return rng.random(n) < 0.5
    dt = np_dtype_of(c_type)
    info = np.iinfo(dt)
    return rng.integers(info.min, info.max, n, dtype=dt, endpoint=True)


WIDE8 = [CTypes.INT64, CTypes.UINT64, CTypes.FLOAT64, CTypes.DATETIME]  # the small kernel's column kinds


def wide8_table(rng, n: int, nc: int, keys=None) -> Table:
    """nc 8-byte columns without bitmaps: an int64 key, then uint64, float64 and DATETIME payloads."""
    k = rng.integers(-(1 << 62), 1 << 62, n) if keys is None else keys
    cols = [_col(k, CTypes.INT64)] + [_col(_values(rng, n, ct), ct) for ct in WIDE8[1:nc]]
    return Table(cols, ["k", "u64", "f64", "ts"][:nc])


def keys_to_dest(O, rng, n_pes: int, wanted, n_candidates=1 << 17):
    """int64 keys whose oracle destination among n_pes is `wanted` (one pool per wanted destination)."""
    cand = rng.integers(-(1 << 62), 1 << 62, n_candidates)
    d = O.hash_to_rank(cand, None, n_pes)
    return [cand[d == w] for w in wanted]


# ---------------------------------------------------------------------------------------------------------------------
# CPU self-checks of the reference
# ---------------------------------------------------------------------------------------------------------------------

def test_reference_equals_oracle_shuffle_partition(oracle):
    rng = np.random.default_rng(1)
    n = 50_021
    keys = rng.integers(-(1 << 62), 1 << 62, n)
    keys[rng.random(n) < 0.3] = 12345  # a heavy key
    valid = rng.random(n) > 0.07
    t = Table([_col(keys, CTypes.INT64, np.packbits(valid, bitorder="little"))])
    for n_pes in (1, 7, 8, 64, 256):
        counts, perm = expected_partition(ref_dest(oracle, t, 1, n_pes), n_pes)
        ecounts, eperm = oracle.shuffle_partition(keys, valid, n_pes)
        np.testing.assert_array_equal(counts, ecounts)
        np.testing.assert_array_equal(perm, eperm)


def test_scalar_reference_equals_oracle_hash_keys_on_int64_columns(oracle):
    rng = np.random.default_rng(2)
    n = 20_011
    ks = [rng.integers(-(1 << 62), 1 << 62, n), rng.integers(0, 50, n), rng.integers(-3, 3, n), rng.integers(0, 1 << 40, n)]
    vs = [rng.random(n) > 0.1, None, rng.random(n) > 0.5, None]
    t = Table([_col(k, CTypes.INT64, None if v is None else np.packbits(v, bitorder="little")) for k, v in zip(ks, vs)])
    for nk in (1, 2, 3, 4):
        np.testing.assert_array_equal(ref_hashes(oracle, t, nk, scalar=True), oracle.hash_keys(ks[:nk], vs[:nk]))


def test_tile_geometry_mirror():
    # the launch of shuffle_partition for a few row counts on a 132-SM card, worked by hand
    assert tile_geometry(1, 132) == (1, CHUNK)
    assert tile_geometry(100_000, 132) == (49, CHUNK)
    assert tile_geometry(1_000_001, 132) == (489, CHUNK)
    assert tile_geometry(8 * 132 * CHUNK + 1, 132) == (4 * 132 + 1, 2 * CHUNK)
    for name in GEOMETRIES:
        for sms in (78, 114, 132):
            geometry_rows(name, sms)


# ---------------------------------------------------------------------------------------------------------------------
# tile geometry: multi-chunk tiles through both kernels
# ---------------------------------------------------------------------------------------------------------------------

@gpu
@pytest.mark.parametrize("geometry", GEOMETRIES)
@pytest.mark.parametrize("n_pes,nc", [(1, 4), (2, 1), (7, 3), (8, 2)])
def test_small_kernel_tile_geometry(gpu_lib, oracle, geometry, n_pes, nc):
    n = geometry_rows(geometry, _sms())
    rng = np.random.default_rng(n + 10 * n_pes + nc)
    check_partition(oracle, wide8_table(rng, n, nc), 1, n_pes)


@gpu
@pytest.mark.parametrize("geometry", GEOMETRIES)
@pytest.mark.parametrize("n_pes", [9, 64, 256])
def test_general_kernel_tile_geometry(gpu_lib, oracle, geometry, n_pes):
    n = geometry_rows(geometry, _sms())
    rng = np.random.default_rng(n + n_pes)
    t = wide8_table(rng, n, 4)
    t = Table(t.columns + [_col(_values(rng, n, CTypes.INT32), CTypes.INT32, _mask(rng, n))], t.names + ["ni32"])
    check_partition(oracle, t, 1, n_pes)


# ---------------------------------------------------------------------------------------------------------------------
# small kernel: every NC, skewed destinations
# ---------------------------------------------------------------------------------------------------------------------

@gpu
@pytest.mark.parametrize("nc", [1, 2, 3, 4])
@pytest.mark.parametrize("n_pes", [1, 3, 4, 5, 8])
def test_small_kernel_every_nc(gpu_lib, oracle, nc, n_pes):
    n = 300_007
    rng = np.random.default_rng(100 * nc + n_pes)
    keys = rng.integers(-(1 << 62), 1 << 62, n)
    keys[rng.random(n) < 0.2] = 7  # one heavy key: long same-destination runs
    check_partition(oracle, wide8_table(rng, n, nc, keys), 1, n_pes)


@gpu
@pytest.mark.parametrize("nc", [1, 2, 3, 4])
@pytest.mark.parametrize("skew", ["all_to_7", "all_to_0", "alternate_2_and_5"])
def test_small_kernel_skewed_destinations(gpu_lib, oracle, nc, skew):
    """All rows to destination 7 of 8 drives a 16-bit field of the high register word to its largest values: 256 for a
    warp's block, 1792 over the earlier warps, 2048 per chunk; two chunks per CTA carry the cursor across chunks."""
    sms = _sms()
    n = geometry_rows("full_grid_plus_one", sms)
    rng = np.random.default_rng(nc)
    if skew == "all_to_7":
        (pool,) = keys_to_dest(oracle, rng, 8, [7])
        keys = rng.choice(pool, n)
        dest = np.full(n, 7, dtype=np.uint8)
    elif skew == "all_to_0":
        (pool,) = keys_to_dest(oracle, rng, 8, [0])
        keys = rng.choice(pool, n)
        dest = np.zeros(n, dtype=np.uint8)
    else:
        lo, hi = keys_to_dest(oracle, rng, 8, [2, 5])
        keys = np.where(np.arange(n) % 2 == 0, rng.choice(lo, n), rng.choice(hi, n))
        dest = np.where(np.arange(n) % 2 == 0, 2, 5).astype(np.uint8)
    t = wide8_table(rng, n, nc, keys)
    np.testing.assert_array_equal(ref_dest(oracle, t, 1, 8), dest)
    check_partition(oracle, t, 1, 8, dest)


# ---------------------------------------------------------------------------------------------------------------------
# general kernel: every width, 5..32 columns, 9..256 destinations
# ---------------------------------------------------------------------------------------------------------------------

ALL_WIDTHS = [CTypes.INT8, CTypes.UINT8, CTypes.INT16, CTypes.UINT16, CTypes.INT32, CTypes.UINT32, CTypes.INT64, CTypes.UINT64,
              CTypes.FLOAT32, CTypes.FLOAT64, CTypes.BOOL, CTypes.DATE, CTypes.DATETIME, CTypes.TIMEDELTA]


def every_width_table(rng, n: int, n_distinct_keys=None) -> Table:
    """An int64 key, then every fixed-width type as a numpy column and as a nullable column with NAs (29 columns)."""
    keys = rng.integers(0, 1000, n) if n_distinct_keys is None else rng.choice(rng.integers(0, 1 << 40, n_distinct_keys), n)
    cols, names = [_col(keys, CTypes.INT64)], ["k"]
    for ct in ALL_WIDTHS:
        cols.append(_col(_values(rng, n, ct), ct))
        cols.append(_col(_values(rng, n, ct), ct, _mask(rng, n)))
        names += [f"t{ct}", f"t{ct}_null"]
    return Table(cols, names)


@gpu
@pytest.mark.parametrize("n_pes,n_distinct_keys", [(9, None), (33, None), (64, None), (255, None), (256, None), (64, 3), (256, 5)])
def test_general_kernel_every_width(gpu_lib, oracle, n_pes, n_distinct_keys):
    n = 250_007
    rng = np.random.default_rng(n_pes * 7 + (n_distinct_keys or 0))
    t = every_width_table(rng, n, n_distinct_keys)
    assert t.n_cols == 29
    part, counts, _ = check_partition(oracle, t, 1, n_pes)
    if n_distinct_keys is not None:  # empty segments between non-empty ones: repeated bitmap byte offsets
        nz = np.flatnonzero(counts)
        assert len(nz) <= n_distinct_keys and nz[-1] + 1 > len(nz)
    # the same call through the C ABI: the library writes n_rows and every column's length / c_type / arr_type itself
    rc, cout, ccounts, outs = raw_partition(gpu_lib, table_to_device(t), 1, n_pes)
    _lib.check(rc, "shuffle partition")
    assert cout.ctab.n_rows == n
    assert [ccounts[d] for d in range(n_pes)] == counts
    for ci, c in enumerate(t.columns):
        oc = cout.cols[ci]
        assert (oc.length, oc.c_type, oc.arr_type) == (n, c.c_type, c.arr_type), ci
        size = np.dtype(np_dtype_of(c.c_type)).itemsize
        assert torch.equal(outs[ci].data[: n * size], part.columns[ci].data.view(torch.uint8)), ci


@gpu
@pytest.mark.parametrize("n_cols,n_pes", [(5, 8), (5, 255), (32, 33), (32, 256)])
def test_general_kernel_column_counts(gpu_lib, oracle, n_cols, n_pes):
    """5 columns is the fewest that leaves the small kernel (even at <= 8 destinations), 32 the most a table may have."""
    n = 150_001
    rng = np.random.default_rng(n_cols * 1000 + n_pes)
    cols = [_col(rng.integers(-(1 << 62), 1 << 62, n), CTypes.INT64)]
    for j in range(1, n_cols):
        ct = CTypes.INT64 if n_cols == 5 else ALL_WIDTHS[j % len(ALL_WIDTHS)]
        cols.append(_col(_values(rng, n, ct), ct, _mask(rng, n) if j % 3 == 0 else None))
    check_partition(oracle, Table(cols), 1, n_pes)


# ---------------------------------------------------------------------------------------------------------------------
# key types and key tuples
# ---------------------------------------------------------------------------------------------------------------------

def _key_column(rng, kind: str, n: int, nullable: bool) -> Column:
    ct = {"int32": CTypes.INT32, "uint32": CTypes.UINT32, "date": CTypes.DATE, "int64": CTypes.INT64,
          "datetime": CTypes.DATETIME, "float64": CTypes.FLOAT64, "float32": CTypes.FLOAT32}[kind]
    if kind in ("float64", "float32"):
        dt = np.float64 if kind == "float64" else np.float32
        x = _float_payload(rng, n, dt)
        small = rng.integers(-20, 20, n).astype(dt)  # repeated keys, integers-as-floats
        x = np.where(rng.random(n) < 0.4, small, x)
        special = np.array([0.0, -0.0, np.nan, np.inf, -np.inf, 2.0 ** 61, -(2.0 ** 61) + 1, 1e-300], dtype=dt)
        pos = rng.random(n) < 0.05
        x[pos] = special[rng.integers(0, len(special), int(pos.sum()))]
    elif kind == "date":
        x = rng.integers(-100_000, 100_000, n).astype(np.int32)
    else:
        x = _values(rng, n, ct)
        x = np.where(rng.random(n) < 0.4, rng.integers(0, 50, n).astype(x.dtype), x)
    return _col(x, ct, _mask(rng, n, 0.15) if nullable else None)


KEY_SETS = [
    (("int32", False),),
    (("uint32", True),),
    (("date", False),),
    (("float64", False),),
    (("float64", True),),
    (("float32", False),),
    (("datetime", False),),
    (("datetime", True),),
    (("float64", False), ("int64", True)),
    (("uint32", False), ("date", True), ("float32", False)),
    (("int32", True), ("float32", True), ("datetime", False), ("float64", True)),
    (("int64", False), ("uint32", False), ("int32", False), ("date", False)),
]


@gpu
@pytest.mark.parametrize("keys", KEY_SETS, ids=lambda ks: "-".join(k + ("_na" if na else "") for k, na in ks))
def test_partition_key_types(gpu_lib, oracle, keys):
    """Every key table against the scalar reference; at 5 destinations a table of 8-byte keys without NAs takes the small
    kernel, at 37 every table takes the general one."""
    n = 60_013
    rng = np.random.default_rng(len(keys) * 100 + sum(na for _, na in keys))
    cols = [_key_column(rng, k, n, na) for k, na in keys]
    cols.append(_col(rng.integers(-(1 << 62), 1 << 62, n), CTypes.INT64))
    t = Table(cols)
    h = ref_hashes(oracle, t, len(keys), scalar=True).astype(np.int64)
    for n_pes in (5, 37):
        check_partition(oracle, t, len(keys), n_pes, (h % n_pes).astype(np.uint8))


# ---------------------------------------------------------------------------------------------------------------------
# receive side, side stream, benchmark shape, hash_keys_table
# ---------------------------------------------------------------------------------------------------------------------

@gpu
@pytest.mark.parametrize("R", [2, 3, 8])
def test_receive_side_reassembly(gpu_lib, oracle, R):
    """Every source partitioned into R destinations (with_schema_validity first, as shuffle_table does), destination d
    concatenating segment d of every source in source order and merging their bitmaps: exactly what exchange_table
    assembles, without the all-to-all.  Expected: the rows of every source whose destination is d, in (source, row) order."""
    sizes = [40_013, 0, 1, 2_049, 100_003, 9, 65_537, 31][:R]
    rng = np.random.default_rng(R)
    hosts, parts = [], []
    for s, n in enumerate(sizes):
        t = Table([_col(rng.integers(0, 5000, n), CTypes.INT64, nullable=True),  # nullable, but no bitmap in this batch
                   _col(_float_payload(rng, n, np.float64), CTypes.FLOAT64),
                   _col(_values(rng, n, CTypes.INT16), CTypes.INT16, _mask(rng, n, 0.3))], ["k", "x", "m"])
        t = with_schema_validity(t)
        assert all(c.validity is not None for c in (t.columns[0], t.columns[2]))
        hosts.append(t)
        parts.append(partition_device(table_to_device(t), 1, R))
    dests = [ref_dest(oracle, t, 1, R) for t in hosts]
    for d in range(R):
        seg_counts = [counts[d] for _, counts in parts]
        for ci in range(3):
            data, bitmaps = [], []
            for part, counts in parts:
                row, byte = sum(counts[:d]), sum((c + 7) // 8 for c in counts[:d])
                col = part.columns[ci]
                data.append(col.data[row: row + counts[d]])
                if col.validity is not None:
                    bitmaps.append(col.validity[byte: byte + (counts[d] + 7) // 8])
            exp = np.concatenate([np.asarray(t.columns[ci].data)[dd == d] for t, dd in zip(hosts, dests)])
            _assert_same_bytes(torch.cat(data).cpu().numpy(), exp, f"destination {d}, column {ci}")
            if ci == 1:
                continue
            merged = merge_segment_bitmaps(torch.cat(bitmaps + [torch.zeros(8, dtype=torch.uint8, device="cuda")]), seg_counts)
            got = np.unpackbits(merged.cpu().numpy(), bitorder="little")[: sum(seg_counts)].astype(bool)
            exp_mask = np.concatenate([t.columns[ci].valid_mask_numpy()[dd == d] for t, dd in zip(hosts, dests)])
            np.testing.assert_array_equal(got, exp_mask, err_msg=f"destination {d}, column {ci} bitmap")


@gpu
def test_side_stream_equals_default_stream(gpu_lib, oracle):
    """The groupby's raw-row path partitions on the current (side) stream."""
    n = geometry_rows("full_grid_plus_one", _sms())
    rng = np.random.default_rng(17)
    t = wide8_table(rng, n, 2)
    t = Table(t.columns + [_col(_values(rng, n, CTypes.UINT16), CTypes.UINT16, _mask(rng, n))], t.names + ["m"])
    dev = table_to_device(t)
    part, counts, perm = check_partition(oracle, t, 1, 16)
    small = table_to_device(wide8_table(rng, n, 3))  # the small kernel on the side stream too
    spart, scounts, sperm = partition_device(small, 1, 8, want_perm=True)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        gpart, gcounts, gperm = partition_device(dev, 1, 16, stream=s.cuda_stream, want_perm=True)
        g2part, g2counts, g2perm = partition_device(small, 1, 8, stream=s.cuda_stream, want_perm=True)
    s.synchronize()
    assert gcounts == counts and g2counts == scounts
    assert torch.equal(gperm, perm) and torch.equal(g2perm, sperm)
    for a, b in list(zip(gpart.columns, part.columns)) + list(zip(g2part.columns, spart.columns)):
        assert torch.equal(a.data.view(torch.uint8), b.data.view(torch.uint8))  # bit patterns: the payloads hold NaNs
        assert (a.validity is None) == (b.validity is None)
        if a.validity is not None:
            assert torch.equal(a.validity, b.validity)


@gpu
def test_benchmark_shape_two_columns_eight_destinations(gpu_lib, oracle):
    """2^26 rows of (int64 key, int64 value) into 8 destinations: scatter_small_kernel<2> with ~30 chunks per CTA.  The
    whole permutation and both columns are compared, so a swap of two rows inside a destination fails here."""
    n = 1 << 26
    n_ctas, tile = tile_geometry(n, _sms())
    assert tile // CHUNK >= 16
    rng = np.random.default_rng(26)
    keys = rng.integers(-(1 << 62), 1 << 62, n)
    dest = torch.from_numpy(oracle.hash_to_rank(keys, None, 8)).cuda()
    k = torch.from_numpy(keys).cuda()
    del keys
    v = torch.randint(-(1 << 62), 1 << 62, (n,), dtype=torch.int64, device="cuda", generator=torch.Generator("cuda").manual_seed(1))
    t = Table([Column(k, None, CTypes.INT64), Column(v, None, CTypes.INT64)])
    eperm = torch.sort(dest, stable=True).indices
    ecounts = torch.bincount(dest, minlength=8).tolist()
    part, counts, perm = partition_device(t, 1, 8, want_perm=True)
    assert counts == ecounts
    assert torch.equal(perm, eperm)
    assert torch.equal(part.columns[0].data, k[eperm]) and torch.equal(part.columns[1].data, v[eperm])
    del part, perm
    part2, counts2 = partition_device(t, 1, 8)
    assert counts2 == ecounts
    assert torch.equal(part2.columns[0].data, k[eperm]) and torch.equal(part2.columns[1].data, v[eperm])


@gpu
def test_hash_keys_table_beyond_one_grid_stride(gpu_lib, oracle):
    """hash_to_rank_kernel runs 8 CTAs of 256 threads per SM and strides over the rest: here each thread takes 2-3 rows."""
    stride = 8 * _sms() * 256
    n = 2 * stride + 4_099
    rng = np.random.default_rng(31)
    ks = [rng.integers(-(1 << 62), 1 << 62, n), rng.integers(0, 1000, n), rng.integers(-5, 5, n)]
    vs = [rng.random(n) > 0.1, None, rng.random(n) > 0.3]
    t = table_to_device(Table([_col(k, CTypes.INT64, None if v is None else np.packbits(v, bitorder="little")) for k, v in zip(ks, vs)]))
    for nk in (1, 2, 3):
        h, dest = hash_keys_table(t, nk, 37)
        exp = oracle.hash_keys(ks[:nk], vs[:nk])
        np.testing.assert_array_equal(h.cpu().numpy().view(np.uint32), exp)
        np.testing.assert_array_equal(dest.cpu().numpy(), (exp % 37).astype(np.int32))


# ---------------------------------------------------------------------------------------------------------------------
# argument errors
# ---------------------------------------------------------------------------------------------------------------------

def _error_case(rng, name):
    n = 1000
    i64 = lambda: _col(rng.integers(0, 100, n), CTypes.INT64)  # noqa: E731
    if name in ("int8_key", "int16_key"):
        ct = CTypes.INT8 if name == "int8_key" else CTypes.INT16
        return Table([_col(_values(rng, n, ct), ct), i64()]), 1, 4, "key columns must be 4- or 8-byte"
    if name == "n_pes_0":
        return Table([i64()]), 1, 0, r"n_pes must be in \[1, 256\]"
    if name == "n_pes_257":
        return Table([i64()]), 1, 257, r"n_pes must be in \[1, 256\]"
    if name == "five_keys":
        return Table([i64() for _ in range(5)]), 5, 4, "between 1 and 4 key columns"
    if name == "33_columns":
        return Table([i64() for _ in range(33)]), 1, 4, "between 1 and 32 columns"
    raise KeyError(name)


@gpu
@pytest.mark.parametrize("name", ["int8_key", "int16_key", "n_pes_0", "n_pes_257", "five_keys", "33_columns"])
def test_partition_argument_errors(gpu_lib, name):
    rng = np.random.default_rng(5)
    host, n_keys, n_pes, msg = _error_case(rng, name)
    dev = table_to_device(host)
    with pytest.raises(_lib.B200Error, match=msg):
        partition_device(dev, n_keys, n_pes, want_perm=True)
    # nothing written: send counts, the output table's fields and every output buffer keep their sentinels
    rc, cout, counts, outs = raw_partition(gpu_lib, dev, n_keys, n_pes)
    with pytest.raises(_lib.B200Error, match=msg):
        _lib.check(rc, "shuffle partition")
    assert list(counts) == [-7] * 260
    assert cout.ctab.n_rows == -1
    for i, o in enumerate(outs):
        assert (cout.cols[i].c_type, cout.cols[i].arr_type, cout.cols[i].length) == (-1, -1, -1)
        assert bool((o.data == 0xA5).all())


@gpu
def test_partition_rejects_host_table(gpu_lib):
    rng = np.random.default_rng(6)
    host = Table([_col(rng.integers(0, 100, 1000), CTypes.INT64), _col(rng.random(1000), CTypes.FLOAT64)])
    with pytest.raises(_lib.B200Error, match="must be device resident"):
        partition_device(host, 1, 4)
    rc, cout, counts, outs = raw_partition(gpu_lib, host, 1, 4)  # the library's own check, past the Python wrapper
    with pytest.raises(_lib.B200Error, match="b200 shuffle: the table must be device resident"):
        _lib.check(rc, "shuffle partition")
    assert list(counts) == [-7] * 260 and cout.ctab.n_rows == -1
    assert all(bool((o.data == 0xA5).all()) for o in outs)
