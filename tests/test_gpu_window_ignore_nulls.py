"""IGNORE NULLS on FIRST_VALUE / LAST_VALUE / NTH_VALUE / LAG / LEAD on the GPU.

A cell is null when count(x) does not count it: invalid, or a float NaN.  The oracle takes each row's frame [lo, hi] (or its
partition [P, pe)) from the helpers of the RESPECT NULLS tests, independently of the device, then walks the frame row by row
(`reference`) for small inputs.  Larger inputs use `reference_vec`, the same definitions through a prefix count of the non-null
rows in numpy, which every small case also checks against `reference`.  Every result is compared bit for bit: no arithmetic
touches the values, so the chosen cell's bits (-0.0, NaN payloads) come back as they are."""

import numpy as np
import pandas as pd
import pytest
import torch

from bodo_b200 import _lib
from bodo_b200._lib import ffi
from bodo_b200.streaming import window as W
from bodo_b200.table import ArrTypes, Column, CTypes, Table
from tests import test_gpu_window_frames as F
from tests import test_gpu_window_ranges as R
from tests.test_gpu_sort import KEY_TYPES, col_mask, make_column
from tests.test_gpu_window_values import TILE, _default_for, _sorted_col, bounds, run

pytestmark = pytest.mark.gpu

FLOATS = (CTypes.FLOAT32, CTypes.FLOAT64)
ROWS_FRAMES = ["range", "rows", "partition", ("rows", -3, 0), ("rows", 0, None), ("rows", 2, 5), ("rows", -6, -4), ("rows", None, 1)]


@pytest.fixture(autouse=True)
def _return_device_memory():
    yield
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    _lib.lib().b200_pool_trim(torch.cuda.current_device(), 0)


def strip(fn):
    """(entry without its marker, IGNORE NULLS)."""
    if len(fn) > 3 and isinstance(fn[-1], str) and fn[-1] in W.NULLS_MARKERS:
        return fn[:-1], fn[-1] == "ignore_nulls"
    return fn, False


def frame_of(fn):
    if fn[1] == "nth_value":
        return fn[4] if len(fn) > 4 else "range"
    return fn[3] if len(fn) > 3 else "range"


def value_column(ct, n, rng, nullable, density):
    """Values of type ct with about `density` null cells: invalid cells (nullable) and NaN (floats), half each when both exist."""
    data = np.asarray(make_column(ct, n, rng, False).data).copy()
    null = rng.random(n) < density
    valid = np.ones(n, bool)
    if ct in FLOATS:
        data[data != data] = 1.5  # only the chosen NaN positions below are NaN
        nan = null & (rng.random(n) < 0.5) if nullable else null
        data[nan] = np.nan
        valid = ~(null & ~nan)
    else:
        assert nullable or density == 0
        valid = ~null
    if not nullable:
        return Column(np.ascontiguousarray(data), None, ct, ArrTypes.NUMPY, n)
    return Column(np.ascontiguousarray(data), np.packbits(valid, bitorder="little"), ct, ArrTypes.NULLABLE_INT_BOOL, n)


def _null(v, m):
    return ~m | np.isnan(v) if v.dtype.kind == "f" else ~m


def _default(fn, v):
    d = fn[4] if len(fn) > 4 else None
    return None if d is None else np.array([d]).astype(v.dtype)[0]


def reference(fn, v, m, P, pe, lo, hi):
    """(values, validity) of one IGNORE NULLS function, walking each row's frame or partition."""
    n, fname = len(v), fn[1]
    null = _null(v, m)
    vals, ok = np.zeros_like(v), np.zeros(n, bool)
    for i in range(n):
        if fname in ("lag", "lead"):
            k, d = fn[3] if len(fn) > 3 else 1, _default(fn, v)
            if k == 0:
                vals[i], ok[i] = v[i], m[i]
                continue
            walk = range(i - 1, P[i] - 1, -1) if fname == "lag" else range(i + 1, pe[i])
            hits = [j for j in walk if not null[j]]
            if len(hits) >= k:
                vals[i], ok[i] = v[hits[k - 1]], True
            elif d is not None:
                vals[i], ok[i] = d, True
            continue
        hits = [j for j in range(lo[i], hi[i] + 1) if not null[j]]
        want = 1 if fname == "first_value" else len(hits) if fname == "last_value" else fn[3]
        if 1 <= want <= len(hits):
            vals[i], ok[i] = v[hits[want - 1]], True
    return vals, ok


def reference_vec(fn, v, m, P, pe, lo, hi):
    """reference() through c = the exclusive prefix count of the non-null rows and pos = their positions."""
    n, fname = len(v), fn[1]
    nn = ~_null(v, m)
    c = np.concatenate([[0], np.cumsum(nn)]).astype(np.int64)
    pos = np.append(np.flatnonzero(nn), 0)
    i = np.arange(n)
    if fname in ("lag", "lead"):
        k, d = fn[3] if len(fn) > 3 else 1, _default(fn, v)
        j = c[i] - k if fname == "lag" else c[i + 1] + k - 1
        ok = j >= c[P] if fname == "lag" else j < c[pe]
        vals = np.where(ok, v[pos[np.where(ok, j, len(pos) - 1)]], d if d is not None else 0).astype(v.dtype)
        ok = ok | (d is not None)
        if k == 0:
            vals, ok = v.copy(), m.copy()
        return vals, ok
    ne = lo <= hi
    c0, c1 = c[np.where(ne, lo, 0)], c[np.where(ne, hi + 1, 0)]
    j = c0 if fname == "first_value" else c1 - 1 if fname == "last_value" else c0 + fn[3] - 1
    ok = ne & (j >= c0) & (j < c1)
    return np.where(ok, v[pos[np.where(ok, j, len(pos) - 1)]], 0).astype(v.dtype), ok


def assert_bits(got, exp, name):
    vals, mask = got[0], got[1]
    np.testing.assert_array_equal(mask, exp[1], err_msg=name)
    e = exp[0].astype(vals.dtype) if exp[0].dtype != vals.dtype else exp[0]
    u = f"u{vals.itemsize}"
    np.testing.assert_array_equal(np.where(mask, vals.view(u), 0), np.where(mask, e.view(u), 0), err_msg=name)


def check(table, part, order, funcs, asc=None, nap=None, vec=False, **kw):
    """Runs funcs and checks every IGNORE NULLS function against the reference (reference_vec when vec); returns the output."""
    part, order = list(part), list(order)
    asc = [True] * len(order) if asc is None else list(asc)
    nap = ["last"] * len(order) if nap is None else list(nap)
    perm, P, pe, ends = bounds(table, part, order, asc, nap)
    got, sizes = run(table, part, order, asc, nap, funcs, **kw)
    for c, (vals, mask, _) in zip(table.columns, got):
        np.testing.assert_array_equal(vals.view(np.uint8), c.values_numpy()[perm].view(np.uint8))
    cache = {}
    for fn, res in zip(funcs, got[table.n_cols:]):
        fn, ign = strip(fn)
        if not ign:
            continue
        oc = res[2]
        ct = table.columns[table.names.index(fn[2])].c_type
        assert (oc.c_type, oc.arr_type) == (ct, ArrTypes.NULLABLE_INT_BOOL), fn
        fr = frame_of(fn)
        key = repr(fr)
        if fn[1] in ("lag", "lead"):
            lo = hi = None
        else:
            if key not in cache:
                cache[key] = (R.range_lo_hi(table, order, asc, nap, fr, perm, P, pe, ends) if isinstance(fr, tuple) and fr[0] == "range_between"
                              else F.lo_hi(fr, P, pe, ends))
            lo, hi = cache[key]
        v, m, _ = _sorted_col(table, fn[2], perm)
        exp = reference_vec(fn, v, m, P, pe, lo, hi)
        if not vec:
            slow = reference(fn, v, m, P, pe, lo, hi)
            assert_bits((exp[0], exp[1]), slow, f"reference_vec {fn}")
        assert_bits(res, exp, str(fn))
    return got, sizes


def nav_funcs(col, ct, frames, marker="ignore_nulls"):
    fs = []
    for j, fr in enumerate(frames):
        fs += [(f"f{j}", "first_value", col, fr, marker), (f"l{j}", "last_value", col, fr, marker),
               (f"n{j}", "nth_value", col, 1 + j % 3, fr, marker)]
    d = _default_for(ct)
    fs += [("lg1", "lag", col, marker), ("ld1", "lead", col, 1, None, marker), ("lg3", "lag", col, 3, d, marker),
           ("ld2", "lead", col, 2, d, marker), ("lg0", "lag", col, 0, d, marker), ("ld0", "lead", col, 0, None, marker)]
    return fs


# ---- every function x every frame x every value type, numpy and nullable ----
@pytest.mark.parametrize("ct", KEY_TYPES)
@pytest.mark.parametrize("nullable", [False, True])
def test_value_types(gpu_lib, ct, nullable):
    rng = np.random.default_rng(2000 + ct * 2 + nullable)
    n = 2500
    density = 0.5 if nullable or ct in FLOATS else 0.0
    g = make_column(CTypes.INT8, n, rng, False)
    o = make_column(CTypes.INT16, n, rng, True, na_frac=0.1)
    t = Table([g, o, value_column(ct, n, rng, nullable, density)], ["g", "o", "x"])
    frames = ROWS_FRAMES[:6] + [("range_between", -3, 0), ("range_between", 0, 2)]
    check(t, ["g"], ["o"], nav_funcs("x", ct, frames)[:29], sizes=(777,))


@pytest.mark.parametrize("density", [0.0, 0.5, 1.0])
def test_null_densities_and_partition_edges(gpu_lib, density):
    """Partitions of 1..200 rows; besides the random nulls: an all-null partition, one with a single non-null cell in its middle,
    and partitions whose first and last rows are null."""
    rng = np.random.default_rng(2100 + int(10 * density))
    sizes = [1, 2, 3, 4, 7, 8, 13, 31, 64, 200, 5, 9, 1, 6]
    g = np.repeat(np.arange(len(sizes)), sizes)
    n = len(g)
    x = value_column(CTypes.FLOAT64, n, rng, True, density)
    valid = col_mask(x).copy()
    data = np.asarray(x.data).copy()
    starts = np.concatenate([[0], np.cumsum(sizes)[:-1]])
    valid[starts[7]:starts[7] + sizes[7]] = False                # all null
    valid[starts[8]:starts[8] + sizes[8]] = False                # one non-null cell
    valid[starts[8] + 20], data[starts[8] + 20] = True, 4.25
    valid[starts[9]], valid[starts[9] + sizes[9] - 1] = False, False  # null at both edges
    valid[starts[10]:starts[10] + 2] = False
    x = Column(data, np.packbits(valid, bitorder="little"), CTypes.FLOAT64, ArrTypes.NULLABLE_INT_BOOL, n)
    perm = rng.permutation(n)
    t = Table([Column(g[perm].astype(np.int64)), Column(np.arange(n, dtype=np.int64)[perm]),
               Column(np.asarray(x.data)[perm], np.packbits(valid[perm], bitorder="little"), CTypes.FLOAT64, ArrTypes.NULLABLE_INT_BOOL, n)],
              ["g", "o", "x"])
    got, _ = check(t, ["g"], ["o"], nav_funcs("x", CTypes.FLOAT64, ROWS_FRAMES)[:29], sizes=(100,))
    if density == 1.0:  # outside the partition with one non-null cell every frame function is NA
        other = np.ones(n, bool)
        other[starts[8]:starts[8] + sizes[8]] = False
        for fn, (vals, mask, _) in zip(nav_funcs("x", CTypes.FLOAT64, ROWS_FRAMES)[:24], got[3:]):
            assert not mask[other].any(), fn


def test_nan_is_null_and_negative_zero_keeps_its_bits(gpu_lib):
    """A valid NaN is skipped under IGNORE NULLS and returned by RESPECT NULLS; -0.0 comes back as -0.0."""
    nan, nz = np.nan, -0.0
    x = np.array([nan, nz, nan, 0.0, 7.0, nan, nz, 3.0, nan, nan], np.float64)
    valid = np.array([1, 1, 0, 1, 1, 1, 1, 0, 1, 1], bool)
    n = len(x)
    t = Table([Column(np.zeros(n, np.int64)), Column(np.arange(n, dtype=np.int64)),
               Column(x, np.packbits(valid, bitorder="little"), CTypes.FLOAT64, ArrTypes.NULLABLE_INT_BOOL, n),
               Column(x.astype(np.float32))], ["g", "o", "x", "y"])
    fs = [("ff", "last_value", "x", "rows", "ignore_nulls"), ("bf", "first_value", "x", ("rows", 0, None), "ignore_nulls"),
          ("rf", "first_value", "x", ("rows", 0, None)), ("lg", "lag", "x", 1, None, "ignore_nulls"),
          ("ffy", "last_value", "y", "rows", "ignore_nulls"), ("n2", "nth_value", "y", 2, "partition", "ignore_nulls")]
    got, _ = check(t, ["g"], ["o"], fs)
    ff, bf, rf, lg = (got[4 + j] for j in range(4))
    assert ff[1].tolist() == [False] + [True] * 9 and bf[1].tolist() == [True] * 7 + [False] * 3
    assert np.signbit(ff[0][1]) and np.signbit(ff[0][2]) and not np.signbit(ff[0][3]) and np.signbit(ff[0][6])
    assert np.isnan(rf[0][0]) and rf[1][0]  # RESPECT NULLS: the NaN is a valid cell
    assert bf[0][0] == 0 and np.signbit(bf[0][0])
    assert lg[1].tolist() == [False, False, True, True, True, True, True, True, True, True]
    assert got[8][1].tolist() == [False] + [True] * 9 and np.signbit(got[8][0][1]) and got[9][0][0] == 0 and not np.signbit(got[9][0][0])


@pytest.mark.parametrize("with_default", [False, True])
def test_lag_lead_offsets(gpu_lib, with_default):
    """k = 0 (the row itself, null or not), 1, 2, 5 and larger than every partition."""
    rng = np.random.default_rng(2200 + with_default)
    n = 3000
    t = Table([make_column(CTypes.INT16, n, rng, False), make_column(CTypes.INT32, n, rng, True, na_frac=0.05),
               value_column(CTypes.INT32, n, rng, True, 0.4), value_column(CTypes.FLOAT32, n, rng, True, 0.4)], ["g", "o", "x", "y"])
    d = 11 if with_default else None
    fs = []
    for col, dd in (("x", d), ("y", 0.5 if with_default else None)):
        for k in (0, 1, 2, 5, 1 << 30):
            fs += [(f"lg{col}{k}", "lag", col, k, dd, "ignore_nulls"), (f"ld{col}{k}", "lead", col, k, dd, "ignore_nulls")]
    check(t, ["g"], ["o"], fs, sizes=(1024,))


@pytest.mark.parametrize("part,order,asc,nap", [([], ["o"], [True], ["last"]), (["g"], [], [], []), (["g", "h"], ["o", "x"], [False, True], ["first", "last"]),
                                                (["g"], ["o"], [False], ["first"]), ([], ["x"], [True], ["first"])])
def test_key_shapes(gpu_lib, part, order, asc, nap):
    """No PARTITION BY, no ORDER BY, several keys, DESC and NA first; the value column may be a key."""
    rng = np.random.default_rng(2300 + len(part) * 3 + len(order))
    n = 3000
    t = Table([make_column(CTypes.INT8, n, rng, True, na_frac=0.1), make_column(CTypes.INT16, n, rng, True, na_frac=0.1),
               make_column(CTypes.UINT8, n, rng, False), value_column(CTypes.FLOAT64, n, rng, True, 0.5)], ["g", "o", "h", "x"])
    frames = ["range", "rows", ("rows", -2, 2)] + ([("range_between", -2, 1)] if len(order) == 1 else [])
    fs = nav_funcs("x", CTypes.FLOAT64, frames)
    fs += [("kf", "last_value", (part + order)[0], "rows", "ignore_nulls")]
    check(t, part, order, fs, asc=asc, nap=nap, sizes=(999,))


@pytest.mark.parametrize("ct", [CTypes.INT32, CTypes.FLOAT64, CTypes.DATETIME])
def test_range_between_order_keys(gpu_lib, ct):
    rng = np.random.default_rng(2400 + ct)
    n = 2000
    o = make_column(ct, n, rng, True, na_frac=0.1)
    if ct == CTypes.DATETIME:
        o.data = np.asarray(o.data) % 50
    off = (lambda k: np.timedelta64(k, "ns")) if ct == CTypes.DATETIME else (lambda k: k)
    frames = [("range_between", off(-3), 0), ("range_between", 0, off(3)), ("range_between", off(-5), off(-2)),
              ("range_between", off(2), off(5)), ("range_between", None, off(-1)), ("range_between", off(1), None),
              ("range_between", 0, 0)]
    t = Table([make_column(CTypes.INT8, n, rng, False), o, value_column(CTypes.INT64, n, rng, True, 0.5)], ["g", "o", "x"])
    fs = []
    for j, fr in enumerate(frames):
        fs += [(f"f{j}", "first_value", "x", fr, "ignore_nulls"), (f"l{j}", "last_value", "x", fr, "ignore_nulls"),
               (f"n{j}", "nth_value", "x", 2, fr, "ignore_nulls"), (f"r{j}", "first_value", "x", fr)]
    check(t, ["g"], ["o"], fs[:28], sizes=(700,))


# ---- tile edges and a large input ----
@pytest.mark.parametrize("n", [TILE - 1, TILE, TILE + 1, 3 * TILE + 5, 70_001])
def test_tile_edges(gpu_lib, n):
    """Null runs of hundreds of rows and partitions that cross the 2048-row tiles."""
    rng = np.random.default_rng(2500 + n)
    runs = np.cumsum(rng.integers(1, 600, n))
    null = (np.searchsorted(runs, np.arange(n), side="right") % 2) == 1
    x = rng.integers(-1000, 1000, n).astype(np.float64)
    x[null & (rng.random(n) < 0.5)] = np.nan
    valid = ~(null & ~np.isnan(x))
    g = np.sort(rng.integers(0, max(2, n // 1500), n))
    t = Table([Column(g.astype(np.int64)), Column(np.arange(n, dtype=np.int64)),
               Column(x, np.packbits(valid, bitorder="little"), CTypes.FLOAT64, ArrTypes.NULLABLE_INT_BOOL, n)], ["g", "o", "x"])
    frames = ["rows", ("rows", 0, None), ("rows", -700, 0), ("rows", -3000, 3000), ("range_between", -900, 900)]
    check(t, ["g"], ["o"], nav_funcs("x", CTypes.FLOAT64, frames), vec=n > 10_000, sizes=(TILE + 7,))


def test_large_input_against_torch(gpu_lib):
    """2^24 + 3 rows: ffill, bfill and lag(1) IGNORE NULLS against torch (cummax / cummin of the non-null positions)."""
    n = (1 << 24) + 3
    rng = np.random.default_rng(2600)
    g = rng.integers(0, 1 << 14, n).astype(np.int64)
    rid = np.arange(n, dtype=np.int64)
    x = rng.standard_normal(n)
    h = (rid.astype(np.uint64) * np.uint64(0x9E3779B97F4A7C15)) >> np.uint64(54)  # a hash of the row id in [0, 1024)
    x[h < 307] = np.nan  # about 30 %
    t = Table([Column(g), Column(rid), Column(x)], ["g", "o", "x"])
    fs = [("ff", "last_value", "x", "rows", "ignore_nulls"), ("bf", "first_value", "x", ("rows", 0, None), "ignore_nulls"),
          ("lg", "lag", "x", 1, None, "ignore_nulls")]
    got, _ = run(t, ["g"], ["o"], [True], ["last"], fs, sizes=(1 << 23,))
    dev = torch.device("cuda")
    sg, so, sx = (torch.as_tensor(got[j][0], device=dev) for j in range(3))
    order = torch.as_tensor(np.lexsort((rid, g)), device=dev)
    assert torch.equal(so, order)
    i = torch.arange(n, device=dev)
    P = torch.cummax(torch.where(torch.cat([torch.ones(1, dtype=torch.bool, device=dev), sg[1:] != sg[:-1]]), i, 0), 0).values
    last = torch.cat([sg[1:] != sg[:-1], torch.ones(1, dtype=torch.bool, device=dev)])
    pe = torch.flip(torch.cummin(torch.flip(torch.where(last, i + 1, n), [0]), 0).values, [0])
    nn = ~torch.isnan(sx)
    prev = torch.cummax(torch.where(nn, i, -1), 0).values
    nxt = torch.flip(torch.cummin(torch.flip(torch.where(nn, i, n), [0]), 0).values, [0])
    before = torch.cat([torch.full((1,), -1, device=dev), prev[:-1]])
    for j, (src, ok) in enumerate(((prev, prev >= P), (nxt, nxt < pe), (before, before >= P))):
        vals, mask = (torch.as_tensor(a, device=dev) for a in got[3 + j][:2])
        assert torch.equal(mask, ok), fs[j]
        exp = sx[src.clamp(0, n - 1)]
        assert torch.equal(torch.where(ok, vals.view(torch.int64), 0), torch.where(ok, exp.view(torch.int64), 0)), fs[j]
    assert 0.25 < float((~nn).double().mean()) < 0.35


# ---- states ----
def test_mixed_state_keeps_old_columns(gpu_lib):
    """IGNORE and RESPECT NULLS over one column next to ranking, scan, frame, range and bivariate functions: every other column
    is bit-identical to a state without the IGNORE NULLS functions."""
    rng = np.random.default_rng(2700)
    n = 10_000
    o = make_column(CTypes.INT32, n, rng, True)
    o.data = np.asarray(o.data) % 2000
    t = Table([make_column(CTypes.INT16, n, rng, True), o, value_column(CTypes.FLOAT64, n, rng, True, 0.4),
               make_column(CTypes.INT64, n, rng, True)], ["g", "o", "x", "z"])
    old = [("rn", "row_number"), ("s", "sum", "x", "rows"), ("lg", "lag", "x", 1, 0.0), ("fv", "first_value", "x", "rows"),
           ("lv", "last_value", "x", ("rows", -3, 0)), ("nv", "nth_value", "x", 2, ("range_between", -20, 0)),
           ("ms", "mean", "x", ("range_between", -20, 0)), ("k", "corr", "x", "z", ("rows", -3, 3)), ("ld", "lead", "z", 2)]
    new = [("ifv", "first_value", "x", "rows", "ignore_nulls"), ("ilv", "last_value", "x", ("rows", -3, 0), "ignore_nulls"),
           ("inv", "nth_value", "x", 2, ("range_between", -20, 0), "ignore_nulls"), ("ilg", "lag", "x", 1, 0.0, "ignore_nulls"),
           ("ild", "lead", "z", 2, "ignore_nulls"), ("ilz", "last_value", "z", ("range_between", -20, 0), "ignore_nulls"),
           ("rlv", "last_value", "x", ("rows", -3, 0), "respect_nulls")]
    alone, _ = run(t, ["g"], ["o"], [True], ["last"], old)
    mixed = [new[0], old[0], old[1], new[1], old[2], new[2], old[3], new[3], old[4], old[5], new[4], old[6], new[5], old[7], old[8], new[6]]
    got, _ = check(t, ["g"], ["o"], mixed)
    for j, f in enumerate(mixed):
        if f in old:
            a, b = alone[4 + old.index(f)], got[4 + j]
            np.testing.assert_array_equal(a[0].view(f"u{a[0].itemsize}"), b[0].view(f"u{b[0].itemsize}"), err_msg=f[0])
            np.testing.assert_array_equal(a[1], b[1], err_msg=f[0])
    r, l = got[4 + mixed.index(new[6])], alone[4 + old.index(old[4])]  # "respect_nulls" is RESPECT NULLS
    np.testing.assert_array_equal(r[0].view(np.uint64), l[0].view(np.uint64))
    np.testing.assert_array_equal(r[1], l[1])


def test_bit_identical_across_batch_splits(gpu_lib):
    rng = np.random.default_rng(2800)
    n = 20_000
    t = Table([make_column(CTypes.INT16, n, rng, True), make_column(CTypes.INT32, n, rng, True, na_frac=0.05),
               value_column(CTypes.FLOAT32, n, rng, True, 0.5)], ["g", "o", "x"])
    fs = nav_funcs("x", CTypes.FLOAT32, ["rows", ("rows", -5, 5), ("range_between", -4, 4)])
    a, _ = run(t, ["g"], ["o"], [True], ["last"], fs, sizes=(1 << 30,))
    for sizes in ((777,), (4096, 1, 13000)):
        b, _ = run(t, ["g"], ["o"], [True], ["last"], fs, sizes=sizes, device=sizes[0] != 777)
        for x, y in zip(a, b):
            np.testing.assert_array_equal(x[0].view(np.uint8), y[0].view(np.uint8))
            np.testing.assert_array_equal(x[1], y[1])


# ---- pandas ----
@pytest.mark.parametrize("dtype", ["float64", "Int64"])
def test_pandas_ffill_bfill(gpu_lib, dtype):
    """groupby().ffill() / ffill(limit=3) / bfill() / bfill(limit=3) are last_value / first_value IGNORE NULLS over ("rows", None,
    0) / ("rows", -3, 0) / ("rows", 0, None) / ("rows", 0, 3), ordered by a row id."""
    from bodo_b200.physical import window

    rng = np.random.default_rng(2900 + (dtype == "Int64"))
    n = 5000
    x = pd.Series(rng.integers(-100, 100, n), dtype=dtype)
    x[rng.random(n) < 0.45] = np.nan if dtype == "float64" else pd.NA
    df = pd.DataFrame({"g": rng.integers(0, 40, n), "r": np.arange(n), "x": x})
    funcs = [("ff", "last_value", "x", "rows", "ignore_nulls"), ("ff3", "last_value", "x", ("rows", -3, 0), "ignore_nulls"),
             ("bf", "first_value", "x", ("rows", 0, None), "ignore_nulls"), ("bf3", "first_value", "x", ("rows", 0, 3), "ignore_nulls")]
    got = window(df, "g", "r", funcs, batch_size=1700)
    order = np.lexsort((df["r"].to_numpy(), df["g"].to_numpy()))
    gb = df.groupby("g")["x"]
    exp = {"ff": gb.ffill(), "ff3": gb.ffill(limit=3), "bf": gb.bfill(), "bf3": gb.bfill(limit=3)}
    np.testing.assert_array_equal(got["r"].to_numpy(), order)
    for k, e in exp.items():
        g = got[k].to_numpy(dtype=np.float64, na_value=np.nan)
        np.testing.assert_array_equal(g, e.to_numpy(dtype=np.float64, na_value=np.nan)[order], err_msg=k)


# ---- the C ABI ----
def _init(L, cts, descs, nulls=None):
    n = len(cts)
    c_types = ffi.new("int8_t[]", cts)
    a_types = ffi.new("int8_t[]", [ArrTypes.NUMPY] * n)
    one = ffi.new("int32_t[]", [1])
    fs = ffi.new("b200_window_func[]", len(descs))
    for d, (code, col, frame, arg), ign in zip(fs, descs, nulls or [0] * len(descs)):
        d.code, d.col, d.frame, d.default_valid, d.arg, d.default_bits, d.ignore_nulls = code, col, frame, 0, arg, 0, ign
    return L.b200_window_state_init(-1, c_types, a_types, n, 1, 1, one, one, fs, len(descs), 1024, 0, ffi.NULL)


def test_abi_flags_and_validation(gpu_lib):
    L = _lib.lib()
    cts = [CTypes.INT64, CTypes.INT64, CTypes.FLOAT64, CTypes.INT32]
    descs = [(0, -1, 0, 0), (11, 2, 2, 0), (12, 2, 3, 0), (13, 2, 0, 1), (14, 3, 0, 2), (15, 2, 1, 2), (6, 2, 2, 0), (22, 2, 2, 3)]
    for nulls in ([0] * 8, [0, 1, 1, 1, 1, 1, 0, 0], [0, 7, -1, 1, 1, 1, 0, 0]):
        h = _init(L, cts, descs, nulls)
        assert h != ffi.NULL, ffi.string(L.b200_last_error()).decode()
        L.b200_delete_sort_state(h)
    for j, (code, *_rest) in enumerate(descs):
        if 11 <= code <= 15:
            continue
        flags = [0] * len(descs)
        flags[j] = 1
        assert _init(L, cts, descs, flags) == ffi.NULL
        assert "IGNORE NULLS takes first_value, last_value, lag, lead and nth_value only" in ffi.string(L.b200_last_error()).decode()
    assert _init(L, cts, [(25, 2, 2, 3)]) == ffi.NULL
    assert "unknown function code" in ffi.string(L.b200_last_error()).decode()


