"""RANGE frames with value offsets (("range_between", start, end)) on the GPU.

The oracle takes each row's [lo, hi] from exact Python arithmetic over the sorted ORDER BY key, per partition and independently
of the device: integers and temporal keys as Python ints (no wrap, so a bound beyond the type's range simply passes every value),
float keys as Python floats (IEEE double, so fl(x -+ k) is what Python computes), with bisect over the partition's non-NA run.
An offset bound at an NA row is the NA peer group's boundary, and at a non-NA row one that no row satisfies leaves the frame
empty.  The functions over [lo, hi] are then evaluated by the per-[lo, hi] evaluators of tests/test_gpu_window_frames.py and
tests/test_gpu_window_moments.py: integers, min / max and gathers bit for bit, float sums within gamma_min(m-1, h) sum|v| with
h = 10 + 3 floor(log2 W), moments within the bound of DESIGN §3c."""

import bisect

import numpy as np
import pandas as pd
import pytest
import torch

from bodo_b200 import _lib
from bodo_b200._lib import ffi
from bodo_b200.streaming import window as W
from bodo_b200.table import ArrTypes, Column, CTypes, Table, np_dtype_of
from tests import test_gpu_window_frames as F
from tests import test_gpu_window_moments as M
from tests.test_gpu_sort import KEY_TYPES, col_mask, make_column
from tests.test_gpu_window_values import CHUNK, TEMPORAL, TILE, _sorted_col, bounds, float_values, out_type, run

pytestmark = pytest.mark.gpu

FLOATS = (CTypes.FLOAT32, CTypes.FLOAT64)
ORDER_TYPES = [ct for ct in KEY_TYPES if ct != CTypes.BOOL]
# every kind pair, empty-frame offsets and (0, 0)
RANGES = [(-3, 0), (0, 3), (-2, 2), (0, 0), (-5, -2), (2, 5), (5, 10), (-10, -5), (None, 3), (-3, None), (0, None), (None, -1),
          (1, None), (-(1 << 40), 1 << 40)]


@pytest.fixture(autouse=True)
def _return_device_memory():
    yield
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    _lib.lib().b200_pool_trim(torch.cuda.current_device(), 0)


def frame_of(fn):
    return fn[4] if fn[1] == "nth_value" else fn[3]


def _py(v, ct):
    return [float(x) for x in v.tolist()] if ct in FLOATS else [int(x) for x in v.tolist()]


def _magnitude(b, ct):
    """The offset's signed value in the key's arithmetic, exactly (days for DATE, ns for DATETIME / TIMEDELTA)."""
    if isinstance(b, (pd.Timedelta, np.timedelta64)):
        ns = pd.Timedelta(b).value
        return ns // 86_400_000_000_000 if ct == CTypes.DATE else ns
    return float(b) if ct in FLOATS else int(b)


def range_lo_hi(table, order, asc, nap, fr, perm, P, pe, ends):
    """Per row [lo, hi] of ("range_between", start, end), from its definition."""
    n = len(perm)
    qe = ends["range"] + 1
    Q = np.zeros(n, np.int64)
    for i in range(1, n):
        Q[i] = Q[i - 1] if qe[i] == qe[i - 1] else i
    _, s, e = fr
    lo, hi = np.empty(n, np.int64), np.empty(n, np.int64)
    if s is not None and s != 0 or e is not None and e != 0:
        v, m, ct = _sorted_col(table, order[0], perm)
        na = ~m | (np.isnan(v) if v.dtype.kind == "f" else False)
        y = _py(v, ct)
        if not asc[0]:
            y = [-x for x in y]  # y grows with the position over each partition's non-NA run
    else:
        na, ct = np.zeros(n, bool), None
    runs = {}
    for i in range(n):
        p0, p1 = int(P[i]), int(pe[i])
        for side, b in ((0, s), (1, e)):
            if b is None:
                r = p0 if side == 0 else p1 - 1
            elif b == 0 or na[i]:
                r = int(Q[i]) if side == 0 else int(qe[i]) - 1
            else:
                if p0 not in runs:
                    ok = [j for j in range(p0, p1) if not na[j]]
                    runs[p0] = (ok[0], [y[j] for j in ok])
                a0, ys = runs[p0]
                Y = y[i] + _magnitude(b, ct)  # y_i - k (PRECEDING) or y_i + k (FOLLOWING), in the key's arithmetic
                if side == 0:
                    j = bisect.bisect_left(ys, Y)
                    r = a0 + j if j < len(ys) else p1
                else:
                    j = bisect.bisect_right(ys, Y) - 1
                    r = a0 + j if j >= 0 else p0 - 1
            (lo if side == 0 else hi)[i] = r
    return lo, hi


def check(table, part, order, funcs, asc=None, nap=None, **kw):
    part, order = list(part), list(order)
    asc = [True] * len(order) if asc is None else asc
    nap = ["last"] * len(order) if nap is None else nap
    perm, P, pe, ends = bounds(table, part, order, asc, nap)
    got, sizes = run(table, part, order, asc, nap, funcs, **kw)
    for c, (vals, mask, _) in zip(table.columns, got):
        np.testing.assert_array_equal(vals.view(np.uint8), c.values_numpy()[perm].view(np.uint8))
    cache = {}
    for fn, (vals, mask, oc) in zip(funcs, got[table.n_cols:]):
        fr = frame_of(fn)
        if fr not in cache:
            cache[fr] = range_lo_hi(table, order, asc, nap, fr, perm, P, pe, ends)
        lo, hi = cache[fr]
        # the evaluators over [lo, hi]: a ("rows", None, None) frame over the "partition" [lo, hi + 1)
        sur = fn[:4] + (("rows", None, None),) if fn[1] == "nth_value" else fn[:3] + (("rows", None, None),)
        if fn[1] in M.MOMENTS:
            assert (oc.c_type, oc.arr_type) == (CTypes.FLOAT64, ArrTypes.NULLABLE_INT_BOOL), fn
            exact, valid, tol, nonfinite = M.expected(table, sur, perm, lo, hi + 1, ends)
            np.testing.assert_array_equal(mask, valid, err_msg=str(fn))
            assert np.isnan(vals[valid & nonfinite]).all(), fn
            ok = valid & ~nonfinite
            assert np.all(np.abs(vals[ok] - exact[ok]) <= tol[ok]), fn
            continue
        ct, at = out_type(table, fn)
        assert (oc.c_type, oc.arr_type) == (ct, at), fn
        assert vals.dtype == np_dtype_of(ct), fn
        exp = F.expected(table, sur, perm, lo, hi + 1, ends)
        np.testing.assert_array_equal(mask, exp[1], err_msg=str(fn))
        if len(exp) == 2:
            e = exp[0].astype(vals.dtype) if exp[0].dtype != vals.dtype else exp[0]
            np.testing.assert_array_equal(np.where(mask, vals.view(f"u{vals.itemsize}"), 0), np.where(mask, e.view(f"u{vals.itemsize}"), 0),
                                          err_msg=str(fn))
        else:
            exact, valid, tol = exp
            g, x, t = vals.astype(np.float64)[valid], exact[valid], tol[valid]
            nf = ~np.isfinite(x)
            np.testing.assert_array_equal(g[nf], x[nf], err_msg=str(fn))
            assert np.all(np.abs(g[~nf] - x[~nf]) <= t[~nf]), fn
    return got, sizes


def range_funcs(col, ct, frames, moments=True):
    fs = []
    for j, (s, e) in enumerate(frames):
        fr = ("range_between", s, e)
        names = ["count", "min", "max", "first_value", "last_value"] + ([] if ct in TEMPORAL else ["sum", "mean"])
        names += list(M.MOMENTS) if moments and ct not in TEMPORAL else []
        fs += [(f"{f}{j}", f, col, fr) for f in names]
        fs += [(f"cz{j}", "count", None, fr), (f"nth{j}", "nth_value", col, 1 + j % 3, fr)]
    return fs


# ---- every function x every range frame, ascending / descending x NA first / last, with many ties ----
@pytest.mark.parametrize("asc", [True, False])
@pytest.mark.parametrize("nap", ["first", "last"])
def test_functions_directions_and_na(gpu_lib, asc, nap):
    rng = np.random.default_rng(1000 + 2 * asc + (nap == "last"))
    n = 1500
    o = make_column(CTypes.INT32, n, rng, True, na_frac=0.1)
    o.data = np.asarray(o.data) % 40  # many ties: CURRENT ROW is the peer group, not the row
    t = Table([make_column(CTypes.INT8, n, rng, False), o, float_values(CTypes.FLOAT64, n, rng, True)], ["g", "o", "x"])
    for chunk in F.in_states(range_funcs("x", CTypes.FLOAT64, RANGES), 3):
        check(t, ["g"], ["o"], chunk, asc=[asc], nap=[nap], sizes=(777,))


def test_without_partition_by_and_integer_values(gpu_lib):
    rng = np.random.default_rng(1010)
    n = 3000
    t = Table([make_column(CTypes.INT64, n, rng, True, na_frac=0.1), make_column(CTypes.INT64, n, rng, True, small=False)], ["o", "x"])
    t.columns[0].data = np.asarray(t.columns[0].data) % 500
    for chunk in F.in_states(range_funcs("x", CTypes.INT64, RANGES[:8]), 2):
        check(t, [], ["o"], chunk)


# ---- every allowed ORDER BY type, numpy and nullable ----
@pytest.mark.parametrize("ct", ORDER_TYPES)
@pytest.mark.parametrize("nullable", [False, True])
def test_order_by_types(gpu_lib, ct, nullable):
    rng = np.random.default_rng(1100 + 2 * ct + nullable)
    n = 1200
    o = float_values(ct, n, rng, nullable) if ct in FLOATS else make_column(ct, n, rng, nullable, na_frac=0.1)
    if ct in FLOATS:
        ks = [(-0.5, 0), (-2.0, 1.0), (0, 3.5), (1.0, 4)]
    elif ct == CTypes.DATE:
        ks = [(-np.timedelta64(3, "D"), 0), (-pd.Timedelta(days=1), pd.Timedelta(days=2)), (np.timedelta64(1, "W"), None)]
    elif ct in (CTypes.DATETIME, CTypes.TIMEDELTA):
        span = int(np.ptp(np.asarray(o.data).astype(np.int64))) or 1
        w = pd.Timedelta(max(span // 50, 20), "ns")
        ks = [(-w, 0), (-w, w), (w // 10, w), (None, -w)]
    else:
        ks = [(-3, 0), (-2, 5), (0, 7), (4, None), (-(1 << 62), -1)]
    t = Table([make_column(CTypes.INT8, n, rng, False), o, make_column(CTypes.INT64, n, rng, True, small=False)], ["g", "o", "x"])
    for chunk in F.in_states(range_funcs("x", CTypes.INT64, ks, moments=False), 3):
        check(t, ["g"], ["o"], chunk, asc=[ct % 2 == 0], nap=["first" if ct % 3 else "last"])


# ---- exactness at the edges of the key's domain ----
def test_integer_extremes(gpu_lib):
    big = (1 << 63) - 1
    i64 = np.array([-(1 << 63), -(1 << 63) + 1, -5, 0, 5, big - 1, big] * 3, dtype=np.int64)
    u64 = np.array([0, 1, 5, 1 << 63, (1 << 64) - 2, (1 << 64) - 1] * 3, dtype=np.uint64)
    for o in (i64, u64):
        n = len(o)
        t = Table([Column(o), Column(np.arange(n, dtype=np.int64))], ["o", "x"])
        frames = [(-1, 0), (-big, 0), (0, big), (-big, big), (-5, 5), (big, None), (None, -big), (-(big - 1), -4)]
        fs = [(f"{f}{j}", f, "x", ("range_between", s, e)) for j, (s, e) in enumerate(frames) for f in ("sum", "count", "min")]
        fs += [(f"c{j}", "count", None, ("range_between", s, e)) for j, (s, e) in enumerate(frames)]
        for asc in (True, False):
            for chunk in F.in_states(fs, 2):
                check(t, [], ["o"], chunk, asc=[asc])


def test_float_extremes(gpu_lib):
    sub = np.finfo(np.float64).smallest_subnormal
    vals = [-np.inf, -1e300, -1.0, -0.0, 0.0, sub, 2 * sub, 1.0, 1e16, 1e16 + 2, 1e300, np.inf, np.nan]
    for dt in (np.float64, np.float32):
        with np.errstate(over="ignore"):  # +-1e300 is +-inf as float32
            o = np.array(vals * 2, dtype=dt)
        n = len(o)
        t = Table([Column(o), Column(np.arange(n, dtype=np.int64))], ["o", "x"])
        frames = [(-1.0, 0), (0, 1.0), (-sub, sub), (-1e300, 0), (-1e308, 1e308), (0.5, 2.0), (-2.0, -0.5), (0, 0)]
        fs = [(f"{f}{j}", f, "x", ("range_between", s, e)) for j, (s, e) in enumerate(frames) for f in ("sum", "first_value", "last_value")]
        for asc in (True, False):
            for nap in ("first", "last"):
                got, _ = check(t, [], ["o"], fs, asc=[asc], nap=[nap])
    # a key of 1e16 with 1.0 FOLLOWING: fl(1e16 + 1) = 1e16, so the frame is the peer group, not the 1e16 + 2 rows
    t = Table([Column(np.array([1e16, 1e16 + 2, 1e16], np.float64)), Column(np.arange(3, dtype=np.int64))], ["o", "x"])
    got, _ = run(t, [], ["o"], [True], ["last"], [("c", "count", None, ("range_between", 0, 1.0)), ("d", "count", None, ("range_between", 0, 2.0))])
    assert got[2][0].tolist() == [2, 2, 1] and got[3][0].tolist() == [3, 3, 1]


def test_na_rows_get_the_na_peer_group(gpu_lib):
    o = pd.array([1, None, 2, None, 3, 10, None], dtype="Int64")
    t = Table([Column(np.asarray(o.fillna(0), np.int64), np.packbits(~np.asarray(o.isna()), bitorder="little")),
               Column(np.arange(7, dtype=np.int64))], ["o", "x"])
    fs = [("c", "count", None, ("range_between", -100, 100)), ("s", "sum", "x", ("range_between", None, -1)),
          ("u", "count", None, ("range_between", 1, None)), ("f", "first_value", "x", ("range_between", -100, 0))]
    for nap in ("first", "last"):
        got, _ = check(t, [], ["o"], fs, nap=[nap])
        na_rows = ~got[0][1]
        assert (got[2][0][na_rows] == 3).all()  # the NA peer group: 3 rows
        ok = ~na_rows
        assert (got[2][0][ok] == 4).all()  # a non-NA row never reaches an NA row


@pytest.mark.parametrize("n", [TILE - 1, TILE + 1, 3 * TILE + 17, 20_000])
def test_tile_edges_and_large_partitions(gpu_lib, n):
    rng = np.random.default_rng(n)
    i = np.arange(n)
    t = Table([Column((i // 9000).astype(np.int64)), Column((i // 3 + rng.integers(0, 2, n)).astype(np.int64)),
               make_column(CTypes.INT32, n, rng, True, small=False), float_values(CTypes.FLOAT64, n, rng, True)], ["g", "o", "x", "f"])
    fs = [("sx", "sum", "x", ("range_between", -700, 1)), ("mx", "max", "x", ("range_between", -683, 0)),
          ("nx", "min", "x", ("range_between", 0, 1700)), ("sf", "sum", "f", ("range_between", -1000, None)),
          ("vf", "var", "f", ("range_between", -400, 400)), ("lf", "last_value", "f", ("range_between", -1, 683)),
          ("c", "count", None, ("range_between", -3, -1)), ("nt", "nth_value", "x", 2049, ("range_between", None, 700))]
    check(t, ["g"], ["o"], fs, sizes=(TILE - 1, TILE, TILE + 1))


def test_large_input_against_torch(gpu_lib):
    """2^24 + 3 rows, DATETIME-like int64 keys uniform in [0, 2^40): lo / hi from torch.searchsorted over the exact composite
    (p << 40) | t; int64 sums against cumsum differences, count(*) against hi - lo + 1."""
    n = CHUNK + 3
    dev = torch.device("cuda", 0)
    g = torch.Generator(device=dev).manual_seed(1200)
    pk = torch.randint(0, 50, (n,), generator=g, device=dev, dtype=torch.int64)
    tk = torch.randint(0, 1 << 40, (n,), generator=g, device=dev, dtype=torch.int64)
    x = torch.randint(-(1 << 40), 1 << 40, (n,), generator=g, device=dev, dtype=torch.int64)
    k1, k2 = 1 << 35, 1 << 34
    funcs = [("s", "sum", "x", ("range_between", -k1, 0)), ("c", "count", None, ("range_between", -k2, k2)),
             ("f", "sum", "x", ("range_between", k2, None))]
    st = W.init_window_state(-1, ["p"], ["t"], [True], ["last"], funcs, ["p", "t", "x"], output_batch_size=1 << 30)
    b = 3_000_000
    for r0 in range(0, n, b):
        t = Table([Column(pk[r0:r0 + b]), Column(tk[r0:r0 + b]), Column(x[r0:r0 + b])], ["p", "t", "x"])
        W.window_build_consume_batch(st, t, r0 + b >= n)
    out, last = W.window_produce_output_batch(st)
    assert last and out.n_rows == n
    got = [torch.as_tensor(c.data, device=dev) for c in out.columns]
    sp, stt, sx = got[0], got[1], got[2]
    comp = (sp << 40) | stt
    assert bool((comp[1:] >= comp[:-1]).all())
    base = sp << 40
    cs = torch.cat([torch.zeros(1, dtype=torch.int64, device=dev), torch.cumsum(sx, 0)])
    lo = torch.searchsorted(comp, base + (stt - k1).clamp(min=0))
    hi = torch.searchsorted(comp, comp, right=True) - 1
    assert torch.equal(got[3], cs[hi + 1] - cs[lo])
    lo = torch.searchsorted(comp, base + (stt - k2).clamp(min=0))
    hi = torch.searchsorted(comp, base + (stt + k2).clamp(max=(1 << 40) - 1), right=True) - 1
    assert torch.equal(got[4], hi - lo + 1)
    lo = torch.searchsorted(comp, base + stt + k2)
    pe = torch.searchsorted(comp, base + (1 << 40))
    ok = lo < pe
    assert torch.equal(torch.as_tensor(col_mask(out.columns[5]), device=dev), ok)
    assert torch.equal(got[5][ok], (cs[pe] - cs[lo])[ok])
    W.delete_window_state(st)


def test_determinism_across_batches(gpu_lib):
    rng = np.random.default_rng(1300)
    n = 30_000
    t = Table([Column(rng.integers(0, 5, n).astype(np.int64)), float_values(CTypes.FLOAT64, n, rng, True),
               float_values(CTypes.FLOAT64, n, rng, True)], ["g", "o", "x"])
    fs = [(f"{f}{j}", f, "x", ("range_between", s, e)) for f in ("sum", "mean", "var", "std_pop")
          for j, (s, e) in enumerate([(-6.0, 0), (-300.0, 300.0), (None, 77.0), (5.0, None), (0, 0)])]
    ref, _ = run(t, ["g"], ["o"], [True], ["last"], fs)
    for sizes, dev in (((1000,), True), ((4096, 17), False), ((TILE,), True)):
        got, _ = run(t, ["g"], ["o"], [True], ["last"], fs, sizes=sizes, device=dev)
        for a, b in zip(ref[3:], got[3:]):
            np.testing.assert_array_equal(a[0].view(np.uint64), b[0].view(np.uint64))
            np.testing.assert_array_equal(a[1], b[1])


def test_current_row_without_order_by_and_with_several_keys(gpu_lib):
    rng = np.random.default_rng(1400)
    n = 5000
    t = Table([Column(rng.integers(0, 4, n).astype(np.int64)), Column(rng.integers(0, 30, n).astype(np.int64)),
               Column(rng.integers(0, 3, n).astype(np.int64)), make_column(CTypes.INT64, n, rng, True, small=False)], ["g", "o", "o2", "x"])
    fs = [("a", "sum", "x", ("range_between", 0, 0)), ("b", "count", None, ("range_between", 0, None)),
          ("c", "max", "x", ("range_between", None, 0)), ("d", "first_value", "x", ("range_between", 0, None))]
    check(t, ["g"], [], fs)
    check(t, ["g"], ["o", "o2"], fs)


def test_mixed_state_keeps_old_columns(gpu_lib):
    rng = np.random.default_rng(1500)
    n = 10_000
    t = Table([make_column(CTypes.INT16, n, rng, True), make_column(CTypes.INT32, n, rng, True), float_values(CTypes.FLOAT64, n, rng, True)],
              ["g", "o", "x"])
    old = [("rn", "row_number"), ("s", "sum", "x", "rows"), ("lg", "lag", "x", 1, 0.0), ("ms", "sum", "x", ("rows", -3, 3)),
           ("nv", "nth_value", "o", 2), ("v", "var", "x", ("rows", -10, 0)), ("fv", "first_value", "x", ("rows", 1, 4))]
    new = [("rs", "sum", "x", ("range_between", -3, 3)), ("rn2", "nth_value", "o", 2, ("range_between", -100, 0)),
           ("rm", "min", "x", ("range_between", -10, 0)), ("rc", "count", None, ("range_between", -3, 3)),
           ("rv", "var", "x", ("range_between", 0, 50))]
    alone, _ = run(t, ["g"], ["o"], [True], ["last"], old)
    mixed = [old[0], new[0], old[1], old[2], new[1], old[3], new[2], old[4], new[3], old[5], new[4], old[6]]
    got, _ = run(t, ["g"], ["o"], [True], ["last"], mixed)
    for j, f in enumerate(mixed):
        if f in old:
            a, b = alone[3 + old.index(f)], got[3 + j]
            np.testing.assert_array_equal(a[0].view(f"u{a[0].itemsize}"), b[0].view(f"u{b[0].itemsize}"), err_msg=f[0])
            np.testing.assert_array_equal(a[1], b[1])
    check(t, ["g"], ["o"], new)


# ---- pandas time-based rolling ----
@pytest.mark.parametrize("with_na", [False, True])
def test_pandas_time_rolling(gpu_lib, with_na):
    """groupby(p).rolling(w, on="t", closed="both") is RANGE BETWEEN w PRECEDING AND CURRENT ROW, and closed="right" is
    (-(w - 1 ns), 0).  pandas ends a window at the current row, not at its last peer, so t is unique within a partition here."""
    from bodo_b200.physical import window

    rng = np.random.default_rng(1600 + with_na)
    n = 20_000
    p = rng.integers(0, 300, n)
    t = (rng.permutation(n).astype(np.int64) * 1_800_000_000 + rng.integers(0, 1_000_000_000, n)).astype("datetime64[ns]")
    f = rng.integers(-2000, 2000, n) / 8.0  # eighths: sums are exact in any order
    if with_na:
        f = np.where(rng.random(n) < 0.2, np.nan, f)
    df = pd.DataFrame({"p": p, "t": t, "f": f})
    w = pd.Timedelta("1h")
    both, right = ("range_between", -w, 0), ("range_between", -(w - pd.Timedelta(1, "ns")), 0)
    hows = ("sum", "mean", "count", "min", "max", "var", "std")
    funcs = [(f"{h}_b", h, "f", both) for h in hows] + [(f"{h}_r", h, "f", right) for h in hows]
    got = window(df, "p", "t", funcs, batch_size=7000)
    srt = df.sort_values(["p", "t"], kind="stable").reset_index(drop=True)
    for closed, sfx in (("both", "_b"), ("right", "_r")):
        r = srt.groupby("p", sort=False).rolling(w, on="t", closed=closed)["f"]
        for h in hows:
            e = getattr(r, h)()  # indexed by (p, t), in the sorted order
            assert (e.index.get_level_values(1) == srt["t"]).all()
            e = e.to_numpy(dtype=np.float64)
            g = got[h + sfx].to_numpy(dtype=np.float64, na_value=np.nan)
            if h == "count":
                e = np.nan_to_num(e)
            np.testing.assert_array_equal(np.isnan(g), np.isnan(e), err_msg=h + sfx)
            np.testing.assert_allclose(g, e, rtol=1e-7, atol=1e-6, err_msg=h + sfx)


# ---- errors ----
def test_device_side_validation(gpu_lib):
    L = _lib.lib()
    one = ffi.new("int32_t[]", [1, 1])

    def init(code, col, frame, kinds=(1, 2), bits=(1, 0), cts=(CTypes.INT64, CTypes.INT64), n_order=1):
        c_types = ffi.new("int8_t[]", list(cts) + [CTypes.INT64])
        a_types = ffi.new("int8_t[]", [ArrTypes.NUMPY] * (len(cts) + 1))
        fs = ffi.new("b200_window_func[]", 1)
        fs[0].code, fs[0].col, fs[0].frame, fs[0].arg = code, col, frame, 1
        fs[0].range.start_kind, fs[0].range.end_kind, fs[0].range.start_bits, fs[0].range.end_bits = kinds[0], kinds[1], bits[0], bits[1]
        np_ = len(cts) - n_order
        h = L.b200_window_state_init(-1, c_types, a_types, len(cts) + 1, np_, n_order, one, one, fs, 1, 1024, 0, ffi.NULL)
        if h != ffi.NULL:
            L.b200_delete_sort_state(h)
            return None
        return ffi.string(L.b200_last_error()).decode()

    dbl = int(np.float64(0.5).view(np.uint64))
    assert init(6, 2, 5) is None and init(15, 2, 5) is None and init(16, 2, 5, (0, 3), (0, 9)) is None
    assert init(7, -1, 5, (2, 4), cts=(CTypes.INT64, CTypes.BOOL)) is None  # no offset: any key
    assert init(6, 2, 5, (1, 3), (dbl, dbl), cts=(CTypes.INT64, CTypes.FLOAT32)) is None
    assert init(6, 2, 5, (1, 1), (5, 5)) is None and init(6, 2, 5, (3, 3), (2, 2)) is None
    for kinds in ((4, 4), (0, 0), (3, 1), (-1, 2), (2, 5)):
        assert "range bound kinds" in init(6, 2, 5, kinds)
    assert "exactly one ORDER BY key" in init(6, 2, 5, n_order=2)
    assert "exactly one ORDER BY key" in init(6, 2, 5, n_order=0)
    assert "not bool" in init(6, 2, 5, cts=(CTypes.INT64, CTypes.BOOL))
    assert "non-negative int64" in init(6, 2, 5, (1, 2), (1 << 63, 0))
    assert "non-negative int64" in init(6, 2, 5, (1, 2), (int(np.float64(-0.5).view(np.uint64)), 0), cts=(CTypes.INT64, CTypes.FLOAT64))
    assert "non-negative int64" in init(6, 2, 5, (1, 2), (int(np.float64(np.inf).view(np.uint64)), 0), cts=(CTypes.INT64, CTypes.FLOAT64))
    assert "start after frame end" in init(6, 2, 5, (1, 1), (2, 5))
    assert "start after frame end" in init(6, 2, 5, (3, 3), (5, 2))
    assert "lag and lead take no frame" in init(13, 2, 5)
    assert "no column and no frame" in init(0, -1, 5)
    assert "unknown frame (1 range, 2 rows, 3 partition, 4 rows between, 5 range between)" in init(6, 2, 6)


def test_type_errors_at_first_consume(gpu_lib):
    n = 10
    t = Table([Column(np.zeros(n, np.int64)), Column(np.arange(n, dtype=np.int64)), Column(np.arange(n, dtype=np.float64))], ["g", "o", "x"])
    f = ("s", "sum", "x", ("range_between", -pd.Timedelta("1h"), 0))
    st = W.init_window_state(-1, ["g"], ["o"], True, "last", [f], t.names)
    with pytest.raises(_lib.B200Error, match="does not fit ORDER BY key 'o'") as e:
        W.window_build_consume_batch(st, t, True)
    assert repr(f) in str(e.value)
    W.delete_window_state(st)
