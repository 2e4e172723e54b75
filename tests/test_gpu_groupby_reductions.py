"""prod, kurtosis, boolor_agg / booland_agg / boolxor_agg, bitor_agg / bitand_agg / bitxor_agg and count_if on the GPU against
references computed here:

  * integer prod: Python ints mod 2^64, bit-exact (uint64 multiplication is exact mod 2^64 in any order);
  * boolean, bitwise and count_if: bit-exact;
  * float prod: |got - exact| <= gamma_(n-1) |exact| against a `fractions` product (any multiplication order), float32 outputs one
    rounding more; powers of two and ±1 bit-exact;
  * kurtosis: the absolute bound kurt_tol against exact rational moments (tests/test_groupby_reductions_host.py), at offsets up to
    1e12 that power sums about 0 would fail, and pandas on ordinary data.

Each runs through the paths of tests/test_gpu_groupby_float_values.py (host, device and 32 768-row batches, a growing table, 3 key
columns, the NA key and INT64_MIN with dropna=False, the sharded exchange at 2 and 3 ranks), plus float keys, a 2^24-row batch into
1 and 30 groups (the warp reduction of prod with every lane on one slot), and all four exchange transports."""

import functools
import math
from fractions import Fraction

import numpy as np
import pandas as pd
import pytest

from bodo_b200 import _lib
from bodo_b200.streaming.groupby import (delete_groupby_state, get_metric, groupby_build_consume_batch,
                                         groupby_produce_output_batch, init_groupby_state)
from bodo_b200.table import Table

from .helpers import table_to_device
from .test_gpu_groupby_exchange import TRANSPORTS, _owned_single, _run, _states
from .test_gpu_groupby_float_values import PATHS, U, _groups, run_path
from .test_groupby_reductions_host import exact_kurt, kurt_tol

pytestmark = pytest.mark.gpu
M64 = (1 << 64) - 1


def gamma(k):
    return k * U / (1 - k * U)


def _vals_na(x):
    """(values, NA mask) of an output column (a Series, or run_path's pair)"""
    if isinstance(x, tuple):
        v, na = x
        if v.dtype == object:  # a nullable bool column: object array with pd.NA
            na = pd.isna(v)
            v = np.where(na, False, v).astype(bool)
        return np.asarray(v), np.asarray(na)
    a = x.array
    if hasattr(a, "_mask"):
        return np.asarray(a._data), np.asarray(a._mask)
    return x.to_numpy(), np.zeros(len(x), dtype=bool)


def _present(s):
    """(values, valid) of an input column; NaN of a float column is NA"""
    v, na = _vals_na(s)
    valid = ~na
    if v.dtype.kind == "f":
        valid &= ~np.isnan(v)
    return v, valid


def expect(f, s, gid, G):
    """The reference of aggregate f over input Series s per group: (values, NA mask), or for float prod (exact Fractions, n)."""
    v, valid = _present(s)
    out, na, ns = [], [], []
    for ix in _groups(gid, G):
        x = v[ix][valid[ix]]
        ns.append(len(x))
        if f == "prod":
            if v.dtype.kind == "f":
                p = Fraction(1)
                for a in x.tolist():
                    p *= Fraction(a)
                out.append(p)
            else:
                p = 1
                for a in x.tolist():
                    p = p * int(a) & M64
                out.append(p)
            na.append(False)
        elif f == "count_if":
            out.append(int(np.count_nonzero(x)))
            na.append(False)
        elif f in ("boolor_agg", "booland_agg", "boolxor_agg"):
            t = np.count_nonzero(x)
            out.append({"boolor_agg": t > 0, "booland_agg": t == len(x), "boolxor_agg": t == 1}[f] if len(x) else False)
            na.append(len(x) == 0)
        elif f in ("bitor_agg", "bitand_agg", "bitxor_agg"):
            r = {"bitor_agg": 0, "bitand_agg": M64, "bitxor_agg": 0}[f]
            for a in x.tolist():
                a = int(a) & M64
                r = r | a if f == "bitor_agg" else r & a if f == "bitand_agg" else r ^ a
            out.append(r)
            na.append(len(x) == 0)
        else:
            raise AssertionError(f)
    return out, np.array(na), np.array(ns)


def check(f, got, s, gid, G, what=""):
    v, na = _vals_na(got)
    exp, exp_na, ns = expect(f, s, gid, G)
    ctx = (f, s.name, what)
    in_dt = s.dtype.numpy_dtype if hasattr(s.dtype, "numpy_dtype") else s.dtype
    np.testing.assert_array_equal(na, exp_na, err_msg=str(ctx))
    ok = ~exp_na
    if f == "prod" and in_dt.kind == "f":
        assert v.dtype == in_dt, ctx
        e = np.array([float(p) for p in exp])
        bound = gamma(np.maximum(ns - 1, 0)) * np.abs(e) * (1 + 1e-15) + (np.abs(e) * 2.0 ** -24 if in_dt == np.float32 else 0)
        assert (np.abs(v.astype(np.float64) - e) <= bound).all(), (ctx, np.flatnonzero(np.abs(v - e) > bound)[:5])
        return
    if f == "prod":
        assert v.dtype == (np.uint64 if in_dt.kind == "u" else np.int64), (ctx, v.dtype)
    elif f == "count_if":
        assert v.dtype == np.int64, ctx
    elif f.startswith("bool"):
        assert v.dtype == np.bool_, (ctx, v.dtype)
    else:
        assert v.dtype == in_dt, (ctx, v.dtype)
    bits = 8 * v.dtype.itemsize
    want = np.array([int(e) & ((1 << bits) - 1) for e in exp], dtype=object)
    have = np.array([int(x) & ((1 << bits) - 1) for x in v.tolist()], dtype=object)
    bad = np.flatnonzero((want != have) & ok)
    assert len(bad) == 0, (ctx, bad[:5], have[bad[:5]], want[bad[:5]])


# ---- data ---------------------------------------------------------------------------------------------------------------

ALL_NA = (3, 4)  # groups whose nullable / float values are all NA


@functools.lru_cache(maxsize=None)
def _data():
    rng = np.random.default_rng(81)
    G, n = 400, 50_000
    # every group has a row; the last 20 groups have exactly one
    gid = np.concatenate([np.arange(G), rng.integers(0, G - 20, n - G)])
    gid = gid[rng.permutation(n)]
    allna = np.isin(gid, ALL_NA)

    def nullable(vals, dtype, p=0.15):
        na = (rng.random(n) < p) | allna
        return pd.arrays.BooleanArray(vals.astype(bool), na) if dtype == "bool" else pd.arrays.IntegerArray(vals.astype(dtype), na)

    def with_nan(x, p):
        x = x.copy()
        x[(rng.random(n) < p) | allna] = np.nan
        return x

    cols = {
        "i64": rng.integers(-(2 ** 62), 2 ** 62, n) * 2 + 1,  # odd: the products stay nonzero
        "u64": rng.integers(0, 2 ** 63, n, dtype=np.uint64) * np.uint64(2) + np.uint64(1),
        "i8": rng.integers(-128, 128, n).astype(np.int8),
        "i32n": nullable(rng.integers(-3, 4, n), "int32"),
        "u16n": nullable(rng.integers(0, 1 << 16, n), "uint16"),
        "b": rng.random(n) < 0.3,
        "bn": nullable(rng.random(n) < 0.02, "bool"),
        "f64": with_nan(rng.choice([0.5, 0.75, 1.0, -1.0, 1.25, -1.5, 2.0, 3.0, 0.1], n) * (rng.random(n) > 0.002), 0.05),
        "f32": with_nan((1.0 + rng.standard_normal(n) * 0.01).astype(np.float32), 0.05),
        "p2": rng.choice([0.5, 2.0, 1.0, -1.0, 0.25, -4.0], n),
        "fz": with_nan(rng.choice([0.0, 0.0, 0.0, 1.5, -2.0], n), 0.1),
    }
    return gid, G, pd.DataFrame(cols)


INT_FUNCS = (("prod", "i64"), ("prod", "u64"), ("prod", "i32n"), ("prod", "b"), ("bitor_agg", "i32n"), ("bitand_agg", "u64"),
             ("bitxor_agg", "i8"), ("bitand_agg", "u16n"), ("boolor_agg", "bn"), ("booland_agg", "i32n"), ("boolxor_agg", "b"),
             ("count_if", "bn"), ("count_if", "b"), ("boolxor_agg", "i8"))
FLOAT_FUNCS = (("prod", "f64"), ("prod", "f32"), ("prod", "p2"), ("boolor_agg", "fz"), ("booland_agg", "fz"), ("boolxor_agg", "fz"),
               ("sum", "f64"), ("mean", "f32"), ("min", "i32n"), ("count", "fz"), ("size", None), ("var", "f64"))


def _run_funcs(path, funcs, extra=()):
    """run_path over _data(); `extra` (first / last: single-column keys) joins on every path but the 3-column keys"""
    gid, G, df = _data()
    funcs = tuple(funcs) + (tuple(extra) if path != "multikey" else ())
    fn = tuple(f for f, _ in funcs)
    cols = tuple(c if c is not None else "i64" for _, c in funcs)  # (run_path gives every function an input column; size ignores it)
    got = run_path(path, gid, G, {c: df[c] for c in df.columns}, fn, cols)
    return gid, G, df, funcs, got


@pytest.mark.parametrize("path", PATHS)
def test_integer_and_bool_inputs_bit_exact(gpu_lib, path):
    gid, G, df, funcs, got = _run_funcs(path, INT_FUNCS)
    for (f, c), g in zip(funcs, got):
        check(f, g, df[c], gid, G, path)
    # one-row groups and all-NA groups
    v, na = _vals_na(got[4])  # bitor_agg of i32n
    assert na[list(ALL_NA)].all()
    v, na = _vals_na(got[11])  # count_if of bn: never NA, 0 for an all-NA group
    assert (v[list(ALL_NA)] == 0).all() and not na.any()


@pytest.mark.parametrize("path", PATHS)
def test_float_inputs_beside_existing_functions(gpu_lib, path):
    gid, G, df, funcs, got = _run_funcs(path, FLOAT_FUNCS, extra=(("first", "f64"), ("last", "i8")))
    p2 = _vals_na(got[2])[0]
    exp = np.array([float(p) for p in expect("prod", df["p2"], gid, G)[0]])
    assert (p2.view(np.int64) == exp.view(np.int64)).all()  # powers of two and ±1: exact in any order
    for (f, c), g in zip(funcs, got):
        if f in ("prod", "boolor_agg", "booland_agg", "boolxor_agg"):
            check(f, g, df[c], gid, G, path)
    # an all-NaN group's product is 1 (valid)
    v, na = _vals_na(got[0])
    assert (v[list(ALL_NA)] == 1.0).all() and not na.any()
    # the existing functions beside them
    v, valid = _present(df["f64"])
    s = np.zeros(G)
    np.add.at(s, gid[valid], v[valid])
    np.testing.assert_allclose(_vals_na(got[6])[0], s, rtol=1e-12, atol=1e-12)
    cnt = np.bincount(gid[_present(df["fz"])[1]], minlength=G)
    np.testing.assert_array_equal(_vals_na(got[9])[0], cnt)
    np.testing.assert_array_equal(_vals_na(got[10])[0], np.bincount(gid, minlength=G))
    var = pd.Series(np.where(valid, v, np.nan)).groupby(gid).var().to_numpy()
    np.testing.assert_allclose(_vals_na(got[11])[0][~np.isnan(var)], var[~np.isnan(var)], rtol=1e-9)


# ---- kurtosis -----------------------------------------------------------------------------------------------------------

OFFSETS = [0.0, 1e3, 1e6, 1e9, 1e12]
SIZES = [3, 4, 5, 7, 31, 1000, 20_000]  # (over 2^15 rows in all: the grow path's table grows)


@functools.lru_cache(maxsize=None)
def _moment_data():
    rng = np.random.default_rng(82)
    gx, gi = [], []
    for o in OFFSETS:
        for s in SIZES:
            x = o + rng.standard_normal(s) * (1.0 if s % 2 else 3.0)
            if s > 7:  # (the small groups keep exactly s values)
                x[rng.random(s) < 0.01] = np.nan
            gx.append(x)
            gi.append(np.int64(o) + rng.integers(-1000, 1000, s))
    special = [np.full(50, 1e9), np.full(4, -2.5), np.array([1.0, 2.0, np.inf, 3.0, 4.0]), np.full(5, np.nan), np.array([4.0]),
               rng.exponential(1.0, 500), rng.standard_t(4, 500)]
    gx += special
    gi += [np.full(len(s), 7, np.int64) for s in special]
    G = len(gx)
    gid = np.concatenate([np.full(len(x), g) for g, x in enumerate(gx)])
    x, i = np.concatenate(gx), np.concatenate(gi)
    perm = rng.permutation(len(gid))
    gid, x, i = gid[perm], x[perm], i[perm]
    groups = _groups(gid, G)
    return gid, G, x, i, [exact_kurt(x[ix]) for ix in groups], [exact_kurt(i[ix].astype(np.float64)) for ix in groups]


def _check_kurt(vals, na, refs, what):
    for g, (k, n, m2, r) in enumerate(refs):
        ctx = (what, g, n, vals[g], k)
        if k is None:
            assert na[g], ctx
            continue
        assert not na[g], ctx
        if math.isnan(k):
            assert math.isnan(vals[g]), ctx
        else:
            assert abs(vals[g] - k) <= kurt_tol(k, n, m2, r), ctx + (kurt_tol(k, n, m2, r),)


@pytest.mark.parametrize("path", PATHS)
def test_kurtosis_against_exact_moments(gpu_lib, path):
    """skew, kurtosis and var on one column share one moment group (five accumulator columns); kurtosis of an integer column too."""
    from .test_gpu_groupby_float_values import exact_moments, skew_tol

    gid, G, x, i, rx, ri = _moment_data()
    fn, cols = ("skew", "kurtosis", "var", "count", "kurtosis"), ("x", "x", "x", "x", "i")
    got = run_path(path, gid, G, {"x": x, "i": i}, fn, cols)
    _check_kurt(*got[1], rx, "x")
    _check_kurt(*got[4], ri, "i")
    groups = _groups(gid, G)
    for g, ix in enumerate(groups):  # skew and var of the same moment group are unchanged by the fourth power sum beside them
        r = exact_moments(x[ix])
        sk, na = got[0][0][g], got[0][1][g]
        assert na == (r["skew"] is None), g
        if r["skew"] is not None and math.isfinite(r["skew"]):
            assert abs(sk - r["skew"]) <= skew_tol(r), (g, sk, r["skew"])
    np.testing.assert_array_equal(got[3][0], [r[1] for r in rx])
    c0 = len(OFFSETS) * len(SIZES)
    assert got[1][0][c0] == 0.0 and got[1][0][c0 + 1] == 0.0 and got[4][0][c0] == 0.0  # constant groups: exactly 0


def test_kurtosis_and_prod_match_pandas_through_groupby_agg(gpu_lib):
    from bodo_b200.physical import groupby_agg

    rng = np.random.default_rng(83)
    n = 200_000
    df = pd.DataFrame({"k": rng.integers(0, 700, n), "x": rng.gamma(2.0, 3.0, n), "y": rng.standard_normal(n),
                       "v": rng.choice([1, -1, 1, 1, 3], n).astype(np.int64), "z": rng.choice([0.5, 2.0, 1.0, -1.0], n)})
    got = groupby_agg(df, "k", [("kx", "x", "kurtosis"), ("ky", "y", "kurtosis"), ("pv", "v", "prod"), ("pz", "z", "prod"),
                                ("bo", "y", "boolor_agg")], batch_size=30_000).sort_values("k").reset_index(drop=True)
    g = df.groupby("k")
    exp = pd.DataFrame({"kx": g.x.apply(pd.Series.kurt), "ky": g.y.apply(pd.Series.kurt), "pv": g.v.prod(), "pz": g.z.prod()}).reset_index()
    np.testing.assert_array_equal(got.k.to_numpy(), exp.k.to_numpy())
    for c in ("kx", "ky"):
        np.testing.assert_allclose(got[c].to_numpy(dtype=np.float64), exp[c].to_numpy(), rtol=1e-9, atol=1e-9, err_msg=c)
    np.testing.assert_array_equal(got.pv.to_numpy(), exp.pv.to_numpy())
    np.testing.assert_array_equal(got.pz.to_numpy(), exp.pz.to_numpy())
    assert got.bo.to_numpy(dtype=bool).all()


# ---- float keys, dropna=False -------------------------------------------------------------------------------------------

@pytest.mark.parametrize("dropna", [False, True])
def test_float_keys_with_nan_key(gpu_lib, dropna):
    gid, G, df = _data()
    key = np.where(gid == 0, np.nan, gid * 0.5 - 3.0)  # group 0: the NaN key
    funcs = (("prod", "i64"), ("kurtosis", "f64"), ("bitxor_agg", "i32n"), ("booland_agg", "fz"), ("count_if", "bn"), ("prod", "f64"))
    t = Table.from_pandas(pd.DataFrame({"k": key.astype(np.float32), **{c: df[c] for c in df.columns}}))
    names = list(t.names)
    st = init_groupby_state(-1, (0,), tuple(f for f, _ in funcs), tuple(range(len(funcs) + 1)), tuple(names.index(c) for _, c in funcs),
                            dropna=dropna, output_batch_size=1 << 30)
    for r0 in range(0, t.n_rows, 20_000):
        b = t.slice(r0, min(t.n_rows, r0 + 20_000))
        groupby_build_consume_batch(st, table_to_device(b) if r0 % 40_000 == 0 else b, r0 + 20_000 >= t.n_rows, True)
    out, _ = groupby_produce_output_batch(st, True)
    out = out.to_pandas()
    delete_groupby_state(st)
    k = out.iloc[:, 0].to_numpy(dtype=np.float64)
    g = np.where(np.isnan(k), 0, np.round((k + 3.0) / 0.5)).astype(np.int64)
    order = np.argsort(g)
    np.testing.assert_array_equal(g[order], np.arange(1 if dropna else 0, G))
    keep = gid != 0 if dropna else np.ones(len(gid), bool)
    sub, gsub = df[keep].reset_index(drop=True), gid[keep]
    if dropna:  # shift group ids so that group 1 is output row 0
        gsub, Gs = gsub - 1, G - 1
    else:
        Gs = G
    for j, (f, c) in enumerate(funcs):
        col = out.iloc[order, 1 + j].reset_index(drop=True)
        if f == "kurtosis":
            v, na = _vals_na(col)
            _check_kurt(v, na, [exact_kurt(sub[c].to_numpy()[ix]) for ix in _groups(gsub, Gs)], "float key")
        else:
            check(f, col, sub[c], gsub, Gs, "float key")


# ---- one 2^24-row batch into 1 and 30 groups ----------------------------------------------------------------------------

@pytest.mark.parametrize("G", [1, 30])
def test_big_batch_few_groups(gpu_lib, G):
    """Every lane of a warp updates one slot: prod's warp reduction and CAS loop, and the word atomics, at 2^24 rows."""
    n = 1 << 24
    rng = np.random.default_rng(84 + G)
    kk = rng.integers(0, G, n)
    r = rng.random(n)
    df = pd.DataFrame({
        "k": kk,
        "v": rng.integers(-(2 ** 62), 2 ** 62, n) * 2 + 1,  # odd: the products stay nonzero
        # powers of two and ±1 whose exponent stays in range: bit-exact in any order
        "z": np.where(r < 1e-4, 2.0, np.where(r < 2e-4, 0.5, np.where(r < 0.6, 1.0, -1.0))),
        "y": 1.0 + (rng.random(n) - 0.5) * 1e-6,
        "b": rng.random(n) < 1e-6})
    t = table_to_device(Table.from_pandas(df))
    funcs = (("prod", 1), ("prod", 2), ("prod", 3), ("boolor_agg", 4), ("count_if", 4), ("bitand_agg", 1), ("booland_agg", 1))
    st = init_groupby_state(-1, (0,), tuple(f for f, _ in funcs), tuple(range(len(funcs) + 1)), tuple(c for _, c in funcs),
                            output_batch_size=1 << 30)
    groupby_build_consume_batch(st, t, True, True)
    out, _ = groupby_produce_output_batch(st, True)
    out = out.to_pandas().sort_values("k").reset_index(drop=True)
    m = {w: get_metric(st, w) for w in (8, 10, 12, 14)}
    delete_groupby_state(st)
    assert all(x == 0 for x in m.values()), m  # the direct kernel
    order = np.argsort(kk, kind="stable")
    starts = np.searchsorted(kk[order], np.arange(G))
    red = lambda ufunc, a: ufunc.reduceat(a[order], starts)
    np.testing.assert_array_equal(out.k.to_numpy(), np.arange(G))
    vu = df.v.to_numpy().view(np.uint64)
    np.testing.assert_array_equal(out.iloc[:, 1].to_numpy().view(np.uint64), red(np.multiply, vu))  # wraps mod 2^64
    zz = df.z.to_numpy()
    np.testing.assert_array_equal(out.iloc[:, 2].to_numpy().view(np.int64), red(np.multiply, zz).view(np.int64))
    yy = red(np.multiply, df.y.to_numpy())  # any order is within gamma_(n-1) of the exact product, so within 2 gamma of this one
    cnt = np.bincount(kk, minlength=G)
    assert (np.abs(out.iloc[:, 3].to_numpy() - yy) <= 2.01 * gamma(cnt - 1) * np.abs(yy)).all()
    bb = df.b.to_numpy()
    nb = np.bincount(kk[bb], minlength=G)
    np.testing.assert_array_equal(_vals_na(out.iloc[:, 4])[0], nb > 0)
    np.testing.assert_array_equal(out.iloc[:, 5].to_numpy(), nb)
    np.testing.assert_array_equal(_vals_na(out.iloc[:, 6])[0].view(np.uint64), red(np.bitwise_and, vu))
    assert _vals_na(out.iloc[:, 7])[0].all()  # odd values are all true


# ---- the sharded exchange, every transport ------------------------------------------------------------------------------

@pytest.mark.parametrize("transport", list(TRANSPORTS))
def test_sharded_every_transport(gpu_lib, oracle, transport):
    gid, G, df = _data()
    R = 3
    funcs = INT_FUNCS[:9] + (("prod", "f64"), ("kurtosis", "f64"), ("skew", "f64"), ("count_if", "b"))  # 16 accumulator columns
    full = pd.concat([pd.DataFrame({"k": gid.astype(np.int64) * 1000003}), df], axis=1)
    names = list(full.columns)
    states = _states(full, 1, tuple(f for f, _ in funcs), tuple(names.index(c) for _, c in funcs), R, expected_groups=16)
    outs, _ = _run(states, transport)
    _owned_single(outs, R, lambda key: oracle.hash_to_rank(key.to_numpy(), None, R))
    got = pd.concat(outs, ignore_index=True)
    g = got.iloc[:, 0].to_numpy() // 1000003
    order = np.argsort(g)
    np.testing.assert_array_equal(g[order], np.arange(G))
    x = df["f64"].to_numpy()
    for j, (f, c) in enumerate(funcs):
        col = got.iloc[order, 1 + j].reset_index(drop=True)
        if f == "kurtosis":
            _check_kurt(*_vals_na(col), [exact_kurt(x[ix]) for ix in _groups(gid, G)], transport)
        elif f == "skew":
            ref = pd.Series(x).groupby(gid).skew().to_numpy()
            v = _vals_na(col)[0]
            ok = ~np.isnan(ref)
            np.testing.assert_allclose(v[ok], ref[ok], rtol=1e-7, atol=1e-9)
        else:
            check(f, col, df[c], gid, G, transport)


# ---- refusals -----------------------------------------------------------------------------------------------------------

REFUSALS = [("prod", "dt", "datetime"), ("prod", "td", "timedelta"), ("prod", "d", "date"), ("boolor_agg", "dt", "datetime"),
            ("booland_agg", "td", "timedelta"), ("boolxor_agg", "d", "date"), ("bitor_agg", "f64", "float64"),
            ("bitand_agg", "f32", "float32"), ("bitxor_agg", "b", "bool"), ("bitor_agg", "dt", "datetime"),
            ("count_if", "i64", "int64"), ("count_if", "f64", "float64")]


@pytest.mark.parametrize("fn,col,tname", REFUSALS)
def test_input_type_refusals(gpu_lib, fn, col, tname):
    import datetime

    import pyarrow as pa

    n = 8
    dates = pd.array([datetime.date(2020, 1, 1 + i) for i in range(n)], dtype=pd.ArrowDtype(pa.date32()))
    df = pd.DataFrame({"k": np.arange(n, dtype=np.int64), "dt": pd.to_datetime(np.arange(n), unit="s"),
                       "td": pd.to_timedelta(np.arange(n), unit="s"), "d": dates,
                       "f64": np.ones(n), "f32": np.ones(n, np.float32), "b": np.ones(n, bool), "i64": np.ones(n, np.int64)})
    t = Table.from_pandas(df)
    st = init_groupby_state(-1, (0,), (fn,), (0, 1), (list(df.columns).index(col),))
    with pytest.raises(_lib.B200Error, match=rf"{fn} does not take a {tname} column"):
        groupby_build_consume_batch(st, t, True, True)
    delete_groupby_state(st)
