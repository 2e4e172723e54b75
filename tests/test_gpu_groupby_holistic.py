"""mode, percentile_cont and percentile_disc on the GPU, bit-exact against the numpy restatement of
tests/test_groupby_holistic_host.py (itself pinned against pandas and numpy): every value type (numpy and nullable), 1..4 key
columns with float keys and dropna both ways, mixed with other aggregates, one-row and empty batches (an empty first batch too),
table growth, a 2^24 + 3-row input with one group holding 90 % of the rows against a torch sort, identical output over runs and
batch splits, and the sharded form on lock-step ranks of one GPU (every key type, the owner of every group, both refusals)."""

import math

import numpy as np
import pytest

from bodo_b200 import _lib
from bodo_b200.streaming.groupby import (delete_groupby_state, get_metric, groupby_build_consume_batch,
                                         groupby_produce_output_batch, init_groupby_state)
from bodo_b200.table import ArrTypes, Column, CTypes, Table

from .helpers import table_to_device
from .test_groupby_holistic_host import bits, present, reference

pytestmark = pytest.mark.gpu
NP = {CTypes.INT8: np.int8, CTypes.UINT8: np.uint8, CTypes.INT16: np.int16, CTypes.UINT16: np.uint16, CTypes.INT32: np.int32,
      CTypes.UINT32: np.uint32, CTypes.INT64: np.int64, CTypes.UINT64: np.uint64, CTypes.FLOAT32: np.float32,
      CTypes.FLOAT64: np.float64, CTypes.BOOL: np.bool_, CTypes.DATE: np.int32, CTypes.DATETIME: np.int64,
      CTypes.TIMEDELTA: np.int64}
INTS = (CTypes.INT8, CTypes.UINT8, CTypes.INT16, CTypes.UINT16, CTypes.INT32, CTypes.UINT32, CTypes.INT64, CTypes.UINT64)
FLOATS = (CTypes.FLOAT32, CTypes.FLOAT64)
TEMPORAL = (CTypes.DATE, CTypes.DATETIME, CTypes.TIMEDELTA)
TAKES = {"percentile_cont": INTS + FLOATS, "percentile_disc": INTS + FLOATS + TEMPORAL,
         "mode": INTS + FLOATS + TEMPORAL + (CTypes.BOOL,)}


@pytest.fixture(scope="module")
def gpu_lib():
    _lib.require_gpu()
    return _lib.lib()


# ================================================================================================ data
def gen(ct, n, rng, nullable, groups=None):
    """n values of c-type ct (few distinct ones, so mode has ties; floats with NaN, ±inf, -0.0 and 0.0) and a validity mask."""
    dt = NP[ct]
    if ct == CTypes.BOOL:
        v = rng.integers(0, 2, n).astype(bool)
    elif ct in FLOATS:
        pool = np.array([np.nan, np.inf, -np.inf, -0.0, 0.0, 1.5, -2.25, 3.0, 1e30, -1e-30], dtype=np.float64)
        v = np.where(rng.random(n) < 0.3, rng.choice(pool, n), np.round(rng.normal(0, 4, n), 1)).astype(dt)
    else:
        info = np.iinfo(dt)
        big = rng.integers(info.min, info.max, n, dtype=dt, endpoint=True)
        small = rng.integers(max(info.min, -5), min(info.max, 5) + 1, n).astype(dt)
        v = np.where(rng.random(n) < 0.5, small, big).astype(dt)
    valid = rng.random(n) > 0.2 if nullable else None
    return v, valid


def column(v, valid, ct):
    if valid is None:
        return Column(np.ascontiguousarray(v), None, ct, ArrTypes.NUMPY)
    return Column(np.ascontiguousarray(v), np.packbits(valid, bitorder="little"), ct, ArrTypes.NULLABLE_INT_BOOL)


def key_canon(vals, valids, float_key):
    """The group of every row as a tuple (None for an NA key; a float key's NaN is NA, -0.0 is 0.0)."""
    n = len(vals[0])
    out = []
    for i in range(n):
        t = []
        for v, ok, fl in zip(vals, valids, float_key):
            x = v[i]
            if (ok is not None and not ok[i]) or (fl and np.isnan(x)):
                t.append(None)
            else:
                t.append(float(x) + 0.0 if fl else int(x))
        out.append(tuple(t))
    return out


# ================================================================================================ running a state
def run_state(t, nk, funcs, percentiles, batches, dropna=True, expected_groups=0, device_every=2, output_batch_size=1 << 30):
    """Consumes host table t cut at `batches` (a list of row counts, zero allowed; every device_every-th non-empty batch is staged on
    the device), produces every output batch.  funcs: (name, logical column).  Returns (columns as (values, valid) lists, state
    metrics)."""
    st = init_groupby_state(-1, tuple(range(nk)), tuple(f for f, _ in funcs), tuple(range(len(funcs) + 1)),
                            tuple(c for _, c in funcs), dropna=dropna, expected_groups=expected_groups,
                            output_batch_size=output_batch_size, device=0, percentiles=percentiles)
    try:
        lo = 0
        for i, n in enumerate(batches):
            b = t.slice(lo, lo + n)
            lo += n
            if n and i % device_every == 0:
                b = table_to_device(b)
            groupby_build_consume_batch(st, b, i == len(batches) - 1, True)
        assert lo == t.n_rows
        cols = None
        while True:
            out, last = groupby_produce_output_batch(st, True)
            part = [(c.values_numpy().copy(), c.valid_mask_numpy(), c.c_type, c.arr_type) for c in out.columns]
            if cols is None:
                cols = [[p] for p in part]
            else:
                for q, p in enumerate(part):
                    cols[q].append(p)
            if last:
                break
        merged = []
        for parts in cols:
            v = np.concatenate([p[0] for p in parts])
            ok = None if parts[0][1] is None else np.concatenate([p[1] for p in parts])
            merged.append((v, ok, parts[0][2], parts[0][3]))
        metrics = {m: get_metric(st, m) for m in (0, 3, 20, 21)}
        return merged, metrics
    finally:
        delete_groupby_state(st)


def expected(t, nk, funcs, percentiles, dropna):
    """{group key tuple: [reference result per holistic function (None = NA)]}, over host table t."""
    keys = [t.columns[j] for j in range(nk)]
    kv = [c.values_numpy() for c in keys]
    kok = [c.valid_mask_numpy() for c in keys]
    fl = [c.c_type in FLOATS for c in keys]
    g = key_canon(kv, kok, fl)
    rows = {}
    for i, k in enumerate(g):
        if dropna and any(x is None for x in k):
            continue
        rows.setdefault(k, []).append(i)
    qs = iter(percentiles or ())
    fq = [(f, c, next(qs) if f in ("percentile_cont", "percentile_disc") else None) for f, c in funcs]
    out = {}
    for k, ix in rows.items():
        ix = np.array(ix)
        res = []
        for f, c, q in fq:
            col = t.columns[c]
            ok = col.valid_mask_numpy()
            res.append(reference(f, present(col.values_numpy()[ix], None if ok is None else ok[ix]), q))
        out[k] = res
    return out


def result_bits(v, ok, i, ct):
    if ok is not None and not ok[i]:
        return None
    x = v[i]
    return bits(float(x)) if ct in FLOATS else int(x)


def check(cols, t, nk, funcs, percentiles, dropna, hol=None):
    """The holistic outputs (function indices `hol`, default: all) equal the reference per group, bit for bit."""
    hol = [j for j, (f, _) in enumerate(funcs) if f in ("mode", "percentile_cont", "percentile_disc")] if hol is None else hol
    want = expected(t, nk, funcs, percentiles, dropna)
    kfl = [cols[j][2] in FLOATS for j in range(nk)]
    got_keys = key_canon([cols[j][0] for j in range(nk)], [cols[j][1] for j in range(nk)], kfl)
    assert len(got_keys) == len(set(got_keys)) == len(want), (len(got_keys), len(want))
    for i, k in enumerate(got_keys):
        for j in hol:
            v, ok, ct, at = cols[nk + j]
            assert at == ArrTypes.NULLABLE_INT_BOOL and ok is not None
            w = want[k][j]
            exp = None if w is None else bits(float(w)) if ct in FLOATS else int(w)
            assert result_bits(v, ok, i, ct) == exp, (funcs[j], k, v[i], w)
            if funcs[j][0] == "percentile_cont":
                assert ct == CTypes.FLOAT64
            else:
                assert ct == t.columns[funcs[j][1]].c_type


def make_table(key_cols, val_cols):
    cols = [column(v, ok, ct) for v, ok, ct in key_cols + val_cols]
    return Table(cols, [f"c{j}" for j in range(len(cols))])


def cuts(n, rng, k):
    c = np.sort(rng.integers(0, n + 1, k - 1))
    return np.diff(np.concatenate([[0], c, [n]])).astype(int).tolist()


# ================================================================================================ value types
@pytest.mark.parametrize("nullable", [False, True])
@pytest.mark.parametrize("ct", INTS + FLOATS + TEMPORAL + (CTypes.BOOL,))
def test_every_value_type(gpu_lib, ct, nullable):
    rng = np.random.default_rng(ct * 2 + nullable)
    n = 6000
    key = rng.integers(0, 150, n).astype(np.int64)
    v, ok = gen(ct, n, rng, nullable)
    t = make_table([(key, None, CTypes.INT64)], [(v, ok, ct)])
    funcs, qs = [], []
    for f, takes in TAKES.items():
        if ct in takes:
            for q in ((0.0, 1 / 3, 0.5, 1.0) if f != "mode" else (None,)):
                funcs.append((f, 1))
                if q is not None:
                    qs.append(q)
    cols, _ = run_state(t, 1, funcs, tuple(qs) or None, cuts(n - 1, rng, 5) + [0, 1, 0])
    check(cols, t, 1, funcs, qs, True)


@pytest.mark.parametrize("f", ["percentile_cont", "percentile_disc"])
def test_type_refusals(gpu_lib, f):
    n = 8
    t = make_table([(np.arange(n, dtype=np.int64), None, CTypes.INT64)], [(np.zeros(n, dtype=bool), None, CTypes.BOOL)])
    with pytest.raises(_lib.B200Error, match=f"{f} does not take a bool column"):
        run_state(t, 1, [(f, 1)], (0.5,), [n])


# ================================================================================================ keys
KEYSETS = {
    "int64": (CTypes.INT64,), "float64": (CTypes.FLOAT64,), "float32": (CTypes.FLOAT32,), "int8": (CTypes.INT8,),
    "2: int32-float64": (CTypes.INT32, CTypes.FLOAT64), "3: uint16-date-int64": (CTypes.UINT16, CTypes.DATE, CTypes.INT64),
    "4: bool-float32-int64-uint8": (CTypes.BOOL, CTypes.FLOAT32, CTypes.INT64, CTypes.UINT8),
}


def gen_key(ct, n, rng, nullable):
    if ct in FLOATS:
        pool = np.array([np.nan, -0.0, 0.0, 1.5, -3.0, np.inf, 2.0, 7.25], dtype=NP[ct])
        return rng.choice(pool, n), None
    if ct == CTypes.BOOL:
        v = rng.integers(0, 2, n).astype(bool)
    else:
        v = rng.integers(0, 9, n).astype(NP[ct])
        v[rng.random(n) < 0.05] = np.iinfo(NP[ct]).min
    return v, (rng.random(n) > 0.1 if nullable else None)


@pytest.mark.parametrize("dropna", [True, False])
@pytest.mark.parametrize("keyset", list(KEYSETS))
def test_keys(gpu_lib, keyset, dropna):
    kts = KEYSETS[keyset]
    rng = np.random.default_rng(len(keyset) * 7 + dropna)
    n = 5000
    keys = [(*gen_key(ct, n, rng, ct not in FLOATS), ct) for ct in kts]
    v, ok = gen(CTypes.FLOAT64, n, rng, True)
    w, wok = gen(CTypes.INT32, n, rng, False)
    t = make_table(keys, [(v, ok, CTypes.FLOAT64), (w, wok, CTypes.INT32)])
    nk = len(kts)
    funcs = [("percentile_cont", nk), ("mode", nk + 1), ("percentile_disc", nk), ("percentile_disc", nk + 1), ("mode", nk)]
    qs = (0.25, 0.9, 0.5)
    cols, _ = run_state(t, nk, funcs, qs, cuts(n, rng, 4), dropna=dropna)
    check(cols, t, nk, funcs, qs, dropna)


# ================================================================================================ mixed states, batches, growth
def test_mixed_with_other_aggregates(gpu_lib):
    rng = np.random.default_rng(5)
    n = 20000
    key = rng.integers(0, 300, n).astype(np.int64)
    v, ok = gen(CTypes.FLOAT64, n, rng, True)
    w = rng.integers(-50, 50, n).astype(np.int64)
    t = make_table([(key, None, CTypes.INT64)], [(v, ok, CTypes.FLOAT64), (w, None, CTypes.INT64)])
    funcs = [("sum", 2), ("percentile_cont", 1), ("mean", 1), ("nunique", 2), ("mode", 2), ("first", 2), ("percentile_disc", 2)]
    qs = (0.5, 0.75)
    cols, _ = run_state(t, 1, funcs, qs, cuts(n, rng, 6))
    check(cols, t, 1, funcs, qs, True)
    kv = cols[0][0]
    for i in rng.integers(0, len(kv), 50):
        ix = key == kv[i]
        assert cols[1][0][i] == w[ix].sum()
        assert cols[4][0][i] == len(np.unique(w[ix]))
        assert cols[6][0][i] == w[ix][0]
        vv = v[ix][ok[ix] & ~np.isnan(v[ix])]
        if len(vv) and np.isfinite(vv).all():
            assert math.isclose(cols[3][0][i], vv.mean(), rel_tol=1e-9, abs_tol=1e-300)


@pytest.mark.parametrize("first", ["empty", "one_row"])
def test_empty_and_one_row_batches_and_growth(gpu_lib, first):
    rng = np.random.default_rng(9)
    n = 300_000
    key = rng.integers(0, 100_000, n).astype(np.int64)
    v, ok = gen(CTypes.INT64, n, rng, True)
    t = make_table([(key, None, CTypes.INT64)], [(v, ok, CTypes.INT64)])
    funcs = [("percentile_cont", 1), ("mode", 1), ("percentile_disc", 1)]
    qs = (0.5, 0.1)
    head = [0, 0] if first == "empty" else [1, 0, 1]
    batches = head + [1, 0] + cuts(n - sum(head) - 1, rng, 7)
    cols, m = run_state(t, 1, funcs, qs, batches, expected_groups=16)
    assert m[3] > 0  # the table grew while ids moved with their slots
    assert m[20] == int(ok.sum())
    check(cols, t, 1, funcs, qs, True)


def test_all_na_groups_and_empty_input(gpu_lib):
    n = 64
    key = np.arange(n, dtype=np.int64) % 4
    v = np.full(n, np.nan)
    v[key == 1] = 2.5
    t = make_table([(key, None, CTypes.INT64)], [(v, None, CTypes.FLOAT64)])
    funcs = [("percentile_cont", 1), ("mode", 1)]
    cols, _ = run_state(t, 1, funcs, (0.5,), [n])
    check(cols, t, 1, funcs, (0.5,), True)
    assert int(cols[1][1].sum()) == 1
    e = t.slice(0, 0)
    cols, m = run_state(e, 1, funcs, (0.5,), [0, 0])
    assert len(cols[0][0]) == 0 and m[21] == 0


def test_identical_over_runs_and_batch_splits(gpu_lib):
    rng = np.random.default_rng(11)
    n = 200_000
    key = rng.integers(0, 5000, n).astype(np.int64)
    v, ok = gen(CTypes.FLOAT32, n, rng, True)
    t = make_table([(key, None, CTypes.INT64)], [(v, ok, CTypes.FLOAT32)])
    funcs = [("percentile_cont", 1), ("mode", 1), ("percentile_disc", 1)]
    qs = (0.3, 0.7)
    runs = [run_state(t, 1, funcs, qs, b)[0] for b in ([n], [n], cuts(n, rng, 9), [n // 2, 0, n - n // 2])]

    def as_dict(cols):
        return {int(cols[0][0][i]): tuple(result_bits(c[0], c[1], i, c[2]) for c in cols[1:]) for i in range(len(cols[0][0]))}

    base = as_dict(runs[0])
    for r in runs[1:]:
        assert as_dict(r) == base
    check(runs[0], t, 1, funcs, qs, True)


# ================================================================================================ skew: one group, 90 % of the rows
def test_one_group_holds_most_rows_against_torch_sort(gpu_lib):
    import torch

    n = (1 << 24) + 3
    g = torch.Generator(device="cuda").manual_seed(3)
    key = torch.randint(1, 1 << 20, (n,), device="cuda", generator=g, dtype=torch.int64)
    key[torch.rand(n, device="cuda", generator=g) < 0.9] = 0
    val = torch.randint(-1000, 1000, (n,), device="cuda", generator=g, dtype=torch.int64)
    t = Table([Column(key, None, CTypes.INT64, ArrTypes.NUMPY, n), Column(val, None, CTypes.INT64, ArrTypes.NUMPY, n)], ["k", "v"])
    funcs = [("percentile_cont", 1), ("percentile_disc", 1), ("mode", 1)]
    qs = (0.5, 0.99)
    st = init_groupby_state(-1, (0,), tuple(f for f, _ in funcs), (0, 1, 2, 3), (1, 1, 1), device=0, percentiles=qs,
                            output_batch_size=1 << 30)
    try:
        groupby_build_consume_batch(st, t, True, True)
        out, last = groupby_produce_output_batch(st, True)
        assert last
        ok_, pc, pd_, md = (c.values_numpy().copy() for c in out.columns)
    finally:
        delete_groupby_state(st)
    # the reference: sort (key, value) with torch, per group read the positions the definitions name
    order = torch.argsort(val, stable=True)
    order = order[torch.argsort(key[order], stable=True)]
    ks, vs = key[order], val[order]
    uk, counts = torch.unique_consecutive(ks, return_counts=True)
    starts = torch.cumsum(counts, 0) - counts
    uk, counts, starts = uk.cpu().numpy(), counts.cpu().numpy(), starts.cpu().numpy()
    vs_h = vs.cpu().numpy()
    pos = {int(k): i for i, k in enumerate(ok_)}
    assert len(pos) == len(uk)
    check_ix = [int(np.argmax(counts))] + list(np.random.default_rng(0).integers(0, len(uk), 2000))
    for j in check_ix:
        s, m = int(starts[j]), int(counts[j])
        V = vs_h[s:s + m]
        i = pos[int(uk[j])]
        assert bits(float(pc[i])) == bits(reference("percentile_cont", V, qs[0]))
        assert int(pd_[i]) == int(reference("percentile_disc", V, qs[1]))
        assert int(md[i]) == int(reference("mode", V))


# ================================================================================================ sharded: lock-step ranks
@pytest.fixture
def lockstep(monkeypatch):
    from tests.test_gpu_join_sharded import LockstepGroup

    return lambda n: LockstepGroup(n).install(monkeypatch)


def run_sharded(lockstep, R, t, nk, funcs, qs, rng, dropna=True):
    """Rank r consumes a random share of t in random batches (empty ones included); returns per rank its output columns."""
    pg = lockstep(R)
    share = np.sort(rng.integers(0, t.n_rows + 1, R - 1))
    bounds = np.concatenate([[0], share, [t.n_rows]]).astype(int)
    per = []
    for r in range(R):
        lo, hi = int(bounds[r]), int(bounds[r + 1])
        bs, at = [], lo
        for c in cuts(hi - lo, rng, 3):
            b = t.slice(at, at + c)
            bs.append(table_to_device(b) if c and r % 2 else b)
            at += c
        per.append(bs)
    n_calls = max(len(b) for b in per) + 1
    empty = t.slice(0, 0)

    def body(r):
        st = init_groupby_state(-1, tuple(range(nk)), tuple(f for f, _ in funcs), tuple(range(len(funcs) + 1)),
                                tuple(c for _, c in funcs), parallel=True, dropna=dropna, device=0, percentiles=qs,
                                output_batch_size=1 << 30)
        try:
            for i in range(n_calls):
                groupby_build_consume_batch(st, per[r][i] if i < len(per[r]) else empty, i == n_calls - 1, True)
            assert st.raw_row_mode and not st.exchanged
            out, last = groupby_produce_output_batch(st, True)
            assert last
            return [(c.values_numpy().copy(), c.valid_mask_numpy(), c.c_type, c.arr_type) for c in out.columns]
        finally:
            delete_groupby_state(st)

    return pg.run(body)


SHARD_KEYS = (CTypes.INT32, CTypes.UINT32, CTypes.INT64, CTypes.UINT64, CTypes.FLOAT32, CTypes.FLOAT64, CTypes.DATE,
              CTypes.DATETIME, CTypes.TIMEDELTA)


@pytest.mark.parametrize("R", [2, 3, 4])
@pytest.mark.parametrize("kct", SHARD_KEYS)
def test_sharded_raw_rows(gpu_lib, lockstep, R, kct):
    from tests.test_gpu_join_sharded import owners

    rng = np.random.default_rng(R * 100 + kct)
    n = 4000
    k, kok = gen_key(kct, n, rng, kct not in FLOATS)
    v, ok = gen(CTypes.FLOAT64, n, rng, True)
    t = make_table([(k, kok, kct)], [(v, ok, CTypes.FLOAT64)])
    funcs = [("percentile_cont", 1), ("mode", 1), ("percentile_disc", 1)]
    qs = (0.5, 0.2)
    res = run_sharded(lockstep, R, t, 1, funcs, qs, rng)
    merged = [(np.concatenate([res[r][j][0] for r in range(R)]),
               None if res[0][j][1] is None else np.concatenate([res[r][j][1] for r in range(R)]), res[0][j][2], res[0][j][3])
              for j in range(len(res[0]))]
    check(merged, t, 1, funcs, qs, True)
    for r in range(R):  # every group sits on the rank the key hash gives it
        kc = res[r][0]
        if len(kc[0]) == 0:
            continue
        ktab = Table([column(kc[0], kc[1], kct)], ["k"])
        assert (owners(ktab, [0], R) == r).all()


def test_sharded_multi_key_and_nunique(gpu_lib, lockstep):
    rng = np.random.default_rng(77)
    n = 3000
    k0, k0ok = gen_key(CTypes.INT64, n, rng, True)
    k1, _ = gen_key(CTypes.FLOAT64, n, rng, False)
    v, ok = gen(CTypes.INT32, n, rng, True)
    t = make_table([(k0, k0ok, CTypes.INT64), (k1, None, CTypes.FLOAT64)], [(v, ok, CTypes.INT32)])
    funcs = [("mode", 2), ("percentile_disc", 2)]
    res = run_sharded(lockstep, 3, t, 2, funcs, (0.5,), rng, dropna=False)
    merged = [(np.concatenate([res[r][j][0] for r in range(3)]),
               None if res[0][j][1] is None else np.concatenate([res[r][j][1] for r in range(3)]), res[0][j][2], res[0][j][3])
              for j in range(len(res[0]))]
    check(merged, t, 2, funcs, (0.5,), False)


@pytest.mark.parametrize("case", ["first", "last", "int16_key", "bool_key"])
def test_sharded_refusals(gpu_lib, lockstep, case):
    pg = lockstep(2)
    n = 16
    kct = {"int16_key": CTypes.INT16, "bool_key": CTypes.BOOL}.get(case, CTypes.INT64)
    k = (np.arange(n) % 2).astype(NP[kct])
    t = make_table([(k, None, kct)], [(np.arange(n, dtype=np.int64), None, CTypes.INT64)])
    funcs = [("mode", 1)] + ([(case, 1)] if case in ("first", "last") else [])
    cause = "first / last" if case in ("first", "last") else "1- or 2-byte key column"

    def body(r):
        st = init_groupby_state(-1, (0,), tuple(f for f, _ in funcs), tuple(range(len(funcs) + 1)), tuple(c for _, c in funcs),
                                parallel=True, device=0)
        try:
            with pytest.raises(_lib.B200Error, match=cause):
                groupby_build_consume_batch(st, t, True, True)
            assert st.handle is None
        finally:
            delete_groupby_state(st)

    pg.run(body)


def test_one_rank_runs_locally(gpu_lib, lockstep):
    pg = lockstep(1)
    n = 500
    rng = np.random.default_rng(1)
    k = rng.integers(0, 7, n).astype(np.int8)  # (a 1-byte key is fine on one rank)
    v, ok = gen(CTypes.FLOAT64, n, rng, False)
    t = make_table([(k, None, CTypes.INT8)], [(v, ok, CTypes.FLOAT64)])
    funcs = [("mode", 1), ("first", 1), ("percentile_cont", 1)]

    def body(r):
        st = init_groupby_state(-1, (0,), ("mode", "first", "percentile_cont"), (0, 1, 2, 3), (1, 1, 1), parallel=True, device=0,
                                percentiles=(0.5,))
        try:
            groupby_build_consume_batch(st, t, True, True)
            out, _ = groupby_produce_output_batch(st, True)
            return [(c.values_numpy().copy(), c.valid_mask_numpy(), c.c_type, c.arr_type) for c in out.columns]
        finally:
            delete_groupby_state(st)

    cols = pg.run(body)[0]
    check(cols, t, 1, funcs, (0.5,), True, hol=[0, 2])
