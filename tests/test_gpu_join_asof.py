"""The as-of join (init_join_state(asof_on=...), physical.merge_asof) against pandas.merge_asof, bit for bit.

The oracle runs pandas.merge_asof on what pandas accepts: both sides' keys become one int64 group id (NA keys one group under
is_na_equal, no group otherwise), rows with an NA `on` cell are dropped and come back unmatched, the build side is sorted stably
by `on` (arrival order among ties) and the probe side too, with the permutation inverted afterwards.  Every output column is then
compared with the build / probe cell the oracle names, bits and validity, in probe order.  The left backward as-of join is also
checked against the window workaround (union both sides, LAST_VALUE(... IGNORE NULLS) over the `on` order, keep the probe rows).

Run time of this file on one H100 80GB HBM3 at its 700 W power limit: 50 s."""

import numpy as np
import pandas as pd
import pytest

from bodo_b200.streaming import join as J
from bodo_b200.table import ArrTypes, Column, CTypes, Table
from tests.helpers import table_to_device

pytestmark = pytest.mark.gpu

NP = {CTypes.INT8: np.int8, CTypes.UINT8: np.uint8, CTypes.INT16: np.int16, CTypes.UINT16: np.uint16, CTypes.INT32: np.int32,
      CTypes.UINT32: np.uint32, CTypes.INT64: np.int64, CTypes.UINT64: np.uint64, CTypes.FLOAT32: np.float32,
      CTypes.FLOAT64: np.float64, CTypes.DATE: np.int32, CTypes.DATETIME: np.int64, CTypes.TIMEDELTA: np.int64}
DIRS = ("backward", "forward", "nearest")


class Side:
    """One side's columns: name -> (numpy values, c-type, bool validity mask or None)."""

    def __init__(self, **cols):
        self.cols = {k: (np.ascontiguousarray(np.asarray(v[0]).astype(NP[v[1]])), v[1], None if len(v) < 3 or v[2] is None else np.asarray(v[2], bool))
                     for k, v in cols.items()}
        self.n = len(next(iter(self.cols.values()))[0])

    def names(self):
        return list(self.cols)

    def table(self, lo, hi, device):
        cols = []
        for vals, ct, valid in self.cols.values():
            v = None if valid is None else np.packbits(valid[lo:hi], bitorder="little")
            cols.append(Column(np.ascontiguousarray(vals[lo:hi]), v, ct, ArrTypes.NULLABLE_INT_BOOL if valid is not None else ArrTypes.NUMPY, hi - lo))
        t = Table(cols, self.names())
        return table_to_device(t) if device else t

    def na(self, name):
        vals, ct, valid = self.cols[name]
        na = np.zeros(self.n, bool) if valid is None else ~valid
        return na | np.isnan(vals) if ct in (CTypes.FLOAT32, CTypes.FLOAT64) else na


def oracle(b, p, bkeys, pkeys, won, von, direction="backward", exact=True, tol=None, na_equal=True):
    """The build row each probe row matches (-1: none), by pandas.merge_asof."""
    def keyframe(side, keys):
        return pd.DataFrame({j: pd.Series(side.cols[k][0]).astype(object).where(~side.na(k), None) for j, k in enumerate(keys)})

    if bkeys:
        allk = pd.concat([keyframe(b, bkeys), keyframe(p, pkeys)], ignore_index=True)
        g = allk.groupby(list(allk.columns), dropna=False, sort=False).ngroup().to_numpy().astype(np.int64)
        na = allk.isna().any(axis=1).to_numpy()
        if not na_equal:
            g[na] = -1 - np.arange(int(na.sum()))
    else:
        g = np.zeros(b.n + p.n, np.int64)
    gb, gp = g[: b.n], g[b.n:]
    bok, pok = ~b.na(won), ~p.na(von)
    w, v = b.cols[won][0], p.cols[von][0]
    R = pd.DataFrame({"w": w[bok], "g": gb[bok], "rid": np.nonzero(bok)[0]}).sort_values("w", kind="stable")
    Lf = pd.DataFrame({"w": v[pok], "g": gp[pok], "pid": np.nonzero(pok)[0]}).sort_values("w", kind="stable")
    m = pd.merge_asof(Lf, R, on="w", by="g", direction=direction, allow_exact_matches=exact, tolerance=tol)
    res = np.full(p.n, -1, np.int64)
    res[m["pid"].to_numpy()] = m["rid"].fillna(-1).to_numpy().astype(np.int64)
    return res


def run(b, p, bkeys, pkeys, won, von, inner=False, b_batches=(), p_batch=None, device=False, used=None, tol=None, **kw):
    """The as-of join in streaming batches; the output columns concatenated as (values, validity mask or None)."""
    st = J.init_join_state(-1, [b.names().index(k) for k in bkeys], [p.names().index(k) for k in pkeys], b.names(), p.names(), False,
                           not inner, asof_on=(won, von), asof_tolerance=tol, **{k: v for k, v in kw.items() if k.startswith("asof_")},
                           is_na_equal=kw.get("na_equal", True))
    cuts = [0, *b_batches, b.n]
    for i in range(len(cuts) - 1):
        J.join_build_consume_batch(st, b.table(cuts[i], cuts[i + 1], device), i == len(cuts) - 2)
    step = p_batch or max(p.n, 1)
    starts = list(range(0, p.n, step)) or [0]
    parts = []
    for s in starts:
        out, _, _ = J.join_probe_consume_batch(st, p.table(s, min(s + step, p.n), device), s == starts[-1], True, used)
        parts.append([(c.values_numpy().copy(), c.valid_mask_numpy()) for c in out.columns])
    J.delete_join_state(st)
    cols = []
    for j in range(len(parts[0])):
        vals = np.concatenate([pt[j][0] for pt in parts])
        masks = [pt[j][1] if pt[j][1] is not None else np.ones(len(pt[j][0]), bool) for pt in parts]
        cols.append((vals, np.concatenate(masks) if any(pt[j][1] is not None for pt in parts) else None))
    return cols


def check(got, b, p, rid_all, inner=False, used=None):
    rows = np.nonzero(rid_all >= 0)[0] if inner else np.arange(p.n)
    rid = rid_all[rows]
    kb, kp = used if used is not None else (list(range(len(b.cols))), list(range(len(p.cols))))
    spec = [(b, c, rid) for c in kb] + [(p, c, rows) for c in kp]
    assert len(got) == len(spec)
    for (vals, mask), (side, c, idx) in zip(got, spec):
        sv, _, svalid = side.cols[side.names()[c]]
        assert len(vals) == len(rows), (side.names()[c], len(vals), len(rows))
        hit = idx >= 0
        exp_valid = hit.copy()
        if svalid is not None:
            exp_valid[hit] = svalid[idx[hit]]
        got_valid = mask if mask is not None else np.ones(len(vals), bool)
        np.testing.assert_array_equal(got_valid, exp_valid, err_msg=f"validity of {side.names()[c]}")
        u = f"u{sv.dtype.itemsize}"
        np.testing.assert_array_equal(vals[exp_valid].view(u), sv[idx[exp_valid]].view(u), err_msg=f"values of {side.names()[c]}")


ON_TYPES = [CTypes.INT8, CTypes.UINT8, CTypes.INT16, CTypes.UINT16, CTypes.INT32, CTypes.UINT32, CTypes.INT64, CTypes.UINT64,
            CTypes.FLOAT32, CTypes.FLOAT64, CTypes.DATE, CTypes.DATETIME, CTypes.TIMEDELTA]


def on_values(rng, ct, n):
    lo, hi = {CTypes.INT8: (-60, 60), CTypes.UINT8: (0, 120)}.get(ct, (0, 1000) if np.issubdtype(NP[ct], np.unsignedinteger) else (-500, 500))
    x = rng.integers(lo, hi, n)
    if ct in (CTypes.FLOAT32, CTypes.FLOAT64):
        x = x / 4.0
        x[rng.random(n) < 0.05] = -0.0
        x[rng.random(n) < 0.03] = np.nan
    return x


@pytest.mark.parametrize("ct", ON_TYPES)
def test_every_on_type_direction_and_tolerance(ct):
    rng = np.random.default_rng(ct)
    nb, npr = 3000, 4000
    bvalid = rng.random(nb) > 0.05
    b = Side(k=(rng.integers(0, 40, nb), CTypes.INT64), w=(on_values(rng, ct, nb), ct, bvalid), x=(rng.integers(-9, 9, nb), CTypes.INT32),
             rid=(np.arange(nb), CTypes.INT64))
    p = Side(k=(rng.integers(0, 45, npr), CTypes.INT64), v=(on_values(rng, ct, npr), ct, rng.random(npr) > 0.05), pid=(np.arange(npr), CTypes.INT64))
    is_float = ct in (CTypes.FLOAT32, CTypes.FLOAT64)
    for direction in DIRS:
        for exact in (True, False):
            for tol in (None, 0, 7.5 if is_float else 7):
                exp = oracle(b, p, ["k"], ["k"], "w", "v", direction, exact, tol)
                for inner in (False, True):
                    got = run(b, p, ["k"], ["k"], "w", "v", inner=inner, b_batches=(1000,), tol=tol, asof_direction=direction,
                              asof_allow_exact_matches=exact)
                    check(got, b, p, exp, inner)


@pytest.mark.parametrize("na_equal", [True, False])
@pytest.mark.parametrize("n_by", [0, 1, 2])
def test_by_keys_nullable_float_and_na(n_by, na_equal):
    rng = np.random.default_rng(10 + n_by)
    nb, npr = 5000, 6000
    def keys(n):
        k0 = rng.integers(0, 12, n)
        k1 = rng.integers(0, 6, n) / 2.0
        k1[rng.random(n) < 0.04] = np.nan
        return dict(k0=(k0, CTypes.INT32, rng.random(n) > 0.05), k1=(k1, CTypes.FLOAT64))
    bk, pk = keys(nb), keys(npr)
    names = ["k0", "k1"][:n_by]
    b = Side(**{k: bk[k] for k in names}, w=(rng.integers(0, 10**6, nb), CTypes.DATETIME), x=(rng.random(nb), CTypes.FLOAT64, rng.random(nb) > 0.1))
    p = Side(**{k: pk[k] for k in names}, v=(rng.integers(0, 10**6, npr), CTypes.DATETIME), y=(rng.integers(0, 99, npr), CTypes.UINT16))
    for direction in DIRS:
        exp = oracle(b, p, names, names, "w", "v", direction, na_equal=na_equal)
        for inner in (False, True):
            for device in (False, True):
                got = run(b, p, names, names, "w", "v", inner=inner, device=device, b_batches=(1700, 1700), asof_direction=direction,
                          na_equal=na_equal)
                check(got, b, p, exp, inner)
    # a pd.Timedelta tolerance on a DATETIME column is in ns
    exp = oracle(b, p, names, names, "w", "v", "nearest", tol=3000, na_equal=na_equal)
    check(run(b, p, names, names, "w", "v", asof_direction="nearest", tol=pd.Timedelta("3us"), na_equal=na_equal), b, p, exp)


def test_ties_within_and_across_build_batches_and_probe_batch_sizes():
    rng = np.random.default_rng(7)
    nb = 4096
    b = Side(k=(rng.integers(0, 3, nb), CTypes.INT64), w=(rng.integers(0, 20, nb), CTypes.INT64), rid=(np.arange(nb), CTypes.INT64))
    for npr in (0, 1, 1023, 1024, 1025):
        p = Side(k=(rng.integers(0, 3, npr), CTypes.INT64), v=(rng.integers(-2, 22, npr), CTypes.INT64), pid=(np.arange(npr), CTypes.INT64))
        for direction in DIRS:
            for exact in (True, False):
                exp = oracle(b, p, ["k"], ["k"], "w", "v", direction, exact)
                for device in (False, True):
                    for pb in (None, 1000):
                        got = run(b, p, ["k"], ["k"], "w", "v", b_batches=(1000, 1001, 3000), p_batch=pb, device=device,
                                  asof_direction=direction, asof_allow_exact_matches=exact)
                        check(got, b, p, exp)


def test_empty_build_groups_of_one_and_used_cols():
    rng = np.random.default_rng(8)
    npr = 3000
    p = Side(k=(rng.integers(0, 500, npr), CTypes.INT64), v=(rng.integers(0, 100, npr), CTypes.INT32), pid=(np.arange(npr), CTypes.INT64))
    empty = Side(k=(np.zeros(0), CTypes.INT64), w=(np.zeros(0), CTypes.INT32), rid=(np.zeros(0), CTypes.INT64))
    for inner in (False, True):
        check(run(empty, p, ["k"], ["k"], "w", "v", inner=inner), empty, p, np.full(npr, -1), inner)
    single = Side(k=(rng.permutation(400), CTypes.INT64), w=(rng.integers(0, 100, 400), CTypes.INT32), rid=(np.arange(400), CTypes.INT64),
                  z=(rng.random(400), CTypes.FLOAT32, rng.random(400) > 0.2))
    for direction in DIRS:
        exp = oracle(single, p, ["k"], ["k"], "w", "v", direction, tol=20)
        check(run(single, p, ["k"], ["k"], "w", "v", asof_direction=direction, tol=20), single, p, exp)
        for used in (([3], [2]), ([], [0, 1]), ([1, 2], []), ([3, 0], [1])):
            for inner in (False, True):
                got = run(single, p, ["k"], ["k"], "w", "v", inner=inner, used=used, asof_direction=direction, tol=20)
                check(got, single, p, exp, inner, used)


def test_integer_extremes_are_exact():
    """Differences near the int64 / uint64 limits: words subtract exactly where int64 arithmetic would overflow."""
    for ct, vals in ((CTypes.INT64, [-2**63, -2**63 + 5, 2**63 - 1, 0]), (CTypes.UINT64, [0, 2**64 - 1, 2**63, 7])):
        w = np.array(vals, dtype=NP[ct])
        b = Side(w=(w, ct), rid=(np.arange(4), CTypes.INT64))
        v = np.array(vals[::-1] + [vals[0] + (3 if ct == CTypes.INT64 else 0)], dtype=NP[ct])
        p = Side(v=(v, ct), pid=(np.arange(5), CTypes.INT64))
        for direction in DIRS:
            for tol in (None, 0, 2**62, 2**63 - 1):
                got = run(b, p, [], [], "w", "v", asof_direction=direction, tol=tol)
                exp = np.full(5, -1)
                for i, x in enumerate(int(a) for a in v):  # brute force over Python ints
                    cands = [(abs(x - int(y)), j, int(y) <= x) for j, y in enumerate(w)]
                    back = [c for c in cands if c[2]]
                    fwd = [c for c in cands if int(w[c[1]]) >= x]
                    bb = max(back, key=lambda c: (int(w[c[1]]), c[1])) if back else None
                    ff = min(fwd, key=lambda c: (int(w[c[1]]), c[1])) if fwd else None
                    pick = bb if direction == "backward" else ff if direction == "forward" else (
                        bb if bb and (not ff or bb[0] <= ff[0]) else ff)
                    if pick and (tol is None or pick[0] <= tol):
                        exp[i] = pick[1]
                check(got, b, p, exp)


def test_one_group_of_2_22_rows_and_a_probe_larger_than_a_grid():
    rng = np.random.default_rng(9)
    nb, npr = 1 << 22, 1 << 20
    b = Side(w=(rng.integers(0, 1 << 40, nb), CTypes.TIMEDELTA), rid=(np.arange(nb), CTypes.INT64))
    p = Side(v=(rng.integers(-1000, (1 << 40) + 1000, npr), CTypes.TIMEDELTA), pid=(np.arange(npr), CTypes.INT64))
    for direction in DIRS:
        exp = oracle(b, p, [], [], "w", "v", direction)
        check(run(b, p, [], [], "w", "v", device=True, b_batches=(1 << 21,), asof_direction=direction), b, p, exp)


def test_build_of_2_25_rows_in_2_22_row_batches():
    rng = np.random.default_rng(11)
    nb, npr = 1 << 25, 1 << 21
    b = Side(k=(rng.integers(0, 1 << 16, nb), CTypes.INT64), w=(rng.integers(0, 1 << 30, nb), CTypes.DATETIME), rid=(np.arange(nb), CTypes.INT64))
    p = Side(k=(rng.integers(0, 1 << 16, npr), CTypes.INT64), v=(rng.integers(0, 1 << 30, npr), CTypes.DATETIME), pid=(np.arange(npr), CTypes.INT64))
    exp = oracle(b, p, ["k"], ["k"], "w", "v", "backward", tol=1 << 14)
    for inner in (False, True):
        got = run(b, p, ["k"], ["k"], "w", "v", inner=inner, device=True, b_batches=tuple(range(1 << 22, nb, 1 << 22)), tol=1 << 14)
        check(got, b, p, exp, inner)


def test_left_backward_equals_the_window_workaround():
    from bodo_b200.physical import window

    rng = np.random.default_rng(12)
    nb, npr = 60_000, 90_000
    quotes = pd.DataFrame({"sym": rng.integers(0, 300, nb), "ts": rng.integers(0, 10**5, nb), "rid": np.arange(nb)})
    trades = pd.DataFrame({"sym": rng.integers(0, 300, npr), "ts": rng.integers(0, 10**5, npr), "pid": np.arange(npr)})
    union = pd.concat([quotes.assign(rid=quotes["rid"].astype("Int64"), pid=pd.array([pd.NA] * nb, dtype="Int64")),
                       trades.assign(rid=pd.array([pd.NA] * npr, dtype="Int64"), pid=trades["pid"].astype("Int64"))], ignore_index=True)
    w = window(union, ["sym"], ["ts"], [("last", "last_value", "rid", "rows", "ignore_nulls")])
    w = w[w["pid"].notna()].sort_values("pid")
    via_window = w["last"].fillna(-1).to_numpy().astype(np.int64)
    b = Side(sym=(quotes["sym"], CTypes.INT64), ts=(quotes["ts"], CTypes.INT64), rid=(quotes["rid"], CTypes.INT64))
    p = Side(sym=(trades["sym"], CTypes.INT64), ts=(trades["ts"], CTypes.INT64), pid=(trades["pid"], CTypes.INT64))
    got = run(b, p, ["sym"], ["sym"], "ts", "ts", device=True, used=([2], [2]))
    check(got, b, p, via_window, used=([2], [2]))
    np.testing.assert_array_equal(via_window, oracle(b, p, ["sym"], ["sym"], "ts", "ts"))


def test_merge_asof_helper_matches_pandas():
    from bodo_b200.physical import merge_asof

    rng = np.random.default_rng(13)
    quotes = pd.DataFrame({"t": np.sort(rng.integers(0, 5000, 2000)), "k": rng.integers(0, 20, 2000), "v": rng.random(2000), "q": rng.integers(0, 9, 2000)})
    trades = pd.DataFrame({"t": np.sort(rng.integers(0, 5000, 3000)), "k": rng.integers(0, 20, 3000), "v": rng.random(3000)})
    for kw in (dict(on="t", by="k"), dict(on="t"), dict(left_on="t", right_on="t", by="k", direction="nearest", tolerance=10),
               dict(on="t", by="k", direction="forward", allow_exact_matches=False, suffixes=("_l", "_r"))):
        got = merge_asof(trades, quotes, batch_size=700, **kw)
        exp = pd.merge_asof(trades, quotes, **kw)
        assert list(got.columns) == list(exp.columns)
        for c in exp.columns:
            np.testing.assert_array_equal(got[c].to_numpy(dtype="float64", na_value=np.nan), exp[c].to_numpy(dtype="float64", na_value=np.nan), err_msg=f"{kw} {c}")
