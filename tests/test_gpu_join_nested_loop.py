"""The nested-loop join (no equi-join key) against an exact numpy cartesian product that never touches the device.

The reference lists every (probe row, build row) pair in probe-major, build-minor order, evaluates the condition on every pair
with the filter-projection reference evaluator (ref_eval in tests/test_gpu_filter_project.py), keeps the pairs whose value is
valid and true (every pair without a condition), then applies the join kind as tests/test_gpu_join_condition.py does: a probe row
without a passing pair is NULL-extended in its place (left / full), kept (anti) or marked false (mark); the build rows without a
passing pair over all probe calls follow the last call in build order (right / full).  The order is part of the contract, so
outputs are compared in order: c-type, array type and bitmap presence per column, then the bits and validity of every cell.
Metrics 8 and 9 must equal the pairs evaluated (n_probe x n_build over the calls) and the pairs passed, and stay 0 without a
condition."""

import numpy as np
import pandas as pd
import pytest

from bodo_b200.expr import build_col, lit, probe_col
from bodo_b200.table import Column, CTypes, Table
from tests.test_gpu_filter_project import ref_eval
from tests.test_gpu_join_condition import expected, small_ints, with_nan
from tests.test_gpu_join_exact import FLAGS, KINDS, _cat, bits_of, col, host_slices, payload, records

CT = CTypes
gpu = pytest.mark.gpu
I64_MIN, I64_MAX, U64_MAX = -(1 << 63), (1 << 63) - 1, (1 << 64) - 1
BAND = (probe_col("x") >= build_col("lo")) & (probe_col("x") < build_col("hi"))
DAY_NS = 86_400 * 10 ** 9


# ---------------------------------------------------------------------------------------------- the reference
def nlj_reference(build, probe, kind, cond, bnames, pnames):
    """(pairs (build row, probe row; -1 on the NULL side) in output order, or the marks of a mark join; pairs evaluated; passed)."""
    bt, pt = _cat(build), _cat(probe)
    nb, npr = bt.n_rows, pt.n_rows
    pi, bi = np.repeat(np.arange(npr), nb), np.tile(np.arange(nb), npr)
    if cond is not None and len(pi):
        cols = {}
        for side, t, names, rows in (("build", bt, bnames, bi), ("probe", pt, pnames, pi)):
            for name, c in zip(names, t.columns):
                cols[(side, name)] = (c.c_type, np.asarray(c.values_numpy())[rows], bits_of(c)[1][rows])
        _, x, v = ref_eval(cond, cols)
        ok = v & (x != 0)
        bi, pi = bi[ok], pi[ok]
    n_eval, n_pass = (npr * nb, len(bi)) if cond is not None else (0, 0)
    has = np.zeros(npr, bool)
    has[pi] = True
    if kind == "mark":
        return has, n_eval, n_pass
    if kind == "anti":
        un = np.flatnonzero(~has)
        return (np.full(len(un), -1, np.int64), un), n_eval, n_pass
    bo, po = FLAGS[kind]
    if po:  # a NULL-extended row in its probe row's place
        un = np.flatnonzero(~has)
        bi, pi = np.concatenate([bi, np.full(len(un), -1)]), np.concatenate([pi, un])
        order = np.argsort(pi, kind="stable")
        bi, pi = bi[order], pi[order]
    if bo:
        matched = np.zeros(nb, bool)
        matched[bi[bi >= 0]] = True
        un = np.flatnonzero(~matched)
        bi, pi = np.concatenate([bi, un]), np.concatenate([pi, np.full(len(un), -1)])
    return (bi.astype(np.int64), pi.astype(np.int64)), n_eval, n_pass


# ---------------------------------------------------------------------------------------------- driving the join
def run(build, probe, kind, cond, bnames, pnames, device=False):
    from bodo_b200.streaming.join import (delete_join_state, get_metric, init_nested_loop_join_state, join_build_consume_batch,
                                          join_probe_consume_batch)
    from tests.helpers import table_to_device

    bo, po = FLAGS[kind]
    st = init_nested_loop_join_state(-1, bnames, pnames, bo, po, cond, is_mark_join=kind == "mark", is_anti_join=kind == "anti")
    dev = table_to_device if device else (lambda t: t)
    try:
        for i, b in enumerate(build):
            join_build_consume_batch(st, dev(b), i == len(build) - 1)
        outs = []
        for i, p in enumerate(probe):
            out, _, _ = join_probe_consume_batch(st, dev(p), i == len(probe) - 1, True)
            outs.append([(c.c_type, c.arr_type, c.validity is not None, bits_of(c)) for c in out.columns])
        metrics = {m: get_metric(st, m) for m in range(10)}
    finally:
        delete_join_state(st)
    return outs, metrics


def compare_in_order(outs, exp_all, kind, what=""):
    assert len(outs) == len(exp_all)
    for q, (got, exp) in enumerate(zip(outs, exp_all)):
        if kind == "mark":  # the mark column's bitmap is there whenever the batch has rows
            exp = [x if x[2] is not None else (x[0], x[1], True if len(x[3][0]) else got[-1][2], x[3]) for x in exp]
        assert [g[:3] for g in got] == [x[:3] for x in exp], (q, what, [g[:3] for g in got], [x[:3] for x in exp])
        g, x = records([c[3] for c in got]), records([c[3] for c in exp])
        assert g.shape == x.shape, (q, what, g.shape, x.shape)
        np.testing.assert_array_equal(g, x, err_msg=f"probe batch {q} ({kind}) {what}")


def check(build, probe, kind, cond, bnames, pnames, device=False):
    outs, m = run(build, probe, kind, cond, bnames, pnames, device)
    res, n_eval, n_pass = nlj_reference(build, probe, kind, cond, bnames, pnames)
    assert (m[8], m[9]) == (n_eval, n_pass), ("metrics 8 / 9: pairs evaluated and passed", m, n_eval, n_pass)
    assert m[5] == 0 and m[6] == 0 and m[7] == 0, m
    compare_in_order(outs, expected(build, probe, kind, res, None), kind)
    return outs, m


# ---------------------------------------------------------------------------------------------- inputs
def bands(n, rng, width=40, span=4000):
    lo = rng.integers(-span // 2, span // 2, n)
    return lo, lo + rng.integers(0, width, n)


def case_none(rng, nb, npr):
    b = Table([payload(CT.INT32, nb, 1, null_every=5), payload(CT.INT64, nb, 2)])
    p = Table([payload(CT.UINT16, npr, 3, null_every=7), payload(CT.INT64, npr, 4)])
    return b, p, ["bc", "bp"], ["pc", "pp"], None


def case_band(rng, nb, npr):
    lo, hi = bands(nb, rng)
    b = Table([col(CT.INT64, lo), col(CT.INT64, hi), payload(CT.INT64, nb, 5)])
    p = Table([col(CT.INT64, rng.integers(-2100, 2100, npr)), payload(CT.INT32, npr, 6, null_every=9)])
    return b, p, ["lo", "hi", "bid"], ["x", "eid"], BAND


def case_na(rng, nb, npr):
    """Nullable columns and NaN floats: the condition is NA for many pairs (Kleene logic and isnull decide the rest)."""
    b = Table([small_ints(CT.INT32, nb, 0, 100, rng, na_every=9), with_nan(CT.FLOAT64, rng.random(nb) * 10, rng), payload(CT.INT64, nb, 7)])
    p = Table([small_ints(CT.INT64, npr, -10, 120, rng, na_every=11), with_nan(CT.FLOAT32, rng.random(npr) * 10, rng, na_every=13),
               payload(CT.UINT16, npr, 8, null_every=7)])
    cond = ((probe_col("t") >= build_col("lo")) & (probe_col("w") < build_col("hi"))) | (probe_col("t").isnull() & (build_col("lo") * 2 < 90))
    return b, p, ["lo", "hi", "bp"], ["t", "w", "pp"], cond


def case_u64_i64(rng, nb, npr):
    bv = np.array([0, 1, 1 << 63, U64_MAX, I64_MAX, (1 << 63) + 5, 5], dtype=object)[rng.integers(0, 7, nb)]
    pv = np.array([I64_MIN, -1, 0, 1, I64_MAX, 5, 6], dtype=object)[rng.integers(0, 7, npr)]
    b = Table([col(CT.UINT64, bv, rng.random(nb) > 0.05), payload(CT.INT64, nb, 9)])
    p = Table([col(CT.INT64, pv, rng.random(npr) > 0.05), payload(CT.INT64, npr, 10)])
    return b, p, ["b", "bp"], ["a", "pp"], (probe_col("a") < build_col("b")) | (probe_col("a") == build_col("b"))


def case_float32(rng, nb, npr):
    b = Table([with_nan(CT.FLOAT32, rng.normal(0, 3, nb), rng), payload(CT.INT64, nb, 11)])
    p = Table([with_nan(CT.FLOAT32, rng.normal(0, 3, npr), rng, na_every=17), payload(CT.INT16, npr, 12)])
    return b, p, ["f", "bp"], ["g", "pp"], (probe_col("g") * 2 <= build_col("f") + lit(1.5)) & (build_col("f") != probe_col("g"))


def case_date_datetime(rng, nb, npr):
    b = Table([col(CT.DATETIME, rng.integers(-3, 12, nb) * DAY_NS + rng.integers(0, DAY_NS, nb), rng.random(nb) > 0.05),
               col(CT.DATE, rng.integers(-3, 12, nb)), payload(CT.INT64, nb, 13)])
    p = Table([col(CT.DATE, rng.integers(-3, 12, npr), rng.random(npr) > 0.05), payload(CT.INT64, npr, 14)])
    cond = (probe_col("a") * DAY_NS >= build_col("b")) & (probe_col("a") < build_col("c") + 2)
    return b, p, ["b", "c", "bp"], ["a", "pp"], cond


CASES = {"none": case_none, "band": case_band, "na": case_na, "u64_i64": case_u64_i64, "float32": case_float32,
         "date_datetime": case_date_datetime}
PROBE_EDGES = [0, 1, 31, 32, 33, 255, 257]  # warp and tile edges; an empty batch


# ================================================================================================ CPU: the reference itself
def test_reference_matches_pandas_cross_merge():
    rng = np.random.default_rng(1)
    b, p, bn, pn, cond = case_band(rng, 300, 700)
    build, probe = [b], host_slices(p, [300, 400])
    bdf = pd.DataFrame({"lo": b.columns[0].data, "hi": b.columns[1].data, "bi": np.arange(300)})
    pdf = pd.DataFrame({"x": p.columns[0].data, "pi": np.arange(700)})
    m = pdf.merge(bdf, how="cross")
    inner = m[(m.x >= m.lo) & (m.x < m.hi)]
    (bi, pi), n_eval, n_pass = nlj_reference(build, probe, "inner", cond, bn, pn)
    assert list(zip(bi.tolist(), pi.tolist())) == list(zip(inner.bi.tolist(), inner.pi.tolist()))
    assert (n_eval, n_pass) == (len(m), len(inner))
    (bi, pi), _, _ = nlj_reference(build, probe, "probe_outer", cond, bn, pn)
    assert pi.tolist() == sorted(pi.tolist()) and sorted(pi[bi < 0].tolist()) == sorted(set(range(700)) - set(inner.pi.tolist()))
    (bi, pi), _, _ = nlj_reference(build, probe, "inner", None, bn, pn)
    assert list(zip(bi.tolist(), pi.tolist())) == list(zip(m.bi.tolist(), m.pi.tolist()))


# ================================================================================================ GPU
@gpu
@pytest.mark.parametrize("device", [False, True])
@pytest.mark.parametrize("case", list(CASES))
@pytest.mark.parametrize("kind", KINDS)
def test_every_kind_and_column_type(gpu_lib, kind, case, device):
    rng = np.random.default_rng(10 * KINDS.index(kind) + list(CASES).index(case))
    b, p, bn, pn, cond = CASES[case](rng, 300, 700)
    check(host_slices(b, [100, 200]), host_slices(p, PROBE_EDGES + [700 - sum(PROBE_EDGES)]), kind, cond, bn, pn, device)


@gpu
@pytest.mark.parametrize("with_cond", [False, True])
@pytest.mark.parametrize("kind", KINDS)
def test_empty_build_side(gpu_lib, kind, with_cond):
    rng = np.random.default_rng(2)
    b, p, bn, pn, cond = case_band(rng, 0, 300)
    check([b], host_slices(p, [0, 1, 299]), kind, cond if with_cond else None, bn, pn)


@gpu
@pytest.mark.parametrize("with_cond", [False, True])
@pytest.mark.parametrize("kind", KINDS)
def test_empty_probe_batches_and_one_build_row(gpu_lib, kind, with_cond):
    rng = np.random.default_rng(3)
    b, p, bn, pn, cond = case_band(rng, 1, 400)
    b = Table([col(CT.INT64, [-1000]), col(CT.INT64, [1000]), payload(CT.INT64, 1, 5)])  # passes about half the probe rows
    check([b], host_slices(p, [0, 0, 1, 0, 399]), kind, cond if with_cond else None, bn, pn)
    check([b], host_slices(p, [0, 0, 0, 400, 0]), kind, cond if with_cond else None, bn, pn)


@gpu
@pytest.mark.parametrize("nb", [1, 255, 256, 257, 511, 513, 4095, 4097, 20001])
@pytest.mark.parametrize("kind", ["inner", "full_outer", "anti", "mark"])
def test_build_sizes_around_the_chunk_and_sub_tile_edges(gpu_lib, kind, nb):
    """Build chunks are multiples of 256 rows, fewer and longer for larger probe batches: builds off those edges, with probe
    batches of 1, 33 and 4097 rows (from many chunks per probe tile to one)."""
    rng = np.random.default_rng(nb)
    b, p, bn, pn, cond = case_band(rng, nb, 4131)
    check([b], host_slices(p, [1, 33, 4097]), kind, cond, bn, pn, device=True)


@gpu
@pytest.mark.parametrize("kind", KINDS)
def test_few_probe_rows_against_many_build_rows(gpu_lib, kind):
    """3 probe rows against 2^20 + 5 build rows: one probe tile served by many build chunks."""
    rng = np.random.default_rng(4)
    b, p, bn, pn, cond = case_band(rng, (1 << 20) + 5, 3)
    check([b], [p], kind, cond, bn, pn, device=True)


@gpu
@pytest.mark.parametrize("with_cond", [False, True])
@pytest.mark.parametrize("kind", KINDS)
def test_many_probe_rows_against_three_build_rows(gpu_lib, kind, with_cond):
    rng = np.random.default_rng(5)
    b, p, bn, pn, cond = case_band(rng, 3, (1 << 20) + 3)
    b = Table([col(CT.INT64, [-2000, -100, 500]), col(CT.INT64, [-1000, 400, 2000]), payload(CT.INT64, 3, 5)])
    check([b], [p], kind, cond if with_cond else None, bn, pn, device=True)


@gpu
@pytest.mark.parametrize("kind", ["build_outer", "full_outer"])
def test_build_row_first_passing_in_a_later_probe_batch(gpu_lib, kind):
    """Bands 0..9 are hit only by the second probe batch and bands 10..19 never: the tail after the last call holds exactly
    bands 10..19, in build order."""
    lo = np.arange(20) * 10
    b = Table([col(CT.INT64, lo), col(CT.INT64, lo + 10), col(CT.INT64, np.arange(20))])
    p1 = Table([col(CT.INT64, [-5, 500, 1000]), col(CT.INT64, [0, 1, 2])])
    p2 = Table([col(CT.INT64, [95, 3, 44, 71, 12, 29, 58, 86, 37, 60, 999]), col(CT.INT64, np.arange(3, 14))])
    outs, _ = check([b], [p1, p2], kind, BAND, ["lo", "hi", "bid"], ["x", "eid"])
    bid_bits, bid_valid = outs[-1][2][3]
    assert bid_bits[-10:].tolist() == list(range(10, 20)) and bid_valid[-10:].all()


@gpu
@pytest.mark.parametrize("with_cond", [False, True])
@pytest.mark.parametrize("kind", KINDS)
def test_deterministic_across_runs_and_probe_splits(gpu_lib, kind, with_cond):
    rng = np.random.default_rng(6)
    b, p, bn, pn, cond = case_na(rng, 2000, 5000)
    cond = cond if with_cond else None
    runs = [run([b], host_slices(p, s), kind, cond, bn, pn, device=True)[0] for s in ([5000], [5000], [1, 2047, 2952], [4097, 903])]

    def concat(outs):
        return records([(np.concatenate([o[j][3][0] for o in outs]), np.concatenate([o[j][3][1] for o in outs])) for j in range(len(outs[0]))])

    first = concat(runs[0])
    for r in runs[1:]:
        np.testing.assert_array_equal(concat(r), first)


@gpu
@pytest.mark.parametrize("kind", KINDS)
def test_equals_the_constant_key_workaround(gpu_lib, kind):
    """The equi-join on an appended constant INT8 key with the same condition joins the same pairs (its order is unspecified)."""
    from bodo_b200.streaming.join import delete_join_state, init_join_state, join_build_consume_batch, join_probe_consume_batch
    from tests.test_gpu_join_exact import sort_records

    rng = np.random.default_rng(7)
    b, p, bn, pn, cond = case_na(rng, 1500, 3000)
    probe = host_slices(p, [1000, 2000])
    outs, _ = run([b], probe, kind, cond, bn, pn)
    with_key = lambda t: Table(list(t.columns) + [Column(np.zeros(max(t.n_rows, 1), np.int8), None, CT.INT8, length=t.n_rows)])
    bo, po = FLAGS[kind]
    st = init_join_state(-1, (3,), (3,), bn + ["k"], pn + ["k"], bo, po, is_mark_join=kind == "mark", is_anti_join=kind == "anti",
                         non_equi_condition=cond)
    try:
        join_build_consume_batch(st, with_key(b), True)
        for i, q in enumerate(probe):
            out, _, _ = join_probe_consume_batch(st, with_key(q), i == len(probe) - 1, True, ([0, 1, 2], [0, 1, 2]))
            got = [(c.c_type, c.arr_type, c.validity is not None, bits_of(c)) for c in out.columns]
            assert [g[:3] for g in got] == [o[:3] for o in outs[i]]
            np.testing.assert_array_equal(sort_records(records([c[3] for c in got])), sort_records(records([c[3] for c in outs[i]])))
    finally:
        delete_join_state(st)


@gpu
def test_cross_join_over_the_output_cap_raises_and_the_state_stays_usable(gpu_lib):
    from bodo_b200._lib import B200Error
    from bodo_b200.streaming.join import (delete_join_state, get_metric, init_nested_loop_join_state, join_build_consume_batch,
                                          join_probe_consume_batch)

    nb = 1 << 16
    b = Table([payload(CT.INT64, nb, 1)])
    big = Table([payload(CT.INT64, (1 << 15) + 1, 2)])
    small = Table([payload(CT.INT64, 3, 3, null_every=2)])  # the probe schema is the first probe call's
    st = init_nested_loop_join_state(-1, ["b"], ["p"], False, False)
    try:
        join_build_consume_batch(st, b, True)
        with pytest.raises(B200Error, match=r"would produce 2147549184 output rows \(32769 probe rows x 65536 build rows\); one probe "
                                            r"call produces at most 2\^31 rows: feed smaller probe batches"):
            join_probe_consume_batch(st, big, False, True)
        assert get_metric(st, 3) == 0
        out, _, _ = join_probe_consume_batch(st, small, True, True)
        got = [bits_of(c) for c in out.columns]
        (bb, bv), (pb, pv) = bits_of(b.columns[0]), bits_of(small.columns[0])
        np.testing.assert_array_equal(got[0][0], np.tile(bb, 3))
        np.testing.assert_array_equal(got[1][0][got[1][1]], np.repeat(pb, nb)[np.repeat(pv, nb)])
        np.testing.assert_array_equal(got[1][1], np.repeat(pv, nb))
    finally:
        delete_join_state(st)


# ---------------------------------------------------------------------------------------------- merge against pandas
@gpu
@pytest.mark.parametrize("sizes", [(7, 5), (0, 4), (300, 0), (1000, 33)])
def test_merge_cross_equals_pandas(gpu_lib, sizes):
    from bodo_b200.physical import merge

    rng = np.random.default_rng(sum(sizes))
    nl, nr = sizes
    left = pd.DataFrame({"a": rng.integers(0, 100, nl), "k": pd.array(np.where(rng.random(nl) < 0.2, None, rng.integers(0, 9, nl)), dtype="Int64"),
                         "f": np.where(rng.random(nl) < 0.1, np.nan, rng.random(nl))})
    right = pd.DataFrame({"k": rng.integers(0, 9, nr).astype(np.int32), "b": rng.random(nr)})
    pd.testing.assert_frame_equal(merge(left, right, how="cross", batch_size=64), left.merge(right, how="cross"))
    pd.testing.assert_frame_equal(merge(left, right, how="cross", suffixes=("_l", "_r")), left.merge(right, how="cross", suffixes=("_l", "_r")))


@gpu
@pytest.mark.parametrize("how", ["inner", "left", "right"])
def test_merge_on_a_condition_alone_equals_pandas_cross_then_filter(gpu_lib, how):
    from bodo_b200.physical import merge

    rng = np.random.default_rng(11)
    events = pd.DataFrame({"x": rng.integers(0, 1000, 700), "eid": np.arange(700)})
    lo = rng.integers(0, 1000, 90)
    bands_df = pd.DataFrame({"lo": lo, "hi": lo + rng.integers(0, 30, 90), "bid": np.arange(90)})
    got = merge(events, bands_df, how=how, non_equi_condition=BAND, batch_size=128)
    m = events.merge(bands_df, how="cross")
    m = m[(m.x >= m.lo) & (m.x < m.hi)]
    if how == "left":  # each event in its place, NULL bands without a partner
        m = pd.concat([m, events[~events.eid.isin(m.eid)]]).sort_values("eid", kind="stable")
    elif how == "right":  # the bands without a partner after the last event
        m = pd.concat([m, bands_df[~bands_df.bid.isin(m.bid)]])
    cols = ["lo", "hi", "bid", "x", "eid"]  # merge's layout: right's columns, then left's
    np.testing.assert_array_equal(got[cols].astype("float64").to_numpy(), m[cols].astype("float64").to_numpy())
