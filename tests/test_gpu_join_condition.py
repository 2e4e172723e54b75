"""The streaming hash join with a non-equi condition against an exact numpy reference that never touches the device.

The reference takes the candidate pairs of the equi-join exactly as tests/test_gpu_join_exact.py does (key_ids / ref_pairs: keys
by value across widths and signedness, float keys with -0.0 = 0.0 and NaN as NA, is_na_equal), evaluates the condition on every
candidate pair with the filter-projection reference evaluator (ref_eval in tests/test_gpu_filter_project.py: NA and NaN cells are
NA, arithmetic and comparisons propagate NA, & / | are Kleene, isnull is never NA, uint64 compares exactly), keeps the pairs whose
value is valid and true, then applies the join kind: a probe row without a passing pair is NULL-extended (left), kept once (anti)
or marked false (mark); a build row without a passing pair over all probe batches goes to the build-outer tail.  Outputs are
compared per probe batch as test_gpu_join_exact.py compares them: c-type, array type and bitmap presence per column, then the
sorted (valid, bits) records; a mark join in order.  Metrics 8 and 9 must equal the reference's candidate and passing pair
counts, and metrics 5, 6 and 7 must stay 0: a condition always takes the CSR form."""

import os
import socket

import numpy as np
import pandas as pd
import pytest

from bodo_b200.expr import build_col, lit, probe_col
from bodo_b200.table import ArrTypes, CTypes, Table
from tests.test_gpu_filter_project import ref_eval
from tests.test_gpu_join_exact import (BATCH_EDGES, FLAGS, KINDS, NULLABLE, _cat, bits_of, canon_key, col, dup_keys, gather, host_slices,
                                       key_ids, payload, records, ref_pairs, sms, sort_records)

CT = CTypes
gpu = pytest.mark.gpu
I64_MIN, I64_MAX, U64_MAX = -(1 << 63), (1 << 63) - 1, (1 << 64) - 1


# ---------------------------------------------------------------------------------------------- the reference
def cond_reference(build, probe, n_keys, kind, na_equal, cond, bnames, pnames):
    """(pairs (build row, probe row; -1 on the NULL side), or the marks of a mark join; candidate pairs; passing pairs).  The key
    columns are the first n_keys of each side, so logical and physical column order agree."""
    bt, pt = _cat(build), _cat(probe)
    bid, pid = key_ids([canon_key(bt.columns[j]) for j in range(n_keys)], [canon_key(pt.columns[j]) for j in range(n_keys)], na_equal)
    bi, pi = ref_pairs(bid, pid, "inner")
    n_cand = len(bi)
    if cond is not None:
        cols = {}
        for side, t, names, rows in (("build", bt, bnames, bi), ("probe", pt, pnames, pi)):
            for name, c in zip(names, t.columns):
                cols[(side, name)] = (c.c_type, np.asarray(c.values_numpy())[rows], bits_of(c)[1][rows])
        _, x, v = ref_eval(cond, cols)
        ok = v & (x != 0)
        bi, pi = bi[ok], pi[ok]
    n_pass = len(bi)
    has = np.zeros(len(pid), bool)
    has[pi] = True
    if kind == "mark":
        return has, n_cand, n_pass
    if kind == "anti":
        un = np.flatnonzero(~has)
        return (np.full(len(un), -1, np.int64), un), n_cand, n_pass
    bo, po = FLAGS[kind]
    if po:
        un = np.flatnonzero(~has)
        bi, pi = np.concatenate([bi, np.full(len(un), -1)]), np.concatenate([pi, un])
    if bo:
        matched = np.zeros(len(bid), bool)
        matched[bi[bi >= 0]] = True
        un = np.flatnonzero(~matched)
        bi, pi = np.concatenate([bi, un]), np.concatenate([pi, np.full(len(un), -1)])
    return (bi.astype(np.int64), pi.astype(np.int64)), n_cand, n_pass


# ---------------------------------------------------------------------------------------------- driving the join
def run(build, probe, n_keys, kind, na_equal, cond, bnames, pnames, used=None, device=False):
    from bodo_b200.streaming.join import (delete_join_state, get_metric, init_join_state, join_build_consume_batch,
                                          join_probe_consume_batch)
    from tests.helpers import table_to_device

    keys = tuple(range(n_keys))
    bo, po = FLAGS[kind]
    st = init_join_state(-1, keys, keys, bnames, pnames, bo, po, is_na_equal=na_equal, is_mark_join=kind == "mark",
                         is_anti_join=kind == "anti", non_equi_condition=cond)
    dev = table_to_device if device else (lambda t: t)
    try:
        for i, b in enumerate(build):
            join_build_consume_batch(st, dev(b), i == len(build) - 1)
        outs = []
        for i, p in enumerate(probe):
            out, _, _ = join_probe_consume_batch(st, dev(p), i == len(probe) - 1, True, used)
            outs.append([(c.c_type, c.arr_type, c.validity is not None, bits_of(c)) for c in out.columns])
        metrics = {m: get_metric(st, m) for m in range(10)}
    finally:
        delete_join_state(st)
    return outs, metrics


def expected(build, probe, kind, res, used):
    """Per probe batch: [(c_type, arr_type, has_bitmap, (bits, valid))] of the general path's output for reference result `res`."""
    bt, pt = _cat(build), _cat(probe)
    bcols = [bits_of(c) for c in bt.columns]
    pcols = [bits_of(c) for c in pt.columns]
    b_has_valid = [any(t.columns[j].validity is not None for t in build) for j in range(bt.n_cols)]
    b_at = [c.arr_type for c in build[0].columns]
    p_at = [c.arr_type for c in probe[0].columns]
    b_ct = [c.c_type for c in build[0].columns]
    p_ct = [c.c_type for c in probe[0].columns]
    bo, po = FLAGS[kind]
    kb = list(range(bt.n_cols)) if used is None else list(used[0])
    kp = list(range(pt.n_cols)) if used is None else list(used[1])
    if kind == "mark":
        kb = []
    starts = np.cumsum([0] + [t.n_rows for t in probe])
    exp_all = []
    for q, pbatch in enumerate(probe):
        s, e = starts[q], starts[q + 1]
        if kind == "mark":
            rows = np.arange(s, e)
            exp = [(p_ct[j], NULLABLE if (pbatch.columns[j].validity is not None or p_at[j] == NULLABLE) else ArrTypes.NUMPY,
                    pbatch.columns[j].validity is not None or p_at[j] == NULLABLE, gather(*pcols[j], rows)) for j in kp]
            exp.append((CT.BOOL, NULLABLE, None, (res[s:e].astype(np.uint64), np.ones(e - s, bool))))
            exp_all.append(exp)
            continue
        bi, pi = res
        sel = ((pi >= s) & (pi < e)) | ((pi < 0) & (q == len(probe) - 1))
        bsel, psel = bi[sel], pi[sel]
        exp = []
        for src in kb:
            nullable = b_has_valid[src] or b_at[src] == NULLABLE or po or kind == "anti"
            exp.append((b_ct[src], NULLABLE if nullable else b_at[src], nullable, gather(*bcols[src], bsel)))
        for src in kp:
            nullable = pbatch.columns[src].validity is not None or p_at[src] == NULLABLE or bo
            exp.append((p_ct[src], NULLABLE if nullable else p_at[src], nullable, gather(*pcols[src], psel)))
        exp_all.append(exp)
    return exp_all


def compare(outs, exp_all, kind, what=""):
    assert len(outs) == len(exp_all)
    for q, (got, exp) in enumerate(zip(outs, exp_all)):
        if kind == "mark":
            exp = [x if x[2] is not None else (x[0], x[1], True if len(x[3][0]) else got[-1][2], x[3]) for x in exp]
            assert [g[:3] for g in got] == [x[:3] for x in exp], (q, [g[:3] for g in got], [x[:3] for x in exp])
            np.testing.assert_array_equal(records([g[3] for g in got]), records([x[3] for x in exp]), err_msg=f"mark batch {q} {what}")
            continue
        assert [g[:3] for g in got] == [x[:3] for x in exp], (q, [g[:3] for g in got], [x[:3] for x in exp])
        g, x = records([c[3] for c in got]), records([c[3] for c in exp])
        assert g.shape == x.shape, (q, what, g.shape, x.shape)
        np.testing.assert_array_equal(sort_records(g), sort_records(x), err_msg=f"probe batch {q} ({kind}) {what}")


def check(build, probe, n_keys, kind, na_equal, cond, bnames, pnames, used=None, device=False):
    outs, m = run(build, probe, n_keys, kind, na_equal, cond, bnames, pnames, used, device)
    res, n_cand, n_pass = cond_reference(build, probe, n_keys, kind, na_equal, cond, bnames, pnames)
    assert m[5] == 0 and m[6] == 0 and m[7] == 0, ("a condition takes the CSR form", m)
    if cond is not None:
        assert (m[8], m[9]) == (n_cand, n_pass), ("metrics 8 / 9: candidate and passing pairs", m, n_cand, n_pass)
    else:
        assert m[8] == 0 and m[9] == 0, m
    compare(outs, expected(build, probe, kind, res, used), kind)
    return outs, m


# ---------------------------------------------------------------------------------------------- inputs
def small_ints(ct, n, lo, hi, rng, na_every=0):
    valid = None
    if na_every:
        valid = rng.random(n) > 1.0 / na_every
    return col(ct, rng.integers(lo, hi, n), valid)


def with_nan(ct, vals, rng, nan_frac=0.05, na_every=0):
    v = np.asarray(vals, dtype=np.float64).copy()
    v[rng.random(len(v)) < nan_frac] = np.nan
    valid = None if not na_every else rng.random(len(v)) > 1.0 / na_every
    return col(ct, v, valid)


def kind_case(n_keys, rng, n_build=3000, n_probe=6000):
    """Duplicated keys with NA keys; a condition over both sides with NA cells and NaN, Kleene logic, isnull and arithmetic."""
    if n_keys == 1:
        bk, pk = [dup_keys(n_build, 1200, rng, na_every=97)], [dup_keys(n_probe, 1600, rng, na_every=89)]
    else:
        bk = [dup_keys(n_build, 40, rng, na_every=101), small_ints(CT.INT32, n_build, 0, 30, rng)]
        pk = [dup_keys(n_probe, 50, rng, na_every=83), small_ints(CT.INT32, n_probe, 0, 40, rng, na_every=30)]
    b = Table(bk + [small_ints(CT.INT32, n_build, 0, 100, rng, na_every=9), with_nan(CT.FLOAT64, rng.random(n_build) * 10, rng),
                    payload(CT.INT64, n_build, 1)])
    p = Table(pk + [small_ints(CT.INT64, n_probe, -10, 120, rng, na_every=11), with_nan(CT.FLOAT32, rng.random(n_probe) * 10, rng, na_every=13),
                    payload(CT.UINT16, n_probe, 2, null_every=7)])
    bnames = [f"bk{j}" for j in range(n_keys)] + ["lo", "hi", "bp"]
    pnames = [f"pk{j}" for j in range(n_keys)] + ["t", "w", "pp"]
    cond = ((probe_col("t") >= build_col("lo")) & (probe_col("w") < build_col("hi"))) | (probe_col("t").isnull() & (build_col("lo") * 2 < 90))
    sizes = BATCH_EDGES + [n_probe - sum(BATCH_EDGES)]
    return [b], host_slices(p, sizes), bnames, pnames, cond


# ================================================================================================ CPU: the reference itself
def test_reference_matches_pandas_merge_and_mask():
    rng = np.random.default_rng(1)
    nb, npr = 400, 900
    b = pd.DataFrame({"k": rng.integers(0, 60, nb), "lo": rng.integers(0, 50, nb), "id": np.arange(nb)})
    p = pd.DataFrame({"k": rng.integers(0, 80, npr), "t": rng.integers(0, 60, npr), "id": np.arange(npr)})
    cond = probe_col("t") > build_col("lo") + 3
    build, probe = [Table([col(CT.INT64, b.k), col(CT.INT64, b.lo), col(CT.INT64, b.id)])], [Table([col(CT.INT64, p.k), col(CT.INT64, p.t), col(CT.INT64, p.id)])]
    m = p.merge(b, on="k", suffixes=("_p", "_b"))
    m = m[m.t > m.lo + 3]
    (bi, pi), n_cand, n_pass = cond_reference(build, probe, 1, "inner", False, cond, ["k", "lo", "id"], ["k", "t", "id"])
    assert sorted(zip(bi.tolist(), pi.tolist())) == sorted(zip(m.id_b.tolist(), m.id_p.tolist()))
    assert n_cand == len(p.merge(b, on="k")) and n_pass == len(m)
    (bi, pi), _, _ = cond_reference(build, probe, 1, "probe_outer", False, cond, ["k", "lo", "id"], ["k", "t", "id"])
    assert sorted(pi[bi < 0].tolist()) == sorted(set(range(npr)) - set(m.id_p.tolist()))
    marks, _, _ = cond_reference(build, probe, 1, "mark", False, cond, ["k", "lo", "id"], ["k", "t", "id"])
    np.testing.assert_array_equal(marks, np.isin(np.arange(npr), m.id_p))


# ================================================================================================ GPU
@gpu
@pytest.mark.parametrize("n_keys", [1, 2])
@pytest.mark.parametrize("device", [False, True])
@pytest.mark.parametrize("na_equal", [False, True])
@pytest.mark.parametrize("kind", KINDS)
def test_every_kind(gpu_lib, kind, na_equal, device, n_keys):
    rng = np.random.default_rng(100 * n_keys + KINDS.index(kind))
    build, probe, bn, pn, cond = kind_case(n_keys, rng)
    check(build, probe, n_keys, kind, na_equal, cond, bn, pn, None, device)


TYPE_CASES = {
    # mixed integer widths and signedness: int8 against uint16, int32 arithmetic
    "int_widths": ((CT.UINT16, [0, 1, 127, 128, 255, 65535, 300, 7]), (CT.INT8, [-128, -1, 0, 1, 127, 100, 7, -7]),
                   lambda: (probe_col("a") < build_col("b")) & (build_col("c") + probe_col("a") > 0)),
    # int64 against uint64 at and above 2^63
    "int64_uint64": ((CT.UINT64, [0, 1, 1 << 63, U64_MAX, I64_MAX, (1 << 63) + 5, 5]), (CT.INT64, [I64_MIN, -1, 0, 1, I64_MAX, 5, 6]),
                     lambda: (probe_col("a") < build_col("b")) | (probe_col("a") == build_col("b"))),
    # float against int: a float64 probe column against an int64 build column, float32 against int16
    "float_int": ((CT.INT64, [-3, 0, 2, 5, 1 << 53, (1 << 53) + 1, I64_MAX]), (CT.FLOAT64, [-2.5, 0.0, -0.0, 2.0, 4.75, 2.0 ** 53, np.nan, np.inf]),
                  lambda: (probe_col("a") <= build_col("b")) & (build_col("c") != probe_col("a") * 2)),
    # DATE (days) against DATETIME (nanoseconds), and a DATE window
    "date_datetime": ((CT.DATETIME, [0, 86_400 * 10 ** 9, 3 * 86_400 * 10 ** 9 - 1, -86_400 * 10 ** 9, 10 ** 18]), (CT.DATE, [-1, 0, 1, 2, 3, 11574]),
                      lambda: (probe_col("a") * 86_400_000_000_000 >= build_col("b")) & (probe_col("a") < build_col("c") + 2)),
}


@gpu
@pytest.mark.parametrize("kind", ["inner", "full_outer", "anti", "mark"])
@pytest.mark.parametrize("case", list(TYPE_CASES))
def test_condition_across_column_types(gpu_lib, case, kind):
    (bt, bvals), (pt, pvals), mk = TYPE_CASES[case]
    rng = np.random.default_rng(7 + list(TYPE_CASES).index(case))
    nb, npr = 900, 2500
    c_ct = {"int_widths": CT.INT32, "int64_uint64": CT.INT16, "float_int": CT.FLOAT32, "date_datetime": CT.DATE}[case]
    bvalid, pvalid = rng.random(nb) > 0.05, rng.random(npr) > 0.05
    b = Table([dup_keys(nb, 60, rng), col(bt, np.array(bvals, dtype=object)[rng.integers(0, len(bvals), nb)], bvalid),
               col(c_ct, rng.integers(-20, 20, nb)), payload(CT.INT64, nb, 3)])
    pv = np.array(pvals, dtype=object)[rng.integers(0, len(pvals), npr)]
    p = Table([dup_keys(npr, 80, rng), col(pt, pv if pt not in (CT.FLOAT64, CT.FLOAT32) else pv.astype(np.float64), pvalid),
               payload(CT.INT64, npr, 4)])
    check([b], host_slices(p, [1000, 1500]), 1, kind, False, mk(), ["k", "b", "c", "bp"], ["k", "a", "pp"])


@gpu
@pytest.mark.parametrize("kind", KINDS)
def test_condition_on_keys_and_dropped_columns(gpu_lib, kind):
    """The condition reads the key columns and columns used_cols drops; the output has only the kept columns."""
    rng = np.random.default_rng(31)
    nb, npr = 2000, 4000
    b = Table([dup_keys(nb, 500, rng, na_every=50), small_ints(CT.INT16, nb, 0, 9, rng, na_every=6), payload(CT.UINT32, nb, 5)])
    p = Table([dup_keys(npr, 700, rng, na_every=40), small_ints(CT.UINT8, npr, 0, 9, rng, na_every=8), payload(CT.INT64, npr, 6)])
    cond = ((build_col("k") * 3 - probe_col("x") > 700) & ~build_col("hidden").isnull()) | (probe_col("k") - build_col("hidden") < 5)
    used = ([2], [2])
    check([b], host_slices(p, [1500, 2500]), 1, kind, True, cond, ["k", "hidden", "bp"], ["k", "x", "pp"], used, True)


@gpu
@pytest.mark.parametrize("kind", KINDS)
def test_always_true_and_always_false(gpu_lib, kind):
    """A condition true on every pair returns what the join without one returns; one that is always false: inner empty, left
    NULL-extends every probe row, right emits every build row in the tail, anti keeps every probe row, every mark is false."""
    rng = np.random.default_rng(41)
    build, probe, bn, pn, _ = kind_case(1, rng, 2000, 5000)
    plain, mp = run(build, probe, 1, kind, True, None, bn, pn)
    assert mp[5] == 0 and mp[7] == 0 and mp[8] == 0 and mp[9] == 0  # duplicated keys: the general path without a condition too
    true_, mt = check(build, probe, 1, kind, True, lit(1) == 1, bn, pn)
    compare(true_, plain, kind, "always true")
    assert mt[8] == mt[9] > 0 and mt[3] == mp[3]
    false_, mf = check(build, probe, 1, kind, True, (probe_col("t") < 0) & (probe_col("t") > 0), bn, pn)
    n_probe, n_build = sum(t.n_rows for t in probe), sum(t.n_rows for t in build)
    rows = mf[3]
    assert mf[9] == 0 and mf[8] == mt[8]
    exp_rows = {"inner": 0, "probe_outer": n_probe, "build_outer": n_build, "full_outer": n_probe + n_build, "anti": n_probe, "mark": n_probe}
    assert rows == exp_rows[kind], (kind, rows)
    if kind == "mark":
        assert not any(batch[-1][3][0].any() for batch in false_)


@gpu
@pytest.mark.parametrize("kind", ["build_outer", "full_outer"])
def test_build_outer_tail_across_probe_batches(gpu_lib, kind):
    """A build row passes only with a probe row of a later batch (need = the probe batch it waits for; 3 = never): it must not
    appear in the tail, and the rows that never pass must."""
    rng = np.random.default_rng(51)
    nb = 1200
    b = Table([dup_keys(nb, 300, rng), col(CT.INT32, rng.integers(0, 4, nb)), payload(CT.INT64, nb, 7)])
    batches = []
    for q in range(3):
        n = 700 + 300 * q
        batches.append(Table([dup_keys(n, 300, rng), col(CT.INT32, np.full(n, q)), payload(CT.INT64, n, 8 + q)]))
    cond = probe_col("batch") == build_col("need")
    check([b], batches, 1, kind, False, cond, ["k", "need", "bp"], ["k", "batch", "pp"])


@gpu
@pytest.mark.parametrize("kind", ["inner", "probe_outer", "anti", "mark"])
def test_ten_thousand_row_duplicate_group(gpu_lib, kind):
    rng = np.random.default_rng(61)
    nb = 10_000 + 500
    bk = np.concatenate([np.full(10_000, 7), rng.integers(100, 300, 500)])
    b = Table([col(CT.INT64, bk), col(CT.INT64, np.concatenate([np.arange(10_000), rng.integers(0, 100, 500)])), payload(CT.INT64, nb, 9)])
    npr = 700
    pk = np.where(rng.random(npr) < 0.3, 7, rng.integers(0, 300, npr))
    p = Table([col(CT.INT64, pk), col(CT.INT64, rng.integers(-100, 10_100, npr), rng.random(npr) > 0.1), payload(CT.INT64, npr, 10)])
    cond = (probe_col("x") > build_col("y")) & (build_col("y") >= 0)
    check([b], host_slices(p, [300, 400]), 1, kind, False, cond, ["k", "y", "bp"], ["k", "x", "pp"])


@gpu
def test_probe_batch_past_one_grid(gpu_lib):
    """grid_for caps the count and gather kernels at 8 CTAs of 256 threads per SM: a larger batch repeats their row loops."""
    G = 8 * sms() * 256
    npr = G + 37
    rng = np.random.default_rng(71)
    nb = 4000
    b = Table([dup_keys(nb, 3000, rng), small_ints(CT.INT64, nb, 0, 100, rng, na_every=10), payload(CT.INT64, nb, 11)])
    p = Table([dup_keys(npr, 6000, rng), small_ints(CT.INT64, npr, 0, 100, rng), payload(CT.INT64, npr, 12)])
    check([b], [p], 1, "probe_outer", False, probe_col("t") >= build_col("lo"), ["k", "lo", "bp"], ["k", "t", "pp"], None, True)


@gpu
def test_unique_keys_take_csr_with_a_condition_and_the_unique_tables_without(gpu_lib):
    """Unique 8-byte bitmap-free build keys take Slot32 without a condition and CSR with one; a bitmap in the build takes Slot16
    without a condition.  The states live in one process, one after the other."""
    from tests.test_gpu_join_exact import check as exact_check

    rng = np.random.default_rng(81)
    nb, npr = 3000, 6000
    keys = rng.permutation(3 * nb)[:nb].astype(np.int64)
    for bitmap in (False, True):
        lo = col(CT.INT64, rng.integers(0, 100, nb), (rng.random(nb) > 0.1) if bitmap else None)
        b = Table([col(CT.INT64, keys), lo, payload(CT.INT64, nb, 13)])
        p = Table([col(CT.INT64, rng.integers(0, 3 * nb, npr)), col(CT.INT64, rng.integers(0, 100, npr)), payload(CT.INT64, npr, 14)])
        probe = host_slices(p, [3000, 3000])
        _, m = exact_check([b], probe, 1, "inner", False, None, True, "slot16" if bitmap else "slot32", None if bitmap else 2)
        assert m[7] == (0 if bitmap else 1)
        check([b], probe, 1, "inner", False, probe_col("t") < build_col("lo"), ["k", "lo", "bp"], ["k", "t", "pp"], None, True)


@gpu
def test_merge_with_a_condition_matches_pandas(gpu_lib):
    """Events into validity windows: merge(events, windows, "acct", "acct", non_equi_condition=...) against pandas merge and a
    boolean mask; how="left" adds every event without a window, NULL-extended."""
    from bodo_b200.physical import merge

    rng = np.random.default_rng(91)
    nw, ne = 3000, 20_000
    acct = rng.integers(0, 500, nw)
    start = rng.integers(0, 10_000, nw)
    windows = pd.DataFrame({"acct": acct, "start": start, "end": start + rng.integers(1, 2_000, nw), "wid": np.arange(nw)})
    events = pd.DataFrame({"acct": rng.integers(0, 600, ne), "ts": rng.integers(0, 12_000, ne), "eid": np.arange(ne)})
    cond = (probe_col("ts") >= build_col("start")) & (probe_col("ts") < build_col("end"))
    m = events.merge(windows, on="acct")
    m = m[(m.ts >= m.start) & (m.ts < m.end)]
    exp_inner = sorted(zip(m.eid.tolist(), m.wid.tolist()))
    lonely = sorted(set(range(ne)) - set(m.eid.tolist()))
    exp_left = sorted(exp_inner + [(e, -1) for e in lonely])
    for how, exp in (("inner", exp_inner), ("left", exp_left)):
        got = merge(events, windows, "acct", "acct", how=how, non_equi_condition=cond, batch_size=7_000)
        wid = pd.Series(got["wid"]).astype("Int64").fillna(-1).astype(np.int64)
        assert sorted(zip(pd.Series(got["eid"]).astype(np.int64).tolist(), wid.tolist())) == exp, how


# ---------------------------------------------------------------------------------------------- sharded
def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _sharded_worker(rank, world, port, q):
    import torch
    import torch.distributed as dist

    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), BODO_BCAST_JOIN_THRESHOLD="0")
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", rank))
    try:
        from bodo_b200.streaming.join import delete_join_state, init_join_state, join_build_consume_batch, join_probe_consume_batch

        windows, events, cond = _sharded_tables()
        res = {}
        for how, bo, po in (("inner", False, False), ("left", False, True), ("right", True, False)):
            st = init_join_state(-1, (0,), (0,), tuple(windows.columns), tuple(events.columns), bo, po, build_parallel=True,
                                 probe_parallel=True, device=rank, is_na_equal=True, non_equi_condition=cond)
            bchunk, pchunk = (len(windows) + world - 1) // world, (len(events) + world - 1) // world
            join_build_consume_batch(st, Table.from_pandas(windows.iloc[rank * bchunk:(rank + 1) * bchunk]), True)
            mine = events.iloc[rank * pchunk:(rank + 1) * pchunk]
            half = len(mine) // 2
            pairs = []
            for i, part in enumerate((mine.iloc[:half], mine.iloc[half:])):
                out, _, _ = join_probe_consume_batch(st, Table.from_pandas(part), i == 1, True)
                df = out.to_pandas()
                pairs += list(zip(df["eid"].astype("Int64").fillna(-1).tolist(), df["wid"].astype("Int64").fillna(-1).tolist()))
            delete_join_state(st)
            res[how] = pairs
        q.put((rank, res))
    except Exception:
        import traceback

        q.put((rank, traceback.format_exc()))
    finally:
        dist.destroy_process_group()


def _sharded_tables():
    rng = np.random.default_rng(101)
    nw, ne = 20_000, 80_000
    start = rng.integers(0, 10_000, nw)
    windows = pd.DataFrame({"acct": rng.integers(0, 3_000, nw), "start": start, "end": start + rng.integers(1, 1_500, nw), "wid": np.arange(nw)})
    events = pd.DataFrame({"acct": rng.integers(0, 3_500, ne), "ts": rng.integers(0, 12_000, ne), "eid": np.arange(ne)})
    return windows, events, (probe_col("ts") >= build_col("start")) & (probe_col("ts") < build_col("end"))


@gpu
@pytest.mark.timeout(600)
def test_sharded_join_with_a_condition_nccl(gpu_lib):
    """build_parallel / probe_parallel: rows are shuffled by key before the local join, so the union of the ranks' outputs is the
    conditional join of the global tables."""
    import torch
    import torch.multiprocessing as mp

    world = min(torch.cuda.device_count(), 4)
    if world < 2:
        pytest.skip("needs at least 2 GPUs")
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_sharded_worker, args=(r, world, port, q)) for r in range(world)]
    for p in procs:
        p.start()
    res = [q.get(timeout=500) for _ in range(world)]
    for p in procs:
        p.join(timeout=60)
    for r in res:
        assert isinstance(r[1], dict), r
    windows, events, _ = _sharded_tables()
    m = events.merge(windows, on="acct")
    m = m[(m.ts >= m.start) & (m.ts < m.end)]
    inner = list(zip(m.eid.tolist(), m.wid.tolist()))
    exp = {"inner": sorted(inner),
           "left": sorted(inner + [(e, -1) for e in sorted(set(range(len(events))) - set(m.eid.tolist()))]),
           "right": sorted(inner + [(-1, w) for w in sorted(set(range(len(windows))) - set(m.wid.tolist()))])}
    for how in exp:
        got = sorted(p for _, r in res for p in r[how])
        assert got == exp[how], how
