"""The streaming hash join against an exact numpy reference, bit for bit, at the paths and edges where its kernels go wrong.

The reference never touches the device.  Each key cell becomes a canonical value: an integer or temporal key is (class, raw 64
bits) with class -1 for a negative signed value, +1 for a uint64 of at least 2^63 and 0 otherwise, so integer keys compare by
value across widths and signedness, as pandas merge compares them; a float key is its canon_float_key (-0.0 is 0.0, NaN is NA).
Key tuples of both sides are factorised together; (build row, probe row) pairs come from a stable argsort of the build ids, then
the NULL-extended rows of the outer kinds are added.  Every expected cell is the input cell's bits and validity (on the unique-key
forms the build key column takes the probe key's, join.cu's documented rule), and a column is nullable exactly when the join's
output plan says so.  The comparison is exact: c-type, array type and bitmap presence per column, then every row as a record of
(valid, bits if valid else 0) per column, lexsorted, per probe batch (the build-outer tail belongs to the last batch).  A mark
join is compared in order.  Payloads are row-unique over 64 bits, so a wrong pairing cannot hide behind equal values.

Each GPU test asserts the table form, the kernel and the geometry it relies on (metrics 1, 5, 6, 7; the SM count), so a change
in the code under it fails the test instead of letting it pass without reaching the path."""

import ctypes
import os
import re

import numpy as np
import pandas as pd
import pytest

from bodo_b200.table import ArrTypes, Column, CTypes, Table

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CT = CTypes
NP_OF = {CT.INT8: np.int8, CT.UINT8: np.uint8, CT.BOOL: np.bool_, CT.INT16: np.int16, CT.UINT16: np.uint16, CT.INT32: np.int32,
         CT.UINT32: np.uint32, CT.FLOAT32: np.float32, CT.DATE: np.int32, CT.INT64: np.int64, CT.UINT64: np.uint64,
         CT.FLOAT64: np.float64, CT.DATETIME: np.int64, CT.TIMEDELTA: np.int64}
TYPE_NAME = {CT.INT8: "int8", CT.UINT8: "uint8", CT.BOOL: "bool", CT.INT16: "int16", CT.UINT16: "uint16", CT.INT32: "int32",
             CT.UINT32: "uint32", CT.FLOAT32: "float32", CT.DATE: "date", CT.INT64: "int64", CT.UINT64: "uint64",
             CT.FLOAT64: "float64", CT.DATETIME: "datetime", CT.TIMEDELTA: "timedelta"}
ALL_TYPES = list(NP_OF)
SIGNED = {CT.INT8, CT.INT16, CT.INT32, CT.INT64, CT.DATE, CT.DATETIME, CT.TIMEDELTA}
FLOATS = {CT.FLOAT32, CT.FLOAT64}
UVIEW = {1: np.uint8, 2: np.uint16, 4: np.uint32, 8: np.uint64}
NULLABLE = ArrTypes.NULLABLE_INT_BOOL
I64_MIN, I64_MAX, U64_MAX = -(1 << 63), (1 << 63) - 1, (1 << 64) - 1
ODD = 0x9E3779B97F4A7C15
KINDS = ("inner", "probe_outer", "build_outer", "full_outer", "anti", "mark")
FLAGS = {"inner": (False, False), "probe_outer": (False, True), "build_outer": (True, False), "full_outer": (True, True),
         "anti": (False, False), "mark": (False, False)}
J_MAX_COLS = 32


# ---------------------------------------------------------------------------------------------- columns
def col(ct, values, valid=None, nullable=False):
    """A host column of type `ct`; `valid` (bool array) gives it a bitmap, `nullable` the nullable array type without one."""
    if isinstance(values, (list, tuple)):  # python ints, exactly (a list mixing 2^64 - 1 and -1 would go through float64)
        values = np.array(values, dtype=object)
    data = np.ascontiguousarray(np.asarray(values).astype(NP_OF[ct]) if ct != CT.BOOL else np.asarray(values).astype(bool))
    bm = None if valid is None else np.packbits(np.asarray(valid, dtype=bool), bitorder="little")
    return Column(data, bm, ct, NULLABLE if (nullable or valid is not None) else ArrTypes.NUMPY, len(data))


def raw_col(ct, bits64, valid=None, nullable=False):
    """A column whose cells are the low bytes of `bits64` (uint64); bool cells keep the low bit."""
    w = np.dtype(NP_OF[ct]).itemsize
    b = np.asarray(bits64, dtype=np.uint64)
    data = (b & np.uint64(1)).astype(bool) if ct == CT.BOOL else b.astype(UVIEW[w]).view(NP_OF[ct])
    return col(ct, data, valid, nullable)


def unique_bits(n, salt):
    """Row-unique 64-bit patterns: (row + salt) * an odd constant over all 64 bits."""
    return (np.arange(n, dtype=np.uint64) + np.uint64(salt)) * np.uint64(ODD)


EDGE_BITS = {  # edge values of each width, placed at the first rows of payload columns
    8: [I64_MIN & U64_MAX, I64_MAX, U64_MAX, 0x7FF8DEADBEEF0001, 0x8000000000000000, 1, 0xFFF0000000000001, 0x7FF0000000000000],
    4: [0x7FC01234, 0x80000000, 1, 0xFFFFFFFF, 0x7FFFFFFF, 0xFF800001],
    2: [0x8000, 0x7FFF, 0xFFFF],
    1: [0x80, 0x7F, 0xFF],
}


def payload(ct, n, salt, nullable=False, null_every=0):
    bits = unique_bits(n, salt)
    w = np.dtype(NP_OF[ct]).itemsize
    e = np.array(EDGE_BITS[w], dtype=np.uint64)[: n]
    bits[: len(e)] = e
    valid = None
    if null_every:
        valid = np.ones(n, bool)
        valid[salt % null_every::null_every] = False
    return raw_col(ct, bits, valid, nullable)


def bits_of(c: Column):
    """(raw bits zero-extended to uint64, validity as bool) of a host or device column."""
    v = np.asarray(c.values_numpy())
    if v.dtype == np.bool_:
        v = v.view(np.uint8)
    b = v.view(UVIEW[v.dtype.itemsize]).astype(np.uint64)
    m = c.valid_mask_numpy()
    return b, (np.ones(len(b), bool) if m is None else m.astype(bool))


def concat_cols(batches, j):
    bits, valid = zip(*(bits_of(t.columns[j]) for t in batches)) if batches else ((), ())
    return np.concatenate(bits) if bits else np.zeros(0, np.uint64), np.concatenate(valid) if valid else np.zeros(0, bool)


def host_slices(t: Table, sizes):
    out, i0 = [], 0
    for s in sizes:
        b = t.slice(i0, i0 + s)
        if s == 0:  # an empty batch carries no bitmap (a device copy of an empty one would be a null pointer)
            b = Table([Column(c.data, None, c.c_type, c.arr_type, 0) for c in b.columns], list(b.names))
        out.append(b)
        i0 += s
    assert i0 == t.n_rows
    return out


# ---------------------------------------------------------------------------------------------- the reference
def canon_key(c: Column):
    """(na, class, value) of each key cell: integers by value, floats as canon_float_key with NaN as NA."""
    ct = c.c_type
    d = np.asarray(c.values_numpy())
    m = c.valid_mask_numpy()
    valid = np.ones(len(d), bool) if m is None else m.astype(bool)
    if ct in FLOATS:
        x = d.astype(np.float64)
        na = ~valid | np.isnan(x)
        x = np.where(x == 0, 0.0, x)
        val = np.ascontiguousarray(x).view(np.uint64).copy()
        cls = np.zeros(len(d), np.int8)
    elif ct in SIGNED:
        v = d.astype(np.int64)
        val, cls, na = v.view(np.uint64).copy(), np.where(v < 0, -1, 0).astype(np.int8), ~valid
    else:
        val = d.astype(np.uint64)
        cls, na = np.where(val >= np.uint64(1 << 63), 1, 0).astype(np.int8), ~valid
    val[na] = 0
    cls[na] = 0
    return na, cls, val


def key_ids(bkeys, pkeys, na_equal):
    """Dense ids of the key tuples of both sides, factorised together (a lexsort over the tuple components gives the ids
    np.unique over a structured array gives, far faster); -1 for a tuple with an NA column when NA does not join NA."""
    nb = len(bkeys[0][0])
    comps = []
    for bk, pk in zip(bkeys, pkeys):
        comps += [np.concatenate([bk[i], pk[i]]) for i in range(3)]
    n = len(comps[0])
    ids = np.full(n, -1, np.int64)
    if n:
        order = np.lexsort(comps[::-1])
        new = np.zeros(n, bool)
        new[0] = True
        for c in comps:
            s = c[order]
            new[1:] |= s[1:] != s[:-1]
        ids[order] = np.cumsum(new) - 1
    if not na_equal:
        anyna = np.logical_or.reduce([np.concatenate([bk[0], pk[0]]) for bk, pk in zip(bkeys, pkeys)])
        ids[anyna] = -1
    return ids[:nb], ids[nb:]


def ref_pairs(bid, pid, kind):
    """(build row, probe row) pairs, -1 on the NULL side; for a mark join the per-probe-row mark."""
    order = np.argsort(bid, kind="stable")
    sb = bid[order]
    lo, hi = np.searchsorted(sb, pid, "left"), np.searchsorted(sb, pid, "right")
    cnt = np.where(pid >= 0, hi - lo, 0)
    if kind == "mark":
        return cnt > 0
    if kind == "anti":
        pi = np.flatnonzero(cnt == 0)
        return np.full(len(pi), -1, np.int64), pi
    total = int(cnt.sum())
    pi = np.repeat(np.arange(len(pid)), cnt)
    within = np.arange(total) - np.repeat(np.cumsum(cnt) - cnt, cnt)
    bi = order[np.repeat(lo, cnt) + within] if total else np.zeros(0, np.int64)
    build_outer, probe_outer = FLAGS[kind]
    if probe_outer:
        un = np.flatnonzero(cnt == 0)
        bi, pi = np.concatenate([bi, np.full(len(un), -1)]), np.concatenate([pi, un])
    if build_outer:
        matched = np.zeros(len(bid), bool)
        matched[bi[bi >= 0]] = True
        un = np.flatnonzero(~matched)
        bi, pi = np.concatenate([bi, un]), np.concatenate([pi, np.full(len(un), -1)])
    return bi.astype(np.int64), pi.astype(np.int64)


def reference(build, probe, n_keys, kind, na_equal):
    bt, pt = _cat(build), _cat(probe)
    bid, pid = key_ids([canon_key(bt.columns[j]) for j in range(n_keys)], [canon_key(pt.columns[j]) for j in range(n_keys)], na_equal)
    return ref_pairs(bid, pid, kind)


def _cat(batches):
    """One host table of the concatenated batches (a batch without a bitmap is all valid)."""
    cols = []
    for j in range(batches[0].n_cols):
        ct = batches[0].columns[j].c_type
        bits, valid = concat_cols(batches, j)
        cols.append(raw_col(ct, bits, valid))
    return Table(cols)


def gather(bits, valid, rows):
    ok = rows >= 0
    r = np.where(ok, rows, 0)
    v = valid[r] & ok if len(bits) else np.zeros(len(rows), bool)
    return np.where(v, bits[r] if len(bits) else 0, np.uint64(0)).astype(np.uint64), v


def records(cols):
    """Rows as records of (valid, bits if valid else 0) per column."""
    if not cols:
        return np.zeros((0, 0), np.uint64)
    return np.stack([x for b, v in cols for x in (v.astype(np.uint64), np.where(v, b, np.uint64(0)).astype(np.uint64))], axis=1)


def sort_records(r):
    return r[np.lexsort(r.T[::-1])] if r.shape[1] else r


# ---------------------------------------------------------------------------------------------- driving the join
def run_join(build, probe, n_keys=1, kind="inner", na_equal=False, used=None, device=False, expected_build_rows=0):
    """Build batches, then probe batches; returns ([(c_type, arr_type, has_bitmap, [(bits, valid)]) per probe batch], metrics)."""
    from bodo_b200.streaming.join import (delete_join_state, get_metric, init_join_state, join_build_consume_batch,
                                          join_probe_consume_batch)
    from tests.helpers import table_to_device

    keys = tuple(range(n_keys))
    bo, po = FLAGS[kind]
    st = init_join_state(-1, keys, keys, [f"b{j}" for j in range(build[0].n_cols)], [f"p{j}" for j in range(probe[0].n_cols)], bo, po,
                         is_na_equal=na_equal, expected_build_rows=expected_build_rows, is_mark_join=kind == "mark",
                         is_anti_join=kind == "anti")
    dev = table_to_device if device else (lambda t: t)
    try:
        for i, b in enumerate(build):
            join_build_consume_batch(st, dev(b), i == len(build) - 1)
        outs = []
        for i, p in enumerate(probe):
            out, _, _ = join_probe_consume_batch(st, dev(p), i == len(probe) - 1, True, used)
            outs.append([(c.c_type, c.arr_type, c.validity is not None, bits_of(c)) for c in out.columns])
        metrics = {m: get_metric(st, m) for m in (0, 1, 5, 6, 7)}
    finally:
        delete_join_state(st)
    return outs, metrics


def expected_cap(n_build):
    cap = 1024
    while cap < 2 * n_build:
        cap <<= 1
    return cap


def check(build, probe, n_keys=1, kind="inner", na_equal=False, used=None, device=False, form="csr", inline=None, expected_build_rows=0):
    """Run the join and compare every probe batch's output with the reference, exactly.  `form`: the table form the build must
    take (csr, slot16 or slot32); `inline`: the number of probe batches the inline kernel must take on slot32."""
    outs, m = run_join(build, probe, n_keys, kind, na_equal, used, device, expected_build_rows)
    n_build = sum(t.n_rows for t in build)
    assert m[0] == n_build and m[1] == expected_cap(n_build), m
    nonempty = sum(1 for t in probe if t.n_rows)
    if form == "csr":
        assert m[5] == 0 and m[7] == 0, ("expected the general (CSR) path", m)
    elif form == "slot16":
        assert m[7] == 0 and m[6] == 0 and m[5] == nonempty, ("expected the Slot16 table and the fast kernel", m)
    else:
        assert m[7] == 1 and m[5] == nonempty, ("expected the inline-built Slot32 table", m)
        if inline is not None:
            assert m[6] == inline, ("inline probe batches", m, inline)
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
    res = reference(build, probe, n_keys, kind, na_equal)
    starts = np.cumsum([0] + [t.n_rows for t in probe])
    for q, got in enumerate(outs):
        s, e = starts[q], starts[q + 1]
        last = q == len(probe) - 1
        pbatch = probe[q]
        if kind == "mark":
            rows = np.arange(s, e)
            exp = [(p_ct[j], NULLABLE if (pbatch.columns[j].validity is not None or p_at[j] == NULLABLE) else ArrTypes.NUMPY,
                    pbatch.columns[j].validity is not None or p_at[j] == NULLABLE, gather(*pcols[j], rows)) for j in kp]
            # the mark column: BOOL, nullable, every row valid (an empty batch may leave it without a bitmap)
            exp.append((CT.BOOL, NULLABLE, True if e > s else got[-1][2], (res[s:e].astype(np.uint64), np.ones(e - s, bool))))
            assert [g[:3] for g in got] == [x[:3] for x in exp], (q, [g[:3] for g in got], [x[:3] for x in exp])
            np.testing.assert_array_equal(records([g[3] for g in got]), records([x[3] for x in exp]), err_msg=f"mark batch {q}")
            continue
        bi, pi = res
        sel = ((pi >= s) & (pi < e)) | ((pi < 0) & last)
        bsel, psel = bi[sel], pi[sel]
        exp = []
        for src in kb:
            unique_key = src == 0 and form != "csr" and n_keys == 1
            if unique_key:
                has_bm = pbatch.columns[0].validity is not None
                cell = gather(*pcols[0], psel)
            else:
                has_bm = b_has_valid[src]
                cell = gather(*bcols[src], bsel)
            nullable = has_bm or b_at[src] == NULLABLE or po or kind == "anti"
            exp.append((b_ct[src], NULLABLE if nullable else b_at[src], nullable, cell))
        for src in kp:
            nullable = pbatch.columns[src].validity is not None or p_at[src] == NULLABLE or bo
            exp.append((p_ct[src], NULLABLE if nullable else p_at[src], nullable, gather(*pcols[src], psel)))
        for x in exp:  # the reference itself: a column without a bitmap has only valid cells
            assert x[2] or x[3][1].all()
        assert [g[:3] for g in got] == [x[:3] for x in exp], (q, [g[:3] for g in got], [x[:3] for x in exp])
        g, x = records([c[3] for c in got]), records([c[3] for c in exp])
        assert g.shape == x.shape, (q, g.shape, x.shape)
        np.testing.assert_array_equal(sort_records(g), sort_records(x), err_msg=f"probe batch {q} ({kind}, {form})")
    return outs, m


def sms():
    import torch

    return torch.cuda.get_device_properties(0).multi_processor_count


def probe_grid(n):
    """CTAs of the fast and inline probe kernels (join.cu probe_unique)."""
    return min(8 * sms(), (n + 1023) // 1024)


BATCH_EDGES = [0, 1, 1023, 1024, 1025]  # probe batch sizes at the tile edges; output counts off multiples of 8 and 32


# ---------------------------------------------------------------------------------------------- xxh3 restated (hash-chain keys)
def seed_hash_join():
    text = open(os.path.join(ROOT, "bodo_b200", "csrc", "common.cuh")).read()
    return int(re.search(r"SEED_HASH_JOIN\s*=\s*(0x[0-9a-fA-F]+)u", text).group(1), 16)


def xxh3_64_short8(keys, seed32):
    """xxh3_64_short(key, 8, seed) of bodo_oracle.c, vectorised over uint64 keys."""
    M = np.uint64(0x9FB21C651E98DF25)
    k = np.asarray(keys).astype(np.int64).view(np.uint64)
    s = seed32 & 0xFFFFFFFF
    sw = int.from_bytes(s.to_bytes(4, "little"), "big")
    seed = s ^ (sw << 32)
    bitflip = np.uint64(((0x1CAD21F72C81017C ^ 0xDB979083E96DD4DE) - seed) & U64_MAX)
    in1, in2 = k & np.uint64(0xFFFFFFFF), k >> np.uint64(32)
    with np.errstate(over="ignore"):
        h = (in2 + (in1 << np.uint64(32))) ^ bitflip
        rot = lambda x, r: (x << np.uint64(r)) | (x >> np.uint64(64 - r))
        h ^= rot(h, 49) ^ rot(h, 24)
        h *= M
        h ^= (h >> np.uint64(35)) + np.uint64(8)
        h *= M
        return h ^ (h >> np.uint64(28))


def home_slot(keys, cap):
    return ((xxh3_64_short8(keys, seed_hash_join()) >> np.uint64(32)) & np.uint64(cap - 1)).astype(np.int64)


def assert_pairs_match_pandas(bk, pk, bi, pi):
    """pandas merge on the same keys gives the same pairs.  pandas meets a uint64 and an int64 key through float64, which rounds
    INT64_MAX onto 2^63, so rows holding INT64_MAX are left out of this comparison (the reference keeps them apart)."""
    bk, pk = np.asarray(bk), np.asarray(pk)
    bok = np.array([int(v) != I64_MAX for v in bk], bool)
    pok = np.array([int(v) != I64_MAX for v in pk], bool)
    m = pd.DataFrame({"k": bk[bok], "bi": np.flatnonzero(bok)}).merge(pd.DataFrame({"k": pk[pok], "pi": np.flatnonzero(pok)}), on="k", how="inner")
    keep = bok[bi] & pok[pi]
    assert sorted(zip(bi[keep].tolist(), pi[keep].tolist())) == sorted(zip(m.bi.tolist(), m.pi.tolist()))


# ================================================================================================ CPU: the reference itself
def test_xxh3_restatement_matches_the_oracle(oracle):
    L = oracle.lib()
    fn = L.oracle_xxh3_64_short
    fn.restype = ctypes.c_uint64
    fn.argtypes = [ctypes.c_uint64, ctypes.c_int, ctypes.c_uint32]
    rng = np.random.default_rng(3)
    keys = np.concatenate([rng.integers(I64_MIN, I64_MAX, 2000, dtype=np.int64, endpoint=True),
                           np.array([0, 1, -1, I64_MIN, I64_MAX], np.int64)])
    seed = seed_hash_join()
    assert seed == 0xB0D01286
    got = xxh3_64_short8(keys, seed)
    exp = np.array([fn(int(k) & U64_MAX, 8, seed) for k in keys], dtype=np.uint64)
    np.testing.assert_array_equal(got, exp)


@pytest.mark.parametrize("na_equal", [False, True])
@pytest.mark.parametrize("kind", KINDS)
def test_reference_matches_the_oracle_on_int64_keys(oracle, kind, na_equal):
    rng = np.random.default_rng(11)
    nb, npr = 3000, 5000
    bk, pk = rng.integers(-400, 400, nb), rng.integers(-600, 600, npr)
    bv, pv = rng.random(nb) > 0.05, rng.random(npr) > 0.05
    build = [Table([col(CT.INT64, bk, bv)])]
    probe = [Table([col(CT.INT64, pk, pv)])]
    bo, po = FLAGS[kind]
    if kind in ("anti", "mark"):
        obi, opi = oracle.hash_join(bk, bv, pk, pv, False, False, na_equal)
        has = np.zeros(npr, bool)
        has[opi] = True
        got = reference(build, probe, 1, kind, na_equal)
        if kind == "mark":
            np.testing.assert_array_equal(got, has)
        else:
            np.testing.assert_array_equal(np.sort(got[1]), np.flatnonzero(~has))
            assert (got[0] == -1).all()
        return
    obi, opi = oracle.hash_join(bk, bv, pk, pv, bo, po, na_equal)
    bi, pi = reference(build, probe, 1, kind, na_equal)
    exp = np.stack([obi, opi], 1)
    got = np.stack([bi, pi], 1)
    np.testing.assert_array_equal(sort_records(got.view(np.uint64)), sort_records(exp.view(np.uint64)))


@pytest.mark.parametrize("pair", [(CT.INT8, CT.UINT8), (CT.INT16, CT.UINT16), (CT.INT32, CT.UINT32), (CT.INT64, CT.UINT64)])
def test_reference_matches_pandas_across_signedness(pair):
    """pandas merge compares integer keys by value: uint64 2^64 - 1 does not meet int64 -1, nor uint32 2^32 - 1 int32 -1."""
    s, u = pair
    w = np.dtype(NP_OF[s]).itemsize * 8
    sv = [-1, 5, -(1 << (w - 1)), (1 << (w - 1)) - 1, 0, 7]
    uv = [(1 << w) - 1, 5, 1 << (w - 1), (1 << (w - 1)) - 1, 0, 9]
    for bt_, bv_, pt_, pv_ in ((u, uv, s, sv), (s, sv, u, uv)):
        build, probe = [Table([col(bt_, bv_)])], [Table([col(pt_, pv_)])]
        bi, pi = reference(build, probe, 1, "inner", False)
        assert_pairs_match_pandas(build[0].columns[0].data, probe[0].columns[0].data, bi, pi)
        assert sorted(pi.tolist()) == [1, 3, 4]  # 5, the largest common signed value, 0; never the top-bit pair


# ================================================================================================ GPU
gpu = pytest.mark.gpu


def side(n, key, n_payload_types, salt, null_every=0, nullable=False):
    """key column + one row-unique payload column per type in n_payload_types."""
    cols = [key] + [payload(ct, n, salt + 97 * j, nullable, null_every) for j, ct in enumerate(n_payload_types)]
    return Table(cols)


def dup_keys(n, n_distinct, rng, na_every=0):
    k = rng.integers(0, n_distinct, n)
    valid = None
    if na_every:
        valid = np.ones(n, bool)
        valid[3::na_every] = False
    return col(CT.INT64, k, valid)


FORMS = ["csr", "slot16", "slot32_nf0", "slot32_nf1", "slot32_nf2", "slot16_from32", "csr_mk"]


def form_case(form, rng, n_build=3000, n_probe=6000):
    """(build batches, probe batches, n_keys, used, expected form, expected inline probe batches)."""
    sizes = BATCH_EDGES + [n_probe - sum(BATCH_EDGES)]
    if form == "csr":
        b = side(n_build, dup_keys(n_build, 1500, rng, na_every=97), [CT.INT32, CT.UINT8], 1, null_every=5)
        p = side(n_probe, dup_keys(n_probe, 2500, rng, na_every=89), [CT.INT64, CT.INT16], 2, null_every=7)
        return [b], host_slices(p, sizes), 1, None, "csr", None
    if form == "csr_mk":
        k0 = dup_keys(n_build, 40, rng, na_every=101)
        b = Table([k0, col(CT.INT32, rng.integers(0, 30, n_build)), payload(CT.UINT64, n_build, 3, null_every=9)])
        p = Table([dup_keys(n_probe, 50, rng, na_every=83), col(CT.INT32, rng.integers(0, 40, n_probe), rng.random(n_probe) > 0.03),
                   payload(CT.FLOAT64, n_probe, 4)])
        return [b], host_slices(p, sizes), 2, None, "csr", None
    keys = (rng.permutation(n_build * 3)[:n_build].astype(np.int64) - n_build) * 7919
    keys[5] = I64_MIN  # the marker key: slot cap + 1
    pk = np.where(rng.random(n_probe) < 0.5, keys[rng.integers(0, n_build, n_probe)], rng.integers(-(1 << 40), 1 << 40, n_probe))
    pk[::211] = I64_MIN
    if form == "slot16":
        kv = np.ones(n_build, bool)
        kv[17] = False  # one NA build key: one row in the NA group
        b = side(n_build, col(CT.INT64, keys, kv), [CT.INT16, CT.FLOAT64], 5, null_every=6)
        pv = rng.random(n_probe) > 0.02
        p = side(n_probe, col(CT.INT64, pk, pv), [CT.UINT32, CT.DATETIME], 6, null_every=4)
        return [b], host_slices(p, sizes), 1, None, "slot16", None
    if form.startswith("slot32"):
        nf = int(form[-1])
        b = side(n_build, col(CT.INT64, keys), [CT.UINT64, CT.FLOAT64][:nf], 7)
        p = side(n_probe, col(CT.INT64, pk), [CT.INT64, CT.FLOAT64, CT.TIMEDELTA], 8)
        nbk = 1 + nf
        used = ([nbk - 1, 0][: 1 + (nf > 0)], [3, 0, 2, 1])  # a subset, reordered: 4 kept probe columns
        return [b], host_slices(p, sizes), 1, used, "slot32", len(sizes) - 1
    assert form == "slot16_from32"
    b = side(n_build, col(CT.INT64, keys), [CT.INT64], 9)
    p = side(n_probe, col(CT.INT64, pk), [CT.FLOAT64], 10)
    ps = host_slices(p, [2000, 2000, 2000])
    mid = ps[1]
    mid.columns[1] = col(CT.FLOAT64, mid.columns[1].data, np.arange(mid.n_rows) % 3 != 0)  # a bitmap: not inline
    return [b], ps, 1, None, "slot32", 2


FORM_KINDS = [(f, k) for f in FORMS for k in (KINDS if f.startswith("csr") else ("inner",))]  # unique-key forms: inner only


@gpu
@pytest.mark.parametrize("device", [False, True])
@pytest.mark.parametrize("na_equal", [False, True])
@pytest.mark.parametrize("form,kind", FORM_KINDS)
def test_every_form_and_kind(gpu_lib, form, kind, na_equal, device):
    rng = np.random.default_rng(10 * FORMS.index(form) + KINDS.index(kind))
    build, probe, nk, used, exp_form, inline = form_case(form, rng)
    check(build, probe, nk, kind, na_equal, used, device, exp_form, inline)


@gpu
@pytest.mark.parametrize("wide", ["build", "probe"])
@pytest.mark.parametrize("form", ["csr", "slot16"])
def test_every_column_width(gpu_lib, form, wide):
    """Every column type on one side, numpy and nullable (with NULLs), through the general gather (full outer: NULL-extended
    cells on both sides) or the fast kernel's packed payload.  Edge bits (INT64_MIN, INT64_MAX, 2^64 - 1, NaN with a payload,
    -0.0, subnormals, float32 NaN) sit in the first rows."""
    rng = np.random.default_rng(21)
    n_build, n_probe = 1500, 4000
    if form == "csr":
        bkey, pkey = dup_keys(n_build, 900, rng, na_every=50), dup_keys(n_probe, 1200, rng, na_every=60)
        kind = "full_outer"
    else:
        bkey = col(CT.INT64, rng.permutation(3 * n_build)[:n_build])
        pkey = col(CT.INT64, rng.integers(0, 3 * n_build, n_probe))
        kind = "inner"
    many = []
    for j, ct in enumerate(ALL_TYPES):
        n = n_build if wide == "build" else n_probe
        many.append(payload(ct, n, 31 * j + 1))
        many.append(payload(ct, n, 31 * j + 2, nullable=True, null_every=3 + j % 4))
    few_b = [payload(ct, n_build, 900 + j) for j, ct in enumerate((CT.INT64, CT.UINT8, CT.FLOAT32))]
    few_p = [payload(ct, n_probe, 910 + j) for j, ct in enumerate((CT.INT64, CT.INT16, CT.DATE))]
    if wide == "build":
        b, p = Table([bkey] + many), Table([pkey] + few_p)
    else:
        b, p = Table([bkey] + few_b), Table([pkey] + many)
    used = (list(range(b.n_cols)), [1, 2, 3]) if wide == "build" else ([0, 1, 2], list(range(p.n_cols)))
    assert len(used[0]) + len(used[1]) == J_MAX_COLS
    probe = host_slices(p, [1000, 1001, 1999])
    check([b], probe, 1, kind, True, used, False, form)


@gpu
@pytest.mark.parametrize("form", ["csr", "slot16", "slot32"])
def test_kept_columns_subset_reordered_repeated(gpu_lib, form):
    rng = np.random.default_rng(5)
    n = 2000
    if form == "csr":
        bkey, kind = dup_keys(n, 800, rng), "probe_outer"
    else:
        bkey, kind = col(CT.INT64, rng.permutation(10 * n)[:n]), "inner"
    pkey = col(CT.INT64, rng.integers(0, 10 * n if form != "csr" else 1000, 3 * n))
    b = side(n, bkey, [CT.INT64, CT.FLOAT64] if form == "slot32" else [CT.INT32, CT.UINT64], 1)
    p = side(3 * n, pkey, [CT.INT64, CT.FLOAT64, CT.UINT64], 2)
    used = ([2, 2, 1], [3, 1, 3]) if form != "slot32" else ([2, 1], [3, 1, 3, 2])  # the keys dropped, a column repeated
    check([b], host_slices(p, [3000, 3000]), 1, kind, False, used, True, form, inline=2 if form == "slot32" else None)


def key_values(ct, n_distinct, rng):
    """Distinct keys of type ct, edge values first: the type's min and max, 0, -1 / the marker pattern."""
    if ct == CT.BOOL:
        return np.array([False, True])
    if ct in FLOATS:
        f = NP_OF[ct]
        bits = [0x8000000000000000, 1, 0x7FF0000000000000, 0xFFF0000000000000] if ct == CT.FLOAT64 else [0x80000000, 1, 0x7F800000, 0xFF800000]
        edge = np.array(bits, dtype=UVIEW[np.dtype(f).itemsize]).view(f)  # -0.0, a subnormal, +-inf
        rest = rng.permutation(1 << 20)[: n_distinct].astype(f) * f(0.5) + f(1.25)
        return np.concatenate([edge, rest])
    info = np.iinfo(NP_OF[ct])
    edge = [info.min, info.max, 0]
    if ct in SIGNED:
        edge.append(-1)
    if ct == CT.UINT64:
        edge.append(1 << 63)  # INT64_MIN's bits
    lo, hi = max(info.min, -(1 << 40)), min(info.max, 1 << 40)
    rest = rng.choice(np.arange(lo, min(hi, lo + 4 * n_distinct + 10)), min(n_distinct, hi - lo - 8), replace=False)
    vals = list(dict.fromkeys([int(v) for v in edge] + [int(v) for v in rest]))
    return np.array(vals, dtype=object).astype(NP_OF[ct])


KEY_FORMS = [(ct, f) for ct in ALL_TYPES for f in ("csr", "slot16", "slot32") if f != "slot32" or np.dtype(NP_OF[ct]).itemsize == 8]


@gpu
@pytest.mark.parametrize("na_equal", [False, True])
@pytest.mark.parametrize("ct,form", KEY_FORMS, ids=[f"{TYPE_NAME[ct]}-{f}" for ct, f in KEY_FORMS])
def test_every_single_key_type(gpu_lib, ct, form, na_equal):
    """One key of each type: edge values (the marker pattern INT64_MIN and uint64 2^63 go to slot cap + 1), NA keys (slot cap),
    NaN / -0.0 float keys; CSR with duplicated keys, Slot16 with unique keys and one NA, Slot32 for the 8-byte types."""
    w = np.dtype(NP_OF[ct]).itemsize
    rng = np.random.default_rng(ct * 7 + 1)
    vals = key_values(ct, 200, rng)
    nb = len(vals)
    if form == "csr":
        bk = np.concatenate([vals, vals[: nb // 2]])
        bvalid = np.ones(len(bk), bool)
        bvalid[1::37] = False
    else:
        bk = vals
        bvalid = np.ones(nb, bool)
        if form == "slot16":
            bvalid[min(4, nb - 1)] = False
    npr = 3000
    pk = vals[rng.integers(0, nb, npr)]
    if ct in FLOATS:
        nan = np.array([0x7FF8DEADBEEF0001 if w == 8 else 0x7FC01234], dtype=UVIEW[w]).view(NP_OF[ct])[0]
        pk = pk.copy()
        pk[::13] = nan
        pk[5::17] = -pk[5::17]  # partly absent values, and -0.0 meets 0.0 among them
        if form != "slot16":
            bk = bk.copy()
            bk[2] = nan  # a NaN build key: NA under the float rule
    pvalid = rng.random(npr) > 0.05
    if form == "slot32":
        bcol_ = col(ct, bk)
        pcol_ = col(ct, pk)
        b = side(len(bk), bcol_, [CT.INT64], 3)
        p = side(npr, pcol_, [CT.UINT64], 4)
        check([b], host_slices(p, [1500, 1500]), 1, "inner", na_equal, None, True, "slot32", inline=2)
        return
    b = side(len(bk), col(ct, bk, bvalid), [CT.INT64], 3)
    p = side(npr, col(ct, pk, pvalid), [CT.UINT64], 4)
    kinds = ["inner"] if form == "slot16" else ["inner", "full_outer", "anti", "mark"]
    for kind in kinds:
        check([b], host_slices(p, [1000, 2000]), 1, kind, na_equal, None, False, form)


CROSS = [(CT.INT8, CT.UINT8), (CT.INT16, CT.UINT16), (CT.INT32, CT.UINT32), (CT.INT64, CT.UINT64), (CT.DATETIME, CT.UINT64),
         (CT.TIMEDELTA, CT.UINT64)]


def cross_values(s, u):
    w = np.dtype(NP_OF[s]).itemsize * 8
    sv = [-1, 5, -(1 << (w - 1)), (1 << (w - 1)) - 1, 0, 7, -2, 11]
    uv = [(1 << w) - 1, 5, 1 << (w - 1), (1 << (w - 1)) - 1, 0, 9, (1 << w) - 2, 11]
    return sv, uv


CROSS_FORMS = [(pr, f) for pr in CROSS for f in ("csr", "slot16", "slot32") if f != "slot32" or np.dtype(NP_OF[pr[0]]).itemsize == 8]


@gpu
@pytest.mark.parametrize("build_unsigned", [True, False])
@pytest.mark.parametrize("pair,form", CROSS_FORMS, ids=[f"{TYPE_NAME[s]}-{TYPE_NAME[u]}-{f}" for (s, u), f in CROSS_FORMS])
def test_integer_keys_join_by_value_across_signedness(gpu_lib, pair, build_unsigned, form):
    """uint64 2^64 - 1 must not meet int64 -1 (nor 2^63 meet INT64_MIN): keys join by value at every width, as pandas merge
    does.  A probe key the build type cannot hold has no partner but is not NA: it is NULL-extended, kept by an anti join, marked
    false, and dropped by the runtime filter, which keeps every row that has a partner."""
    from bodo_b200.streaming.join import (delete_join_state, init_join_state, join_build_consume_batch, runtime_join_filter)
    from tests.helpers import table_to_device

    s, u = pair
    sv, uv = cross_values(s, u)
    bt_, pt_ = (u, s) if build_unsigned else (s, u)
    bvals, pvals = (uv, sv) if build_unsigned else (sv, uv)
    rep = 40
    pk = np.array(pvals * rep, dtype=object)
    bk = list(bvals) + ([bvals[1]] if form == "csr" else [])  # a duplicate key for the CSR form
    b = side(len(bk), col(bt_, np.array(bk, dtype=object).astype(NP_OF[bt_])), [CT.INT64], 1)
    p = Table([col(pt_, pk.astype(NP_OF[pt_])), col(CT.INT64, np.arange(len(pk)))])  # the payload is the row id
    probe = host_slices(p, [len(pk) // 2, len(pk) - len(pk) // 2])
    if form == "slot32":
        check([b], probe, 1, "inner", False, None, True, "slot32", inline=0)  # such batches take the fast kernel
    elif form == "slot16":
        b.columns[1] = payload(CT.INT64, b.n_rows, 1, null_every=3)  # a bitmap: not inline
        check([b], probe, 1, "inner", False, None, True, "slot16")
    else:
        for kind in ("inner", "probe_outer", "anti", "mark"):
            check([b], probe, 1, kind, False, None, True, "csr")
    # pandas merge agrees on the pairs
    bi, pi = reference([b], probe, 1, "inner", False)
    assert_pairs_match_pandas(b.columns[0].data, p.columns[0].data, bi, pi)
    # the runtime filter: keeps every row with a partner, drops every row whose key the build type cannot hold
    st = init_join_state(-1, (0,), (0,), ["k", "v"], ["k", "v"], False, False)
    try:
        join_build_consume_batch(st, table_to_device(b), True)
        kept = runtime_join_filter((st,), table_to_device(p), ((0,),))
        kept_rows = np.sort(bits_of(kept.columns[1])[0].astype(np.int64))
    finally:
        delete_join_state(st)
    partner = np.zeros(p.n_rows, bool)
    partner[pi] = True
    assert np.isin(np.flatnonzero(partner), kept_rows).all()
    top = np.array([int(v) < 0 or int(v) >= 1 << 63 for v in pk]) if np.dtype(NP_OF[s]).itemsize == 8 else np.zeros(len(pk), bool)
    assert not np.isin(np.flatnonzero(top), kept_rows).any()


@gpu
@pytest.mark.parametrize("kind", ["inner", "probe_outer", "anti", "mark"])
def test_multi_key_joins_by_value_across_signedness(gpu_lib, kind):
    """Key position 1 is uint64 on the build side and int64 on the probe side."""
    rng = np.random.default_rng(8)
    sv, uv = cross_values(CT.INT64, CT.UINT64)
    b = Table([col(CT.INT32, np.repeat(np.arange(3), len(uv))), col(CT.UINT64, np.array(uv * 3, dtype=object).astype(np.uint64)),
               payload(CT.INT64, 3 * len(uv), 1)])
    n = 600
    p = Table([col(CT.INT32, rng.integers(0, 4, n)), col(CT.INT64, np.array(sv, dtype=object)[rng.integers(0, len(sv), n)].astype(np.int64)),
               payload(CT.INT64, n, 2)])
    check([b], host_slices(p, [300, 300]), 2, kind, False, None, True, "csr")


@gpu
def test_fast_and_inline_probes_past_one_grid_and_inline_build_past_one_grid(gpu_lib):
    """A probe batch of more than 8 * SMs * 1024 rows repeats the fast and the inline kernels' tile loop, and an inline build of
    more than that many rows repeats join_build_inline_kernel's loop."""
    G = 8 * sms() * 1024
    n_build, n_probe = G + 11, G + 37
    assert probe_grid(n_probe) * 1024 < n_probe and min((n_build + 1023) // 1024, 8 * sms()) * 1024 < n_build
    rng = np.random.default_rng(1)
    keys = rng.permutation(3 * n_build)[:n_build].astype(np.int64) * 5 - 7
    keys[9] = I64_MIN
    b = side(n_build, col(CT.INT64, keys), [CT.INT64, CT.FLOAT64], 1)
    pk = rng.integers(-10, 15 * n_build, n_probe)
    pk[::777] = I64_MIN
    p_inl = side(n_probe, col(CT.INT64, pk), [CT.INT64], 2)
    p_fast = side(n_probe, col(CT.INT64, pk, rng.random(n_probe) > 0.01), [CT.INT64], 3)
    check([b], [p_inl, p_fast], 1, "inner", False, None, True, "slot32", inline=1)


@gpu
def test_fast_probe_past_one_grid_on_slot16(gpu_lib):
    G = 8 * sms() * 1024
    n_probe = G + 37
    assert probe_grid(n_probe) * 1024 < n_probe
    rng = np.random.default_rng(2)
    n_build = 400_000
    b = side(n_build, col(CT.INT64, rng.permutation(2 * n_build)[:n_build]), [CT.INT16, CT.INT32], 1, null_every=11)
    p = side(n_probe, col(CT.INT64, rng.integers(0, 2 * n_build, n_probe)), [CT.UINT8], 2)
    check([b], [p], 1, "inner", False, None, True, "slot16")


@gpu
def test_general_probe_and_build_outer_tail_past_2_21_scan_elements(gpu_lib):
    """The offsets scan's single-CTA tile_carry_kernel gives each thread more than one tile only past 2^21 elements: a general-path
    probe batch of more than 2^21 rows, and a build-outer tail over more than 2^21 build rows."""
    n_probe = (1 << 21) + 5 + 1000
    n_build = (1 << 21) + 3
    assert (n_probe - 1000 + 1 + 2047) // 2048 > 1024 and (n_build + 1 + 2047) // 2048 > 1024
    rng = np.random.default_rng(3)
    b = side(n_build, col(CT.INT64, rng.integers(0, 3 * n_build, n_build)), [CT.INT32], 1)
    p = side(n_probe, col(CT.INT64, rng.integers(0, 3 * n_build, n_probe)), [CT.INT64], 2)
    check([b], host_slices(p, [n_probe - 1000, 1000]), 1, "full_outer", False, ([1], [1]), True, "csr")  # keys dropped: less host memory


def chain_keys(cap, rng):
    """Build keys whose home slots are the last slots of a cap-slot table (chains wrap to slot 0), with a cluster of 64 keys that
    share home slot cap - 1, and absent keys with those home slots."""
    cand = rng.integers(I64_MIN + 1, I64_MAX, 1 << 21, dtype=np.int64)
    hs = home_slot(cand, cap)
    cluster = cand[hs == cap - 1][:80]
    tail = np.concatenate([cand[hs == cap - 1 - d][:3] for d in range(1, 6)])
    head = np.concatenate([cand[hs == d][:2] for d in range(0, 4)])  # displaced by the wrapped chain
    assert len(cluster) == 80
    build = np.concatenate([cluster[:64], tail, head])
    absent = np.concatenate([cluster[64:], cand[hs == cap - 2][3:10]])
    assert len(np.unique(build)) == len(build)
    return build, absent


@gpu
@pytest.mark.parametrize("form", ["csr", "slot16", "slot32"])
def test_probe_chains_that_wrap_the_table(gpu_lib, form):
    cap = 1024
    rng = np.random.default_rng(6)
    bk, absent = chain_keys(cap, rng)
    hs = home_slot(bk, cap)
    assert (hs[:64] == cap - 1).all() and 2 * len(bk) + 2 <= cap
    bkeys = np.concatenate([bk, bk[:50]]) if form == "csr" else bk
    npr = 4000
    pk = np.concatenate([bk, absent])[rng.integers(0, len(bk) + len(absent), npr)]
    if form == "slot32":
        b = side(len(bkeys), col(CT.INT64, bkeys), [CT.INT64, CT.FLOAT64], 1)
        p = side(npr, col(CT.INT64, pk), [CT.INT64], 2)
        check([b], host_slices(p, [2000, 2000]), 1, "inner", False, None, True, "slot32", inline=2)
        return
    b = side(len(bkeys), col(CT.INT64, bkeys), [CT.INT32], 1, null_every=5 if form == "slot16" else 0)
    p = side(npr, col(CT.INT64, pk), [CT.INT64], 2)
    for kind in (["inner"] if form == "slot16" else ["inner", "full_outer", "anti"]):
        check([b], host_slices(p, [2000, 2000]), 1, kind, False, None, True, form)


@gpu
@pytest.mark.parametrize("ebr", ["below", "equal", "above"])
@pytest.mark.parametrize("kind", ["inner", "full_outer"])
def test_build_stream(gpu_lib, kind, ebr):
    """Many build batches: empty ones, one that brings the first bitmap, a nullable-typed batch without a bitmap; the column
    reservation of expected_build_rows below, at and above the real count."""
    rng = np.random.default_rng(7)
    n = 5000
    keys = rng.permutation(4 * n)[:n] if kind == "inner" else rng.integers(0, n, n)
    b = side(n, col(CT.INT64, keys), [CT.INT32, CT.FLOAT64], 1)
    batches = host_slices(b, [0, 700, 0, 1300, 1, 999, 0, 2000])
    v = np.arange(1300) % 4 != 0
    batches[3].columns[1] = col(CT.INT32, batches[3].columns[1].data, v)  # the first bitmap
    batches[5].columns[2] = Column(batches[5].columns[2].data, None, CT.FLOAT64, NULLABLE, 999)  # nullable type, no bitmap
    exp_rows = {"below": n // 3, "equal": n, "above": 3 * n}[ebr]
    p = side(8000, col(CT.INT64, rng.integers(0, 4 * n, 8000)), [CT.INT64], 2)
    check(batches, host_slices(p, [4000, 4000]), 1, kind, False, None, False, "slot16" if kind == "inner" else "csr",
          expected_build_rows=exp_rows)


@gpu
@pytest.mark.parametrize("kind", ["inner", "probe_outer", "full_outer", "anti", "mark"])
def test_probe_call_that_keeps_no_columns(gpu_lib, kind):
    """A batch is a list of columns, so a probe call that keeps none could not say how many rows it produced (COUNT(*) over it
    would read 0): it is refused, naming used_cols.  A mark join always has its mark column."""
    from bodo_b200._lib import B200Error
    from bodo_b200.streaming.join import delete_join_state, init_join_state, join_build_consume_batch, join_probe_consume_batch

    rng = np.random.default_rng(9)
    b = side(100, col(CT.INT64, rng.integers(0, 50, 100)), [CT.INT64], 1)
    p = side(300, col(CT.INT64, rng.integers(0, 80, 300)), [CT.INT64], 2)
    bo, po = FLAGS[kind]
    st = init_join_state(-1, (0,), (0,), ["k", "v"], ["k", "v"], bo, po, is_mark_join=kind == "mark", is_anti_join=kind == "anti")
    try:
        join_build_consume_batch(st, b, True)
        if kind == "mark":
            out, _, _ = join_probe_consume_batch(st, p, True, True, ([], []))
            assert out.n_cols == 1 and out.n_rows == 300
            has = np.isin(p.columns[0].data, b.columns[0].data)
            np.testing.assert_array_equal(bits_of(out.columns[0])[0].astype(bool), has)
        else:
            with pytest.raises(B200Error, match="used_cols"):
                join_probe_consume_batch(st, p, True, True, ([], []))
    finally:
        delete_join_state(st)
