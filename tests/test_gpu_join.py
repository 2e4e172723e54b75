"""GPU parity tests for the streaming hash join: row-set equality under sort against the CPU oracle and pandas
(join output order is unspecified in the reference as well; its tests sort before comparing)."""

import numpy as np
import pandas as pd
import pytest

from bodo_b200.streaming.join import (delete_join_state, init_join_state, join_build_consume_batch,
                                      join_probe_consume_batch)
from bodo_b200.table import Table
from tests.helpers import table_to_device

pytestmark = pytest.mark.gpu


def stream_join(build_df, probe_df, build_outer=False, probe_outer=False, batch_size=None, to_device=False, used_cols=None, is_na_equal=True):
    """Reference-shaped streaming loop (bodo/tests/test_streaming/test_join.py): build batches, then probe batches."""
    bt, pt = Table.from_pandas(build_df), Table.from_pandas(probe_df)
    st = init_join_state(-1, (0,), (0,), tuple(build_df.columns), tuple(probe_df.columns), build_outer, probe_outer, is_na_equal=is_na_equal)
    bs = batch_size or max(bt.n_rows, pt.n_rows, 1)
    it, last = 0, False
    while not last:
        b = bt.slice(it * bs, (it + 1) * bs)
        last = (it + 1) * bs >= bt.n_rows
        it += 1
        join_build_consume_batch(st, table_to_device(b) if to_device else b, last)
    outs, it, last = [], 0, False
    while not last:
        p = pt.slice(it * bs, (it + 1) * bs)
        last = (it + 1) * bs >= pt.n_rows
        it += 1
        out, out_last, _ = join_probe_consume_batch(st, table_to_device(p) if to_device else p, last, True, used_cols)
        outs.append(out.to_pandas())
    delete_join_state(st)
    return pd.concat(outs, ignore_index=True)


def oracle_join_frame(oracle, build_df, probe_df, build_outer=False, probe_outer=False, is_na_equal=True):
    def kv(s):
        if hasattr(s.array, "_mask"):
            return np.asarray(s.array._data, dtype=np.int64), ~np.asarray(s.array._mask)
        return s.to_numpy(dtype=np.int64), None
    bk, bv = kv(build_df.iloc[:, 0])
    pk, pv = kv(probe_df.iloc[:, 0])
    bi, pi = oracle.hash_join(bk, bv, pk, pv, build_outer, probe_outer, is_na_equal)
    out = {}
    for name in build_df.columns:
        col = build_df[name].astype("Float64" if build_df[name].dtype.kind == "f" else "Int64")
        vals = col.take(np.where(bi >= 0, bi, 0)).reset_index(drop=True)
        vals[bi < 0] = pd.NA
        out[f"b_{name}"] = vals
    for name in probe_df.columns:
        col = probe_df[name].astype("Float64" if probe_df[name].dtype.kind == "f" else "Int64")
        vals = col.take(np.where(pi >= 0, pi, 0)).reset_index(drop=True)
        vals[pi < 0] = pd.NA
        out[f"p_{name}"] = vals
    return pd.DataFrame(out)


def canon(df):
    df = df.copy()
    df.columns = [f"c{i}" for i in range(df.shape[1])]
    for c in df.columns:
        df[c] = df[c].to_numpy(dtype="float64", na_value=np.nan)
    return df.sort_values(list(df.columns), na_position="last").reset_index(drop=True)


def assert_rowset_equal(got, exp):
    g, e = canon(got), canon(exp)
    assert g.shape == e.shape, (g.shape, e.shape)
    np.testing.assert_array_equal(g.to_numpy(), e.to_numpy())


@pytest.mark.parametrize("build_outer,probe_outer", [(False, False), (True, True), (True, False), (False, True)])
@pytest.mark.parametrize("to_device", [False, True])
def test_hash_join_non_nullable_outer_fixture(gpu_lib, oracle, build_outer, probe_outer, to_device):
    # fixture of test_hash_join_non_nullable_outer (bodo/tests/test_streaming/test_join.py:922-940):
    # many-to-many duplicates (key 2 -> 25 x 25 rows), unmatched keys on both sides
    df1 = pd.DataFrame({"A": [1, 2, 3, 4, 5] * 25, "B": np.array([1, 2, 3, 4, 5] * 25, dtype=np.int32)})
    df2 = pd.DataFrame({"C": [2, 6] * 25, "D": np.array([2, 6] * 25, dtype=np.int8)})
    got = stream_join(df1, df2, build_outer, probe_outer, batch_size=40, to_device=to_device)
    exp = oracle_join_frame(oracle, df1, df2, build_outer, probe_outer)
    assert_rowset_equal(got, exp)
    how = {(False, False): "inner", (True, True): "outer", (True, False): "left", (False, True): "right"}[(build_outer, probe_outer)]
    pexp = df1.merge(df2, left_on="A", right_on="C", how=how)
    assert_rowset_equal(got, pexp)


def test_shuffle_batching_fixture(gpu_lib):
    # test_shuffle_batching (bodo/tests/test_streaming/test_join.py:4803-4816): 60 000-row 1:1 join
    build = pd.DataFrame({"A": np.arange(60000), "B": [1, 2, 3, 4, 5, 6] * 10000})
    probe = pd.DataFrame({"C": np.arange(60000), "D": [1, 2, 3, 4, 5, 6] * 10000})
    got = stream_join(build, probe, batch_size=4096)
    exp = pd.DataFrame({"A": np.arange(60000), "B": [1, 2, 3, 4, 5, 6] * 10000, "C": np.arange(60000), "D": [1, 2, 3, 4, 5, 6] * 10000})
    assert_rowset_equal(got, exp)


@pytest.mark.parametrize("how", ["inner", "left", "right", "outer"])
def test_merge_nullable_keys(gpu_lib, how):
    # test_merge fixture (bodo/tests/test_df_lib/test_end_to_end.py:1255-1286): nullable Int64 keys [2,2,3] vs [2,3,8];
    # NA keys match NA keys (pandas semantics)
    left = pd.DataFrame({"A": pd.array([2, 2, 3, None, None], dtype="Int64"), "B": [1.5, 2.5, 3.5, 4.5, 5.5]})
    right = pd.DataFrame({"C": pd.array([2, 3, 8, None], dtype="Int64"), "D": pd.array([10, None, 30, 40], dtype="Int64")})
    # reference convention: right table = build side
    bo, po = {"inner": (False, False), "left": (False, True), "right": (True, False), "outer": (True, True)}[how]
    got = stream_join(right, left, bo, po, batch_size=2)
    exp = right.merge(left, left_on="C", right_on="A", how={"left": "right", "right": "left"}.get(how, how))
    assert_rowset_equal(got, exp)


def test_empty_sides(gpu_lib):
    b = pd.DataFrame({"A": np.array([], dtype=np.int64), "B": np.array([], dtype=np.float64)})
    p = pd.DataFrame({"C": np.arange(10, dtype=np.int64), "D": np.arange(10, dtype=np.float64)})
    assert len(stream_join(b, p)) == 0
    assert len(stream_join(b, p, probe_outer=True)) == 10
    assert len(stream_join(p, b)) == 0
    assert len(stream_join(p, b, build_outer=True)) == 10


def test_synthetic_join_vs_oracle(gpu_lib, oracle):
    rng = np.random.default_rng(5)
    nb, npr = 200_000, 1_000_000
    build = pd.DataFrame({"k": rng.permutation(nb).astype(np.int64), "b1": rng.integers(0, 1 << 40, nb), "b2": rng.random(nb)})
    probe = pd.DataFrame({"k": rng.integers(0, nb * 2, npr).astype(np.int64), "p1": rng.integers(0, 1 << 40, npr), "p2": rng.random(npr)})
    got = stream_join(build, probe, batch_size=300_000, to_device=True)
    exp = oracle_join_frame(oracle, build, probe)
    assert_rowset_equal(got, exp)
    # kept columns: drop the probe key and b2
    got2 = stream_join(build, probe, batch_size=300_000, to_device=True, used_cols=([0, 1], [1, 2]))
    assert_rowset_equal(got2, exp.iloc[:, [0, 1, 4, 5]])


@pytest.mark.parametrize("build_outer,probe_outer", [(False, False), (True, True), (True, False), (False, True)])
def test_na_keys_never_match_on_the_streaming_door(gpu_lib, oracle, build_outer, probe_outer):
    # is_na_equal=False is what join_state_init_py_entry constructs (bodo/libs/streaming/_join.cpp:4087-4136, NA build keys
    # filtered at :3180): NA keys match nothing and survive only as NULL-extended rows of an outer side
    build = pd.DataFrame({"A": pd.array([2, None, 3, None, 7], dtype="Int64"), "B": [1.5, 2.5, 3.5, 4.5, 5.5]})
    probe = pd.DataFrame({"C": pd.array([2, 3, None, 8, None, 2], dtype="Int64"), "D": pd.array([10, None, 30, 40, 50, 60], dtype="Int64")})
    got = stream_join(build, probe, build_outer, probe_outer, batch_size=2, is_na_equal=False)
    exp = oracle_join_frame(oracle, build, probe, build_outer, probe_outer, is_na_equal=False)
    assert_rowset_equal(got, exp)
    n_inner = 3  # 2-2, 2-2 (probe has two 2s), 3-3
    n_exp = n_inner + (3 if build_outer else 0) + (3 if probe_outer else 0)  # unmatched: build {NA, NA, 7}, probe {NA, 8, NA}
    assert len(got) == n_exp


@pytest.mark.parametrize("n_payload", [0, 1, 2])
def test_inline_payload_probe_matches_oracle(gpu_lib, oracle, n_payload, monkeypatch):
    """All-8-byte bitmap-free schemas with <= 2 build payload columns probe a Slot32 table (key + payload in one 32-byte
    sector, join_probe_inline_kernel, metric 6); same rows as the oracle and as the two-sector fast kernel (B200_JOIN_INLINE=0).
    The marker key (INT64_MIN, the table's free-slot value) is present on both sides."""
    from bodo_b200.streaming.join import get_metric
    rng = np.random.default_rng(9)
    nb, npr = 150_000, 700_001
    bk = rng.permutation(nb).astype(np.int64) * 3
    bk[7] = np.iinfo(np.int64).min
    build = pd.DataFrame({"k": bk})
    for j in range(n_payload):
        build[f"b{j}"] = rng.integers(-(1 << 50), 1 << 50, nb) if j == 0 else rng.random(nb)
    pk = rng.integers(0, nb * 4, npr).astype(np.int64)
    pk[::1000] = np.iinfo(np.int64).min
    probe = pd.DataFrame({"k": pk, "p1": rng.integers(0, 1 << 40, npr), "p2": rng.random(npr)})
    exp = oracle_join_frame(oracle, build, probe)

    def run(used_cols=None):
        bt, pt = Table.from_pandas(build), Table.from_pandas(probe)
        st = init_join_state(-1, (0,), (0,), tuple(build.columns), tuple(probe.columns), False, False)
        join_build_consume_batch(st, table_to_device(bt), True)
        outs = []
        for i0 in range(0, npr, 250_000):
            out, _, _ = join_probe_consume_batch(st, table_to_device(pt.slice(i0, i0 + 250_000)), i0 + 250_000 >= npr, True, used_cols)
            outs.append(out.to_pandas())
        m = get_metric(st, 6)
        delete_join_state(st)
        return pd.concat(outs, ignore_index=True), m

    got, used = run()
    assert used >= 1, "the inline-payload probe kernel was expected to run for this schema"
    assert_rowset_equal(got, exp)
    nbc = 1 + n_payload
    got2, used2 = run(([0] if n_payload == 0 else [nbc - 1], [2, 1]))  # kept subset, probe columns reordered
    assert used2 >= 1
    assert_rowset_equal(got2, exp.iloc[:, [0 if n_payload == 0 else nbc - 1, nbc + 2, nbc + 1]])
    monkeypatch.setenv("B200_JOIN_INLINE", "0")
    got3, used3 = run()
    assert used3 == 0
    assert_rowset_equal(got3, exp)


@pytest.mark.parametrize("is_na_equal", [False, True])
@pytest.mark.parametrize("to_device", [False, True])
def test_anti_and_mark_joins_vs_pandas(gpu_lib, is_na_equal, to_device):
    """LEFT ANTI (probe rows without a partner, NULL build columns dropped by the caller) and MARK joins (every probe row + a
    boolean "has a partner" column), reference: is_anti_join / is_mark_join of HashJoinState (_join.cpp:763-767, 3668-3693).
    Duplicated build keys must not duplicate output rows; NA probe keys match NA build keys only under is_na_equal."""
    rng = np.random.default_rng(21)
    nb, npr = 5_000, 40_000
    build = pd.DataFrame({"k": pd.array(rng.integers(0, 3_000, nb), dtype="Int64"), "b1": rng.integers(0, 100, nb)})
    build.loc[::500, "k"] = pd.NA
    probe = pd.DataFrame({"k": pd.array(rng.integers(0, 6_000, npr), dtype="Int64"), "p1": rng.random(npr), "p2": rng.integers(0, 1 << 40, npr)})
    probe.loc[::777, "k"] = pd.NA
    pna = probe.k.isna().to_numpy()
    has = np.where(pna, is_na_equal, probe.k.fillna(-1).isin(build.k.dropna()).to_numpy())

    def run(**kind):
        bt, pt = Table.from_pandas(build), Table.from_pandas(probe)
        st = init_join_state(-1, (0,), (0,), tuple(build.columns), tuple(probe.columns), False, False, is_na_equal=is_na_equal, **kind)
        join_build_consume_batch(st, table_to_device(bt) if to_device else bt, True)
        outs = []
        for i0 in range(0, npr, 15_000):
            p = pt.slice(i0, i0 + 15_000)
            out, _, _ = join_probe_consume_batch(st, table_to_device(p) if to_device else p, i0 + 15_000 >= npr, True, ([], [0, 1, 2]))
            outs.append(out.to_pandas())
        delete_join_state(st)
        return pd.concat(outs, ignore_index=True)

    anti = run(is_anti_join=True)
    exp_anti = probe[~has].reset_index(drop=True)
    assert_rowset_equal(anti, exp_anti)
    markdf = run(is_mark_join=True)
    assert markdf.shape == (npr, 4)
    # a mark join keeps the probe rows in order: row i of the output is probe row i
    np.testing.assert_array_equal(markdf.iloc[:, 3].to_numpy(dtype=bool), has)
    np.testing.assert_array_equal(markdf.iloc[:, 2].to_numpy(dtype=np.int64), probe.p2.to_numpy())


def test_runtime_join_filter_has_no_false_negatives(gpu_lib):
    """runtime_join_filter (bodo/libs/streaming/join.py:1392-1415): rows outside the build keys' [min, max] and bloom misses are
    dropped before the probe; no row with a partner may be lost, and the false-positive rate of the ~8 bits / key split-block
    bloom filter stays small."""
    from bodo_b200.streaming.join import build_runtime_filter, runtime_join_filter
    rng = np.random.default_rng(4)
    nb, npr = 200_000, 1_000_000
    bk = rng.choice(np.arange(1_000_000, 3_000_000), nb, replace=False).astype(np.int64)
    build = pd.DataFrame({"k": bk, "b1": rng.integers(0, 100, nb)})
    pk = rng.integers(0, 4_000_000, npr).astype(np.int64)
    probe = pd.DataFrame({"p0": rng.random(npr), "k": pd.array(pk, dtype="Int64")})
    probe.loc[::1000, "k"] = pd.NA
    st = init_join_state(-1, (0,), (1,), tuple(build.columns), tuple(probe.columns), False, False)
    join_build_consume_batch(st, table_to_device(Table.from_pandas(build)), True)
    words, [(mn, mx)] = build_runtime_filter(st)
    assert (mn, mx) == (int(bk.min()), int(bk.max())) and words.numel() == (nb // 32 + 1) * 8
    kept = runtime_join_filter((st,), table_to_device(Table.from_pandas(probe)), ((1,),)).to_pandas()
    partner = probe.k.isin(bk).fillna(False).to_numpy()
    kept_keys = kept.iloc[:, 1].to_numpy(dtype="float64", na_value=np.nan)
    assert np.isin(pk[partner], kept_keys[~np.isnan(kept_keys)].astype(np.int64)).all()
    assert len(kept) >= partner.sum() and not np.isnan(kept_keys).any()
    in_range = (pk >= mn) & (pk <= mx) & ~probe.k.isna().to_numpy()
    false_pos = len(kept) - partner.sum()
    assert false_pos <= 0.08 * (in_range.sum() - partner.sum()), (false_pos, in_range.sum(), partner.sum())
    # the join over the filtered rows equals the join over all rows
    out_f, _, _ = join_probe_consume_batch(st, kept_table := runtime_join_filter((st,), table_to_device(Table.from_pandas(probe)), ((1,),)), True, True)
    delete_join_state(st)
    assert out_f.n_rows == partner.sum()
