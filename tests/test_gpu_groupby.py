"""GPU parity tests for the streaming hash groupby (call through the C ABI; compare with the CPU oracle
and with pandas, the reference's own oracle).  Bar: integer aggregates bit-exact; float aggregates within
rtol=1e-5 / atol=1e-8 (bodo/tests/utils.py:179-180)."""

import numpy as np
import pandas as pd
import pytest

from bodo_b200.table import Table
from tests.helpers import (assert_frames_equal, oracle_groupby_frame, positional, stream_groupby)

pytestmark = pytest.mark.gpu


def _basic_df(use_np_data):
    # test_groupby_basic fixture (bodo/tests/test_streaming/test_groupby.py:83-96)
    groups = [1, 2, 1, 1, 2, 0, 1, 2] * 100
    data = [1, 3, 5, 11, 1, 3, 5, 3] * 100
    return pd.DataFrame({"A": groups, "B": np.array(data, dtype=np.int32) if use_np_data else data})


@pytest.mark.parametrize("func_name", ["sum", "mean", "count", "min", "max", "size"])
@pytest.mark.parametrize("use_np_data", [True, False])
@pytest.mark.parametrize("to_device", [False, True])
def test_groupby_basic(gpu_lib, oracle, func_name, use_np_data, to_device):
    df = _basic_df(use_np_data)
    t = Table.from_pandas(df)
    got = stream_groupby(t, (0,), (func_name,), (0, 1), (1,), batch_size=3 if not to_device else 96, to_device=to_device)
    exp = df.groupby("A", as_index=False).agg(func_name) if func_name != "size" else df.groupby("A", as_index=False).size()
    assert_frames_equal(positional(got), positional(exp))
    assert_frames_equal(positional(got), oracle_groupby_frame(oracle, t, 0, [func_name], [1], batch_size=3))


def test_groupby_key_reorder(gpu_lib):
    # key is not the first column (bodo/tests/test_streaming/test_groupby.py:180-245)
    df = pd.DataFrame({"B": np.arange(800, dtype=np.int64) * 3, "A": [1, 2, 1, 1, 2, 0, 1, 2] * 100, "C": np.arange(800, dtype=np.float64)})
    t = Table.from_pandas(df)
    got = stream_groupby(t, (1,), ("sum", "mean"), (0, 1, 2), (0, 2), batch_size=7)
    exp = df.groupby("A", as_index=False).agg(B=("B", "sum"), C=("C", "mean"))
    assert_frames_equal(positional(got), positional(exp))


def test_quickstart_example(gpu_lib):
    # README / test_quickstart_docs.py:29-63 shape: 2000 rows % 30 groups, max
    df = pd.DataFrame({"A": np.arange(2000) % 30, "B": np.arange(2000)})
    got = stream_groupby(Table.from_pandas(df), (0,), ("max",), (0, 1), (1,), batch_size=512)
    assert_frames_equal(positional(got), positional(df.groupby("A", as_index=False).B.max()))


@pytest.mark.parametrize("dropna", [True, False])
def test_nullable_keys_and_values(gpu_lib, oracle, dropna):
    # test_series_groupby / test_dataframe_groupby fixtures (bodo/tests/test_df_lib/test_end_to_end.py:1606-1660)
    df = pd.DataFrame({
        "A": pd.array([1, 2, None, 2147483647, 1, None, 2, 1] * 40, dtype="Int64"),
        "B": pd.array([1.5, None, 3.0, 4.0, None, 6.0, 7.5, 8.0] * 40, dtype="Float64"),
        "C": pd.array([1, 2, 3, None, 5, 6, None, 8] * 40, dtype="Int32"),
    })
    t = Table.from_pandas(df)
    fn = ("sum", "mean", "count", "min", "max", "sum", "count", "min", "max", "size")
    offs = tuple(range(len(fn))) + (len(fn) - 1,)
    cols = (1, 1, 1, 1, 1, 2, 2, 2, 2)
    got = stream_groupby(t, (0,), fn, offs, cols, batch_size=64, dropna=dropna)
    exp = oracle_groupby_frame(oracle, t, 0, list(fn), list(cols) + [None], dropna=dropna, batch_size=64)
    assert_frames_equal(positional(got), exp)
    g = df.groupby("A", dropna=dropna)
    pexp = pd.DataFrame({"key": g.B.sum().index.to_numpy(dtype="float64", na_value=np.nan), "f0": g.B.sum().to_numpy(dtype="float64"),
                         "f1": g.B.mean().to_numpy(dtype="float64", na_value=np.nan), "f2": g.B.count().to_numpy()})
    pgot = positional(got)[["key", "f0", "f1", "f2"]]
    pgot["key"] = pgot["key"].to_numpy(dtype="float64", na_value=np.nan)
    assert_frames_equal(pgot, pexp)


def test_int64_sum_wraps_and_extreme_keys(gpu_lib, oracle):
    # int64 SUM accumulates in int64 with wraparound (casted_aggfunc, -fwrapv); INT64_MIN is the table's
    # free-slot marker, so it exercises the dedicated slot.
    keys = np.array([np.iinfo(np.int64).min, np.iinfo(np.int64).max, 0, -1, np.iinfo(np.int64).min, 0] * 50, dtype=np.int64)
    vals = np.array([2**62, 2**62, 2**62, -(2**62), 2**62, 2**62] * 50, dtype=np.int64)
    t = Table.from_pandas(pd.DataFrame({"k": keys, "v": vals}))
    got = stream_groupby(t, (0,), ("sum", "count"), (0, 1, 2), (1, 1), batch_size=100)
    assert_frames_equal(positional(got), oracle_groupby_frame(oracle, t, 0, ["sum", "count"], [1, 1], batch_size=100))


def test_empty_and_ragged_batches(gpu_lib):
    df = pd.DataFrame({"A": np.array([5, 5, 7], dtype=np.int64), "B": np.array([1.0, 2.0, 4.0])})
    t = Table.from_pandas(df)
    from bodo_b200.streaming.groupby import (delete_groupby_state, groupby_build_consume_batch,
                                             groupby_produce_output_batch, init_groupby_state)
    st = init_groupby_state(-1, (0,), ("sum",), (0, 1), (1,))
    groupby_build_consume_batch(st, t.slice(0, 0), False, True)   # empty batch first
    groupby_build_consume_batch(st, t.slice(0, 2), False, True)
    groupby_build_consume_batch(st, t.slice(2, 3), False, True)
    last, _ = groupby_build_consume_batch(st, t.slice(3, 3), True, True)  # empty last batch
    assert last
    out, out_last = groupby_produce_output_batch(st, True)
    assert out_last
    assert_frames_equal(positional(out.to_pandas()), positional(df.groupby("A", as_index=False).B.sum()))
    delete_groupby_state(st)
    # a state that never saw a row produces an empty table
    st = init_groupby_state(-1, (0,), ("sum",), (0, 1), (1,))
    groupby_build_consume_batch(st, t.slice(0, 0), True, True)
    out, out_last = groupby_produce_output_batch(st, True)
    assert out_last and out.n_rows == 0
    delete_groupby_state(st)


@pytest.mark.parametrize("n_groups", [1, 30, 5000, 300000])
def test_synthetic_vs_oracle_table_growth(gpu_lib, oracle, n_groups):
    # seeded synthetic rows (same generator as bench.py); small expected_groups forces fail-list replays
    # and table rebuilds (the reference's threshold-exceeded retry path, _groupby.cpp:3309-3341)
    n = 1_000_000
    k, v = oracle.synth_fill(0, n, n_groups, 7)
    t = Table.from_pandas(pd.DataFrame({"k": k, "v": v}))
    got = stream_groupby(t, (0,), ("sum", "count"), (0, 1, 2), (1, 1), batch_size=250_000, to_device=True, expected_groups=16,
                         output_batch_size=4096)
    exp = oracle_groupby_frame(oracle, t, 0, ["sum", "count"], [1, 1])
    assert len(got) == min(n_groups, len(np.unique(k)))
    assert_frames_equal(positional(got), exp)


def test_float_sum_mean_tolerance(gpu_lib, oracle):
    rng = np.random.default_rng(3)
    n = 400_000
    k = rng.integers(0, 1000, n).astype(np.int64)
    v = rng.random(n)
    v[rng.random(n) < 0.01] = np.nan
    df = pd.DataFrame({"k": k, "v": v})
    t = Table.from_pandas(df)
    got = stream_groupby(t, (0,), ("sum", "mean", "min", "max", "count"), (0, 1, 2, 3, 4, 5), (1, 1, 1, 1, 1), batch_size=100_000)
    exp = df.groupby("k", as_index=False).agg(f0=("v", "sum"), f1=("v", "mean"), f2=("v", "min"), f3=("v", "max"), f4=("v", "count"))
    # float SUM/MEAN: atomics reorder the additions -> tolerance rtol 1e-5 / atol 1e-8 (bodo/tests/utils.py:179-180)
    assert_frames_equal(positional(got), positional(exp), rtol=1e-5, atol=1e-8)


def test_unsupported_function_fails_loudly(gpu_lib):
    from bodo_b200 import B200Error
    from bodo_b200.streaming.groupby import init_groupby_state
    with pytest.raises(B200Error, match="unsupported aggregate function"):
        init_groupby_state(-1, (0,), ("median",), (0, 1), (1,))


@pytest.mark.timeout(300)
@pytest.mark.parametrize("n_groups,hint", [(1000, 0), (50_000, 50_000), (1_000_000, 1_000_000), (3_000_000, 16), (3_000_000, 3_000_000)])
@pytest.mark.parametrize("funcs", [("sum", "count"), ("count", "sum"), ("sum",), ("size",)])
def test_sm_partitioned_path_vs_oracle(gpu_lib, oracle, n_groups, hint, funcs):
    # >= 1 Mi-row device batches of the headline shape take the SM-partitioned kernel (when its estimate of the
    # cardinality fits shared memory); 3 M groups with a tiny hint overflows the shared tables and the global table,
    # exercising the in-kernel direct path and the retry list.  Result must be bit-exact either way.
    from bodo_b200.streaming.groupby import get_metric
    n = 2_600_001
    k, v = oracle.synth_fill(0, n, n_groups, 13)
    t = Table.from_pandas(pd.DataFrame({"k": k, "v": v}))
    nf = len(funcs)
    from bodo_b200.streaming.groupby import (delete_groupby_state, groupby_build_consume_batch,
                                             groupby_produce_output_batch, init_groupby_state)
    from tests.helpers import table_to_device
    st = init_groupby_state(-1, (0,), funcs, tuple(range(nf + 1)) if "size" not in funcs else (0, 0), (1,) * (0 if funcs == ("size",) else nf),
                            expected_groups=hint, output_batch_size=1 << 30)
    dt = table_to_device(t)
    groupby_build_consume_batch(st, dt, True, True)
    used = {m: get_metric(st, m) for m in (8, 10, 14, 15)}
    out, last = groupby_produce_output_batch(st, True)
    got = out.to_pandas()
    delete_groupby_state(st)
    exp = oracle_groupby_frame(oracle, t, 0, list(funcs), [None if f == "size" else 1 for f in funcs])
    assert_frames_equal(positional(got), exp)
    # synth_fill keys and values fit 32 bits: an estimate of at most 1024 groups (the 1000-group prefix, the hint 16) takes the
    # low-cardinality kernel (metric 10), any other the narrow-row pair (metric 14); the 16-byte pair (metric 15) never runs
    lowcard = (hint or n_groups) <= 1024
    assert used[10 if lowcard else 14] >= 1 and used[15] == 0, f"expected the {'low-cardinality' if lowcard else 'narrow-row'} kernels, metrics {used}"


@pytest.mark.timeout(300)
@pytest.mark.parametrize("n_groups", [1, 30, 700, 3000])
def test_low_cardinality_warp_aggregated_path_exact(gpu_lib, oracle, n_groups):
    # few hot keys -> the low-cardinality kernel (match_any + REDUX limb sums + leader upsert); extreme int64 values
    # exercise the 16-bit limb recombination and the carry into the high word: SUM must be exact mod 2^64
    from bodo_b200.streaming.groupby import (delete_groupby_state, get_metric, groupby_build_consume_batch,
                                             groupby_produce_output_batch, init_groupby_state)
    from tests.helpers import table_to_device
    rng = np.random.default_rng(n_groups)
    n = 1_300_003
    k = rng.integers(0, n_groups, n).astype(np.int64) * 7919 - 5
    v = rng.integers(-(2**62), 2**62, n).astype(np.int64)
    v[::3] = rng.integers(-500, 500, len(v[::3]))
    t = Table.from_pandas(pd.DataFrame({"k": k, "v": v}))
    st = init_groupby_state(-1, (0,), ("sum", "count"), (0, 1, 2), (1, 1), expected_groups=n_groups, output_batch_size=1 << 30)
    groupby_build_consume_batch(st, table_to_device(t), True, True)
    lc = get_metric(st, 10)
    out, last = groupby_produce_output_batch(st, True)
    got = out.to_pandas()
    delete_groupby_state(st)
    assert_frames_equal(positional(got), oracle_groupby_frame(oracle, t, 0, ["sum", "count"], [1, 1]))
    if n_groups <= 1024:
        assert lc >= 1, "the low-cardinality kernel was expected to run"


@pytest.mark.timeout(300)
def test_sm_partitioned_path_skewed_keys(gpu_lib, oracle):
    # Zipf-like keys: a few owners receive far more rows than their bucket holds, so K1 sends the excess through the
    # direct global path; hot keys hammer single shared-memory slots in K2.  Result must still be bit-exact.
    from bodo_b200.streaming.groupby import (delete_groupby_state, get_metric, groupby_build_consume_batch,
                                             groupby_produce_output_batch, init_groupby_state)
    from tests.helpers import table_to_device
    rng = np.random.default_rng(99)
    n = 3_000_000
    k = np.minimum(rng.zipf(1.2, n), 200_000).astype(np.int64) * 31 + 7
    v = rng.integers(-(2**40), 2**40, n).astype(np.int64)
    t = Table.from_pandas(pd.DataFrame({"k": k, "v": v}))
    st = init_groupby_state(-1, (0,), ("sum", "count"), (0, 1, 2), (1, 1), expected_groups=100_000, output_batch_size=1 << 30)
    groupby_build_consume_batch(st, table_to_device(t), True, True)
    assert get_metric(st, 8) >= 1
    out, last = groupby_produce_output_batch(st, True)
    got = out.to_pandas()
    delete_groupby_state(st)
    assert_frames_equal(positional(got), oracle_groupby_frame(oracle, t, 0, ["sum", "count"], [1, 1]))


@pytest.mark.timeout(300)
@pytest.mark.parametrize("fnames", [("sum",), ("count",), ("size", "sum")])
def test_sm_partitioned_heavy_hitters(gpu_lib, oracle, fnames):
    # heavy hitters are aggregated inside K1 (per-CTA shared accumulators) from a table sampled at the first launch.
    # Two batches: the second one brings a hot key the sample has never seen (it must simply take the ordinary route),
    # a hot key whose values cancel to zero (the group has to exist when only SUM is asked for) and values with
    # non-zero high words (carry path of the 32-bit limb accumulators).
    from bodo_b200.streaming.groupby import (delete_groupby_state, get_metric, groupby_build_consume_batch,
                                             groupby_produce_output_batch, init_groupby_state)
    from tests.helpers import table_to_device
    rng = np.random.default_rng(5)
    n = 2_500_000
    def batch(hot, seed):
        r = np.random.default_rng(seed)
        k = r.integers(0, 150_000, n).astype(np.int64) * 13 - 77
        u = r.random(n)
        k[u < 0.30] = hot[0]
        k[(u >= 0.30) & (u < 0.45)] = hot[1]
        k[(u >= 0.45) & (u < 0.47)] = hot[2]
        v = r.integers(-(2**40), 2**40, n).astype(np.int64)
        v[k == hot[1]] = 0                       # sums to zero
        v[k == hot[0]] = 2**62                   # wraps: 30 % of 2.5 M rows x 2^62
        return pd.DataFrame({"k": k, "v": v})
    d1, d2 = batch((123456789, -5, 42), 1), batch((987654321, -5, 123456789), 2)
    offs, cols = [0], []
    for f in fnames:
        if f != "size":
            cols.append(1)
        offs.append(len(cols))
    st = init_groupby_state(-1, (0,), fnames, tuple(offs), tuple(cols), expected_groups=200_000, output_batch_size=1 << 30)
    groupby_build_consume_batch(st, table_to_device(Table.from_pandas(d1)), False, True)
    groupby_build_consume_batch(st, table_to_device(Table.from_pandas(d2)), True, True)
    assert get_metric(st, 8) >= 2
    out, last = groupby_produce_output_batch(st, True)
    got = out.to_pandas()
    delete_groupby_state(st)
    both = Table.from_pandas(pd.concat([d1, d2], ignore_index=True))
    assert_frames_equal(positional(got), oracle_groupby_frame(oracle, both, 0, list(fnames), [1 if f != "size" else None for f in fnames]))


def test_groupby_drop_duplicates_reference_fixture(gpu_lib):
    # test_groupby_drop_duplicates (bodo/tests/test_streaming/test_groupby.py:111-177): two key columns, zero functions
    df = pd.DataFrame({"A": [1, 1, 2, 4, 4, 2], "B": [1, 1, 3, 6, 6, 3]})
    got = stream_groupby(Table.from_pandas(df), (0, 1), (), (0,), (), batch_size=3)
    exp = df.drop_duplicates().reset_index(drop=True)
    assert list(got.columns) == ["A", "B"]
    g = got.sort_values(["A", "B"]).reset_index(drop=True)
    np.testing.assert_array_equal(g.to_numpy(), exp.sort_values(["A", "B"]).to_numpy())


@pytest.mark.parametrize("dropna", [True, False])
def test_multi_key_groupby_vs_pandas(gpu_lib, dropna):
    rng = np.random.default_rng(17)
    n = 200_000
    df = pd.DataFrame({
        "k1": pd.array(rng.integers(0, 300, n), dtype="Int64"),
        "v": rng.integers(-1000, 1000, n).astype(np.int64),
        "k2": rng.integers(-5, 5, n).astype(np.int32),
        "k3": pd.array(rng.integers(0, 3, n), dtype="Int32"),
        "f": rng.random(n),
    })
    df.loc[rng.random(n) < 0.02, "k1"] = pd.NA
    df.loc[rng.random(n) < 0.02, "k3"] = pd.NA
    t = Table.from_pandas(df)
    # keys = (k1, k2, k3) at logical columns (0, 2, 3); tiny expected_groups forces table rebuilds of the multi-key table
    got = stream_groupby(t, (0, 2, 3), ("sum", "count", "mean", "max", "size"), (0, 1, 2, 3, 4, 4), (1, 1, 4, 4), batch_size=37_000,
                         dropna=dropna, expected_groups=8, output_batch_size=4096)
    exp = df.groupby(["k1", "k2", "k3"], dropna=dropna, as_index=False).agg(f0=("v", "sum"), f1=("v", "count"), f2=("f", "mean"), f3=("f", "max"),
                                                                          f4=("v", "size"))
    assert len(got) == len(exp)
    got.columns = list(exp.columns)
    def canon(d):
        d = d.copy()
        for c in d.columns:
            d[c] = d[c].to_numpy(dtype="float64", na_value=np.nan)
        return d.sort_values(list(d.columns[:3]), na_position="last").reset_index(drop=True)
    g, e = canon(got), canon(exp)
    for c in ("k1", "k2", "k3", "f0", "f1", "f4"):
        np.testing.assert_array_equal(g[c].to_numpy(), e[c].to_numpy(), err_msg=c)
    for c in ("f2", "f3"):
        np.testing.assert_allclose(g[c].to_numpy(), e[c].to_numpy(), rtol=1e-5, atol=1e-8, err_msg=c)


def test_float32_sum_mean_stated_tolerance(gpu_lib, oracle):
    """float32 SUM: the reference accumulates in float32 (aggfunc<float, sum>, bodo/libs/groupby/_groupby_agg_funcs.h:159-173,
    in batch / combine order); the device accumulates every group in float64 (atomics reorder additions, so a float32
    accumulator would not be reproducible anyway) and narrows once at eval.  The two differ by float32 rounding of the
    running sum: |device - reference| <= n_g * 2^-24 * sum|v| per group — the bound asserted here, with the oracle
    (float32 accumulation in the reference's order) as the reference value.  Against the exact (float64) sum the device
    result is within ONE float32 rounding, i.e. it is the more accurate of the two."""
    rng = np.random.default_rng(17)
    n, ng = 200_000, 97
    k = rng.integers(0, ng, n).astype(np.int64)
    v = (rng.random(n) * 100.0 - 20.0).astype(np.float32)
    df = pd.DataFrame({"k": k, "v": v})
    t = Table.from_pandas(df)
    got = positional(stream_groupby(t, (0,), ("sum", "mean", "count"), (0, 1, 2, 3), (1, 1, 1), batch_size=4096, to_device=True))
    got = got.sort_values("key").reset_index(drop=True)
    assert got["f0"].dtype == np.float32  # SUM(float32) stays float32 (get_groupby_output_dtype, _groupby_common.cpp:567-619)
    exp = oracle_groupby_frame(oracle, t, 0, ["sum", "mean", "count"], [1, 1, 1], batch_size=4096).sort_values("key").reset_index(drop=True)
    g64 = df.assign(v=df.v.astype(np.float64)).groupby("k").v
    exact, cnt, abs_sum = g64.sum().to_numpy(), g64.count().to_numpy(), g64.apply(lambda s: s.abs().sum()).to_numpy()
    np.testing.assert_array_equal(got["f2"].to_numpy(), cnt)
    bound_ref = cnt * 2.0 ** -24 * abs_sum
    assert (np.abs(got["f0"].to_numpy().astype(np.float64) - exp["f0"].to_numpy().astype(np.float64)) <= bound_ref).all()
    # one float32 rounding of the exact sum
    assert (np.abs(got["f0"].to_numpy().astype(np.float64) - exact) <= 2.0 ** -24 * np.abs(exact) * 1.0000001).all()
    np.testing.assert_allclose(got["f1"].to_numpy(), exact / cnt, rtol=1e-12)  # MEAN is float64 throughout (mean_agg :673-689)


@pytest.mark.parametrize("nullable", [False, True])
def test_var_std_skew_against_pandas_and_reference_formulas(gpu_lib, nullable):
    """var / std / var_pop / std_pop / skew (Bodo_FTypes 24 / 25 / 22 / 23 / 27; the reference's GPU test matrix,
    bodo/tests/test_df_lib/test_gpu/test_gpu_end_to_end.py:68-110).  Reference: Welford (count, mean, M2) for var / std
    (groupby/_groupby_agg_funcs.h:694-719), power sums for skew (:723-745), eval in _groupby_eval.h:71-137.  The device carries
    power sums about a per-group shift for all of them; tolerance = the reference's test tolerance (rtol 1e-5).  The shift keeps
    the error independent of |mean| / std (tests/test_gpu_groupby_float_values.py states the bound and checks it up to offsets
    of 1e12)."""
    rng = np.random.default_rng(23)
    n, ng = 60_000, 211
    k = rng.integers(0, ng, n).astype(np.int64)
    k[:3] = [ng, ng + 1, ng + 1]  # groups with one / two rows: var NaN for n < 2, skew NaN for n < 3
    x = rng.standard_normal(n) * 3.0 + 10.0
    i = rng.integers(-1000, 1000, n).astype(np.int64)
    df = pd.DataFrame({"k": k, "x": x, "i": i})
    if nullable:
        df["x"] = pd.array(x, dtype="Float64")
        df["i"] = pd.array(i, dtype="Int64")
        df.loc[rng.random(n) < 0.07, "x"] = pd.NA
        df.loc[rng.random(n) < 0.07, "i"] = pd.NA
    t = Table.from_pandas(df)
    fn = ("var", "std", "skew", "var_pop", "std_pop", "var", "skew", "mean")
    cols = (1, 1, 1, 1, 1, 2, 2, 1)
    got = positional(stream_groupby(t, (0,), fn, tuple(range(len(fn) + 1)), cols, batch_size=7000, to_device=True)).sort_values("key").reset_index(drop=True)
    g = df.astype({"x": "float64", "i": "float64"}).groupby("k")
    exp = pd.DataFrame({"key": sorted(df.k.unique()), "f0": g.x.var().to_numpy(), "f1": g.x.std().to_numpy(), "f2": g.x.skew().to_numpy(),
                        "f3": g.x.var(ddof=0).to_numpy(), "f4": g.x.std(ddof=0).to_numpy(), "f5": g.i.var().to_numpy(),
                        "f6": g.i.skew().to_numpy(), "f7": g.x.mean().to_numpy()})
    assert len(got) == len(exp)
    for c in exp.columns[1:]:
        np.testing.assert_allclose(got[c].to_numpy(dtype="float64", na_value=np.nan), exp[c].to_numpy(dtype="float64"), rtol=1e-5, atol=1e-8,
                                   equal_nan=True, err_msg=c)


@pytest.mark.parametrize("to_device", [False, True])
def test_streaming_batches_are_coalesced_into_fast_path_launches(gpu_lib, oracle, to_device):
    """The reference's streaming batch size is 32 768 rows (bodo/libs/streaming/_shuffle.h:27-31): such batches are buffered on the
    device and reach the SM-partitioned / low-cardinality kernels in >= 2^20-row launches (metric 8 / 10 > 0, metric 11 counts the
    coalesced batches); result bit-exact against the oracle."""
    from bodo_b200.streaming.groupby import (delete_groupby_state, get_metric, groupby_build_consume_batch, groupby_produce_output_batch,
                                             init_groupby_state)
    from tests.helpers import table_to_device
    n, ng, bs = 3_000_000 + 12_345, 40_000, 32_768
    k, v = oracle.synth_fill(0, n, ng, 31)
    t = Table.from_pandas(pd.DataFrame({"k": k, "v": v}))
    st = init_groupby_state(-1, (0,), ("sum", "count"), (0, 1, 2), (1, 1), output_batch_size=1 << 30)
    for r0 in range(0, n, bs):
        b = t.slice(r0, r0 + bs)
        groupby_build_consume_batch(st, table_to_device(b) if to_device else b, r0 + bs >= n, True)
    out, last = groupby_produce_output_batch(st, True)
    got = out.to_pandas()
    fast_launches, coalesced = get_metric(st, 8) + get_metric(st, 10), get_metric(st, 11)
    delete_groupby_state(st)
    assert coalesced >= 90 and fast_launches >= 1, (coalesced, fast_launches)
    assert_frames_equal(positional(got), oracle_groupby_frame(oracle, t, 0, ["sum", "count"], [1, 1]))


@pytest.mark.timeout(600)
@pytest.mark.parametrize("key_dtype,val_dtype", [("Int64", "Int64"), ("Int32", "Int32"), ("int32", "int64"), ("int64", "Int32")])
@pytest.mark.parametrize("funcs", [("mean", "min", "max"), ("sum", "count", "size"), ("min",), ("size", "mean", "sum", "count", "max")])
@pytest.mark.parametrize("dropna", [True, False])
def test_generic_sm_partitioned_path_nullable_int32_mean_min_max(gpu_lib, oracle, key_dtype, val_dtype, funcs, dropna):
    """SPG-G (spgg.cuh): >= 2^20-row device batches with nullable / 4-byte keys and values and mean / min / max take the
    SM-partitioned kernels too (metric 12).  Integer results bit-exact against pandas, mean within rtol 1e-5
    (bodo/tests/utils.py:179-180).  Covers NA keys (dropped or grouped), NA values (the group must still exist, count for
    size only), values whose sum needs the high word, and a hint-less state that overflows the global table (retry list)."""
    from bodo_b200.streaming.groupby import (delete_groupby_state, get_metric, groupby_build_consume_batch,
                                             groupby_produce_output_batch, init_groupby_state)
    from tests.helpers import table_to_device
    rng = np.random.default_rng(7)
    n, n_groups = 2_400_003, 60_000
    k = rng.integers(-n_groups // 2, n_groups // 2, n)
    big = val_dtype.lower() == "int64"
    v = rng.integers(-(1 << 40) if big else -(1 << 31), (1 << 40) if big else (1 << 31) - 1, n)
    ks = pd.Series(k).astype(key_dtype.lower())
    vs = pd.Series(v).astype(val_dtype.lower())
    if key_dtype[0] == "I":
        ks = ks.astype(key_dtype).mask(rng.random(n) < 0.03)
    if val_dtype[0] == "I":
        vs = vs.astype(val_dtype).mask(rng.random(n) < 0.10)
        # one group whose values are all NA: must exist, with NA aggregates and size > 0
        vs = vs.mask(ks == 17)
    df = pd.DataFrame({"k": ks, "v": vs})
    t = Table.from_pandas(df)
    nf = len(funcs)
    offs, cols, c = [0], [], 0
    for f in funcs:
        if f != "size":
            cols.append(1); c += 1
        offs.append(c)
    st = init_groupby_state(-1, (0,), funcs, tuple(offs), tuple(cols), expected_groups=0, output_batch_size=1 << 30, dropna=dropna)
    groupby_build_consume_batch(st, table_to_device(t), True, True)
    used = get_metric(st, 12)
    out, _ = groupby_produce_output_batch(st, True)
    got = out.to_pandas()
    delete_groupby_state(st)
    g = df.groupby("k", as_index=False, dropna=dropna)
    exp = g.size()[["k"]]
    for j, f in enumerate(funcs):
        col = g.size()["size"] if f == "size" else g.agg(x=("v", f))["x"]
        exp[f"o{j}"] = col.values
    assert used >= 1, "the generic SM-partitioned kernels were expected to run for this shape"
    assert_frames_equal(positional(got), positional(exp))


@pytest.mark.timeout(600)
@pytest.mark.parametrize("n_groups,nullable", [(1_200_000, False), (1_200_000, True), (2_400_000, True)])
def test_generic_sm_partitioned_path_multi_pass(gpu_lib, n_groups, nullable):
    """More groups than the owners' shared tables hold at once (min / max slots are 32 B): K2g runs several passes.  With
    2 passes K1g partitions into owners x passes buckets (each row read once); with more, every pass scans the owner's
    bucket and tests the rows' pass (the class table of K1g has no room for owners x passes + owners buckets)."""
    from bodo_b200.streaming.groupby import (delete_groupby_state, get_metric, groupby_build_consume_batch,
                                             groupby_produce_output_batch, init_groupby_state)
    from tests.helpers import table_to_device
    rng = np.random.default_rng(11)
    n = 4_200_001
    k = rng.integers(0, n_groups, n)
    v = rng.integers(-(1 << 45), 1 << 45, n)
    ks, vs = pd.Series(k), pd.Series(v)
    if nullable:
        ks = ks.astype("Int64").mask(rng.random(n) < 0.02)
        vs = vs.astype("Int64").mask(rng.random(n) < 0.15)
    df = pd.DataFrame({"k": ks, "v": vs})
    funcs = ("size", "sum", "min", "max", "mean", "count")
    st = init_groupby_state(-1, (0,), funcs, (0, 0, 1, 2, 3, 4, 5), (1, 1, 1, 1, 1), expected_groups=n_groups, output_batch_size=1 << 30)
    groupby_build_consume_batch(st, table_to_device(Table.from_pandas(df)), True, True)
    used = get_metric(st, 12)
    out, _ = groupby_produce_output_batch(st, True)
    got = out.to_pandas()
    delete_groupby_state(st)
    g = df.groupby("k", as_index=False)
    exp = g.size()[["k"]]
    for j, f in enumerate(funcs):
        exp[f"o{j}"] = (g.size()["size"] if f == "size" else g.agg(x=("v", f))["x"]).values
    assert used >= 1
    assert_frames_equal(positional(got), positional(exp))


@pytest.mark.parametrize("to_device", [False, True])
@pytest.mark.parametrize("dropna", [True, False])
def test_first_last_in_row_order_vs_pandas(gpu_lib, to_device, dropna):
    """first / last = the first / last non-NA value of the group in ROW order (aggfunc<first / last>,
    bodo/libs/groupby/_groupby_agg_funcs.h:594-611), across batch boundaries and table growth; a group without a non-NA value
    gives NA; float NaN counts as NA."""
    rng = np.random.default_rng(3)
    n, ng = 300_007, 40_000
    df = pd.DataFrame({
        "k": pd.array(rng.integers(0, ng, n), dtype="Int64").copy(),
        "i": pd.array(rng.integers(-(1 << 50), 1 << 50, n), dtype="Int64"),
        "f": rng.random(n),
        "s": rng.integers(-1000, 1000, n).astype(np.int32),
    })
    df.loc[rng.random(n) < 0.02, "k"] = pd.NA
    df.loc[rng.random(n) < 0.3, "i"] = pd.NA
    df.loc[rng.random(n) < 0.3, "f"] = np.nan
    df.loc[df.k == 5, "i"] = pd.NA   # a group whose values are all NA
    t = Table.from_pandas(df)
    fn = ("first", "last", "first", "last", "first", "last", "size")
    got = stream_groupby(t, (0,), fn, (0, 1, 2, 3, 4, 5, 6, 6), (1, 1, 2, 2, 3, 3), batch_size=70_001, to_device=to_device, dropna=dropna)
    g = df.groupby("k", as_index=False, dropna=dropna)
    exp = g.size()[["k"]]
    for j, (c, f) in enumerate(zip(("i", "i", "f", "f", "s", "s"), fn)):
        exp[f"o{j}"] = g.agg(x=(c, f))["x"].values
    exp["o6"] = g.size()["size"].values
    assert_frames_equal(positional(got), positional(exp))


@pytest.mark.parametrize("to_device", [False, True])
@pytest.mark.parametrize("dropna", [True, False])
def test_nunique_vs_pandas(gpu_lib, to_device, dropna):
    """nunique = distinct non-NA values per group (nunique_computation, bodo/libs/groupby/_groupby_col_set.cpp:1771-1810), mixed
    with other aggregates, over nullable and plain columns, across batches; the reference's GPU matrix lists it
    (bodo/tests/test_df_lib/test_gpu/test_gpu_end_to_end.py:68-110)."""
    rng = np.random.default_rng(12)
    n, ng = 250_003, 9_000
    df = pd.DataFrame({
        "k": pd.array(rng.integers(0, ng, n), dtype="Int64"),
        "a": pd.array(rng.integers(0, 40, n), dtype="Int64"),
        "b": rng.integers(-5, 5, n).astype(np.int32),
    })
    df.loc[rng.random(n) < 0.02, "k"] = pd.NA
    df.loc[rng.random(n) < 0.2, "a"] = pd.NA
    df.loc[df.k == 7, "a"] = pd.NA  # a group without a non-NA value: nunique 0
    t = Table.from_pandas(df)
    fn = ("nunique", "sum", "nunique", "size", "nunique")
    got = stream_groupby(t, (0,), fn, (0, 1, 2, 3, 3, 4), (1, 1, 2, 1), batch_size=60_001, to_device=to_device, dropna=dropna)
    g = df.groupby("k", as_index=False, dropna=dropna)
    exp = g.size()[["k"]]
    exp["o0"] = g.agg(x=("a", "nunique"))["x"].values
    exp["o1"] = g.agg(x=("a", "sum"))["x"].values
    exp["o2"] = g.agg(x=("b", "nunique"))["x"].values
    exp["o3"] = g.size()["size"].values
    exp["o4"] = exp["o0"]
    assert_frames_equal(positional(got), positional(exp))


@pytest.mark.timeout(300)
@pytest.mark.parametrize("funcs", [("sum", "count"), ("sum",), ("size",)])
def test_narrow_row_sm_partitioned_path_exact_with_wide_stragglers(gpu_lib, oracle, funcs):
    """SPG-N (spgn.cuh): when the sampled rows all fit (int32 key, int32 value) the owner buckets carry 8-byte rows (metric 14).
    Rows that do not fit — here a few thousand the sample cannot see: keys beyond 2^40, the key INT32_MIN, values beyond 2^35,
    negative everything — take the direct path inside K1n; the result is bit-exact either way (int64 sums wrap mod 2^64)."""
    from bodo_b200.streaming.groupby import (delete_groupby_state, get_metric, groupby_build_consume_batch,
                                             groupby_produce_output_batch, init_groupby_state)
    from tests.helpers import table_to_device
    rng = np.random.default_rng(8)
    n, ng = 32768 * 80, 200_000   # the sampler looks at 32 blocks of 1024 rows: [b * n / 32, b * n / 32 + 1024)
    k = rng.integers(-ng // 2, ng // 2, n).astype(np.int64)
    v = rng.integers(-(1 << 31), (1 << 31) - 1, n).astype(np.int64)
    idx = np.arange(n)
    w = (idx % 80 == 3) & (idx < 400_000) & (idx % (n // 32) >= 1024)  # ~5000 rows outside the narrow format, none of them sampled
    k[w & (idx % 3 == 0)] += 1 << 41
    k[w & (idx % 3 == 1)] = np.iinfo(np.int32).min
    v[w & (idx % 3 == 2)] = (1 << 36) + idx[w & (idx % 3 == 2)]
    v[w & (idx % 7 == 0)] = -(1 << 62)             # sums wrap
    t = Table.from_pandas(pd.DataFrame({"k": k, "v": v}))
    nf = len(funcs)
    st = init_groupby_state(-1, (0,), funcs, tuple(range(nf + 1)) if "size" not in funcs else (0, 0), (1,) * (0 if funcs == ("size",) else nf),
                            expected_groups=ng, output_batch_size=1 << 30)
    groupby_build_consume_batch(st, table_to_device(t), True, True)
    used, wide = get_metric(st, 14), get_metric(st, 15)
    out, _ = groupby_produce_output_batch(st, True)
    got = out.to_pandas()
    delete_groupby_state(st)
    assert used >= 1 and wide == 0, "the narrow-row kernels (and not the 16-byte ones) were expected to run for this shape"
    assert_frames_equal(positional(got), oracle_groupby_frame(oracle, t, 0, list(funcs), [None if f == "size" else 1 for f in funcs]))
