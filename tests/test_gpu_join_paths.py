"""Which probe path a join state takes, and the array type and bitmap of every output column on each path: the inline-payload
kernel (Slot32 table), the two-sector fast kernel on Slot16 tables (built from the key table, or derived from Slot32 when a
batch does not qualify for the inline kernel) and the general count / scan / gather path with its build-outer tail.  Row sets
are compared with the CPU oracle; metrics 5 / 6 / 7 (fast probes, inline probes, inline builds) name the path."""

import numpy as np
import pandas as pd
import pytest

from bodo_b200.streaming.join import (delete_join_state, get_metric, init_join_state, join_build_consume_batch,
                                      join_probe_consume_batch)
from bodo_b200.table import ArrTypes, Table
from tests.helpers import table_to_device
from tests.test_gpu_join import assert_rowset_equal, oracle_join_frame

pytestmark = pytest.mark.gpu

PLAIN, NULLABLE = (ArrTypes.NUMPY, False), (ArrTypes.NULLABLE_INT_BOOL, True)  # (arr_type, has a bitmap)


def run_join(build_batches, probe_batches, build_outer=False):
    """One join state fed the device-resident build batches, then the probe batches.  Per probe batch: the output frame, the
    (arr_type, has a bitmap) of every output column, and metrics 0..7 after the batch."""
    st = init_join_state(-1, (0,), (0,), tuple(build_batches[0].columns), tuple(probe_batches[0].columns), build_outer, False)
    for i, b in enumerate(build_batches):
        join_build_consume_batch(st, table_to_device(Table.from_pandas(b)), i == len(build_batches) - 1)
    res = []
    for i, p in enumerate(probe_batches):
        out, _, _ = join_probe_consume_batch(st, table_to_device(Table.from_pandas(p)), i == len(probe_batches) - 1)
        kinds = [(c.arr_type, c.validity is not None) for c in out.columns]
        res.append((out.to_pandas(), kinds, [get_metric(st, m) for m in range(8)]))
    delete_join_state(st)
    return res


def unique_build(rng, nb):
    return pd.DataFrame({"k": rng.permutation(nb).astype(np.int64), "b1": rng.integers(-(1 << 40), 1 << 40, nb)})


def test_inline_build_with_a_bitmap_batch_between_inline_batches(gpu_lib, oracle):
    # a probe column with a bitmap does not qualify for the inline kernel: that batch takes the fast kernel on Slot16 tables
    # derived from the Slot32 table, and the next bitmap-free batch is inline again
    rng = np.random.default_rng(31)
    nb = 20_000
    build = unique_build(rng, nb)

    def probe(n, with_bitmap):
        df = pd.DataFrame({"k": rng.integers(0, 2 * nb, n).astype(np.int64), "p1": rng.integers(0, 1 << 40, n)})
        if with_bitmap:
            df["p1"] = df["p1"].astype("Int64").mask(rng.random(n) < 0.2)
        return df

    probes = [probe(30_000, False), probe(30_000, True), probe(30_000, False)]
    res = run_join([build], probes)
    for (got, _, _), p in zip(res, probes):
        assert_rowset_equal(got, oracle_join_frame(oracle, build, p))
    assert [kinds for _, kinds, _ in res] == [[PLAIN] * 4, [PLAIN] * 3 + [NULLABLE], [PLAIN] * 4]
    assert [m[5:] for _, _, m in res] == [[1, 1, 1], [2, 1, 1], [3, 2, 1]]


def test_inline_build_probed_with_an_int32_column(gpu_lib, oracle):
    rng = np.random.default_rng(32)
    nb = 20_000
    build = unique_build(rng, nb)
    probe = pd.DataFrame({"k": rng.integers(0, 2 * nb, 30_000).astype(np.int64), "p1": rng.integers(-1000, 1000, 30_000).astype(np.int32)})
    [(got, kinds, m)] = run_join([build], [probe])
    assert_rowset_equal(got, oracle_join_frame(oracle, build, probe))
    assert kinds == [PLAIN] * 4
    assert m[5:] == [1, 0, 1]


def test_unique_keys_with_nullable_and_int32_payload(gpu_lib, oracle):
    # not an inline schema: Slot16 tables built from the key table, fast kernel
    rng = np.random.default_rng(33)
    nb = 20_000
    build = unique_build(rng, nb)
    build["b1"] = build["b1"].astype("Int64").mask(rng.random(nb) < 0.1)
    build["b2"] = rng.integers(-1000, 1000, nb).astype(np.int32)
    probe = pd.DataFrame({"k": rng.integers(0, 2 * nb, 30_000).astype(np.int64), "p1": rng.random(30_000)})
    [(got, kinds, m)] = run_join([build], [probe])
    assert_rowset_equal(got, oracle_join_frame(oracle, build, probe))
    assert kinds == [PLAIN, NULLABLE, PLAIN, PLAIN, PLAIN]
    assert m[5:] == [1, 0, 0]


@pytest.mark.parametrize("duplicate_key", [False, True])
def test_build_key_validity_on_the_unique_and_general_paths(gpu_lib, oracle, duplicate_key):
    # The build key column: a first batch without a bitmap (so its array type stays NUMPY), then one with a bitmap and an NA.
    # The probe key: a bitmap (and NAs) in the first batch, none in the second.  On the unique-key path the build key output
    # column carries the probe key's bitmap; on the general path (one duplicated key) it carries the build key's.
    rng = np.random.default_rng(34)
    nb = 4_000
    keys = rng.permutation(nb).astype(np.int64)
    if duplicate_key:
        keys[-1] = keys[0]
    b1 = pd.DataFrame({"k": keys[: nb // 2], "b1": rng.integers(0, 1000, nb // 2)})
    b2 = pd.DataFrame({"k": pd.array(keys[nb // 2:], dtype="Int64"), "b1": rng.integers(0, 1000, nb - nb // 2)})
    b2.loc[5, "k"] = pd.NA
    p1 = pd.DataFrame({"k": pd.array(rng.integers(0, nb, 3_000), dtype="Int64"), "p1": rng.integers(0, 1000, 3_000)})
    p1.loc[::100, "k"] = pd.NA
    p2 = pd.DataFrame({"k": rng.integers(0, nb, 3_000).astype(np.int64), "p1": rng.integers(0, 1000, 3_000)})
    res = run_join([b1, b2], [p1, p2])
    build = pd.concat([b1, b2], ignore_index=True)
    for (got, _, _), p in zip(res, [p1, p2]):
        assert_rowset_equal(got, oracle_join_frame(oracle, build, p, is_na_equal=False))
    second_build_key = NULLABLE if duplicate_key else PLAIN
    assert [kinds for _, kinds, _ in res] == [[NULLABLE, PLAIN, NULLABLE, PLAIN], [second_build_key, PLAIN, NULLABLE, PLAIN]]
    assert [m[5:] for _, _, m in res] == ([[0, 0, 0], [0, 0, 0]] if duplicate_key else [[1, 0, 0], [2, 0, 0]])


def test_build_outer_tail_regrows_the_outputs_of_a_small_last_batch(gpu_lib, oracle):
    # the last probe batch gathers 5 rows, then ~1.5 M unmatched build rows follow: the output columns (data and validity
    # bytes) are regrown past any pooled block's slack and must keep the 5 gathered rows
    rng = np.random.default_rng(35)
    nb = 1_500_000
    build = pd.DataFrame({"k": np.arange(nb, dtype=np.int64), "b1": pd.array(rng.integers(0, 1000, nb), dtype="Int64")})
    build.loc[::7, "b1"] = pd.NA
    p1 = pd.DataFrame({"k": np.arange(1_000, dtype=np.int64), "p1": rng.integers(0, 1000, 1_000)})
    p2 = pd.DataFrame({"k": np.arange(1_000, 1_005, dtype=np.int64), "p1": rng.integers(0, 1000, 5)})
    res = run_join([build], [p1, p2], build_outer=True)
    assert [len(got) for got, _, _ in res] == [1_000, 5 + nb - 1_005]
    got = pd.concat([got for got, _, _ in res], ignore_index=True)
    assert_rowset_equal(got, oracle_join_frame(oracle, build, pd.concat([p1, p2], ignore_index=True), build_outer=True))
    assert [kinds for _, kinds, _ in res] == [[PLAIN, NULLABLE, NULLABLE, NULLABLE]] * 2
    assert [m[5:] for _, _, m in res] == [[0, 0, 0], [0, 0, 0]]
