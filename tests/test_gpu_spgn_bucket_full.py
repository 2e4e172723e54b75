"""SPG-N (spgn.cuh) when an owner's bucket overflows: K1n's bucket-full branch sends the rows past the end of a bucket through the
direct path.  Uniform keys never get there, and skewed keys with heavy hitters run the 16-byte HOT kernel instead, so this input
puts half the rows on owner 0 through ~10^5 distinct keys, none of which crosses the heavy-hitter share (1/1024 of the rows)."""

import numpy as np
import pandas as pd
import pytest

from bodo_b200.table import Table
from tests.helpers import assert_frames_equal, oracle_groupby_frame, positional

pytestmark = pytest.mark.gpu


def _owner(keys, n_owners):
    """spg_owner(spg_hash(key), n_owners) of groupby.cu: (x ^ (x >> 29)) * 0x9E3779B97F4A7C15, owner = umulhi(high word, owners)."""
    x = keys.astype(np.int64).view(np.uint64)
    with np.errstate(over="ignore"):
        h = (x ^ (x >> np.uint64(29))) * np.uint64(0x9E3779B97F4A7C15)
    return ((h >> np.uint64(32)) * np.uint64(n_owners)) >> np.uint64(32)


@pytest.mark.timeout(300)
def test_narrow_rows_overflowing_one_owner_bucket_are_exact(gpu_lib, oracle):
    import torch

    from bodo_b200.streaming.groupby import (delete_groupby_state, get_metric, groupby_build_consume_batch,
                                             groupby_produce_output_batch, init_groupby_state)
    from tests.helpers import table_to_device

    sms = torch.cuda.get_device_properties(0).multi_processor_count
    rng = np.random.default_rng(21)
    cand = np.arange(1, 20_000_000, dtype=np.int64)
    owner0 = cand[_owner(cand, sms) == 0][:100_000]
    assert len(owner0) == 100_000
    n, ng = 1 << 22, 300_000
    k = rng.integers(-ng, ng, n).astype(np.int64)
    skew = rng.random(n) < 0.5
    k[skew] = owner0[rng.integers(0, len(owner0), int(skew.sum()))]
    v = rng.integers(-(1 << 31), (1 << 31) - 1, n).astype(np.int64)
    t = Table.from_pandas(pd.DataFrame({"k": k, "v": v}))
    st = init_groupby_state(-1, (0,), ("sum", "count"), (0, 1, 2), (1, 1), expected_groups=len(np.unique(k)), output_batch_size=1 << 30)
    groupby_build_consume_batch(st, table_to_device(t), True, True)
    used = get_metric(st, 14)
    out, _ = groupby_produce_output_batch(st, True)
    got = out.to_pandas()
    delete_groupby_state(st)
    assert used >= 1, "the narrow-row kernels were expected to run for this shape"
    assert_frames_equal(positional(got), oracle_groupby_frame(oracle, t, 0, ["sum", "count"], [1, 1]))
