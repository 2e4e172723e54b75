"""Full-size parity checks (BASELINE.json configs[1]: 2 B rows, 1 M groups, SUM+COUNT on one H100).

The CPU oracle cannot finish 2 B rows inside a test, so the result is pinned two ways that do not depend on size:
  * an independent device-side recomputation with torch (bincount / index_add_ per 2^28-row chunk) — every group's COUNT and
    SUM must be bit-identical;
  * checksums: sum of COUNTs == number of rows, sum of SUMs == sum of the value column (mod 2^64), one output row per key.
The same rows at oracle-sized prefixes are compared against the oracle itself in test_gpu_groupby.py.
"""
import pytest

pytestmark = pytest.mark.gpu


@pytest.mark.timeout(900)
def test_c2_full_size_matches_independent_scatter_add(gpu_lib):
    import torch

    from bodo_b200 import synth
    from bodo_b200.streaming.groupby import (delete_groupby_state, get_metric, groupby_build_consume_batch,
                                             groupby_produce_output_batch, init_groupby_state)
    from bodo_b200.table import Column, Table

    n, g = 2_000_000_000, 1_000_000
    free, _total = torch.cuda.mem_get_info(0)
    if free < 70e9:
        pytest.skip("needs ~60 GB of free device memory (32 GB of rows + scratch)")
    dev = torch.device("cuda", 0)
    keys = torch.empty(n, dtype=torch.int64, device=dev)
    vals = torch.empty(n, dtype=torch.int64, device=dev)
    synth.device_fill(keys, vals, 0, g, 1)
    torch.cuda.synchronize()

    st = init_groupby_state(-1, (0,), ("sum", "count"), (0, 1, 2), (1, 1), expected_groups=g, output_batch_size=1 << 30, device=0)
    step = 500_000_000
    for r0 in range(0, n, step):
        r1 = min(n, r0 + step)
        t = Table([Column(keys[r0:r1]), Column(vals[r0:r1])], ["k", "v"])
        groupby_build_consume_batch(st, t, r1 == n, True)
    assert get_metric(st, 8) >= 4  # the SM-partitioned path ran
    ks, ss, cs = [], [], []
    while True:
        out, last = groupby_produce_output_batch(st, True)
        if out.n_rows:
            ks.append(torch.as_tensor(out.columns[0].data, device=dev).clone())
            ss.append(torch.as_tensor(out.columns[1].data, device=dev).clone())
            cs.append(torch.as_tensor(out.columns[2].data, device=dev).clone())
        if last:
            break
    delete_groupby_state(st)
    k, s, c = torch.cat(ks), torch.cat(ss), torch.cat(cs)

    # independent recomputation
    cnt = torch.zeros(g, dtype=torch.int64, device=dev)
    sm = torch.zeros(g, dtype=torch.int64, device=dev)
    chunk = 1 << 28
    for r0 in range(0, n, chunk):
        r1 = min(n, r0 + chunk)
        cnt += torch.bincount(keys[r0:r1], minlength=g)
        sm.index_add_(0, keys[r0:r1], vals[r0:r1])
    assert k.numel() == int((cnt > 0).sum().item()) == g
    assert torch.unique(k).numel() == g           # one output row per key
    assert torch.equal(cnt[k], c)
    assert torch.equal(sm[k], s)
    # checksums
    assert int(c.sum().item()) == n
    assert int(s.sum().item()) == int(vals.sum().item())
