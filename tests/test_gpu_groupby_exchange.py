"""The sharded groupby's partial-aggregate exchange on ONE GPU: R ranks are simulated by R C states on one device
(parallel=1, n_pes=R, rank=r) that share the default stream, so stream order stands in for the barrier between the pack and
the combine.  Each state consumes its slice of the same global rows (rank-major, as first / last order them), mixing device
and host batches; the states are then exchanged in the fused form (receive slabs as plain device tensors), in the fused form
with a slab too small for the rows (finalize returns -2, the NCCL form follows), or in the NCCL form directly (the test does
the all-to-all itself).  The union of the states' outputs must equal pandas, and every group a state outputs must be owned by
it (hash_to_rank of the key, as shuffle_table places its rows)."""

import numpy as np
import pandas as pd
import pytest
import torch

from bodo_b200 import _lib
from bodo_b200._lib import ffi
from bodo_b200.streaming.groupby import FTYPES, GroupbyState, groupby_produce_output_batch
from bodo_b200.table import CTable, Table

from .helpers import table_to_device
from .test_gpu_groupby_float_keys import SPECIAL

pytestmark = pytest.mark.gpu

SEED = 0xB0D01289  # SEED_HASH_PARTITION
BIG_SLAB, TINY_SLAB = 16 << 20, 8192
# (nested nunique states, outer state): slab bytes of the fused form, or None for the NCCL form directly
TRANSPORTS = {"fused": (BIG_SLAB, BIG_SLAB), "overflow": (TINY_SLAB, TINY_SLAB), "nccl": (None, None),
              "fused-then-overflow": (BIG_SLAB, TINY_SLAB)}


def _states(df: pd.DataFrame, n_keys, fnames, in_cols, R, dropna=True, expected_groups=0):
    """R simulated ranks: one Python handle per rank around a C state with n_pes=R, rank=r; rank r consumes the r-th slice
    of df in three batches (device, host, device)."""
    L = _lib.lib()
    offs, cols = [0], []
    for c in in_cols:
        cols += [] if c is None else [c]
        offs.append(len(cols))
    n, chunk = len(df), (len(df) + R - 1) // R
    states = []
    for r in range(R):
        mine = Table.from_pandas(df.iloc[r * chunk:min(n, (r + 1) * chunk)].reset_index(drop=True))
        st = GroupbyState(-1, range(n_keys), fnames, offs, cols, False, dropna, 1 << 30, expected_groups, 0, 0, None)
        ct, at = ffi.new("int8_t[]", [c.c_type for c in mine.columns]), ffi.new("int8_t[]", [c.arr_type for c in mine.columns])
        h = L.b200_groupby_state_init(-1, ct, at, mine.n_cols, ffi.new("int32_t[]", [FTYPES[f] for f in fnames]),
                                      ffi.new("int32_t[]", offs), ffi.new("int32_t[]", cols or [0]), len(fnames), n_keys, 1 << 30,
                                      1, int(dropna), 0, R, r, expected_groups, ffi.NULL)
        st.handle = _lib.check_ptr(h, "groupby state")
        st.build_indices = list(range(mine.n_cols))
        st.out_names = [f"k{j}" for j in range(n_keys)] + [f"f{j}" for j in range(len(fnames))]
        cuts = [0, mine.n_rows // 3, 2 * mine.n_rows // 3, mine.n_rows]
        for b in range(3):
            part = mine.slice(cuts[b], cuts[b + 1])
            batch = CTable(part if b == 1 else table_to_device(part))
            _lib.check(L.b200_groupby_build_consume_batch(st.handle, batch.ptr, int(b == 2), 1, ffi.new("int32_t*")), "consume")
        states.append(st)
    return states


def _fused(L, handles, slab_bytes):
    """pack -> (stream order) -> combine -> finalize on every rank; returns the finalize results and the slabs."""
    R = len(handles)
    cap_rows = (slab_bytes - 256) // (R * int(L.b200_groupby_exchange_row_bytes(handles[0])))
    slabs = [torch.zeros(slab_bytes, dtype=torch.uint8, device="cuda:0") for _ in range(R)]
    peers = torch.tensor([s.data_ptr() for s in slabs], dtype=torch.int64, device="cuda:0")
    for h in handles:
        _lib.check(L.b200_groupby_exchange_pack(h, ffi.cast("void* const*", peers.data_ptr()), cap_rows, ffi.NULL), "fused pack")
    for h, s in zip(handles, slabs):
        _lib.check(L.b200_groupby_exchange_combine(h, ffi.cast("void*", s.data_ptr()), cap_rows, ffi.NULL), "fused combine")
    return [int(L.b200_groupby_finalize(h)) for h in handles], [slabs, peers]


def _nccl(L, handles, counted):
    """The NCCL form, with the all-to-all done by torch on the one device; `counted`: a fused pack already counted the rows."""
    R = len(handles)
    words = int(L.b200_groupby_exchange_row_bytes(handles[0])) // 8
    counts, sends = [], []
    for h in handles:
        if not counted:
            _lib.check(L.b200_groupby_exchange_pack(h, ffi.NULL, 0, ffi.NULL), "count")
        c = ffi.new("int64_t[]", R)
        _lib.check(L.b200_groupby_exchange_counts(h, c), "counts")
        counts.append(list(c))
        send = torch.empty((max(sum(counts[-1]), 1), words), dtype=torch.int64, device="cuda:0")
        _lib.check(L.b200_groupby_exchange_pack(h, ffi.NULL, 0, ffi.cast("void*", send.data_ptr())), "pack")
        sends.append(send)
    recvs = []
    for d, h in enumerate(handles):
        pieces = [sends[s][sum(counts[s][:d]):sum(counts[s][:d + 1])] for s in range(R)]
        recv = torch.cat(pieces + [torch.empty((1, words), dtype=torch.int64, device="cuda:0")])
        _lib.check(L.b200_groupby_exchange_combine(h, ffi.cast("void*", recv.data_ptr()), 0, ffi.new("int64_t[]", [counts[s][d] for s in range(R)])),
                   "combine")
        recvs.append(recv)
    for h in handles:  # (the receive buffers stay alive until finalize returned: a replay reads them)
        _lib.check(int(L.b200_groupby_finalize(h)), "finalize")
    return recvs


def _exchange(L, handles, slab_bytes):
    """The sharded groupby's routine for one state per rank: fused when there are slabs, NCCL without or after -2."""
    keep = []
    if slab_bytes is not None:
        rcs, keep = _fused(L, handles, slab_bytes)
        assert len(set(rc == -2 for rc in rcs)) == 1 and min(rcs) >= -2, rcs  # every rank sees the same overflow flags
        if rcs[0] != -2:
            return "fused", keep
    return "nccl", keep + _nccl(L, handles, counted=slab_bytes is not None)


def _run(states, transport):
    """Exchanges the nested nunique states, then the outer ones; returns every rank's output and table rebuilds (metric 3)."""
    L = _lib.lib()
    inner_slab, outer_slab = TRANSPORTS[transport]
    handles = [st.handle for st in states]
    for i in range(int(L.b200_groupby_num_inner_states(handles[0]))):
        path, keep = _exchange(L, [_lib.check_ptr(L.b200_groupby_inner_state(h, i)) for h in handles], inner_slab)
        assert path == ("fused" if inner_slab == BIG_SLAB else "nccl"), path
    path, keep = _exchange(L, handles, outer_slab)
    assert path == ("fused" if outer_slab == BIG_SLAB else "nccl"), path
    outs, rebuilds = [], []
    for st in states:
        out, last = groupby_produce_output_batch(st, True)
        assert last
        outs.append(out.to_pandas())
        rebuilds.append(int(L.b200_groupby_get_metric(st.handle, 3)))
        L.b200_delete_groupby_state(st.handle)
        st.handle = None
    return outs, rebuilds


def _canon(df, n_keys):
    df = df.copy()
    for c in df.columns:
        df[c] = df[c].to_numpy(dtype="float64", na_value=np.nan) + 0.0  # (-0.0 and 0.0 are one group)
    return df.sort_values(list(df.columns[:n_keys]), na_position="last").reset_index(drop=True)


def _check_union(outs, exp, n_keys, exact, approx):
    got = pd.concat(outs, ignore_index=True)
    got.columns = list(exp.columns)
    g, e = _canon(got, n_keys), _canon(exp, n_keys)
    assert g.shape == e.shape, (g.shape, e.shape)
    for c in list(exp.columns[:n_keys]) + list(exact):
        np.testing.assert_array_equal(g[c].to_numpy(), e[c].to_numpy(), err_msg=c)
    for c in approx:
        np.testing.assert_allclose(g[c].to_numpy(), e[c].to_numpy(), rtol=1e-5, atol=1e-8, equal_nan=True, err_msg=c)


def _owned_single(outs, R, owner):
    for r, o in enumerate(outs):
        k = o.iloc[:, 0]
        assert (owner(k) == r).all(), f"rank {r} outputs a group it does not own"


@pytest.mark.parametrize("transport", ["fused", "overflow", "nccl"])
@pytest.mark.parametrize("R", [2, 3, 4])
def test_int64_key_every_aggregate_and_growth(gpu_lib, oracle, R, transport):
    """sum / count / mean / min / max / var / first / last; the key ranges make each rank's table grow while it combines."""
    rng = np.random.default_rng(100 + R)
    span, per = 24_000, 60_000
    k = np.concatenate([np.where(rng.random(per) < 0.85, r * span + rng.integers(0, span, per), rng.integers(0, R * span, per)) for r in range(R)])
    v = rng.integers(-1000, 1000, len(k)).astype(np.int64)
    vf = rng.standard_normal(len(k))
    df = pd.DataFrame({"k": k.astype(np.int64), "v": v, "vf": vf})
    fn = ("sum", "count", "mean", "min", "max", "var", "first", "last")
    states = _states(df, 1, fn, (1, 1, 2, 1, 2, 2, 1, 1), R, expected_groups=64)
    rebuilds_before = [int(gpu_lib.b200_groupby_get_metric(st.handle, 3)) for st in states]
    outs, rebuilds = _run(states, transport)
    assert any(a > b for a, b in zip(rebuilds, rebuilds_before)), (rebuilds_before, rebuilds)  # a table grew while combining
    gv = df.groupby("k")
    exp = pd.DataFrame({"sum": gv.v.sum(), "count": gv.v.count(), "mean": gv.vf.mean(), "min": gv.v.min(), "max": gv.vf.max(),
                        "var": gv.vf.var(), "first": gv.v.first(), "last": gv.v.last()}).reset_index()
    _check_union(outs, exp, 1, ("sum", "count", "min", "first", "last"), ("mean", "max", "var"))
    _owned_single(outs, R, lambda key: oracle.hash_to_rank(key.to_numpy(), None, R))


@pytest.mark.parametrize("transport", ["fused", "overflow", "nccl"])
@pytest.mark.parametrize("R", [2, 3, 4])
def test_float64_key_special_values(gpu_lib, oracle, R, transport):
    """±0.0 (0.0 and the INT64_MIN bit pattern), its neighbours ±5e-324, NaN (dropna=False keeps its group), infinities."""
    rng = np.random.default_rng(200 + R)
    n = 90_000
    pool = np.concatenate([SPECIAL, rng.standard_normal(3000) * 10.0 ** rng.integers(-5, 5, 3000)])
    df = pd.DataFrame({"k": pool[rng.integers(0, len(pool), n)], "w": rng.integers(-9, 9, n).astype(np.int64)})
    outs, _ = _run(_states(df, 1, ("sum", "count", "min"), (1, 1, 1), R, dropna=False), transport)
    exp = df.groupby("k", dropna=False).agg(sum=("w", "sum"), count=("w", "count"), min=("w", "min")).reset_index()
    _check_union(outs, exp, 1, ("sum", "count", "min"), ())
    L = oracle.lib()
    _owned_single(outs, R, lambda key: np.array([L.oracle_hash_inner_32_f64(float(x), SEED) % R for x in key]))


@pytest.mark.parametrize("transport", ["fused", "overflow", "nccl"])
@pytest.mark.parametrize("R", [2, 3, 4])
def test_nullable_int32_key_with_na_owned_where_shuffle_table_sends_it(gpu_lib, R, transport):
    """An int32 key's owner is the hash of its 4 raw bytes (hash_keys_table, pinned against the oracle in test_gpu_shuffle.py),
    as shuffle_table places its rows, not the hash of its widened 8-byte value."""
    rng = np.random.default_rng(300 + R)
    n = 80_000
    k = pd.array(rng.integers(-5000, 5000, n).astype(np.int32), dtype="Int32")
    k[rng.random(n) < 0.05] = pd.NA
    df = pd.DataFrame({"k": k, "w": rng.integers(-100, 100, n).astype(np.int64)})
    outs, _ = _run(_states(df, 1, ("sum", "count", "max"), (1, 1, 1), R, dropna=False), transport)
    exp = df.groupby("k", dropna=False).agg(sum=("w", "sum"), count=("w", "count"), max=("w", "max")).reset_index()
    _check_union(outs, exp, 1, ("sum", "count", "max"), ())

    def owner(key):
        from bodo_b200.shuffle import hash_keys_table

        _, dest = hash_keys_table(table_to_device(Table.from_pandas(key.to_frame())), 1, R)
        return dest.cpu().numpy()
    _owned_single(outs, R, owner)


def _mk_frame(rng, n, nk):
    cols = {"a0": rng.integers(0, 40, n).astype(np.int64),
            "a1": pd.array(rng.integers(-3, 4, n).astype(np.int32), dtype="Int32"),
            "a2": np.array([0.0, -0.0, np.nan, 1.5, -2.25])[rng.integers(0, 5, n)],
            "a3": pd.array(rng.integers(0, 3, n), dtype="Int64")}
    cols["a1"][rng.random(n) < 0.1] = pd.NA
    cols["a3"][rng.random(n) < 0.1] = pd.NA
    keys = {c: cols[c] for c in list(cols)[:nk]}
    return pd.DataFrame({**keys, "w": rng.integers(-50, 50, n).astype(np.int64), "x": rng.standard_normal(n)})


@pytest.mark.parametrize("transport", ["fused", "overflow", "nccl"])
@pytest.mark.parametrize("R,nk", [(2, 2), (3, 3), (4, 4), (4, 2)])
def test_multi_column_keys_with_na(gpu_lib, R, nk, transport):
    from bodo_b200.shuffle import hash_keys_table

    rng = np.random.default_rng(400 + 10 * R + nk)
    df = _mk_frame(rng, 70_000, nk)
    keys = list(df.columns[:nk])
    outs, _ = _run(_states(df, nk, ("sum", "count", "max", "mean"), (nk, nk, nk, nk + 1), R, dropna=False), transport)
    exp = df.groupby(keys, dropna=False).agg(sum=("w", "sum"), count=("w", "count"), max=("w", "max"), mean=("x", "mean")).reset_index()
    _check_union(outs, exp, nk, ("sum", "count", "max"), ("mean",))
    for r, o in enumerate(outs):
        if len(o):
            kt = table_to_device(Table.from_pandas(o.iloc[:, :nk]))
            _, dest = hash_keys_table(kt, nk, R)
            assert (dest.cpu().numpy() == r).all(), f"rank {r} outputs a key tuple it does not own"


@pytest.mark.parametrize("transport", ["fused", "overflow", "nccl", "fused-then-overflow"])
@pytest.mark.parametrize("R", [2, 3, 4])
def test_nunique(gpu_lib, oracle, R, transport):
    """nunique's nested (key, value) states are exchanged first (owned where the key is owned), then the outer state."""
    rng = np.random.default_rng(500 + R)
    n = 90_000
    df = pd.DataFrame({"k": rng.integers(0, 6000, n).astype(np.int64), "u": rng.integers(0, 7, n).astype(np.int64)})
    outs, _ = _run(_states(df, 1, ("nunique", "count", "sum"), (1, 1, 1), R), transport)
    gu = df.groupby("k").u
    exp = pd.DataFrame({"nunique": gu.nunique(), "count": gu.count(), "sum": gu.sum()}).reset_index()
    _check_union(outs, exp, 1, ("nunique", "count", "sum"), ())
    _owned_single(outs, R, lambda key: oracle.hash_to_rank(key.to_numpy(), None, R))
