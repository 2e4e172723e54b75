"""The sharded streaming hash join (build_parallel / probe_parallel, streaming/dist_join.py) against the exact join reference, on
one GPU, with the ranks simulated as threads of this process.

The lock-step process group.  R ranks run as R threads, each with a thread-local rank, and the torch.distributed functions the
library calls (is_initialized, get_world_size, get_rank, all_reduce with SUM / MIN / MAX, all_gather_into_tensor and
all_to_all_single with or without split sizes, barrier) are replaced through monkeypatch.  A collective called with async_op=True
runs at its barrier as any other and returns a completed handle whose wait() returns at once: a schedule more synchronous than
the real one, never less.  The ranks take turns: between two collectives
rank 0 runs, then rank 1, ..., so no two ranks are ever inside the library at once (the real system runs one process per GPU) and
every run is deterministic.  A collective stores its input, hands the turn on and waits on a threading.Barrier(R) whose action
runs the collective once for all ranks with torch ops on the ranks' tensors and gives the turn back to rank 0.  A rank that
raises aborts the barrier and the turn, the other ranks stop, and the test fails naming the rank and its exception; ranks that
call different collectives, or one that returns while others wait in a collective, fail the same way.  The threads are daemon
threads joined with a timeout.

The reference.  tests/test_gpu_join_exact.py's reference (and tests/test_gpu_join_condition.py's for a non-equi condition) joins
the global tables: the rank slices of a row-distributed side concatenated in rank order, the one table of a replicated side.
Every reference row is assigned to the rank that must emit it and to the probe batch it belongs to: a probe row is probed where
its key's owner is (hash_keys_table, which tests/test_gpu_shuffle.py pins against the oracle) when the build side is partitioned,
and where it was fed otherwise (broadcast build, or replicated build of a join without a build-outer tail); the build-outer tail
comes from the owner of the build key, in the last probe batch.  Each rank's output is then compared with its share exactly:
c-type, array type and bitmap presence per column, and the multiset of (valid, bits) records.  On the unique-key table forms a
rank's build key column takes the probe key's bits and bitmap (join.cu's documented rule); the rule is applied per rank, from
that rank's table form (metrics 5 and 7 of its local state).  The metrics are checked as well: where the build rows live
(build_rows_local, broadcast) and the OR-ed runtime filter of a partitioned inner join.

Float keys: a numpy NaN and a nullable NA can go to different ranks (the documented placement limitation), so no test mixes the
two in one key column when is_na_equal is True.

The GPU part (about 450 tests) took 157 s on one H100 80GB HBM3 (700 W power limit); its budget is 5 minutes."""

import threading
import time

import numpy as np
import pytest
import torch

from bodo_b200.table import ArrTypes, Column, CTypes, Table
from tests.test_gpu_join_exact import (ALL_TYPES, FLAGS, FLOATS, KINDS, NP_OF, NULLABLE, TYPE_NAME, UVIEW, _cat, bits_of, col,
                                       cross_values, dup_keys, gather, key_values, payload, records, reference, sort_records)

CT = CTypes
gpu = pytest.mark.gpu
RANK_TIMEOUT = 300.0  # seconds a run of all ranks may take before the test fails


# ================================================================================================ the lock-step process group
class RankError(AssertionError):
    """A rank raised: `rank` and `error` name the first rank that failed and its exception."""

    def __init__(self, rank, error, msg=None):
        super().__init__(msg or f"rank {rank} raised {type(error).__name__}: {error}")
        self.rank, self.error = rank, error


class _Aborted(Exception):
    """Raised in a rank that stops because another rank failed."""


class _Completed:
    """The work handle of an async_op collective: it already ran."""

    def wait(self, timeout=None):
        return True

    def is_completed(self):
        return True


class LockstepGroup:
    """R ranks as R threads that take turns (see the module docstring); `install` patches torch.distributed, `run` runs them."""

    def __init__(self, n_ranks, timeout=RANK_TIMEOUT):
        self.n = n_ranks
        self.timeout = timeout
        self.cond = threading.Condition()
        self.turn = 0
        self.failed = False
        self.finished = set()
        self.local = threading.local()
        self.inputs = [None] * n_ranks
        self.calls = []  # the collectives run, in order
        self.barrier = threading.Barrier(n_ranks, action=self._collective, timeout=timeout)

    # ---- torch.distributed, as the library calls it
    def install(self, monkeypatch):
        import torch.distributed as dist

        monkeypatch.setattr(dist, "is_initialized", lambda: True)
        monkeypatch.setattr(dist, "get_world_size", lambda group=None: self._check_group(group) or self.n)
        monkeypatch.setattr(dist, "get_rank", lambda group=None: self._check_group(group) or self.rank)
        monkeypatch.setattr(dist, "all_reduce", self.all_reduce)
        monkeypatch.setattr(dist, "all_gather_into_tensor", self.all_gather_into_tensor)
        monkeypatch.setattr(dist, "all_to_all_single", self.all_to_all_single)
        monkeypatch.setattr(dist, "barrier", self.barrier_collective)
        return self

    @staticmethod
    def _check_group(group):
        if group is not None:
            raise NotImplementedError("the lock-step group is the default group only")
        return 0

    @property
    def rank(self):
        r = getattr(self.local, "rank", None)
        if r is None:
            raise RuntimeError("torch.distributed called outside a rank thread")
        return r

    def all_reduce(self, tensor, op=None, group=None, async_op=False):
        import torch.distributed as dist

        return self._enter("all_reduce", group, async_op, tensor=tensor, op=dist.ReduceOp.SUM if op is None else op)

    def all_gather_into_tensor(self, output_tensor, input_tensor, group=None, async_op=False):
        return self._enter("all_gather_into_tensor", group, async_op, output=output_tensor, input=input_tensor)

    def all_to_all_single(self, output, input, output_split_sizes=None, input_split_sizes=None, group=None, async_op=False):
        return self._enter("all_to_all_single", group, async_op, output=output, input=input,
                           out_splits=None if output_split_sizes is None else [int(x) for x in output_split_sizes],
                           in_splits=None if input_split_sizes is None else [int(x) for x in input_split_sizes])

    def barrier_collective(self, group=None, async_op=False, device_ids=None):
        """torch.distributed.barrier: every rank waits until all ranks arrived (also the device-side barrier of a stand-in for
        the fused exchange's symmetric-memory handle)."""
        return self._enter("barrier", group, async_op)

    # ---- turns and collectives
    def _enter(self, name, group, async_op, **args):
        self._check_group(group)
        r = self.rank
        with self.cond:
            if self.finished:
                raise RuntimeError(f"rank {r} calls {name} after rank(s) {sorted(self.finished)} returned")
            self.inputs[r] = (name, args)
            self.turn = r + 1
            self.cond.notify_all()
        try:
            self.barrier.wait()
        except threading.BrokenBarrierError:
            raise _Aborted(f"rank {r}: {name} was abandoned") from None
        self._wait_turn(r)
        return _Completed() if async_op else None

    def _wait_turn(self, r):
        with self.cond:
            ok = self.cond.wait_for(lambda: self.failed or self.turn == r, self.timeout)
            if self.failed:
                raise _Aborted(f"rank {r} stopped: another rank failed")
            if not ok:
                raise TimeoutError(f"rank {r} waited {self.timeout} s for its turn")

    def _abort(self):
        with self.cond:
            self.failed = True
            self.cond.notify_all()
        self.barrier.abort()

    def _collective(self):
        """The barrier's action: every rank has stored its input; run the collective once for all of them."""
        names = [x[0] for x in self.inputs]
        if len(set(names)) != 1:
            raise RuntimeError(f"the ranks called different collectives: {names}")
        args = [x[1] for x in self.inputs]
        getattr(self, "_run_" + names[0])(args)
        self.calls.append(names[0])
        self.inputs = [None] * self.n
        with self.cond:
            self.turn = 0
            self.cond.notify_all()

    def _run_barrier(self, args):
        pass

    def _run_all_reduce(self, args):
        import torch.distributed as dist

        ts = [a["tensor"] for a in args]
        ops = [a["op"] for a in args]
        assert all(o == ops[0] for o in ops), ops
        assert all(t.shape == ts[0].shape and t.dtype == ts[0].dtype for t in ts), [(t.shape, t.dtype) for t in ts]
        st = torch.stack([t.detach() for t in ts])
        if ops[0] == dist.ReduceOp.SUM:
            res = st.sum(0).to(ts[0].dtype)
        elif ops[0] == dist.ReduceOp.MIN:
            res = st.amin(0)
        elif ops[0] == dist.ReduceOp.MAX:
            res = st.amax(0)
        else:
            raise NotImplementedError(f"all_reduce {ops[0]}")
        for t in ts:
            t.copy_(res)

    def _run_all_gather_into_tensor(self, args):
        ins = [a["input"] for a in args]
        assert all(x.shape == ins[0].shape and x.dtype == ins[0].dtype for x in ins), [(x.shape, x.dtype) for x in ins]
        res = torch.cat([x.reshape(-1) for x in ins])
        for a in args:
            assert a["output"].numel() == res.numel() and a["output"].dtype == res.dtype, (a["output"].shape, res.shape)
            a["output"].copy_(res.view(a["output"].shape))

    def _run_all_to_all_single(self, args):
        n = self.n
        splits = []
        for a in args:
            x = a["input"]
            if a["in_splits"] is None:
                assert x.shape[0] % n == 0, ("equal splits need a multiple of the world size", x.shape)
                s = [x.shape[0] // n] * n
            else:
                s = a["in_splits"]
                assert len(s) == n and sum(s) == x.shape[0], (s, x.shape)
            splits.append(s)
        recv = []
        for d in range(n):
            parts = []
            for s in range(n):
                off = sum(splits[s][:d])
                parts.append(args[s]["input"].narrow(0, off, splits[s][d]))
            got = [splits[s][d] for s in range(n)]
            o = args[d]["output"]
            exp = args[d]["out_splits"] if args[d]["out_splits"] is not None else [o.shape[0] // n] * n
            assert exp == got and sum(exp) == o.shape[0], (f"rank {d} expects {exp} rows per source (output {tuple(o.shape)}), "
                                                           f"the sources send {got}")
            recv.append(torch.cat(parts) if parts else None)
        for d in range(n):
            if recv[d] is not None and recv[d].shape[0]:
                args[d]["output"].copy_(recv[d])

    def run(self, fn):
        """fn(rank) on every rank; returns [fn(0), ..., fn(R - 1)] or raises RankError for the first rank that failed."""
        results, errors = [None] * self.n, [None] * self.n

        def main(r):
            self.local.rank = r
            try:
                self._wait_turn(r)
                results[r] = fn(r)
            except BaseException as e:  # noqa: BLE001 (reported by run)
                errors[r] = e
                self._abort()
                return
            with self.cond:
                if self.barrier.n_waiting:
                    errors[r] = RuntimeError(f"rank {r} returned while {self.barrier.n_waiting} rank(s) wait in a collective")
                else:
                    self.finished.add(r)
                    self.turn = r + 1
                    self.cond.notify_all()
                    return
            self._abort()

        threads = [threading.Thread(target=main, args=(r,), name=f"rank{r}", daemon=True) for r in range(self.n)]
        for t in threads:
            t.start()
        deadline = time.monotonic() + self.timeout
        for t in threads:
            t.join(max(0.0, deadline - time.monotonic()))
        alive = [t.name for t in threads if t.is_alive()]
        if alive:
            self._abort()
            for t in threads:
                t.join(10.0)
            raise AssertionError(f"ranks {alive} still ran after {self.timeout} s")
        for r, e in enumerate(errors):
            if e is not None and not isinstance(e, _Aborted):
                raise RankError(r, e) from e
        if any(e is not None for e in errors):
            raise AssertionError(f"ranks stopped without a failing rank (a collective timed out): {errors}")
        return results


@pytest.fixture
def lockstep(monkeypatch):
    """lockstep(R) -> a LockstepGroup of R ranks, installed as torch.distributed for this test."""
    return lambda n: LockstepGroup(n).install(monkeypatch)


# ================================================================================================ CPU: the harness itself
@pytest.mark.parametrize("R", [2, 3, 5])
def test_collectives_match_hand_computed_results(lockstep, R):
    import torch.distributed as dist

    pg = lockstep(R)

    def body(r):
        out = {"world": dist.get_world_size(), "rank": dist.get_rank(), "init": dist.is_initialized()}
        t = torch.tensor([r + 1, 10 - 3 * r, -r], dtype=torch.int64)
        for name, op in (("sum", dist.ReduceOp.SUM), ("min", dist.ReduceOp.MIN), ("max", dist.ReduceOp.MAX)):
            x = t.clone()
            dist.all_reduce(x, op=op)
            out[name] = x.tolist()
        x = t.clone()
        dist.all_reduce(x)  # the default op is SUM
        out["default"] = x.tolist()
        g = torch.empty(2 * R, dtype=torch.uint8)
        dist.all_gather_into_tensor(g, torch.tensor([r, 200 + r], dtype=torch.uint8))
        out["gather"] = g.tolist()
        eq = torch.arange(2 * R, dtype=torch.int32) + 100 * r  # equal splits: 2 rows to every rank
        eo = torch.empty(2 * R, dtype=torch.int32)
        dist.all_to_all_single(eo, eq)
        out["equal"] = eo.tolist()
        sc = [(r * 7 + 3 * d) % 4 for d in range(R)]  # uneven, zeros included
        sc_t = torch.tensor(sc, dtype=torch.int64)
        rc_t = torch.empty(R, dtype=torch.int64)
        dist.all_to_all_single(rc_t, sc_t)
        rc = rc_t.tolist()
        x = torch.arange(sum(sc), dtype=torch.float64) + 1000 * r
        y = torch.empty(sum(rc), dtype=torch.float64)
        dist.all_to_all_single(y, x, output_split_sizes=rc, input_split_sizes=sc)
        out["counts"], out["v"] = rc, y.tolist()
        return out

    res = pg.run(body)
    t = [[r + 1, 10 - 3 * r, -r] for r in range(R)]
    sc = [[(s * 7 + 3 * d) % 4 for d in range(R)] for s in range(R)]
    for r, o in enumerate(res):
        assert (o["world"], o["rank"], o["init"]) == (R, r, True)
        assert o["sum"] == o["default"] == [sum(c) for c in zip(*t)]
        assert o["min"] == [min(c) for c in zip(*t)] and o["max"] == [max(c) for c in zip(*t)]
        assert o["gather"] == [v for s in range(R) for v in (s, 200 + s)]
        assert o["equal"] == [100 * s + 2 * r + i for s in range(R) for i in range(2)]
        assert o["counts"] == [sc[s][r] for s in range(R)]
        assert o["v"] == [1000.0 * s + sum(sc[s][:r]) + i for s in range(R) for i in range(sc[s][r])]
    assert pg.calls == ["all_reduce"] * 4 + ["all_gather_into_tensor"] + ["all_to_all_single"] * 3


@pytest.mark.parametrize("R", [2, 3, 5])
def test_async_collectives_return_a_completed_handle(lockstep, R):
    """async_op=True: the collective has run when the call returns (the output is already there), and wait() returns at once."""
    import torch.distributed as dist

    pg = lockstep(R)

    def body(r):
        x = torch.tensor([r + 1, 2 * r], dtype=torch.int64)
        w1 = dist.all_reduce(x, async_op=True)
        after_reduce = x.tolist()  # read before wait(): the collective ran already
        g = torch.empty(2 * R, dtype=torch.int64)
        w2 = dist.all_gather_into_tensor(g, torch.tensor([r, 7 * r], dtype=torch.int64), async_op=True)
        after_gather = g.tolist()
        y = torch.empty(R, dtype=torch.int64)
        w3 = dist.all_to_all_single(y, torch.arange(R, dtype=torch.int64) + 10 * r, async_op=True)
        t0 = time.monotonic()
        for w in (w1, w2, w3):
            w.wait()
        assert time.monotonic() - t0 < 1.0
        assert dist.all_reduce(torch.zeros(1)) is None  # (a synchronous call still returns None)
        return after_reduce, after_gather, y.tolist(), all(w.is_completed() for w in (w1, w2, w3))

    res = pg.run(body)
    for r, (red, gat, a2a, done) in enumerate(res):
        assert red == [R * (R + 1) // 2, R * (R - 1)]
        assert gat == [v for s in range(R) for v in (s, 7 * s)]
        assert a2a == [10 * s + r for s in range(R)] and done
    assert pg.calls == ["all_reduce", "all_gather_into_tensor", "all_to_all_single", "all_reduce"]


def test_barrier_waits_for_every_rank(lockstep):
    """barrier(): no rank passes it before every rank arrived; a sync and an async barrier match one another."""
    import torch.distributed as dist

    R = 3
    pg = lockstep(R)
    log = []

    def body(r):
        log.append(("before", r))
        dist.barrier()
        log.append(("after", r))
        w = dist.barrier(async_op=(r == 1))
        if w is not None:
            w.wait()
        log.append(("end", r))

    pg.run(body)
    assert log == [(p, r) for p in ("before", "after", "end") for r in range(R)]
    assert pg.calls == ["barrier", "barrier"]
    mixed = lockstep(2)

    def other(r):
        if r == 0:
            dist.barrier()
        else:
            dist.all_reduce(torch.zeros(1))

    with pytest.raises(RankError, match="different collectives"):
        mixed.run(other)


def test_ranks_take_turns_in_rank_order(lockstep):
    import torch.distributed as dist

    R = 4
    pg = lockstep(R)
    log = []

    def body(r):
        for step in range(3):
            log.append((step, r))
            dist.all_reduce(torch.zeros(1))
        log.append((3, r))

    pg.run(body)
    assert log == [(step, r) for step in range(4) for r in range(R)]


def test_a_rank_that_raises_fails_the_run_promptly(lockstep):
    import torch.distributed as dist

    pg = lockstep(3)

    def body(r):
        dist.all_reduce(torch.zeros(1))
        if r == 1:
            raise ValueError("rank 1 gives up")
        dist.all_reduce(torch.zeros(1))

    t0 = time.monotonic()
    with pytest.raises(RankError, match="rank 1 raised ValueError: rank 1 gives up") as ei:
        pg.run(body)
    assert ei.value.rank == 1 and time.monotonic() - t0 < 10
    assert not any(t.name.startswith("rank") and t.is_alive() for t in threading.enumerate())


@pytest.mark.parametrize("how", ["different collectives", "returns early", "calls after a rank returned"])
def test_a_protocol_mismatch_fails_the_run(lockstep, how):
    import torch.distributed as dist

    pg = lockstep(3)

    def body(r):
        if how == "different collectives" and r == 2:
            dist.all_gather_into_tensor(torch.zeros(3), torch.zeros(1))
        elif how == "returns early" and r == 2:
            return
        elif how == "calls after a rank returned" and r == 0:
            return
        dist.all_reduce(torch.zeros(1))

    t0 = time.monotonic()
    with pytest.raises(RankError) as ei:
        pg.run(body)
    msg = {"different collectives": "different collectives", "returns early": "returned while", "calls after a rank returned": "after rank"}[how]
    assert msg in str(ei.value) and time.monotonic() - t0 < 10


@pytest.mark.parametrize("R", [2, 3, 5])
def test_exchange_table_on_cpu_tensors(lockstep, oracle, R):
    """shuffle.exchange_table through the lock-step group, with tests/test_dist_gloo.py's oracle partition and numpy bitmap merge
    standing in for the CUDA kernels: rank r receives the rows whose destination is r, ordered by source rank, then input order."""
    from bodo_b200.shuffle import exchange_table, with_schema_validity
    from tests.test_dist_gloo import _numpy_merge_bitmaps, _oracle_partition

    pg = lockstep(R)
    parts = []
    for r in range(R):
        rng = np.random.default_rng(40 + r)
        n = [0, 13, 1000, 77, 5][r]
        k = rng.integers(0, 50, n)
        parts.append(Table([col(CT.INT64, k), payload(CT.UINT16, n, 3 + r), payload(CT.FLOAT64, n, 9 + r, nullable=True, null_every=3),
                            Column(payload(CT.INT32, n, r).data, None, CT.INT32, NULLABLE, n)]))  # nullable, no bitmap: one travels

    def body(r):
        part, counts = _oracle_partition(with_schema_validity(parts[r]), 1, R)
        out = exchange_table(part, counts, merge_bitmaps=_numpy_merge_bitmaps)
        return [(c.c_type, c.arr_type, c.validity is not None, bits_of(c)) for c in out.columns]

    res = pg.run(body)
    dests = [oracle.hash_to_rank(p.columns[0].data, None, R) for p in parts]
    for r in range(R):
        for j in range(4):
            exp_b = np.concatenate([bits_of(parts[s].columns[j])[0][dests[s] == r] for s in range(R)])
            exp_v = np.concatenate([bits_of(parts[s].columns[j])[1][dests[s] == r] for s in range(R)])
            ct, at, has, (b, v) = res[r][j]
            assert (ct, at, has) == (parts[0].columns[j].c_type, parts[0].columns[j].arr_type, j >= 2), (r, j)
            np.testing.assert_array_equal(v, exp_v)
            np.testing.assert_array_equal(np.where(v, b, 0), np.where(exp_v, exp_b, 0))


def test_sharded_operators_that_are_not_supported_are_refused(lockstep):
    """A sharded full sort, window and min_row_number_filter raise their B200Error on the first consume call of a 2-rank group."""
    from bodo_b200._lib import B200Error
    from bodo_b200.streaming import sort as S
    from bodo_b200.streaming import window as W
    from bodo_b200.streaming.groupby import groupby_build_consume_batch
    from tests.test_groupby_mrnf_host import mrnf_state

    t = Table([col(CT.INT64, np.arange(10)), col(CT.INT64, np.arange(10))], ["k", "o"])
    cases = {
        "a sharded full sort is not supported": lambda: S.sort_build_consume_batch(
            S.init_stream_sort_state(-1, None, 0, ["k"], [True], ["last"], ["k", "o"], parallel=True, full=True), t, True),
        "a sharded window is not supported": lambda: W.window_build_consume_batch(
            W.init_window_state(-1, ["k"], [], True, "last", [("rn", "row_number")], ["k", "o"], parallel=True), t, True),
        "a sharded min_row_number_filter is not supported": lambda: groupby_build_consume_batch(mrnf_state(parallel=True), t, True, True),
    }
    for msg, call in cases.items():
        with pytest.raises(RankError) as ei:
            lockstep(2).run(lambda r: call())
        assert ei.value.rank == 0 and isinstance(ei.value.error, B200Error) and msg in str(ei.value.error), ei.value


# ================================================================================================ driving the sharded join
PLACEMENTS = ["partitioned", "broadcast_forced", "broadcast_by_size", "partitioned_build_replicated_probe",
              "replicated_build_partitioned_probe"]


def placement_args(placement, monkeypatch):
    """(build_parallel, probe_parallel, force_broadcast), with BODO_BCAST_JOIN_THRESHOLD set for the placement."""
    monkeypatch.setenv("BODO_BCAST_JOIN_THRESHOLD", "1000000000" if placement == "broadcast_by_size" else "0")
    return {"partitioned": (True, True, False), "broadcast_forced": (True, True, True), "broadcast_by_size": (True, True, False),
            "partitioned_build_replicated_probe": (True, False, False),
            "replicated_build_partitioned_probe": (False, True, False)}[placement]


def to_dev(t):
    from tests.helpers import table_to_device

    return table_to_device(t)


def rank_batches(t, R, rng, n_batches=3, empty_ranks=(), on_device=True):
    """A host table split into R rank slices (the ranks in empty_ranks get none) of n_batches batches each, at uneven sizes with
    zero-row batches; every other batch is staged on the device."""
    live = [r for r in range(R) if r not in empty_ranks]
    cuts = np.sort(rng.integers(0, t.n_rows + 1, len(live) - 1)) if live else []
    bounds = np.concatenate([[0], cuts, [t.n_rows]]).astype(int)
    from tests.test_gpu_join_exact import host_slices

    out = []
    for r in range(R):
        if r in empty_ranks:
            lo = hi = 0
        else:
            i = live.index(r)
            lo, hi = bounds[i], bounds[i + 1]
        n = hi - lo
        c = np.sort(rng.integers(0, n + 1, n_batches - 1))
        sizes = np.diff(np.concatenate([[0], c, [n]])).astype(int).tolist()
        if r % 2 and n_batches > 1:
            sizes = [0] + sizes[:-2] + [sizes[-2] + sizes[-1]]  # a leading empty batch
        part = t.slice(lo, hi)
        bs = host_slices(part, sizes)
        out.append([to_dev(b) if on_device and (q + r) % 2 and b.n_rows else b for q, b in enumerate(bs)])
    return out


def owners(t, keys, R):
    """hash_keys_table's destination rank of every row of host table t over the key columns `keys` (in key order)."""
    from bodo_b200.shuffle import hash_keys_table
    from bodo_b200.table import to_device

    if t.n_rows == 0:
        return np.zeros(0, np.int64)
    kt = to_device(t.select(list(keys)), 0)
    _, dest = hash_keys_table(kt, len(keys), R)
    torch.cuda.synchronize()
    return dest.cpu().numpy().astype(np.int64)


def run_sharded(lockstep, monkeypatch, R, build, probe, bkeys, pkeys, kind, na_equal, placement, used=None, cond=None, bnames=None,
                pnames=None):
    """Every rank feeds its build batches, then its probe batches; returns per rank ([(c_type, arr_type, has_bitmap, (bits, valid))
    per column] per probe batch, st.metrics, {local metric: value})."""
    from bodo_b200.streaming.join import (delete_join_state, get_metric, init_join_state, join_build_consume_batch,
                                          join_probe_consume_batch)

    bp, pp, force = placement_args(placement, monkeypatch)
    bo, po = FLAGS[kind]
    bnames = bnames or [f"b{j}" for j in range(build[0][0].n_cols)]
    pnames = pnames or [f"p{j}" for j in range(probe[0][0].n_cols)]
    pg = lockstep(R)

    def body(r):
        st = init_join_state(-1, tuple(bkeys), tuple(pkeys), bnames, pnames, bo, po, force_broadcast=force, non_equi_condition=cond,
                             build_parallel=bp, probe_parallel=pp, is_na_equal=na_equal, is_mark_join=kind == "mark",
                             is_anti_join=kind == "anti", device=0)
        try:
            for i, b in enumerate(build[r]):
                join_build_consume_batch(st, b, i == len(build[r]) - 1)
            outs = []
            for i, p in enumerate(probe[r]):
                out, _, _ = join_probe_consume_batch(st, p, i == len(probe[r]) - 1, True, used)
                outs.append([(c.c_type, c.arr_type, c.validity is not None, bits_of(c)) for c in out.columns])
            return outs, dict(st.metrics), {m: get_metric(st, m) for m in (0, 1, 5, 6, 7)}
        finally:
            delete_join_state(st)

    return pg.run(body)


def _global(parts, parallel):
    """The global table of a side: the rank slices in rank order, or the one table of a replicated side; with each row's
    (source rank, batch index)."""
    ranks = range(len(parts)) if parallel else [0]
    batches, src, bq = [], [], []
    for r in ranks:
        for q, b in enumerate(parts[r]):
            batches.append(b)
            src.append(np.full(b.n_rows, r))
            bq.append(np.full(b.n_rows, q))
    return _cat(batches), np.concatenate(src).astype(np.int64), np.concatenate(bq).astype(np.int64)


def check_sharded(lockstep, monkeypatch, R, build, probe, bkeys, pkeys, kind="inner", na_equal=False, placement="partitioned",
                  used=None, cond=None, bnames=None, pnames=None):
    """Run the sharded join and compare every rank's every probe batch with its share of the reference join of the global tables,
    exactly; check the placement metrics.  build / probe: per rank, a list of batches (the same list on every rank for a
    replicated side).  Returns (per-rank results, global probe table, reference result)."""
    from tests.test_gpu_join_condition import cond_reference

    res = run_sharded(lockstep, monkeypatch, R, build, probe, bkeys, pkeys, kind, na_equal, placement, used, cond, bnames, pnames)
    bp, pp, force = placement_args(placement, monkeypatch)
    bo, po = FLAGS[kind]
    bt, _, _ = _global(build, bp)
    pt, psrc, pq = _global(probe, pp)
    nk = len(bkeys)
    bnames = bnames or [f"b{j}" for j in range(bt.n_cols)]
    pnames = pnames or [f"p{j}" for j in range(pt.n_cols)]
    border = list(bkeys) + [j for j in range(bt.n_cols) if j not in bkeys]
    porder = list(pkeys) + [j for j in range(pt.n_cols) if j not in pkeys]
    if cond is None:
        ref = reference([bt.select(border)], [pt.select(porder)], nk, kind, na_equal)
    else:
        ref = cond_reference([bt.select(border)], [pt.select(porder)], nk, kind, na_equal, cond, [bnames[j] for j in border],
                             [pnames[j] for j in porder])[0]
    # where the build rows live, and who probes each probe row
    broadcast = bp and pp and not bo and (force or placement == "broadcast_by_size")
    partitioned_build = (bp and not broadcast) or (pp and bo)
    mets = [m for _, m, _ in res]
    locs = [lm for _, _, lm in res]
    assert [m["broadcast"] for m in mets] == [int(broadcast)] * R, mets
    n_build = bt.n_rows
    if partitioned_build:
        bown = owners(bt, bkeys, R)
        pown = owners(pt, pkeys, R)
        assert [m["build_rows_local"] for m in mets] == [int((bown == r).sum()) for r in range(R)], (mets, np.bincount(bown, minlength=R))
        prank = pown
    else:
        bown = None
        prank = psrc
        if broadcast:
            assert [m["build_rows_local"] for m in mets] == [n_build] * R, mets
    if partitioned_build and pp and kind in ("inner", "build_outer"):
        assert [m.get("filter", 0) for m in mets] == [1] * R, mets  # the OR-ed bloom filter and global key bounds
    else:
        assert all("filter" not in m for m in mets), mets
    for r in range(R):
        assert locs[r][0] == (mets[r]["build_rows_local"] if partitioned_build or broadcast else n_build), (r, locs[r], mets[r])

    b_at = [c.arr_type for c in build[0][0].columns]
    p_at = [c.arr_type for c in probe[0][0].columns]
    b_ct = [c.c_type for c in build[0][0].columns]
    p_ct = [c.c_type for c in probe[0][0].columns]
    bcols = [bits_of(c) for c in bt.columns]
    pcols = [bits_of(c) for c in pt.columns]
    kb = list(range(bt.n_cols)) if used is None else list(used[0])
    kp = list(range(pt.n_cols)) if used is None else list(used[1])
    if kind == "mark":
        kb = []
    n_q = len(probe[0])
    unique_rule = kind == "inner" and nk == 1 and cond is None
    for r in range(R):
        outs = res[r][0]
        assert len(outs) == n_q
        unique = locs[r][7] == 1 or locs[r][5] > 0
        unknown_form = unique_rule and not unique and not (prank == r).any()
        for q, got in enumerate(outs):
            last = q == n_q - 1
            if kind == "mark":
                rows = np.flatnonzero((prank == r) & (pq == q))
                exp = [(p_ct[j], p_at[j] == NULLABLE, gather(*pcols[j], rows)) for j in kp]
                exp.append((CT.BOOL, True if len(rows) else None, (ref[rows].astype(np.uint64), np.ones(len(rows), bool))))
            else:
                bi, pi = ref
                sel = ((pi >= 0) & (prank[np.maximum(pi, 0)] == r) & (pq[np.maximum(pi, 0)] == q))
                if bown is not None:
                    sel |= (pi < 0) & last & (bown[np.maximum(bi, 0)] == r)
                else:
                    assert not ((pi < 0) & last).any() or not bo
                bsel, psel = bi[sel], pi[sel]
                exp = []
                for src in kb:
                    cell = gather(*bcols[src], bsel)
                    nullable = b_at[src] == NULLABLE or po or kind == "anti"
                    if unique_rule and src == bkeys[0] and (unique or unknown_form):
                        pk = pkeys[0]
                        local_bitmap = p_at[pk] == NULLABLE if partitioned_build else probe[r][q].columns[pk].validity is not None
                        pcell = gather(*pcols[pk], psel)
                        cell = (np.where(bsel >= 0, pcell[0], cell[0]), np.where(bsel >= 0, pcell[1], cell[1]))
                        nullable = (local_bitmap or b_at[src] == NULLABLE) if unique else None
                    exp.append((b_ct[src], nullable, cell))
                for src in kp:
                    exp.append((p_ct[src], p_at[src] == NULLABLE or bo, gather(*pcols[src], psel)))
            assert len(got) == len(exp), (r, q, len(got), len(exp))
            for j, (g, x) in enumerate(zip(got, exp)):
                # nullable: a bitmap and the nullable array type; None: either (an empty batch's mark column, or the build key
                # column of a rank that saw no probe row, whose table form its metrics cannot tell)
                allowed = {True: [(NULLABLE, True)], False: [(ArrTypes.NUMPY, False)],
                           None: [(NULLABLE, True), (NULLABLE, False), (ArrTypes.NUMPY, False)]}[x[1]]
                assert g[0] == x[0] and tuple(g[1:3]) in allowed, (f"rank {r} batch {q} column {j}: got (c_type, arr_type, bitmap) "
                                                                   f"{g[:3]}, expected c_type {x[0]}, nullable {x[1]}")
            g, x = records([c[3] for c in got]), records([c[2] for c in exp])
            assert g.shape == x.shape, (f"rank {r} batch {q} ({kind}, {placement}): {g.shape[0]} rows, expected {x.shape[0]}")
            np.testing.assert_array_equal(sort_records(g), sort_records(x), err_msg=f"rank {r} batch {q} ({kind}, {placement})")
    return res, pt, ref


# ================================================================================================ GPU: the matrix
RS = [2, 3, 4, 7]


def basic_tables(rng, n_build=2500, n_probe=6000, n_distinct=1500):
    """Duplicated int64 keys with NA keys, probe keys partly outside the build keys' range; a numpy and a nullable payload a side."""
    b = Table([payload(CT.INT32, n_build, 1, nullable=True, null_every=5), dup_keys(n_build, n_distinct, rng, na_every=97),
               payload(CT.UINT64, n_build, 2)])
    pk = rng.integers(-300, n_distinct + 600, n_probe)
    pv = np.ones(n_probe, bool)
    pv[5::89] = False
    p = Table([col(CT.INT64, pk, pv), payload(CT.FLOAT64, n_probe, 3), payload(CT.INT16, n_probe, 4, nullable=True, null_every=7)])
    return b, p


def sides(b, p, R, rng, placement, build_kw=None, probe_kw=None):
    """Per-rank batches of the build and probe tables: rank slices of a row-distributed side, the same batches on every rank for a
    replicated one (empty_ranks applies to row-distributed sides only)."""
    bp, pp = {"partitioned_build_replicated_probe": (True, False), "replicated_build_partitioned_probe": (False, True)}.get(
        placement, (True, True))

    def split(t, parallel, kw):
        kw = dict(kw or {})
        if parallel:
            return rank_batches(t, R, rng, **kw)
        kw.pop("empty_ranks", None)
        return [rank_batches(t, 1, rng, **kw)[0]] * R

    return split(b, bp, build_kw), split(p, pp, probe_kw)


@gpu
@pytest.mark.timeout(900)
@pytest.mark.parametrize("na_equal", [False, True])
@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("placement", PLACEMENTS)
@pytest.mark.parametrize("R", RS)
def test_every_kind_and_placement(gpu_lib, lockstep, monkeypatch, R, placement, kind, na_equal):
    """Rank R - 1 has no build rows and rank 0 no probe rows in a partitioned side; a replicated side is the same batches on every
    rank.  A replicated build against a partitioned probe with a build-outer tail must still emit each unmatched build row once."""
    rng = np.random.default_rng(1000 * R + 10 * PLACEMENTS.index(placement) + KINDS.index(kind))
    b, p = basic_tables(rng)
    build, probe = sides(b, p, R, rng, placement, {"empty_ranks": (R - 1,)}, {"empty_ranks": (0,)})
    check_sharded(lockstep, monkeypatch, R, build, probe, [1], [0], kind, na_equal, placement)


KEY_CASES = [(ct, nullable) for ct in ALL_TYPES for nullable in (False, True)]


@gpu
@pytest.mark.timeout(900)
@pytest.mark.parametrize("na_equal", [False, True])
@pytest.mark.parametrize("ct,nullable", KEY_CASES, ids=[f"{TYPE_NAME[c]}-{'nullable' if n else 'numpy'}" for c, n in KEY_CASES])
def test_every_single_key_type(gpu_lib, lockstep, monkeypatch, ct, nullable, na_equal):
    """One key of each type with its edge values, NA keys in the nullable form and NaN in the numpy form of a float key (never both
    in one column), -0.0 meeting 0.0.  Keys of 1 and 2 bytes cannot be hash-partitioned (the shuffle hashes 4- and 8-byte keys):
    the placements that shuffle refuse them, the others join them."""
    from bodo_b200._lib import B200Error

    R = 3
    w = np.dtype(NP_OF[ct]).itemsize
    rng = np.random.default_rng(ct * 7 + 3)
    vals = key_values(ct, 150, rng)
    bk = np.concatenate([vals, vals[: len(vals) // 2]])
    pk = vals[rng.integers(0, len(vals), 3000)]
    bvalid = pvalid = None
    if ct in FLOATS:
        pk = pk.copy()
        pk[5::17] = -pk[5::17]  # -0.0 meets 0.0 among them
        if not nullable:
            nan = np.array([0x7FF8DEADBEEF0001 if w == 8 else 0x7FC01234], dtype=UVIEW[w]).view(NP_OF[ct])[0]
            pk[::13] = nan
            bk = bk.copy()
            bk[2] = nan
    if nullable:
        bvalid = np.ones(len(bk), bool)
        bvalid[1::37] = False
        pvalid = rng.random(len(pk)) > 0.05
    b = Table([col(ct, bk, bvalid, nullable), payload(CT.INT64, len(bk), 3)])
    p = Table([col(ct, pk, pvalid, nullable), payload(CT.UINT64, len(pk), 4)])
    for placement in ("partitioned", "broadcast_forced", "replicated_build_partitioned_probe"):
        for kind in ("inner", "full_outer", "anti", "mark"):
            build, probe = sides(b, p, R, rng, placement)
            shuffles = placement == "partitioned" or FLAGS[kind][0]  # a build-outer tail keeps the build partitioned
            if w < 4 and shuffles:
                with pytest.raises(RankError) as ei:
                    run_sharded(lockstep, monkeypatch, R, build, probe, [0], [0], kind, na_equal, placement)
                assert isinstance(ei.value.error, B200Error) and "4- or 8-byte" in str(ei.value.error), ei.value
                continue
            check_sharded(lockstep, monkeypatch, R, build, probe, [0], [0], kind, na_equal, placement)


@gpu
@pytest.mark.timeout(900)
@pytest.mark.parametrize("n_keys", [2, 3, 4])
@pytest.mark.parametrize("placement", PLACEMENTS)
@pytest.mark.parametrize("R", [3, 4])
def test_multi_column_keys(gpu_lib, lockstep, monkeypatch, R, placement, n_keys):
    """2 to 4 key columns (int64, nullable int32, float64, date), not first, in a different order on the two sides."""
    rng = np.random.default_rng(50 * R + 5 * PLACEMENTS.index(placement) + n_keys)
    nb, npr = 2000, 5000
    kt = [CT.INT64, CT.INT32, CT.FLOAT64, CT.DATE][:n_keys]

    def keycols(n, na):
        cols = []
        for j, ct in enumerate(kt):
            v = rng.integers(0, [30, 4, 3, 2][j], n)
            if ct == CT.FLOAT64:
                v = np.where(v == 0, -0.0, v * 0.5)
                cols.append(col(ct, v))
            else:
                cols.append(col(ct, v, (rng.random(n) > 0.04) if (j == 1 and na) else None, nullable=j == 1))
        return cols

    bkc, pkc = keycols(nb, True), keycols(npr, True)
    # build: payload, keys in order 1, 0, 2, ...; probe: keys reversed, a payload in between
    border = [1, 0] + list(range(2, n_keys))
    b = Table([payload(CT.UINT32, nb, 1, nullable=True, null_every=4)] + [bkc[j] for j in border] + [payload(CT.INT64, nb, 2)])
    bkeys = [1 + border.index(j) for j in range(n_keys)]
    prev = list(range(n_keys))[::-1]
    p = Table([pkc[prev[0]], payload(CT.FLOAT32, npr, 3)] + [pkc[j] for j in prev[1:]])
    ppos = [0] + list(range(2, n_keys + 1))
    pkeys = [ppos[prev.index(j)] for j in range(n_keys)]
    for kind in KINDS:
        build, probe = sides(b, p, R, rng, placement)
        check_sharded(lockstep, monkeypatch, R, build, probe, bkeys, pkeys, kind, kind in ("inner", "anti"), placement)


CROSS_PAIRS = [(CT.INT64, CT.UINT64), (CT.DATETIME, CT.UINT64)]


@gpu
@pytest.mark.timeout(900)
@pytest.mark.parametrize("placement", PLACEMENTS)
@pytest.mark.parametrize("build_unsigned", [True, False])
@pytest.mark.parametrize("pair", CROSS_PAIRS, ids=[f"{TYPE_NAME[s]}-{TYPE_NAME[u]}" for s, u in CROSS_PAIRS])
def test_keys_join_by_value_across_signedness(gpu_lib, lockstep, monkeypatch, pair, build_unsigned, placement):
    """uint64 2^64 - 1 does not meet int64 -1 on any rank; equal values meet whatever side and rank they come from."""
    R = 3
    s, u = pair
    sv, uv = cross_values(s, u)
    rng = np.random.default_rng(7 + build_unsigned)
    bt_, pt_ = (u, s) if build_unsigned else (s, u)
    bvals, pvals = (uv, sv) if build_unsigned else (sv, uv)
    bk = np.array(list(bvals) * 3, dtype=object).astype(NP_OF[bt_])
    pk = np.array(pvals, dtype=object)[rng.integers(0, len(pvals), 1200)].astype(NP_OF[pt_])
    b = Table([col(bt_, bk), payload(CT.INT64, len(bk), 1)])
    p = Table([col(pt_, pk), col(CT.INT64, np.arange(len(pk)))])
    for kind in ("inner", "probe_outer", "full_outer", "anti", "mark"):
        build, probe = sides(b, p, R, rng, placement)
        check_sharded(lockstep, monkeypatch, R, build, probe, [0], [0], kind, False, placement)


@gpu
@pytest.mark.timeout(900)
@pytest.mark.parametrize("wide", ["build", "probe"])
@pytest.mark.parametrize("placement", ["partitioned", "broadcast_forced", "partitioned_build_replicated_probe"])
@pytest.mark.parametrize("R", [3, 7])
def test_every_column_width(gpu_lib, lockstep, monkeypatch, R, placement, wide):
    """Every column type on one side, numpy and nullable with NULLs and edge bits, through the all-to-all and the merge of segment
    bitmaps whose lengths are not multiples of 8 (full outer: NULL-extended cells on both sides); used_cols keeps a subset."""
    rng = np.random.default_rng(R + 3 * ["build", "probe"].index(wide))
    nb, npr = 1500, 4000
    many = []
    n = nb if wide == "build" else npr
    for j, ct in enumerate(ALL_TYPES):
        many.append(payload(ct, n, 31 * j + 1))
        many.append(payload(ct, n, 31 * j + 2, nullable=True, null_every=3 + j % 4))
    bkey, pkey = dup_keys(nb, 900, rng, na_every=50), dup_keys(npr, 1200, rng, na_every=60)
    few_b = [payload(ct, nb, 900 + j) for j, ct in enumerate((CT.INT64, CT.UINT8, CT.FLOAT32))]
    few_p = [payload(ct, npr, 910 + j) for j, ct in enumerate((CT.INT64, CT.INT16, CT.DATE))]
    b, p = (Table([bkey] + many), Table([pkey] + few_p)) if wide == "build" else (Table([bkey] + few_b), Table([pkey] + many))
    used = (list(range(b.n_cols)), [1, 2, 3]) if wide == "build" else ([0, 1, 2], list(range(p.n_cols)))
    kind = "full_outer" if placement != "broadcast_forced" else "probe_outer"
    build, probe = sides(b, p, R, rng, placement)
    check_sharded(lockstep, monkeypatch, R, build, probe, [0], [0], kind, True, placement, used)
    used2 = ([2, 0], [1, 0]) if wide == "build" else ([1], [5, 0, 5])  # a subset, reordered, a column repeated
    check_sharded(lockstep, monkeypatch, R, build, probe, [0], [0], "inner", False, placement, used2)


@gpu
@pytest.mark.timeout(900)
@pytest.mark.parametrize("n_keys", [1, 2])
@pytest.mark.parametrize("kind", ["inner", "probe_outer", "build_outer", "full_outer", "anti", "mark"])
@pytest.mark.parametrize("placement", PLACEMENTS)
def test_non_equi_condition(gpu_lib, lockstep, monkeypatch, placement, kind, n_keys):
    """tests/test_gpu_join_condition.py's case (NA cells, NaN, Kleene logic, isnull, arithmetic) through DistJoinState."""
    from tests.test_gpu_join_condition import kind_case

    R = 3
    rng = np.random.default_rng(100 * n_keys + KINDS.index(kind) + 7 * PLACEMENTS.index(placement))
    (b,), probe_batches, bn, pn, cond = kind_case(n_keys, rng, 2000, 4000)
    p = _cat(probe_batches)
    p = Table([col(c.c_type, *_host_cell(c, pc)) for c, pc in zip(p.columns, probe_batches[0].columns)])
    build, probe = sides(b, p, R, rng, placement)
    keys = list(range(n_keys))
    check_sharded(lockstep, monkeypatch, R, build, probe, keys, keys, kind, True, placement, None, cond, bn, pn)


def _host_cell(c, like):
    """(values, validity or None, nullable) of a _cat column, with the array type of the column it came from."""
    v = np.asarray(c.values_numpy())
    m = c.valid_mask_numpy()
    keep = like.arr_type == NULLABLE
    return v, (m if keep else None), keep


@gpu
@pytest.mark.timeout(900)
@pytest.mark.parametrize("kind", ["inner", "build_outer", "full_outer", "anti"])
@pytest.mark.parametrize("R", [2, 4, 7])
def test_skewed_and_empty_inputs(gpu_lib, lockstep, monkeypatch, R, kind):
    """One distinct build key: one rank owns every build row and the others build on empty tables (their runtime-filter bounds are
    the empty sentinel).  Ranks feed different numbers of non-empty batches and keep calling with empty ones until is_last; the
    build arrives in several batches (concat_device) where one batch of a nullable column has a bitmap and another has none."""
    rng = np.random.default_rng(R * 10 + KINDS.index(kind))
    nb, npr = 900, 4000
    b = Table([col(CT.INT64, np.full(nb, 42)), payload(CT.INT32, nb, 1, nullable=True, null_every=3), payload(CT.FLOAT64, nb, 2)])
    pk = np.where(rng.random(npr) < 0.3, 42, rng.integers(-50, 100, npr))
    p = Table([col(CT.INT64, pk), payload(CT.UINT8, npr, 3, nullable=True, null_every=4)])
    for placement in ("partitioned", "replicated_build_partitioned_probe", "partitioned_build_replicated_probe"):
        build, probe = sides(b, p, R, rng, placement, {"n_batches": 4}, {"n_batches": 5, "empty_ranks": (1,)})
        for r in range(R):  # a nullable column without a bitmap in some batches: concat_device gives the whole build one
            for q, t in enumerate(build[r]):
                if q % 2 == 0 and t.n_rows:
                    c = t.columns[1]
                    t.columns[1] = Column(c.data, None, c.c_type, NULLABLE, c.length)
        res, pt, _ = check_sharded(lockstep, monkeypatch, R, build, probe, [0], [0], kind, False, placement)
        if placement == "partitioned":
            mets = [m for _, m, _ in res]
            assert sorted(m["build_rows_local"] for m in mets) == [0] * (R - 1) + [nb], mets
    # the build side on one rank only, the probe side on another rank only
    from tests.test_gpu_join_exact import host_slices

    build = [host_slices(b.slice(0, 0), [0, 0]) for _ in range(R)]
    build[R - 1] = host_slices(b, [nb // 2, nb - nb // 2])
    probe = [host_slices(p.slice(0, 0), [0, 0, 0]) for _ in range(R)]
    probe[0] = host_slices(p, [100, 0, npr - 100])
    check_sharded(lockstep, monkeypatch, R, build, probe, [0], [0], kind, False, "partitioned")


@gpu
@pytest.mark.timeout(900)
@pytest.mark.parametrize("R", [2, 3, 7])
def test_runtime_filter_drops_probe_rows_outside_the_global_bounds(gpu_lib, lockstep, monkeypatch, R):
    """Partitioned inner join: the ranks' bloom filters are OR-ed and the key bounds taken over all ranks; every probe row with a
    partner survives (the result is complete) and every probe row whose key lies outside the global bounds is dropped."""
    rng = np.random.default_rng(R)
    nb, npr = 3000, 20000
    bk = rng.integers(1000, 5000, nb)
    b = Table([col(CT.INT64, bk), payload(CT.INT64, nb, 1)])
    pk = rng.integers(-4000, 10000, npr)
    p = Table([col(CT.INT64, pk), payload(CT.INT64, npr, 2)])
    build, probe = sides(b, p, R, rng, "partitioned")
    res, _, _ = check_sharded(lockstep, monkeypatch, R, build, probe, [0], [0], "inner", False, "partitioned")
    mets = [m for _, m, _ in res]
    after = sum(m.get("probe_rows_after_filter", 0) for m in mets)
    outside = int(((pk < bk.min()) | (pk > bk.max())).sum())
    partner = int(np.isin(pk, bk).sum())
    assert outside > npr // 3 and partner <= after <= npr - outside, (after, outside, partner)
    assert sum(m["probe_rows_local"] for m in mets) == after


@gpu
def test_runtime_filter_keeps_rows_as_they_are(gpu_lib):
    """runtime_join_filter returns the kept rows unchanged: every column type, numpy or nullable, 16 columns (its limit); a NaN
    stays a valid NaN with its payload bits and a numpy column stays numpy.  The sharded join filters probe batches before it
    exchanges them, so every rank must see the same schema, whether its batch went through the filter or not."""
    from bodo_b200.streaming.join import delete_join_state, init_join_state, join_build_consume_batch, runtime_join_filter

    rng = np.random.default_rng(12)
    nb, npr = 2000, 5000
    b = Table([col(CT.INT64, rng.integers(0, 4000, nb)), payload(CT.INT64, nb, 1)])
    cols = [col(CT.INT64, rng.integers(-2000, 8000, npr)), col(CT.INT64, np.arange(npr))]
    for j, ct in enumerate(ALL_TYPES):
        cols.append(payload(ct, npr, 31 * j + 1, nullable=j % 2 == 1, null_every=3 if j % 2 else 0))
    p = Table(cols)
    assert p.n_cols == 16
    st = init_join_state(-1, (0,), (0,), ["k", "v"], [f"p{j}" for j in range(p.n_cols)], False, False)
    try:
        join_build_consume_batch(st, to_dev(b), True)
        kept = runtime_join_filter((st,), to_dev(p), ((0,),))
        got = [(c.c_type, c.arr_type, c.validity is not None, bits_of(c)) for c in kept.columns]
    finally:
        delete_join_state(st)
    rows = got[1][3][0].astype(np.int64)
    assert np.isin(np.flatnonzero(np.isin(p.columns[0].data, b.columns[0].data)), rows).all() and len(rows) < npr
    for j, (c, g) in enumerate(zip(p.columns, got)):
        assert g[:3] == (c.c_type, c.arr_type, c.validity is not None), (j, g[:3])
        eb, ev = bits_of(c)
        np.testing.assert_array_equal(g[3][1], ev[rows], err_msg=f"column {j} validity")
        np.testing.assert_array_equal(np.where(g[3][1], g[3][0], 0), np.where(ev[rows], eb[rows], 0), err_msg=f"column {j}")


# ================================================================================================ GPU: shuffle_table, top-k
@gpu
@pytest.mark.timeout(900)
@pytest.mark.parametrize("n_keys", [1, 2])
@pytest.mark.parametrize("R", [2, 3, 5, 8])
def test_shuffle_table_at_r_ranks(gpu_lib, lockstep, R, n_keys):
    """Rank r receives exactly the rows whose destination is r, ordered by source rank, then input order; data and validity bit for
    bit at every column width; empty destinations and segment lengths that are not multiples of 8."""
    from bodo_b200.shuffle import shuffle_table

    rng = np.random.default_rng(R * 3 + n_keys)
    host = []
    for r in range(R):
        n = [1003, 0, 17, 4099, 1, 250, 8, 77][r]
        keys = [col(CT.INT64, rng.integers(0, 3 if r == 2 else 400, n), rng.random(n) > 0.1)]  # rank 2: few keys, empty destinations
        if n_keys == 2:
            keys.append(col(CT.INT32, rng.integers(0, 5, n)))
        pays = [payload(ct, n, 17 * j + r, nullable=j % 2 == 1, null_every=3 if j % 2 else 0) for j, ct in enumerate(ALL_TYPES)]
        host.append(Table(keys + pays))
    parts = [to_dev(t) if r % 2 and t.n_rows else t for r, t in enumerate(host)]
    dests = [owners(h, list(range(n_keys)), R) for h in host]

    def body(r):
        from bodo_b200.table import to_device

        out = shuffle_table(to_device(parts[r], 0), n_keys)
        return [(c.c_type, c.arr_type, c.validity is not None, bits_of(c)) for c in out.columns]

    res = lockstep(R).run(body)
    for r in range(R):
        assert len(res[r]) == host[0].n_cols
        for j, (ct, at, has, (b, v)) in enumerate(res[r]):
            exp_b = np.concatenate([bits_of(h.columns[j])[0][d == r] for h, d in zip(host, dests)])
            exp_v = np.concatenate([bits_of(h.columns[j])[1][d == r] for h, d in zip(host, dests)])
            assert (ct, at, has) == (host[0].columns[j].c_type, host[0].columns[j].arr_type, host[0].columns[j].arr_type == NULLABLE), (r, j)
            np.testing.assert_array_equal(v, exp_v, err_msg=f"rank {r} column {j} validity")
            np.testing.assert_array_equal(np.where(v, b, 0), np.where(exp_v, exp_b, 0), err_msg=f"rank {r} column {j}")


@gpu
@pytest.mark.timeout(900)
@pytest.mark.parametrize("case", ["base", "past_the_end", "empty_rank"])
@pytest.mark.parametrize("R", [2, 3, 4])
def test_sharded_topk(gpu_lib, lockstep, R, case):
    """tests/test_gpu_sort.py's sharded top-k case at R ranks on one GPU: the stable top-k of the rank inputs in rank order on
    rank 0, one empty batch on the others; limit + offset beyond the global row count; a rank without rows."""
    from bodo_b200.streaming import sort as S
    from tests.test_gpu_sort import _sharded_data, batches_of, col_mask, oracle_perm

    parts = [_sharded_data(r) for r in range(R)]
    parts = [p.slice(0, 20_000 + 3000 * r) for r, p in enumerate(parts)]
    if case == "empty_rank":
        parts[1] = parts[1].slice(0, 0)
    n_total = sum(p.n_rows for p in parts)
    limit, offset = (500, 9) if case != "past_the_end" else (n_total, 1000)

    def body(r):
        st = S.init_stream_sort_state(-1, limit, offset, ["k", "f"], [False, True], ["first", "last"], parts[r].names, parallel=True, device=0)
        try:
            bs = batches_of(parts[r], [7_000], 2)
            for i, b in enumerate(bs):
                S.sort_build_consume_batch(st, to_dev(b) if i % 2 and b.n_rows else b, i == len(bs) - 1)
            rows = []
            while True:
                out, last = S.produce_output_batch(st)
                rows.append([(c.values_numpy().copy(), col_mask(c)) for c in out.columns])
                if last:
                    break
            return [(np.concatenate([x[c][0] for x in rows]), np.concatenate([x[c][1] for x in rows])) for c in range(3)]
        finally:
            S.delete_stream_sort_state(st)

    res = lockstep(R).run(body)
    cols = []
    for c in range(3):
        cs = [p.columns[c] for p in parts]
        v = np.concatenate([x.values_numpy() for x in cs])
        m = np.concatenate([col_mask(x) for x in cs])
        cols.append(Column(v, np.packbits(m, bitorder="little") if cs[0].validity is not None else None, cs[0].c_type, cs[0].arr_type, len(v)))
    full = Table(cols, ["k", "f", "p"])
    perm = oracle_perm(full, ["k", "f"], [False, True], ["first", "last"])[offset:offset + limit]
    assert len(perm) == min(limit, max(n_total - offset, 0))
    for c in range(3):
        vals, mask = res[0][c]
        np.testing.assert_array_equal(vals.view(np.uint8), full.columns[c].values_numpy()[perm].view(np.uint8))
        np.testing.assert_array_equal(mask, col_mask(full.columns[c])[perm])
    for r in range(1, R):
        assert all(len(v) == 0 for v, _ in res[r])
