"""Host side of the sampled evaluation (Master.local_sampled_*, core/Master.scala:109-118) on CPU: the rank split of the
sample, the draw key, the empty-sample decisions, and a 2-process gloo run of the SPMD Master over a stand-in device
context that records what each rank would ask the GPU for."""
import math
import os
import socket
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LAM = 0.5


def _free_port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def _counts_of_positions(lo, hi):
    """Stand-in counters of positions [lo, hi): hinge p % 3 per position, correct when p is even."""
    p = np.arange(lo, hi)
    return int((p % 3).sum()), int((p % 2 == 0).sum())


def _counts_of_ids(ids):
    ids = np.asarray(ids, dtype=np.int64)
    return int((ids % 3).sum()), int((ids % 2 == 0).sum())


class RecordingCtx:
    """Stands in for NativeCtx: records the sampled-evaluation calls and answers with counters that depend on what was
    asked for, so that sums over ranks can be checked."""

    def __init__(self, dim):
        self.dim, self.calls = dim, []

    def eval_sampled_counts(self, row_begin, row_end, key, pos_begin, pos_end, w=None):
        self.calls.append(("sampled", int(row_begin), int(row_end), int(key), int(pos_begin), int(pos_end)))
        return (*_counts_of_positions(pos_begin, pos_end), 4.0)

    def eval_samples_counts(self, samples, w=None):
        samples = np.array(samples, dtype=np.int64)
        self.calls.append(("samples", samples.tolist()))
        return (*_counts_of_ids(samples), 4.0)

    def comm_init(self, uid):
        pass


class RecordingSlave:
    def __init__(self, world, n_train, n_test, dim):
        self.ctx, self.world, self.is_async = RecordingCtx(dim), world, False
        self.n_train, self.n_test, self.dim = n_train, n_test, dim


def _stub(n, dim):
    from distributed_sgd_b200.utils.dataset import Data
    return Data(np.arange(n + 1, dtype=np.int64), np.zeros(n, np.int32), np.ones(n, np.float32), np.ones(n, np.int8), dim)


def _master(n_train=101, n_test=40, dim=16, jvm_exact=False, group=None, world=1, seed=3):
    from distributed_sgd_b200.core.master import MasterSync
    from distributed_sgd_b200.ml import SparseSVM
    slave = RecordingSlave(world, n_train, n_test, dim)
    m = MasterSync(0, _stub(n_train, dim), _stub(n_test, dim), SparseSVM(LAM), world, slave=slave, group=group, seed=seed,
                   jvm_exact=jvm_exact)
    return m, slave.ctx


def test_sample_shard_covers_every_position_once():
    from distributed_sgd_b200.core.master import sample_shard
    for W in range(1, 9):
        for k in range(0, 301):
            shards = [sample_shard(k, W, r) for r in range(W)]
            assert shards[0][0] == 0 and shards[-1][1] == k
            assert all(shards[r][1] == shards[r + 1][0] for r in range(W - 1))        # contiguous, no overlap, no gap
            sizes = [hi - lo for lo, hi in shards]
            assert min(sizes) >= 0 and max(sizes) - min(sizes) <= 1 and sum(sizes) == k


def test_sampled_key_is_deterministic_and_differs_per_draw():
    from distributed_sgd_b200.core.master import sampled_key
    for seed in (0, 1, 42, 2**63 + 5, -1):
        keys = [sampled_key(seed, t) for t in range(2000)]
        assert keys == [sampled_key(seed, t) for t in range(2000)]
        assert len(set(keys)) == len(keys)
        assert all(0 <= k < 2**64 for k in keys)
    assert sampled_key(0, 0) != sampled_key(1, 0)


def test_empty_sample_is_decided_on_the_host():
    from distributed_sgd_b200.core.master import sampled_key
    from distributed_sgd_b200.native import DsgdEmpty
    m, ctx = _master(n_test=0)
    for count in (0, -3):
        with pytest.raises(DsgdEmpty):
            m.local_sampled_loss(None, count)
        with pytest.raises(DsgdEmpty):
            m.local_sampled_loss_accuracy(None, count)
        assert math.isnan(m.local_sampled_accuracy(None, count))
    with pytest.raises(DsgdEmpty):                               # no test rows: take(k) of an empty range
        m.local_sampled_loss(None, 5, test_data=True)
    assert math.isnan(m.local_sampled_accuracy(None, 5, test_data=True))
    assert ctx.calls == []                                       # nothing reached the device
    m.local_sampled_accuracy(None, 10)                           # the first real draw still uses t = 0
    assert ctx.calls == [("sampled", 0, 101, sampled_key(3, 0), 0, 10)]


def test_one_rank_loss_accuracy_and_fresh_keys():
    from distributed_sgd_b200.core.master import sampled_key
    m, ctx = _master()
    loss, acc = m.local_sampled_loss_accuracy(None, 37)
    h, c = _counts_of_positions(0, 37)
    assert (loss, acc) == (LAM * 4.0 + h / 37, c / 37)
    assert m.local_sampled_loss(None, 500, test_data=True) == LAM * 4.0 + _counts_of_positions(0, 40)[0] / 40   # take(k)
    m.local_sampled_accuracy(None, 5)
    assert ctx.calls == [("sampled", 0, 101, sampled_key(3, 0), 0, 37), ("sampled", 101, 141, sampled_key(3, 1), 0, 40),
                         ("sampled", 0, 101, sampled_key(3, 2), 0, 5)]


def test_jvm_exact_draws_take_from_the_fit_stream():
    from distributed_sgd_b200.utils.jvm_random import JvmRandom
    m, ctx = _master(jvm_exact=True, seed=0)
    ref = JvmRandom(0)
    m.local_sampled_accuracy(None, 9, test_data=True)
    assert ctx.calls[-1] == ("samples", (ref.shuffle(np.arange(40))[:9] + 101).tolist())
    m.local_sampled_accuracy(None, 0)                            # empty, but the reference shuffles before `take`
    ref.shuffle(np.arange(101))
    assert len(ctx.calls) == 1
    m.local_sampled_loss(None, 7)
    assert ctx.calls[-1] == ("samples", ref.shuffle(np.arange(101))[:7].tolist())
    assert m.jvm.next_int() == ref.next_int()                    # both streams are at the same place


def _worker(rank, world, port, jvm_exact, q):
    sys.path.insert(0, ROOT)
    import torch.distributed as dist
    from distributed_sgd_b200.core import Group, master as master_mod
    dist.init_process_group("gloo", init_method=f"tcp://127.0.0.1:{port}", rank=rank, world_size=world)
    master_mod.NativeCtx.comm_unique_id = staticmethod(lambda: bytes(range(128)))
    m, ctx = _master(jvm_exact=jvm_exact, group=Group(), world=world, seed=0)
    out = [m.local_sampled_loss_accuracy(None, 37), m.local_sampled_loss_accuracy(None, 3, test_data=True),
           m.local_sampled_loss_accuracy(None, 1000, test_data=True), (m.local_sampled_accuracy(None, 1),)]
    q.put({"rank": rank, "calls": ctx.calls, "out": out})
    dist.destroy_process_group()


def _run_two_ranks(jvm_exact):
    import torch.multiprocessing as mp
    ctxmp = mp.get_context("spawn")
    q = ctxmp.Queue()
    port = _free_port()
    procs = [ctxmp.Process(target=_worker, args=(r, 2, port, jvm_exact, q)) for r in range(2)]
    for p in procs:
        p.start()
    res = sorted([q.get(timeout=120) for _ in procs], key=lambda r: r["rank"])
    for p in procs:
        p.join(timeout=30)
    return res


# (rows, k) of the four evaluations _worker makes: 37 train rows, 3 and all 40 test rows, 1 train row
CASES = [((0, 101), 37), ((101, 141), 3), ((101, 141), 40), ((0, 101), 1)]


def test_two_ranks_split_one_device_drawn_sample():
    r0, r1 = _run_two_ranks(jvm_exact=False)
    assert r0["out"] == r1["out"]
    calls = {0: iter(r0["calls"]), 1: iter(r1["calls"])}
    for i, ((b, e), k) in enumerate(CASES):
        got = {}
        for r in (0, 1):
            lo, hi = (k * r) // 2, (k * (r + 1)) // 2
            if hi > lo:                                          # k = 1: rank 0's share is empty and it skips the call
                got[r] = next(calls[r])
        assert all(c[0] == "sampled" for c in got.values())
        assert {(c[1], c[2]) for c in got.values()} == {(b, e)}   # the same rows ...
        assert len({c[3] for c in got.values()}) == 1            # ... and the same key on both ranks
        shares = sorted((c[4], c[5]) for c in got.values())
        assert shares[0][0] == 0 and shares[-1][1] == k and all(a[1] == b_[0] for a, b_ in zip(shares, shares[1:]))
        h, c = _counts_of_positions(0, k)
        loss, acc = r0["out"][i] if i < 3 else (None, r0["out"][i][0])
        if loss is not None:
            assert loss == LAM * 4.0 + h / k
        assert acc == c / k
    assert next(calls[0], None) is None and next(calls[1], None) is None
    keys = [c[3] for c in r1["calls"]]
    assert len(set(keys)) == len(keys)                           # a fresh draw per call


def test_two_ranks_split_one_jvm_exact_list():
    from distributed_sgd_b200.utils.jvm_random import JvmRandom
    r0, r1 = _run_two_ranks(jvm_exact=True)
    assert r0["out"] == r1["out"]
    ref = JvmRandom(0)
    calls = {0: iter(r0["calls"]), 1: iter(r1["calls"])}
    for i, ((b, e), k) in enumerate(CASES):
        ids = (ref.shuffle(np.arange(e - b))[:k] + b).tolist()
        parts = []
        for r in (0, 1):
            lo, hi = (k * r) // 2, (k * (r + 1)) // 2
            if hi > lo:
                c = next(calls[r])
                assert c == ("samples", ids[lo:hi])
                parts += c[1]
        assert parts == ids
        h, c = _counts_of_ids(ids)
        if i < 3:
            assert r0["out"][i] == (LAM * 4.0 + h / k, c / k)
        else:
            assert r0["out"][i] == (c / k,)
    assert next(calls[0], None) is None and next(calls[1], None) is None
