"""Several Hogwild workers on one GPU, against the fp64 oracle through the C ABI.

Every update of a worker goes to its own replica, to every peer's and to the master's, which counts it.  Hogwild workers
never wait for each other, so K async contexts can share one GPU, in one process or in several.

- Turn-taking replays (dsgd_async_replay from the resident replica, one worker after another): every replica receives the
  same deltas in the same order, so the oracle is Oracle.async_run over the merged schedule.  lambda = 0: every replica
  and the master bit for bit; lambda > 0: replicas bit-identical to each other and within the async tolerance of the
  oracle.  Outboxes hold exactly each worker's own deltas.  The filter edges with their updates dealt to different
  workers: a residual leaves every replica, and a worker reads c from the S slot a peer's update moved.
- Concurrent free-running loops on exact data: replicas and master bit-identical, nothing lost or counted twice.
- The replica table at its edges: 16 workers and the master fill all 17 slots, async worlds above 16 and attaches to a
  running loop are refused, and dsgd_update_grad stays on its own replica.
- Across processes: replicas exchanged as CUDA IPC handles, and MasterAsync.fit with two worker processes.
"""
import multiprocessing as mp
import os
import socket
import sys
import time

import numpy as np
import pytest

from helpers import FILTER_CASES, async_workers, conservation_rows, csr, edge_rows, filter_case, filter_expect

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LR = 0.125
TIMEOUT = 120


def _oracle(data, lam, d):
    from oracle.oracle import Oracle
    orc = Oracle(data.row_ptr, data.col, data.val, data.label, data.dim, lam)
    orc.set_dim_sparsity(d)
    return orc


def schedule(K, n_updates, seed):
    """Turns (worker, updates) of 1 to 7 updates each, n_updates in all: every worker once in a shuffled order, then
    workers drawn at random (a worker may follow itself)."""
    rng = np.random.default_rng(seed)
    first = [int(k) for k in rng.permutation(K)]
    turns, total = [], 0
    while total < n_updates:
        k = first.pop(0) if first else int(rng.integers(K))
        n = min(int(rng.integers(1, 8)), n_updates - total)
        turns.append((k, n))
        total += n
    assert {k for k, _ in turns} == set(range(K)), "every worker takes a turn"
    return turns


def batches(seed, n_rows, batch, n_updates):
    rng = np.random.default_rng(seed)
    return np.stack([rng.choice(n_rows, size=batch, replace=False) for _ in range(n_updates)]).astype(np.int32)


def replay_turns(ctxs, turns, idx, batch, lr):
    """Worker k replays its turn's updates idx[pos:pos + n] from its resident replica (peers' pushes included)."""
    pos = 0
    for k, n in turns:
        ctxs[k].async_replay(None, idx[pos:pos + n].reshape(-1), batch, lr)
        pos += n


def _close(ctxs):
    for c in ctxs:
        c.close()


@pytest.fixture(scope="module")
def edge_data():
    """Dyadic rows of 0 to 2000 pairs (tests/helpers.py edge_rows), w0, and the dimSparsity of all rows."""
    data, w0 = edge_rows(21)
    d = _oracle(data, 0.0, np.zeros(data.dim)).dim_sparsity(data.n_rows)
    return data, w0, d


def _n_updates(K, batch):
    return max({1: 240, 4: 96, 33: 32}[batch], 8 * K)


# ---- A. turn-taking replays in one process ----------------------------------------------------------------------------

@pytest.mark.parametrize("lam", [0.0, 1e-3])
@pytest.mark.parametrize("batch", [1, 4, 33])
@pytest.mark.parametrize("K", [2, 3, 16])
def test_turns_match_oracle(edge_data, K, batch, lam):
    """Batch 1 runs k_async_worker_b1, 4 and 33 k_async_worker.  With K = 16 the master fills the 17th replica slot.  At
    lambda > 0 each worker forms c from its own replica's S slot (the others' pushes keep it incrementally), but it sends
    the same delta to every replica: the replicas stay bit-identical."""
    data, w0, d = edge_data
    n = _n_updates(K, batch)
    turns = schedule(K, n, seed=10 * K + batch)
    idx = batches(1000 * K + batch, data.n_rows, batch, n)
    ctxs = async_workers(data, lam, d, K, w0)
    try:
        replay_turns(ctxs, turns, idx, batch, LR)
        ws = [c.get_weights() for c in ctxs]
        masters = [c.async_master_weights() for c in ctxs]   # hosted by rank 0, attached by the others
        counts = [c.async_updates() for c in ctxs]
    finally:
        _close(ctxs)
    w_ref = _oracle(data, lam, d).async_run(w0, idx.reshape(-1), batch, LR)
    assert np.count_nonzero(w_ref != w0) > 100                 # the run moved many columns (not a vacuous pass)
    assert counts == [n] * K                                   # the master counted every worker's updates
    for r in range(K):
        np.testing.assert_array_equal(masters[r], masters[0], err_msg=f"rank {r} reads another master")
    for r, w in enumerate(ws + masters[:1]):
        what = f"replica {r}" if r < K else "the master"
        if lam == 0.0:
            np.testing.assert_array_equal(w, w_ref, err_msg=what)
        else:
            np.testing.assert_array_equal(w, ws[0], err_msg=f"{what} differs from replica 0")
    if lam != 0.0:
        assert (ws[0] == 0).tolist() == (w_ref == 0).tolist()
        np.testing.assert_allclose(ws[0], w_ref, rtol=1e-9, atol=1e-13)


@pytest.mark.parametrize("batch", [1, 4])
@pytest.mark.parametrize("K", [2, 3, 15])
def test_turns_outboxes(edge_data, K, batch):
    """Every worker's outbox holds minus the sum of its own deltas, in the order it made them; the outboxes together hold
    w_final - w0.  Dyadic values and power-of-two batches keep every sum exact.  K = 15: the master and the outbox fill
    all 17 replica slots."""
    data, w0, d = edge_data
    n = _n_updates(K, batch)
    turns = schedule(K, n, seed=20 * K + batch)
    idx = batches(2000 * K + batch, data.n_rows, batch, n)
    ctxs = async_workers(data, 0.0, d, K, w0, outbox=True)
    try:
        replay_turns(ctxs, turns, idx, batch, LR)
        ws = [c.get_weights() for c in ctxs]
        wm = ctxs[0].async_master_weights()
        outs = [c.async_outbox_read() for c in ctxs]
        count = ctxs[0].async_updates()
    finally:
        _close(ctxs)
    orc = _oracle(data, 0.0, d)
    w, expect, pos = w0.copy(), [np.zeros(data.dim) for _ in range(K)], 0
    for k, m in turns:
        for u in range(pos, pos + m):
            expect[k] -= orc.async_delta(w, idx[u], LR)
            w = orc.async_run(w, idx[u], batch, LR)
        pos += m
    assert count == n
    # a worker whose every row fails the gate sends nothing; most send something (not a vacuous pass)
    assert sum(bool(np.any(e != 0)) for e in expect) > K // 2
    for r in range(K):
        np.testing.assert_array_equal(ws[r], w, err_msg=f"replica {r}")
        np.testing.assert_array_equal(outs[r], expect[r], err_msg=f"outbox of worker {r}")
    np.testing.assert_array_equal(wm, w)
    np.testing.assert_array_equal(np.sum(outs, axis=0), w - w0)


@pytest.mark.parametrize("batch", [1, 2])
@pytest.mark.parametrize("name", FILTER_CASES)
def test_filter_cases_across_workers(name, batch):
    """The 1e-20 filter edges of test_gpu_async_edges.py with update u made by worker 1 + u % 2 of three (rank 0 hosts the
    master).  residual: the entry lands on exactly 0 in every replica and the master.  cancel and tiny_delta: the second
    update is made by a worker that only received the first: it reads c from the S slot the first update's -sum(delta d)
    push moved (or, for tiny_delta, left alone) in its own replica."""
    rows, labels, dim, d, lam, lr, w0 = filter_case(name)
    data = csr(rows, np.asarray(labels, np.int8), dim)
    ctxs = async_workers(data, lam, d, 3, w0)
    try:
        for u in range(len(rows)):
            ctxs[1 + u % 2].async_replay(None, np.full(batch, u, np.int32), batch, lr)
        ws = [c.get_weights() for c in ctxs] + [ctxs[0].async_master_weights()]
        count = ctxs[0].async_updates()
    finally:
        _close(ctxs)
    w_ref = _oracle(data, lam, d).async_run(w0, np.repeat(np.arange(len(rows), dtype=np.int32), batch), batch, lr)
    expect = filter_expect(name)
    assert count == len(rows)
    for r, w in enumerate(ws):
        what = f"replica {r}" if r < 3 else "the master"
        for j, v in expect.items():
            assert w_ref[j] == v, (j, w_ref[j], v)             # the case is what it says on the oracle
            assert w[j] == v, (what, j, w[j], v)
        np.testing.assert_array_equal(w, w_ref, err_msg=what)


# ---- B. concurrent free-running loops in one process ------------------------------------------------------------------

@pytest.fixture(scope="module")
def conservation():
    return conservation_rows()


def _wait_idle(ctxs):
    t0 = time.time()
    while any(c.async_running() for c in ctxs) and time.time() - t0 < 60:
        time.sleep(0.002)
    assert not any(c.async_running() for c in ctxs), "a loop did not finish"
    for c in ctxs:
        c.stop_async()


@pytest.mark.parametrize("batch", [1, 8])
@pytest.mark.parametrize("lanes", [1, 32])
@pytest.mark.parametrize("K", [2, 4, 16])
def test_concurrent_workers_conserve(conservation, K, lanes, batch):
    """K loops run at once, worker r for its own max_updates.  Every entry is 2^-4, y = +1, w0 = 2^10, lr = 2^-6: every
    partial sum is exact in any order, so replicas, master, counter, outboxes and the total decrease must all be exact.
    K = 16 runs without outboxes: 16 workers and the master fill all 17 replica slots."""
    data, k = conservation
    w0 = np.full(data.dim, 1024.0)
    lr = 2.0 ** -6
    U = [1000 + 250 * r for r in range(K)]
    outbox = K < 16
    assigned = np.arange(data.n_rows, dtype=np.int32)
    ctxs = async_workers(data, 0.0, np.zeros(data.dim), K, w0)
    try:
        # one short run each first: it sizes the loop's scratch, whose growth (cudaFree) would otherwise wait for the
        # loops already running and serialise the workers
        for r, c in enumerate(ctxs):
            c.start_async(None, assigned, batch, lr, concurrency=lanes, max_updates=lanes, seed=r)
            _wait_idle([c])
        for c in ctxs:
            c.set_weights(w0)
            if outbox:
                c.async_outbox_enable()
        ctxs[0].async_host_master(w0)
        for r, c in enumerate(ctxs):
            c.start_async(None, assigned, batch, lr, concurrency=lanes, max_updates=U[r], seed=100 * r + lanes + batch)
        _wait_idle(ctxs)
        ws = [c.get_weights() for c in ctxs]
        wm = ctxs[0].async_master_weights()
        count = ctxs[K - 1].async_updates()
        outs = [c.async_outbox_read() for c in ctxs] if outbox else None
    finally:
        _close(ctxs)
    for r in range(K):
        np.testing.assert_array_equal(ws[r], ws[0], err_msg=f"replica {r}")
    np.testing.assert_array_equal(wm, ws[0])
    assert count == sum(U)
    assert (w0 - ws[0]).sum() == sum(U) * lr * k * 2.0 ** -4
    if outbox:
        np.testing.assert_array_equal(np.sum(outs, axis=0), ws[0] - w0)


@pytest.mark.parametrize("K", [2, 16])
def test_loops_finish_while_another_runs(conservation, K):
    """Worker 0 runs batch 1 until it is stopped; workers 1..K-1 run bounded batch-8 loops, which must all finish while
    worker 0's loop still runs (the workers really overlap: nothing they launch waits for the other loops).  Then the
    replicas and the master are bit-identical, and the total decrease is exactly what the master counted."""
    data, k = conservation
    w0 = np.full(data.dim, 1024.0)
    lr = 2.0 ** -6
    U = [0] + [500 + 100 * r for r in range(1, K)]
    batch = [1] + [8] * (K - 1)
    assigned = np.arange(data.n_rows, dtype=np.int32)
    ctxs = async_workers(data, 0.0, np.zeros(data.dim), K, w0)
    try:
        for r, c in enumerate(ctxs):   # sizes every worker's scratch before any loop runs (see above)
            c.start_async(None, assigned, batch[r], lr, concurrency=8, max_updates=8, seed=r)
            _wait_idle([c])
        for c in ctxs:
            c.set_weights(w0)
        ctxs[0].async_host_master(w0)
        for r, c in enumerate(ctxs):
            c.start_async(None, assigned, batch[r], lr, concurrency=8, max_updates=U[r], seed=200 + r)
        t0 = time.time()
        while any(c.async_running() for c in ctxs[1:]) and time.time() - t0 < 60:
            time.sleep(0.002)
        others_done = not any(c.async_running() for c in ctxs[1:])
        still_running = ctxs[0].async_running()
        ctxs[0].stop_async()
        _wait_idle(ctxs)
        ws = [c.get_weights() for c in ctxs]
        wm = ctxs[0].async_master_weights()
        count = ctxs[0].async_updates()
    finally:
        for c in ctxs:
            c.stop_async()
        _close(ctxs)
    assert others_done and still_running, (others_done, still_running)
    for r in range(K):
        np.testing.assert_array_equal(ws[r], ws[0], err_msg=f"replica {r}")
    np.testing.assert_array_equal(wm, ws[0])
    assert count > sum(U)
    assert (w0 - ws[0]).sum() == count * lr * k * 2.0 ** -4


# ---- C. the replica table at its edges --------------------------------------------------------------------------------

def test_sixteen_workers_leave_no_slot_for_an_outbox(edge_data):
    """Own replica, 15 peers and the master: an outbox would be an 18th target.  The launch is refused and nothing moves."""
    from distributed_sgd_b200.native import DsgdInvalid
    data, w0, d = edge_data
    ctxs = async_workers(data, 0.0, d, 16, w0, outbox=True)
    try:
        for r in (0, 9):
            with pytest.raises(DsgdInvalid, match="no replica slot left"):
                ctxs[r].async_replay(None, np.arange(4, dtype=np.int32), 1, LR)
        ws = [c.get_weights() for c in ctxs] + [ctxs[0].async_master_weights()]
        count = ctxs[0].async_updates()
    finally:
        _close(ctxs)
    for w in ws:
        np.testing.assert_array_equal(w, w0)
    assert count == 0


def test_async_world_above_sixteen_is_refused():
    """A 17th worker's replica would have no slot in the table, and the master would sit at peer_rank 17, where no worker
    can reach it: async worlds above 16 are refused.  Sync mode has no such table."""
    from distributed_sgd_b200.native import DsgdInvalid, NativeCtx
    for rank in (0, 16):
        with pytest.raises(DsgdInvalid, match="at most 16 workers"):
            NativeCtx(0, 64, 0.0, rank=rank, world=17, is_async=True)
    NativeCtx(0, 64, 0.0, rank=15, world=16, is_async=True).close()
    NativeCtx(0, 64, 0.0, rank=16, world=17).close()


def test_attach_refused_while_the_loop_runs(conservation):
    """The running loop copied its replica table at launch: an attach then would never receive a delta."""
    from distributed_sgd_b200.native import REPLICA_MASTER, DsgdState
    data, _ = conservation
    w0 = np.full(data.dim, 1024.0)
    a, b = ctxs = async_workers(data, 0.0, np.zeros(data.dim), 2, w0, master=False)
    try:
        b.async_host_master(w0)
        a.start_async(None, np.arange(data.n_rows, dtype=np.int32), 1, 2.0 ** -6, concurrency=1, max_updates=0, seed=1)
        try:
            with pytest.raises(DsgdState, match="running"):
                a.peer_attach(2, b, REPLICA_MASTER)
            with pytest.raises(DsgdState, match="running"):
                a.ipc_import(1, b.ipc_export())
        finally:
            a.stop_async()
        a.peer_attach(2, b, REPLICA_MASTER)                     # allowed once the loop has stopped
    finally:
        _close(ctxs)


def test_update_grad_stays_on_its_replica(edge_data):
    """SlaveImpl.updateGrad (core/Slave.scala:177-185) applies a colleague's delta to this worker's replica only: no peer
    and not the master (which counts nothing for it)."""
    data, w0, d = edge_data
    ctxs = async_workers(data, 0.0, d, 3, w0)
    try:
        ctxs[1].update_grad([5, 17, 4098], [0.25, -0.5, 2.0 ** -6])
        ws = [c.get_weights() for c in ctxs]
        wm = ctxs[0].async_master_weights()
        count = ctxs[2].async_updates()
    finally:
        _close(ctxs)
    expect = w0.copy()
    expect[[5, 17, 4098]] -= [0.25, -0.5, 2.0 ** -6]
    np.testing.assert_array_equal(ws[1], expect)
    for w in (ws[0], ws[2], wm):
        np.testing.assert_array_equal(w, w0)
    assert count == 0


# ---- D. across processes on one GPU -----------------------------------------------------------------------------------

def _ipc_worker(rank, K, batch, turns, idx, d, barrier, q_in, q_out):
    """Rank `rank` of K in its own process: exchanges CUDA IPC handles through the parent, then replays its turns of the
    schedule with a barrier between turns, and reports its replica, the master and the counter."""
    sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]
    ctx = None
    try:
        from distributed_sgd_b200.native import REPLICA_MASTER, REPLICA_SELF, NativeCtx
        from helpers import edge_rows
        data, w0 = edge_rows(21)
        ctx = NativeCtx(0, data.dim, 0.0, rank=rank, world=K, is_async=True)
        ctx.load_csr(data.row_ptr, data.col, data.val, data.label)
        ctx.set_dim_sparsity(d)
        ctx.set_weights(w0)
        if rank == 0:
            ctx.async_host_master(w0)
        q_out.put(("handle", rank, ctx.ipc_export(REPLICA_SELF), ctx.ipc_export(REPLICA_MASTER) if rank == 0 else b""))
        handles, master = q_in.get(timeout=TIMEOUT)
        for q, h in enumerate(handles):
            if q != rank:
                ctx.ipc_import(q, h)
        if rank != 0:
            ctx.ipc_import(K, master)
        pos = 0
        for k, n in turns:
            barrier.wait(timeout=TIMEOUT)
            if k == rank:
                ctx.async_replay(None, idx[pos:pos + n].reshape(-1), batch, LR)
            pos += n
        barrier.wait(timeout=TIMEOUT)
        q_out.put(("result", rank, ctx.get_weights(), ctx.async_master_weights(), ctx.async_updates()))
        barrier.wait(timeout=TIMEOUT)                      # every rank has read the replicas before any is freed
    except BaseException as e:  # noqa: BLE001 -- reported to the parent
        barrier.abort()
        q_out.put(("error", rank, repr(e)))
    finally:
        if ctx is not None:
            ctx.close()


def _run_procs(target, args_of, n, on_message):
    """Starts n spawned processes target(*args_of(i)), hands every message of the shared queue to on_message(msg, queues),
    and joins them; whatever still runs at the end is terminated."""
    ctxmp = mp.get_context("spawn")
    q_out = ctxmp.Queue()
    q_in = [ctxmp.Queue() for _ in range(n)]
    barrier = ctxmp.Barrier(n)
    procs = [ctxmp.Process(target=target, args=args_of(i, barrier, q_in[i], q_out)) for i in range(n)]
    try:
        for p in procs:
            p.start()
        while not on_message(q_out.get(timeout=TIMEOUT), q_in):
            pass
        for p in procs:
            p.join(timeout=TIMEOUT)
        assert all(p.exitcode == 0 for p in procs), [p.exitcode for p in procs]
    finally:
        for p in procs:
            if p.is_alive():
                p.terminate()
                p.join(timeout=10)


@pytest.mark.parametrize("batch", [1, 4])
@pytest.mark.parametrize("K", [2, 3])
def test_ipc_turns_match_oracle(edge_data, K, batch):
    """K processes on one GPU, every replica and the master mapped with dsgd_ipc_export / dsgd_ipc_import, replaying in
    turns: replicas, master and counter bit for bit as the oracle (lambda = 0)."""
    data, w0, d = edge_data
    n = _n_updates(K, batch)
    turns = schedule(K, n, seed=30 * K + batch)
    idx = batches(3000 * K + batch, data.n_rows, batch, n)
    handles, results = {}, {}

    def on_message(msg, q_in):
        if msg[0] == "error":
            raise AssertionError(f"rank {msg[1]}: {msg[2]}")
        if msg[0] == "handle":
            handles[msg[1]] = (msg[2], msg[3])
            if len(handles) == K:
                for q in q_in:
                    q.put(([handles[r][0] for r in range(K)], handles[0][1]))
            return False
        results[msg[1]] = msg[2:]
        return len(results) == K

    _run_procs(_ipc_worker, lambda r, barrier, q_in, q_out: (r, K, batch, turns, idx, d, barrier, q_in, q_out), K, on_message)
    w_ref = _oracle(data, 0.0, d).async_run(w0, idx.reshape(-1), batch, LR)
    assert np.count_nonzero(w_ref != w0) > 100
    for r in range(K):
        w, wm, count = results[r]
        np.testing.assert_array_equal(w, w_ref, err_msg=f"replica of rank {r}")
        np.testing.assert_array_equal(wm, w_ref, err_msg=f"master as rank {r} sees it")
        assert count == n, (r, count)


def _free_port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def _fit_worker(rank, port, barrier, q_in, q_out):
    """Rank `rank` of a two-worker MasterAsync.fit on device 0 (gloo for the host collectives)."""
    sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]
    slave = None
    try:
        import torch.distributed as dist
        from distributed_sgd_b200 import MasterAsync, Slave, SparseSVM
        from distributed_sgd_b200.utils import synthetic_rcv1
        dist.init_process_group("gloo", init_method=f"tcp://127.0.0.1:{port}", rank=rank, world_size=2)
        synth = synthetic_rcv1(n_rows=5000, seed=9)
        train, test = synth.split_at(4000)
        model = SparseSVM(1e-5)
        slave = Slave(rank, 0, train, model, is_async=True, world=2, device=0, test_data=test)
        master = MasterAsync(rank, train, test, model, 2, slave=slave)
        state = master.fit(np.zeros(synth.dim), max_epoch=2, batch_size=1, learning_rate=0.1,
                           stopping_criterion=lambda losses: False, check_every=2000, concurrency=8,
                           poll_seconds=0.001)
        acc = master.local_loss_accuracy(state.grad, test_data=True)[1]
        q_out.put(("result", rank, slave.ctx.get_weights(), slave.ctx.async_master_weights(), slave.ctx.async_updates(),
                   acc, master.history["ended_by"]))
        barrier.wait(timeout=TIMEOUT)                      # every rank has read the replicas before any is freed
        dist.destroy_process_group()
    except BaseException as e:  # noqa: BLE001 -- reported to the parent
        barrier.abort()
        q_out.put(("error", rank, repr(e)))
    finally:
        if slave is not None:
            slave.stop()


def test_master_async_fit_two_workers_one_gpu():
    """MasterAsync.fit with W = 2 in two processes on one GPU: handles exchanged by _attach_replicas over a gloo group,
    rank 0's counter polled while both loops run, ended by max_steps = n_train * max_epoch.  Each fresh process evaluates
    the master's weights for the first time while its loop runs: the kernels the library loads before the first async
    loop keep that evaluation from waiting for the loop.  The three replicas agree up to the order of the fp64 sums."""
    port = _free_port()
    results = {}

    def on_message(msg, q_in):
        if msg[0] == "error":
            raise AssertionError(f"rank {msg[1]}: {msg[2]}")
        results[msg[1]] = msg[2:]
        return len(results) == 2

    _run_procs(_fit_worker, lambda r, barrier, q_in, q_out: (r, port, barrier, q_in, q_out), 2, on_message)
    max_steps = 4000 * 2
    w0, wm0, count0, acc0, ended0 = results[0]
    w1, wm1, count1, acc1, ended1 = results[1]
    np.testing.assert_array_equal(wm0, wm1)                    # one master, seen by both ranks
    assert np.abs(w0 - wm0).max() <= 1e-12 and np.abs(w1 - wm0).max() <= 1e-12
    assert np.count_nonzero(wm0) > 0
    assert count0 == count1 >= max_steps
    assert ended0 == ended1 == "max_steps"
    assert acc0 == acc1 > 0.5
