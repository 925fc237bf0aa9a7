"""The L1 penalty of the sync steps on the device (dsgd_set_l1, dsgd_weights_l1, SparseSVM / SparseLogistic(l1=...)).

Every step soft-thresholds every column at tau = lr_t * lambda1 after its update; the checker is oracle/l1.py (the C
restatement, itself tested against the literal one in tests/test_oracle_l1.py).  Checked:

1. Dyadic rows, dyadic lambda, lambda1 and rates (every sum exact): weights and losses bit for bit on every
   path -- the persistent kernel's L1 form at batches 1 to 32 G and grid limits 1, 2 and S, the per-step path at 32 G + 1
   (the launch counts show which path ran), two virtual workers, the logistic model on rows whose sigma is 0 or 1,
   averaging with a rate table that has zero entries on both paths, one call of 20 steps against four of 5, calls that
   alternate the two paths, and turning the penalty on after steps without it.
2. RCV1-shaped fp32 rows over 20 steps: max |dw| <= 1e-11 max |w|, supports equal but for columns at the threshold.
3. The number of zero weights grows with lambda1; set_l1(0) gives the bits of a context that never set it.
4. weights_l1: exact against math.fsum on dyadic weights, and the same bits for resident and host weights.
5. Refusals: lambda1 < 0 or not finite, an async ctx, ranks wired with the peer exchange only.
6. MasterSync.fit with l1 > 0 against a replay of the checker; two GPUs over NCCL (skipped with fewer).
"""
import math
import os
import socket
import sys

import numpy as np
import pytest

from helpers import data_from_csr, make_pair

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LAM, LAM1, LR = 2.0 ** -8, 2.0 ** -7, 2.0 ** -3
STEPS = 20


@pytest.fixture(scope="module")
def S():
    from distributed_sgd_b200.native import NativeCtx
    ctx = NativeCtx(0, 8, 0.0)
    s = int(ctx.info()["sm_count"])
    ctx.close()
    return s


def _dyadic(dim, n_rows, seed):
    """Rows of 1 to 40 distinct columns with values k / 16, weights k / 8 on 40 % of the columns, and dimSparsity 0, so that
    c = 0 while lambda > 0 still enters every loss: every weight stays a multiple of lr * lambda1 / 2^k below 2^12 and every
    sum is exact, so the trajectories are the checker's bit for bit.  (A non-zero c would put ever finer bits into the
    weights at every step, and sums of those round in the order of their terms.)"""
    rng = np.random.default_rng(seed)
    nnz = rng.integers(1, 41, size=n_rows)
    rp = np.concatenate([[0], np.cumsum(nnz)])
    col = np.concatenate([rng.choice(dim, size=k, replace=False) for k in nnz])
    val = rng.integers(1, 33, size=int(rp[-1])) / 16.0 * rng.choice([-1, 1], size=int(rp[-1]))
    lab = rng.choice([-1, 1], size=n_rows)
    w0 = rng.integers(-32, 33, size=dim) / 8.0 * (rng.random(dim) < 0.4)
    d = np.zeros(dim)
    return data_from_csr(rp, col, val, lab, dim), w0, d


def _pair(data, d, lam=LAM, logistic=False):
    from distributed_sgd_b200.native import NativeCtx
    from oracle.logistic import LogisticOracle
    from oracle.oracle import Oracle
    ctx = NativeCtx(0, data.dim, lam, logistic=logistic)
    ctx.load_csr(data.row_ptr, data.col, data.val, data.label)
    ctx.set_dim_sparsity(d)
    orc = (LogisticOracle if logistic else Oracle)(data.row_ptr, data.col, data.val, data.label, data.dim, lam)
    orc.set_dim_sparsity(d)
    return ctx, orc


def _ids(rng, n_rows, steps, batch):
    return np.stack([rng.choice(n_rows, size=batch, replace=False) for _ in range(steps)]).astype(np.int32)


def _call(ctx, ids, lr):
    ids = np.ascontiguousarray(ids, np.int32)
    if np.ndim(lr):
        return ctx.sync_steps_lr(ids.reshape(-1), ids.shape[1], np.asarray(lr, np.float64))
    return ctx.sync_steps(ids.reshape(-1), ids.shape[1], ids.shape[0], float(lr))


def _same(a, b, what):
    a, b = np.asarray(a), np.asarray(b)
    diff = np.flatnonzero(a != b)
    assert diff.size == 0, f"{what}: {diff.size} differ, first at {diff[0]}: {a[diff[0]]!r} against {b[diff[0]]!r}"


@pytest.fixture(scope="module")
def dy(S):
    data, w0, d = _dyadic(2 * 6 * 32 * S + 1, 40 * S + 400, 1)
    ctx, orc = _pair(data, d)
    ctx.set_l1(LAM1)
    yield data, w0, ctx, orc
    ctx.close()


# ---- 1. dyadic rows, bit for bit ---------------------------------------------------------------------------------------

@pytest.mark.parametrize("grid", ["1", "2", "S"])
@pytest.mark.parametrize("batch", ["1", "64", "32G", "32G+1"])
def test_dyadic_bit_for_bit(dy, S, grid, batch):
    from oracle import l1 as L1
    data, w0, ctx, orc = dy
    G = {"1": 1, "2": 2, "S": S}[grid]
    B = {"1": 1, "64": 64, "32G": 32 * G, "32G+1": 32 * G + 1}[batch]
    ids = _ids(np.random.default_rng(G * 1000 + B), data.n_rows, STEPS, B)
    ctx.set_grid_limit(G)
    try:
        ctx.set_weights(w0)
        n0 = ctx.launch_count()
        losses = _call(ctx, ids, LR)
        launches = ctx.launch_count() - n0
    finally:
        ctx.set_grid_limit(0)
    # the persistent kernel (k_rec_init + one launch) up to 32 rows per CTA, else k_rows + k_update<..., kL1> per step
    assert launches == (2 if B <= 32 * G else 2 * STEPS), launches
    w_ref, l_ref = L1.sync_steps(orc, w0, ids.reshape(-1), [B], np.full(STEPS, LR), LAM1)
    _same(ctx.get_weights(), w_ref, "weights")
    _same(losses, l_ref, "losses")
    assert ctx.weights_l1() == (L1.l1_norm(w_ref), int(np.count_nonzero(w_ref)))


def test_dyadic_virtual_workers(dy):
    from oracle import l1 as L1
    data, w0, _, orc = dy
    counts = [40, 24]
    ids = _ids(np.random.default_rng(7), data.n_rows, STEPS, sum(counts))
    ctx, _ = _pair(data, orc.d)                                   # its own context: it keeps the worker split
    try:
        ctx.set_l1(LAM1)
        ctx.set_weights(w0)
        ctx.set_workers(counts, len(counts))
        losses = _call(ctx, ids, LR)
        w = ctx.get_weights()
    finally:
        ctx.close()
    w_ref, l_ref = L1.sync_steps(orc, w0, ids.reshape(-1), counts, np.full(STEPS, LR), LAM1)
    _same(w, w_ref, "weights")
    _same(losses, l_ref, "losses")


def test_dyadic_averaging_with_a_table_with_zero_entries(dy, S):
    from oracle import l1 as L1
    data, w0, ctx, orc = dy
    lrs = 2.0 ** -(2 + np.arange(STEPS) % 3)
    lrs[1::4] = 0.0
    A, w_ref = np.zeros(data.dim), w0
    ctx.set_weights(w0)
    ctx.average_begin()
    try:
        for B in (64, 32 * S + 1):                                # a batch of each side of 32 G
            ids = _ids(np.random.default_rng(B), data.n_rows, STEPS, B)
            losses = _call(ctx, ids, lrs)
            w_ref, l_ref = L1.sync_steps(orc, w_ref, ids.reshape(-1), [B], lrs, LAM1, avg_sum=A)
            _same(losses, l_ref, f"losses at batch {B}")
        avg, n = ctx.average_weights()
    finally:
        ctx.average_end()
    _same(ctx.get_weights(), w_ref, "weights")
    assert n == 2 * STEPS
    v = A / n
    _same(avg, np.where(np.abs(v) > 1e-20, v, 0.0), "average")


def test_one_call_equals_four(dy):
    data, w0, ctx, orc = dy
    ids = _ids(np.random.default_rng(3), data.n_rows, STEPS, 64)
    ctx.set_weights(w0)
    l_one = _call(ctx, ids, LR)
    w_one = ctx.get_weights()
    ctx.set_weights(w0)
    l_four = np.concatenate([_call(ctx, ids[5 * k:5 * (k + 1)], LR) for k in range(4)])
    _same(ctx.get_weights(), w_one, "weights")
    _same(l_four, l_one, "losses")


def test_alternating_persistent_and_fallback_batches(dy, S):
    from oracle import l1 as L1
    data, w0, ctx, orc = dy
    rng = np.random.default_rng(11)
    w_ref = w0
    ctx.set_weights(w0)
    for k in range(6):
        B = 64 if k % 2 == 0 else 32 * S + 1
        ids = _ids(rng, data.n_rows, 4, B)
        n0 = ctx.launch_count()
        losses = _call(ctx, ids, LR)
        assert ctx.launch_count() - n0 == (2 if B == 64 else 8)          # persistent, per-step, persistent, ...
        w_ref, l_ref = L1.sync_steps(orc, w_ref, ids.reshape(-1), [B], np.full(4, LR), LAM1)
        _same(losses, l_ref, f"losses of call {k}")
    _same(ctx.get_weights(), w_ref, "weights")


def test_turning_the_penalty_on_after_steps_without_it(dy, S):
    """Steps without the penalty (the persistent kernel, which keeps no ||w||_1), then set_l1: the per-step path's first
    loss needs ||w||_1 of the weights those steps left."""
    from oracle import l1 as L1
    data, w0, _, orc = dy
    ctx, _ = _pair(data, orc.d)
    try:
        ids = _ids(np.random.default_rng(5), data.n_rows, 8, 64)
        ctx.set_weights(w0)
        _call(ctx, ids, LR)
        w_mid, _ = L1.sync_steps(orc, w0, ids.reshape(-1), [64], np.full(8, LR), 0.0)
        _same(ctx.get_weights(), w_mid, "weights without the penalty")
        ctx.set_l1(LAM1)
        ids = _ids(np.random.default_rng(6), data.n_rows, 4, 32 * S + 1)
        losses = _call(ctx, ids, LR)
        w_ref, l_ref = L1.sync_steps(orc, w_mid, ids.reshape(-1), [32 * S + 1], np.full(4, LR), LAM1)
        _same(losses, l_ref, "losses")
        _same(ctx.get_weights(), w_ref, "weights")
    finally:
        ctx.close()


def test_dyadic_logistic_bit_for_bit():
    """Rows whose sigma is 0 or 1 (test_gpu_logistic_exact.py), lambda = 0: every weight stays a multiple of tau = 2^-10.
    (With lambda > 0 the bias columns at +-2048 pick up the bits of c, their squares no longer fit a double, and the order
    of the ||w||^2 sum shows in the last bit of the loss.)"""
    from oracle import l1 as L1
    from test_gpu_logistic_exact import LR_D, _dyadic_data
    data, w0, d = _dyadic_data(4000, 500, 4, with_half=False)
    ctx, orc = _pair(data, d, lam=0.0, logistic=True)
    try:
        ctx.set_l1(2.0 ** -4)
        for counts in ([64], [32, 32], [1]):
            tot = sum(counts)
            ids = _ids(np.random.default_rng(tot + len(counts)), data.n_rows, STEPS, tot)
            ctx.set_weights(w0)
            ctx.set_workers(counts, len(counts))
            try:
                losses = _call(ctx, ids, LR_D)
            finally:
                ctx.set_workers([], 0)
            w_ref, l_ref = L1.sync_steps(orc, w0, ids.reshape(-1), counts, np.full(STEPS, LR_D), 2.0 ** -4, logistic=True)
            z = data.label * np.array([float(np.dot(data.val[a:b].astype(np.float64), w_ref[data.col[a:b]]))
                                       for a, b in zip(data.row_ptr[:-1], data.row_ptr[1:])])
            assert (np.abs(z) >= 800.0).all()                   # the run stayed where sigma is 0 or 1
            _same(ctx.get_weights(), w_ref, f"weights {counts}")
            _same(losses, l_ref, f"losses {counts}")
    finally:
        ctx.close()


# ---- 2. RCV1-shaped fp32 rows ------------------------------------------------------------------------------------------

@pytest.fixture(scope="module")
def rcv1():
    from distributed_sgd_b200.utils import synthetic_rcv1
    data = synthetic_rcv1(n_rows=6000, seed=21)
    ctx, orc = make_pair(data, 1e-5)
    yield data, ctx, orc
    ctx.close()


@pytest.mark.parametrize("logistic", [False, True])
@pytest.mark.parametrize("batch", [64, 1024, 5000])
def test_rcv1_shaped_within_tolerance(rcv1, logistic, batch):
    from oracle import l1 as L1
    from oracle.logistic import LogisticOracle
    data, ctx0, orc0 = rcv1
    lam1 = 2e-4
    if logistic:
        ctx, orc = _pair(data, orc0.d, lam=1e-5, logistic=True)
    else:
        ctx, orc = ctx0, orc0
    try:
        ctx.set_l1(lam1)
        ids = _ids(np.random.default_rng(batch), data.n_rows, STEPS, batch)
        ctx.set_weights(np.zeros(data.dim))
        losses = _call(ctx, ids, 0.5)
        w = ctx.get_weights()
        w_ref, l_ref = L1.sync_steps(orc, np.zeros(data.dim), ids.reshape(-1), [batch], np.full(STEPS, 0.5), lam1,
                                     logistic=logistic)
        scale = np.abs(w_ref).max()
        assert scale > 0 and np.abs(w - w_ref).max() <= 1e-11 * scale
        off = np.flatnonzero((w == 0) != (w_ref == 0))
        # a support can differ only where |u| lies within rounding of tau: the non-zero side is then tiny
        assert off.size <= max(2, data.dim // 10000), off.size
        assert (np.maximum(np.abs(w[off]), np.abs(w_ref[off])) <= 1e-11 * scale).all()
        np.testing.assert_allclose(losses, l_ref, rtol=1e-11)
        assert (w == 0).sum() > 0
    finally:
        ctx.set_l1(0.0)
        if logistic:
            ctx.close()


# ---- 3. sparsity and switching off ---------------------------------------------------------------------------------------

def test_zero_weights_grow_with_lambda1(rcv1):
    data, ctx, orc = rcv1
    ids = _ids(np.random.default_rng(2), data.n_rows, 40, 256)
    nnz = []
    try:
        for lam1 in (0.0, 1e-5, 1e-4, 1e-3):
            ctx.set_l1(lam1)
            ctx.set_weights(np.zeros(data.dim))
            _call(ctx, ids, 0.5)
            nnz.append(ctx.weights_l1()[1])
    finally:
        ctx.set_l1(0.0)
    assert nnz[0] > nnz[1] > nnz[2] > nnz[3], nnz


def test_set_l1_zero_is_bit_identical_to_never_setting_it(rcv1, S):
    from distributed_sgd_b200.native import NativeCtx
    data, ctx, orc = rcv1
    fresh = NativeCtx(0, data.dim, 1e-5)
    try:
        fresh.load_csr(data.row_ptr, data.col, data.val, data.label)
        fresh.set_dim_sparsity(orc.d)
        ctx.set_l1(1e-4)
        ctx.set_l1(0.0)
        assert ctx.info()["lambda1"] == 0.0
        for B in (64, 32 * S + 1):
            ids = _ids(np.random.default_rng(B), data.n_rows, STEPS, B)
            out = []
            for c in (ctx, fresh):
                c.set_weights(np.zeros(data.dim))
                n0 = c.launch_count()
                out.append((_call(c, ids, 0.5), c.get_weights(), c.launch_count() - n0))
            _same(out[0][0], out[1][0], "losses")
            _same(out[0][1], out[1][1], "weights")
            assert out[0][2] == out[1][2]                        # the same kernels: the persistent one at batch 64
    finally:
        fresh.close()


# ---- 4. weights_l1 ------------------------------------------------------------------------------------------------------

def test_weights_l1_exact_and_resident_equals_host(rcv1):
    data, ctx, orc = rcv1
    rng = np.random.default_rng(4)
    # multiples of 2^-20 below 2^10: the sum needs fewer than 53 bits, so fsum and the device both give it exactly
    w = rng.integers(-2 ** 10, 2 ** 10, size=data.dim) * 2.0 ** -rng.integers(0, 21, size=data.dim) * (rng.random(data.dim) < 0.5)
    assert ctx.weights_l1(w) == (math.fsum(np.abs(w)), int(np.count_nonzero(w)))
    ctx.set_weights(w)
    assert ctx.weights_l1() == ctx.weights_l1(w)
    w = rng.standard_normal(data.dim) * 10.0 ** rng.integers(-15, 3, size=data.dim)
    ctx.set_weights(w)
    l1, nnz = ctx.weights_l1()
    assert (l1, nnz) == ctx.weights_l1(w) and nnz == data.dim
    assert abs(l1 - math.fsum(np.abs(w))) <= 2.0 ** -52 * l1


# ---- 5. refusals -----------------------------------------------------------------------------------------------------------

def test_refusals(rcv1):
    from distributed_sgd_b200.native import DsgdInvalid, DsgdState, NativeCtx
    data, ctx, orc = rcv1
    for bad in (-1e-9, float("inf"), float("nan")):
        with pytest.raises(DsgdInvalid):
            ctx.set_l1(bad)
    assert ctx.info()["lambda1"] == 0.0
    a = NativeCtx(0, 64, 0.1, is_async=True)
    try:
        with pytest.raises(DsgdState):
            a.set_l1(1e-3)
        with pytest.raises(DsgdState):
            a.weights_l1()
    finally:
        a.close()


def test_exchange_only_ranks_refuse_before_launching():
    """Two ranks on one GPU wired with the peer exchange only: without L1 the fused kernel could take the step; with L1
    the call fails before anything is launched (one thread: nothing waits for the other rank)."""
    from distributed_sgd_b200.native import DsgdState
    from distributed_sgd_b200.utils import synthetic_rcv1
    data = synthetic_rcv1(n_rows=2000, seed=5)
    ctxs = [make_pair(data, 1e-5, rank=r, world=2)[0] for r in range(2)]
    try:
        ctxs[0].xchg_attach(1, ctxs[1])
        ctxs[1].xchg_attach(0, ctxs[0])
        ctxs[0].set_l1(1e-4)
        n0 = ctxs[0].launch_count()
        with pytest.raises(DsgdState, match="L1"):
            ctxs[0].sync_steps(np.arange(32, dtype=np.int32), 32, 1, 0.5)
        assert ctxs[0].launch_count() == n0
    finally:
        for c in ctxs:
            c.close()


# ---- 6. MasterSync.fit and two GPUs ---------------------------------------------------------------------------------------

def test_master_sync_fit_matches_checker_replay():
    from distributed_sgd_b200 import EarlyStopping, Master, Slave, SparseSVM
    from distributed_sgd_b200.core import Group
    from distributed_sgd_b200.core.master import EpochDraw
    from distributed_sgd_b200.ml import SplitStrategy
    from distributed_sgd_b200.utils import synthetic_rcv1
    from oracle import l1 as L1
    from oracle.oracle import Oracle
    data = synthetic_rcv1(n_rows=6000, seed=8)
    train, test = data.split_at(4800)
    lam, lam1 = 1e-5, 1e-4
    model = SparseSVM(lam, None, lam1)
    slave = Slave(0, 0, train, model, False, device=0, test_data=test)
    try:
        m = Master.create(0, train, test, model, False, 1, slave=slave, group=Group(), seed=5)
        batch, lr, epochs = 64, 0.5, 2
        w0 = np.zeros(data.dim)
        state = m.fit(w0, epochs, batch, lr, EarlyStopping.no_improvement(patience=5, min_delta=0.0))
        orc = Oracle(data.row_ptr, data.col, data.val, data.label, data.dim, lam)
        orc.set_dim_sparsity(model.dim_sparsity)
        w, losses, nnz = w0, [], []
        for e in range(epochs):
            draw = EpochDraw.draw(5, e, SplitStrategy.vanilla(4800, 1), batch)
            w, _ = L1.sync_steps(orc, w, draw.ids.reshape(-1), [batch], np.full(draw.ids.shape[0], lr), lam1)
            loss, _ = orc.loss_acc(w, begin=0, n=4800)
            losses.append(loss + lam1 * math.fsum(np.abs(w)))
            nnz.append(int(np.count_nonzero(w)))
        assert np.abs(state.grad - w).max() <= 1e-11 * np.abs(w).max()
        np.testing.assert_allclose(m.history["losses"], losses, rtol=1e-11)
        assert m.history["nnz"] == nnz and nnz[-1] < data.dim
    finally:
        slave.stop()


def _free_port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def _nccl_worker(rank, world, port, q):
    sys.path.insert(0, ROOT)
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    import torch
    import torch.distributed as dist
    from distributed_sgd_b200.core import Group
    from distributed_sgd_b200.native import NativeCtx
    from oracle import l1 as L1
    from oracle.oracle import Oracle

    torch.cuda.set_device(rank)
    dist.init_process_group("gloo", init_method=f"tcp://127.0.0.1:{port}", rank=rank, world_size=world)
    group = Group()
    data, w0, d = _dyadic(3000, 4000, 6)
    batch, steps = 48, STEPS
    ctx = NativeCtx(rank, data.dim, LAM, rank=rank, world=world)
    ctx.load_csr(data.row_ptr, data.col, data.val, data.label)
    ctx.set_dim_sparsity(d)
    ctx.set_l1(LAM1)
    uid = NativeCtx.comm_unique_id() if rank == 0 else b""
    ctx.comm_init(group.broadcast_bytes(uid, 0))
    rng = np.random.default_rng(9)
    per = data.n_rows // world
    idx = np.stack([np.concatenate([k * per + rng.choice(per, size=batch, replace=False) for k in range(world)])
                    for _ in range(steps)]).astype(np.int32)
    mine = idx.reshape(steps, world, batch)[:, rank, :]
    ctx.set_weights(w0)
    losses = ctx.sync_steps(mine.reshape(-1), batch, steps, LR)
    w = ctx.get_weights()
    orc = Oracle(data.row_ptr, data.col, data.val, data.label, data.dim, LAM)
    orc.set_dim_sparsity(d)
    w_ref, l_ref = L1.sync_steps(orc, w0, idx.reshape(-1), [batch] * world, np.full(steps, LR), LAM1)
    q.put((rank, bool(np.array_equal(losses, l_ref)), bool(np.array_equal(w, w_ref))))
    ctx.close()
    dist.destroy_process_group()


def test_two_gpu_nccl_dyadic_bit_for_bit():
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    import torch.multiprocessing as mp
    ctxmp = mp.get_context("spawn")
    q = ctxmp.Queue()
    port = _free_port()
    procs = [ctxmp.Process(target=_nccl_worker, args=(r, 2, port, q)) for r in range(2)]
    for p in procs:
        p.start()
    res = [q.get(timeout=300) for _ in procs]
    for p in procs:
        p.join(timeout=60)
    for rank, same_losses, same_w in res:
        assert same_losses, f"rank {rank}: step losses differ from the checker"
        assert same_w, f"rank {rank}: weights differ from the checker"
