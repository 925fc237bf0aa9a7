"""SparseLogistic on the GPU against the fp64 oracle: gradient requests of every size, evaluation passes (range, device-drawn
sample, list), the per-step sync path (one worker, virtual workers, two GPUs over NCCL), MasterSync.fit, and the refusals.

Tolerances: predictions, correct counts and gradient supports are exact.  Logistic summands are not fp32 values, so batch
sums are not exact and a relative error means nothing for entries that cancel: gradients are checked per entry against
1e-12 * (sum_i |sigma_i x_ij| + |c|).  Losses: rtol 1e-12, the oracle's sum taken with math.fsum for passes of 1e4 rows or
more.  Trajectories: max |dw| <= 1e-11 * max |w|."""
import math
import os
import socket
import sys

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LAM = 1e-5


@pytest.fixture(scope="module")
def setup():
    from distributed_sgd_b200.native import NativeCtx
    from distributed_sgd_b200.utils import synthetic_rcv1
    from oracle.logistic import LogisticOracle
    data = synthetic_rcv1(n_rows=12000, seed=21)
    n_train = 10000
    ctx = NativeCtx(0, data.dim, LAM, logistic=True)
    ctx.load_csr(data.row_ptr, data.col, data.val, data.label)
    d = ctx.compute_dim_sparsity(n_train)
    orc = LogisticOracle(data.row_ptr, data.col, data.val, data.label, data.dim, LAM)
    orc.set_dim_sparsity(d)
    yield data, n_train, ctx, orc
    ctx.close()


def _weights(dim, seed, scale=0.5):
    rng = np.random.default_rng(seed)
    return np.where(rng.random(dim) < 0.3, scale * rng.standard_normal(dim), 0.0)


def _abs_bound(data, w, idx, c):
    """sum_i |sigma_i x_ij| + |c| per column (the scale of each gradient entry's rounding)."""
    b = np.zeros(data.dim)
    for r in idx:
        lo, hi = data.row_ptr[r], data.row_ptr[r + 1]
        cols, vals = data.col[lo:hi], data.val[lo:hi].astype(np.float64)
        z = float(data.label[r]) * float(np.dot(vals, w[cols]))
        s = 1.0 / (1.0 + math.exp(-z)) if z >= 0 else math.exp(z) / (1.0 + math.exp(z))
        b[cols] += np.abs(vals) * s
    return b + abs(c)


def _check_grad(g, g_ref, bound):
    assert ((g == 0) == (g_ref == 0)).all(), "gradient support differs"
    assert (np.abs(g - g_ref) <= 1e-12 * bound).all(), float(np.max(np.abs(g - g_ref) / np.maximum(bound, 1e-300)))


def test_info_reports_the_model(setup):
    assert setup[2].info()["model"] == "logistic"


@pytest.mark.parametrize("n", [1, 7, 256, 2047, 2048, 5000])
@pytest.mark.parametrize("resident", [False, True])
def test_gradient_and_loss(setup, n, resident):
    data, n_train, ctx, orc = setup
    w = _weights(data.dim, n)
    idx = np.random.default_rng(n).choice(n_train, size=n, replace=False).astype(np.int32)
    if resident:
        ctx.set_weights(w)
        g, loss = ctx.gradient(idx, None, want_loss=True)
    else:
        g, loss = ctx.gradient(idx, w, want_loss=True)
    g_ref, c = orc.gradient(w, idx)
    _check_grad(g, g_ref, _abs_bound(data, w, idx, c))
    loss_ref = LAM * float(np.dot(w, w)) + math.fsum(orc.sample_losses(w, idx)) / n
    assert abs(loss - loss_ref) <= 1e-12 * loss_ref


def test_zero_weights_known_answers(setup):
    data, n_train, ctx, orc = setup
    w = np.zeros(data.dim)
    for r in (0, 17, 4242):   # one row: sigma = 1/2 exactly, loss = log 2 exactly, gradient = y * x / 2 exactly
        g, loss = ctx.gradient([r], w, want_loss=True)
        lo, hi = data.row_ptr[r], data.row_ptr[r + 1]
        ref = np.zeros(data.dim)
        ref[data.col[lo:hi]] = 0.5 * float(data.label[r]) * data.val[lo:hi].astype(np.float64)
        assert np.array_equal(g, ref)
        assert abs(loss - math.log(2.0)) <= 2.3e-16 * math.log(2.0)   # log1p(1) on the device: last ulp at most
    s, correct, n2 = ctx.eval_sums(0, n_train, w)
    assert correct == 0 and n2 == 0.0 and abs(s - n_train * math.log(2.0)) <= 1e-15 * s
    loss, acc = ctx.eval(0, n_train, w)
    assert acc == 0.0 and abs(loss - math.log(2.0)) <= 1e-15


def _tiny_ctx(rows, dim=8):
    """One column per row: row r holds (col r % dim, val) with label y; returns (ctx, oracle)."""
    from distributed_sgd_b200.native import NativeCtx
    from oracle.logistic import LogisticOracle
    n = len(rows)
    rp = np.arange(n + 1, dtype=np.int64)
    col = np.array([r % dim for r in range(n)], dtype=np.int32)
    val = np.array([v for v, _ in rows], dtype=np.float32)
    lab = np.array([y for _, y in rows], dtype=np.int8)
    ctx = NativeCtx(0, dim, LAM, logistic=True)
    ctx.load_csr(rp, col, val, lab)
    ctx.set_dim_sparsity(np.zeros(dim))
    orc = LogisticOracle(rp, col, val, lab, dim, LAM)
    return ctx, orc


@pytest.mark.parametrize("z", [700.0, -700.0, 800.0, -800.0, 1e4, -1e4])
def test_extreme_margins(z):
    ctx, orc = _tiny_ctx([(1.0, 1), (1.0, -1)], dim=2)
    try:
        w = np.array([z, -z])            # both rows at margin z
        g, loss = ctx.gradient([0, 1], w, want_loss=True)
        g_ref, _ = orc.gradient(w, [0, 1])
        assert np.isfinite(g).all() and np.isfinite(loss)
        assert np.array_equal(g == 0, g_ref == 0)
        np.testing.assert_allclose(g, g_ref, rtol=1e-12, atol=0)
        loss_ref = orc.loss_acc(w, idx=[0, 1])[0]
        assert abs(loss - loss_ref) <= 1e-12 * loss_ref
    finally:
        ctx.close()


def test_product_filter_edges():
    """sigma(z) * x crosses 1e-20 near z = -46: products on both sides, each >= 1e-9 (relative) from the threshold."""
    zs = [-45.0, -45.9, -46.0, -46.05, -46.2, -47.0]
    ctx, orc = _tiny_ctx([(1.0, 1)] * len(zs), dim=len(zs))
    try:
        w = np.array(zs)
        for r, z in enumerate(zs):
            prod = math.exp(z) / (1.0 + math.exp(z))
            assert abs(prod - 1e-20) >= 1e-9 * 1e-20
        g, _ = ctx.gradient(list(range(len(zs))), w, want_loss=True)
        g_ref, _ = orc.gradient(w, list(range(len(zs))))
        assert np.array_equal(g == 0, g_ref == 0) and (g != 0).any() and (g == 0).any()
        np.testing.assert_allclose(g, g_ref, rtol=1e-12, atol=0)
    finally:
        ctx.close()


def test_regularize_threshold_of_c():
    """c = 2 lambda (w . d) at exactly 1e-20 is not added; one ulp above it is.  The row's gradient entry sigma(-45.9) * 1
    ~ 1.2e-20 is of the same size, so whether c was added shows in the result."""
    from distributed_sgd_b200.native import NativeCtx
    from oracle.logistic import LogisticOracle
    rp = np.array([0, 1], dtype=np.int64)
    col, val, lab = np.array([0], np.int32), np.array([1.0], np.float32), np.array([1], np.int8)
    d = np.array([0.0, 0.0, 1.0, 0.0])
    p = 1e-10
    got = []
    for target in (1e-20, float(np.nextafter(1e-20, 1.0))):
        lam = target / (2.0 * p)
        for _ in range(8):                        # the lambda whose c = lambda * 2 * p rounds to the target
            if lam * 2.0 * p == target:
                break
            lam = float(np.nextafter(lam, np.inf if lam * 2.0 * p < target else 0.0))
        assert lam * 2.0 * p == target
        w = np.array([-45.9, 0.0, p, 0.0])
        ctx = NativeCtx(0, 4, lam, logistic=True)
        try:
            ctx.load_csr(rp, col, val, lab)
            ctx.set_dim_sparsity(d)
            orc = LogisticOracle(rp, col, val, lab, 4, lam)
            orc.set_dim_sparsity(d)
            g = ctx.gradient([0], w)
            g_ref, c_ref = orc.gradient(w, [0])
            assert c_ref == target
            assert np.array_equal(g == 0, g_ref == 0)
            np.testing.assert_allclose(g, g_ref, rtol=1e-14, atol=0)
            got.append(g[0])
        finally:
            ctx.close()
    assert got[1] > 1.5 * got[0]                  # c was added above the threshold only


def test_eval_and_sums(setup):
    data, n_train, ctx, orc = setup
    w = _weights(data.dim, 99)
    n = data.n_rows - n_train
    loss, acc = ctx.eval(n_train, data.n_rows, w)
    losses = orc.sample_losses(w, begin=n_train, n=n)
    ref_acc = orc.loss_acc(w, begin=n_train, n=n)[1]
    assert acc == ref_acc
    assert abs(loss - (LAM * float(np.dot(w, w)) + math.fsum(losses) / n)) <= 1e-12 * loss
    s, correct, n2 = ctx.eval_sums(0, n_train, w)
    s_ref = math.fsum(orc.sample_losses(w, begin=0, n=n_train))
    assert abs(s - s_ref) <= 1e-12 * s_ref and abs(n2 - float(np.dot(w, w))) <= 1e-14 * n2
    assert correct / n_train == orc.loss_acc(w, begin=0, n=n_train)[1]
    # device-drawn sample, split over two position shards that add up to the whole
    from distributed_sgd_b200.core.master import sample_shard
    from distributed_sgd_b200.native import host_lib
    k, key = 3001, 0x1234ABCD
    whole = ctx.eval_sampled_sums(0, n_train, key, 0, k, w)
    parts = [ctx.eval_sampled_sums(0, n_train, key, *sample_shard(k, 2, r), w) for r in range(2)]
    assert parts[0][1] + parts[1][1] == whole[1]
    assert abs(parts[0][0] + parts[1][0] - whole[0]) <= 1e-13 * whole[0]
    # the host reproduces the device draw (dsgd_feistel_pos, the same source): the list form of the same ids gives the same
    # bits, and the oracle the same numbers
    ids = np.fromiter((host_lib().dsgd_feistel_pos(p, n_train, key) for p in range(k)), dtype=np.int64, count=k)
    lst = ctx.eval_samples_sums(ids.astype(np.int32), w)
    assert lst[0] == whole[0] and lst[1] == whole[1]
    assert abs(whole[0] - math.fsum(orc.sample_losses(w, idx=ids))) <= 1e-12 * whole[0]
    assert whole[1] == round(orc.loss_acc(w, idx=ids)[1] * k)
    # a list with repeats: every occurrence counts
    rep = np.array([5, 5, 9, 5, 123, 9], dtype=np.int32)
    s, correct, _ = ctx.eval_samples_sums(rep, w)
    s_ref = math.fsum(orc.sample_losses(w, idx=rep))
    assert abs(s - s_ref) <= 1e-12 * s_ref
    assert correct == round(orc.loss_acc(w, idx=rep)[1] * len(rep))


def test_loss_sum_does_not_depend_on_row_order(setup):
    data, n_train, ctx, orc = setup
    w = _weights(data.dim, 7)
    s_range = ctx.eval_sums(0, n_train, w)
    ids = np.arange(n_train, dtype=np.int32)
    s_rev = ctx.eval_samples_sums(ids[::-1].copy(), w)
    s_shuf = ctx.eval_samples_sums(np.random.default_rng(3).permutation(ids), w)
    assert s_range[0] == s_rev[0] == s_shuf[0] and s_range[1] == s_rev[1] == s_shuf[1]


def test_counts_calls_refused(setup):
    from distributed_sgd_b200.native import DsgdState
    data, n_train, ctx, _ = setup
    with pytest.raises(DsgdState):
        ctx.eval_counts(0, 100)
    with pytest.raises(DsgdState):
        ctx.eval_sampled_counts(0, 100, 1, 0, 10)
    with pytest.raises(DsgdState):
        ctx.eval_samples_counts([1, 2, 3])


def _check_traj(w, w_ref, losses, losses_ref):
    np.testing.assert_allclose(losses, losses_ref, rtol=1e-12, atol=0)
    assert np.abs(w - w_ref).max() <= 1e-11 * np.abs(w_ref).max()


def _sm_count():
    from distributed_sgd_b200.native import NativeCtx
    with NativeCtx(0, 16, 0.1) as c:
        return int(c.info()["sm_count"])


@pytest.mark.parametrize("batch", [1, 64, 256, 1024, "33S"])
def test_sync_steps_one_worker(setup, batch):
    data, n_train, ctx, orc = setup
    if batch == "33S":
        batch = 33 * _sm_count()
    steps, lr = 50, 0.5
    rng = np.random.default_rng(batch)
    idx = np.concatenate([rng.choice(n_train, size=batch, replace=False) for _ in range(steps)]).astype(np.int32)
    w0 = _weights(data.dim, 1, scale=0.05)
    ctx.set_weights(w0)
    ctx.set_workers([batch], 1)
    n0 = ctx.launch_count()
    h = steps // 2
    l1 = ctx.sync_steps(idx[:h * batch], batch, h, lr)
    assert ctx.launch_count() - n0 == 2 * h          # row kernel + k_update per step: never the persistent kernel
    l2 = ctx.sync_steps(idx[h * batch:], batch, steps - h, lr)
    w_ref, losses_ref = orc.sync_steps(w0, idx, [batch], lr, n_steps=steps)
    _check_traj(ctx.get_weights(), w_ref, np.concatenate([l1, l2]), losses_ref)
    ctx.set_workers([], 0)


@pytest.mark.parametrize("counts", [[40, 24], [50, 31, 7]])
def test_sync_steps_virtual_workers(setup, counts):
    data, n_train, ctx, orc = setup
    steps, lr, tot = 30, 0.5, sum(counts)
    rng = np.random.default_rng(len(counts))
    idx = np.concatenate([rng.choice(n_train, size=tot, replace=False) for _ in range(steps)]).astype(np.int32)
    w0 = np.zeros(data.dim)
    ctx.set_weights(w0)
    ctx.set_workers(counts, len(counts))
    try:
        losses = ctx.sync_steps(idx, tot, steps, lr)
    finally:
        ctx.set_workers([], 0)
    w_ref, losses_ref = orc.sync_steps(w0, idx, counts, lr, n_steps=steps)
    _check_traj(ctx.get_weights(), w_ref, losses, losses_ref)


def test_world2_without_communicator_refused():
    from distributed_sgd_b200.native import DsgdState, NativeCtx
    rp = np.array([0, 1, 2], dtype=np.int64)
    with NativeCtx(0, 4, LAM, rank=0, world=2, logistic=True) as ctx:
        ctx.load_csr(rp, np.array([0, 1], np.int32), np.array([1.0, 1.0], np.float32), np.array([1, -1], np.int8))
        ctx.set_dim_sparsity(np.ones(4))
        n0 = ctx.launch_count()
        with pytest.raises(DsgdState):
            ctx.sync_steps(np.array([0], np.int32), 1, 1, 0.5)
        assert ctx.launch_count() == n0


def test_master_sync_fit_matches_oracle_replay():
    from distributed_sgd_b200 import EarlyStopping, Master, Slave, SparseLogistic
    from distributed_sgd_b200.core import Group
    from distributed_sgd_b200.core.master import EpochDraw
    from distributed_sgd_b200.ml import SplitStrategy
    from distributed_sgd_b200.utils import synthetic_rcv1
    from oracle.logistic import LogisticOracle
    data = synthetic_rcv1(n_rows=6000, seed=8)
    train, test = data.split_at(4800)
    model = SparseLogistic(1e-4)
    slave = Slave(0, 0, train, model, False, device=0, test_data=test)
    try:
        m = Master.create(0, train, test, model, False, 1, slave=slave, group=Group(), seed=5)
        batch, lr, epochs = 64, 0.5, 2
        w0 = np.zeros(data.dim)
        state = m.fit(w0, epochs, batch, lr, EarlyStopping.no_improvement(patience=5, min_delta=0.0))
        orc = LogisticOracle(data.row_ptr, data.col, data.val, data.label, data.dim, 1e-4)
        orc.set_dim_sparsity(model.dim_sparsity)
        groups = SplitStrategy.vanilla(4800, 1)
        w = w0
        losses = []
        for e in range(epochs):
            draw = EpochDraw.draw(5, e, groups, batch)
            assert (draw.counts == batch).all()
            w, _ = orc.sync_steps(w, draw.ids.reshape(-1), [batch], lr, n_steps=draw.ids.shape[0])
            losses.append(1e-4 * float(np.dot(w, w)) + math.fsum(orc.sample_losses(w, begin=0, n=4800)) / 4800)
        assert np.abs(state.grad - w).max() <= 1e-11 * np.abs(w).max()
        np.testing.assert_allclose(m.history["losses"], losses, rtol=1e-11)
        assert m.history["losses"][1] < m.history["losses"][0]
    finally:
        slave.stop()


def _free_port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def _worker(rank, world, port, q):
    sys.path.insert(0, ROOT)
    import torch
    import torch.distributed as dist
    from distributed_sgd_b200.core import Group
    from distributed_sgd_b200.native import NativeCtx
    from distributed_sgd_b200.utils import synthetic_rcv1
    from oracle.logistic import LogisticOracle

    torch.cuda.set_device(rank)
    dist.init_process_group("gloo", init_method=f"tcp://127.0.0.1:{port}", rank=rank, world_size=world)
    group = Group()
    data = synthetic_rcv1(n_rows=6000, seed=3)
    n_train, lam, lr, batch, steps = 4800, 0.01, 0.5, 48, 20
    ctx = NativeCtx(rank, data.dim, lam, rank=rank, world=world, logistic=True)
    ctx.load_csr(data.row_ptr, data.col, data.val, data.label)
    d = ctx.compute_dim_sparsity(n_train)
    uid = NativeCtx.comm_unique_id() if rank == 0 else b""
    ctx.comm_init(group.broadcast_bytes(uid, 0))
    rng = np.random.default_rng(5)
    per = n_train // world
    idx = np.stack([np.concatenate([k * per + rng.choice(per, size=batch, replace=False) for k in range(world)])
                    for _ in range(steps)]).astype(np.int32)
    mine = idx.reshape(steps, world, batch)[:, rank, :]
    ctx.set_weights(np.zeros(data.dim))
    losses = ctx.sync_steps(mine.reshape(-1), batch, steps, lr)
    w = ctx.get_weights()
    orc = LogisticOracle(data.row_ptr, data.col, data.val, data.label, data.dim, lam)
    orc.set_dim_sparsity(d)
    w_ref, losses_ref = orc.sync_steps(np.zeros(data.dim), idx.reshape(-1), [batch] * world, lr, n_steps=steps)
    ok = bool(np.allclose(losses, losses_ref, rtol=1e-12, atol=0) and np.abs(w - w_ref).max() <= 1e-11 * np.abs(w_ref).max())
    blobs = group.all_gather_bytes(w.tobytes())
    q.put((rank, ok, all(b == blobs[0] for b in blobs)))
    ctx.close()
    dist.destroy_process_group()


def test_two_gpu_nccl_logistic():
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    import torch.multiprocessing as mp
    ctxmp = mp.get_context("spawn")
    q = ctxmp.Queue()
    port = _free_port()
    procs = [ctxmp.Process(target=_worker, args=(r, 2, port, q)) for r in range(2)]
    for p in procs:
        p.start()
    res = [q.get(timeout=300) for _ in procs]
    for p in procs:
        p.join(timeout=60)
    for rank, ok, same in res:
        assert ok, f"rank {rank}: trajectory differs from the oracle"
        assert same, "weight replicas differ across GPUs"
