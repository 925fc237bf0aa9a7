"""SparseSquaredHinge and SparseModifiedHuber on the GPU against the margin checker (oracle/dsgd_oracle_margin.c), each model
in each weighting.

Both losses are piecewise polynomials of the activity with no exp or log, and the library is built with --fmad=false, so
wherever the device and the checker start from the same dot product they agree bit for bit:
  * single rows: loss, gradient, prediction and probability from the device's own margin (dsgd_margins, the row fold that
    decides the row on every path), restated in numpy, whose float64 operations are correctly rounded;
  * evaluation sums: S = sum R(c_i L_i) of those per-row losses, through tests/loss_sum_model.py; range, device-drawn and
    listed passes over one multiset give the same bits;
  * dyadic rows of at most two entries on columns of their own, with lambda = 0 (disjoint_problem): gradients and 50-step
    trajectories are the checker's bits.
Against the checker's serial dot product on RCV1-shaped rows: gradient entries within 1e-12 * (sum_i |s_i x_ij| + |c|) (the
logistic rule), loss sums rtol 1e-12, trajectories max |dw| <= 1e-11 * max |w| and losses rtol 1e-12."""
import os
import socket
import sys

import numpy as np
import pytest

from loss_sum_model import device_model
from oracle import margin as M
from oracle.oracle import Oracle
from test_oracle_sample_weight import dyadic_weights

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LAM = 1e-5
MODELS = ("squared_hinge", "modified_huber")
WEIGHTINGS = ("none", "class", "sample")


def np_row(model, z):
    """L(z) and s(z) elementwise, in the kernel's order of operations."""
    z = np.asarray(z, dtype=np.float64)
    t = 1.0 + z
    if model == "squared_hinge":
        return np.where(z <= -1.0, 0.0, t * t), np.where(z <= -1.0, 0.0, 2.0 * t)
    return (np.where(z <= -1.0, 0.0, np.where(z <= 1.0, t * t, 4.0 * z)),
            np.where(z <= -1.0, 0.0, np.where(z <= 1.0, 2.0 * t, 4.0)))


def filt(v):
    return np.where(np.abs(v) > 1e-20, v, 0.0)


@pytest.fixture(scope="module")
def data():
    from distributed_sgd_b200.utils import synthetic_rcv1
    return synthetic_rcv1(n_rows=110000, seed=31), 100000


@pytest.fixture(scope="module", params=MODELS)
def setup(request, data):
    from distributed_sgd_b200.native import NativeCtx
    data, n_train = data
    ctx = NativeCtx(0, data.dim, LAM, model=request.param)
    ctx.load_csr(data.row_ptr, data.col, data.val, data.label)
    d = ctx.compute_dim_sparsity(n_train)
    orc = Oracle(data.row_ptr, data.col, data.val, data.label, data.dim, LAM)
    orc.set_dim_sparsity(d)
    yield request.param, data, n_train, ctx, orc, d
    ctx.close()


def _weights(dim, seed, scale=0.5):
    rng = np.random.default_rng(seed)
    return np.where(rng.random(dim) < 0.3, scale * rng.standard_normal(dim), 0.0)


def _set_weighting(ctx, weighting, n_rows, seed=0):
    """Installs the weighting; returns (w_pos, w_neg, sw) for the checker."""
    if weighting == "none":
        return 1.0, 1.0, None
    ctx.set_class_weights(2.0, 0.5)
    if weighting == "class":
        return 2.0, 0.5, None
    sw = np.random.default_rng(seed).integers(0, 9, size=n_rows) / 4.0
    ctx.set_sample_weights(sw)
    return 2.0, 0.5, sw


def _clear_weighting(ctx):
    ctx.set_class_weights(1.0, 1.0)
    ctx.set_sample_weights(None)


def _row_weights(label, ids, w_pos, w_neg, sw, weighting):
    """c_i of the rows ids (None: unweighted)"""
    wy = np.where(label[ids] > 0, w_pos, w_neg)
    if weighting == "sample":
        return wy * sw[ids]
    return wy if weighting == "class" else None


def test_info_names_the_model(setup):
    model, _, _, ctx, _, _ = setup
    assert ctx.info()["model"] == model


# ---- single rows, bit for bit --------------------------------------------------------------------------------------------

@pytest.mark.parametrize("weighting", WEIGHTINGS)
def test_single_rows_bit_for_bit(setup, weighting):
    """One-row losses, gradients, predictions and probabilities from the device's margin, at margins spread over every branch."""
    model, data, n_train, ctx, orc, d = setup
    rng = np.random.default_rng(3)
    ids = rng.choice(n_train, size=40, replace=False).astype(np.int32)
    w = _weights(data.dim, 4, scale=3.0)
    w_pos, w_neg, sw = _set_weighting(ctx, weighting, data.n_rows, seed=5)
    ctx.set_dim_sparsity(np.zeros(data.dim))   # c = 0: a one-row gradient is its scatter alone
    try:
        dots = ctx.margins(ids, w)
        z = data.label[ids] * dots
        assert (z <= -1).any() and ((z > -1) & (z <= 1)).any() and (z > 1).any(), "margins miss a branch"
        L, s = np_row(model, z)
        ref_l, ref_s = zip(*(M.row(model, float(v)) for v in z))
        assert np.array_equal(L, ref_l) and np.array_equal(s, ref_s)
        c = _row_weights(data.label, ids, w_pos, w_neg, sw, weighting)
        for k, r in enumerate(ids):
            g = ctx.gradient([r], w)
            lo, hi = data.row_ptr[r], data.row_ptr[r + 1]
            y = float(data.label[r])
            v = y * s[k] if c is None else (y * s[k]) * c[k]
            ref = np.zeros(data.dim)
            if s[k] != 0.0:
                ref[data.col[lo:hi]] = filt(filt(data.val[lo:hi].astype(np.float64)) * v)
            assert np.array_equal(g, ref), (r, z[k])
            we = ctx.eval_samples_weighted([r], w) if weighting == "sample" else None
            if we is not None:
                assert we.loss_sum == device_model([c[k] * L[k]])
            assert ctx.eval_samples_sums([r], w)[0] == device_model([L[k]])
        np.testing.assert_array_equal(ctx.forward(ids, w), -np.sign(dots))
        np.testing.assert_array_equal(ctx.forward(ids, w), orc.forward(w, ids))
        from distributed_sgd_b200.native import DsgdState
        if model == "modified_huber":
            m = np.clip(-dots, -1.0, 1.0)
            assert np.array_equal(ctx.probabilities(ids, w), (m + 1.0) / 2.0)
        else:
            with pytest.raises(DsgdState, match="squared_hinge"):
                ctx.probabilities(ids, w)
    finally:
        ctx.set_dim_sparsity(d)
        _clear_weighting(ctx)


# ---- evaluation sums ----------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("n", [1, 7, 1000, 100000])
def test_eval_sums_forms_agree_and_match_the_oracle(setup, n):
    model, data, n_train, ctx, orc, _ = setup
    w = _weights(data.dim, 6, scale=2.0)
    ids = np.arange(n, dtype=np.int32)
    shuffled = np.random.default_rng(n).permutation(ids).astype(np.int32)
    s_range, ok_range, n2 = ctx.eval_sums(0, n, w)
    s_list, ok_list, _ = ctx.eval_samples_sums(shuffled, w)
    s_drawn, ok_drawn, _ = ctx.eval_sampled_sums(0, n, 12345, 0, n, w)   # every position of a permutation of [0, n)
    assert s_range == s_list == s_drawn and ok_range == ok_list == ok_drawn
    dots = ctx.margins(ids, w)
    L, _ = np_row(model, data.label[:n] * dots)
    assert s_range == device_model(L)
    assert ok_range == int(np.sum(-np.sign(dots) == data.label[:n]))
    _, _, s_orc, ok_orc = M.loss_acc(orc, model, w, ids)
    assert s_range == pytest.approx(s_orc, rel=1e-12, abs=1e-300) and ok_range == ok_orc
    loss, acc = ctx.eval(0, n, w)
    assert loss == pytest.approx(LAM * n2 + s_range / n, rel=1e-15) and acc == ok_range / n


@pytest.mark.parametrize("weighting", ["class", "sample"])
def test_weighted_evaluations(setup, weighting):
    model, data, n_train, ctx, orc, _ = setup
    w = _weights(data.dim, 7, scale=2.0)
    n = 5000
    ids = np.arange(n, dtype=np.int32)
    w_pos, w_neg, sw = _set_weighting(ctx, weighting, data.n_rows, seed=8)
    try:
        dots = ctx.margins(ids, w)
        y = data.label[:n]
        L, _ = np_row(model, y * dots)
        ok = -np.sign(dots) == y
        if weighting == "class":
            ce = ctx.eval_class(0, n, w)
            assert ce.loss_pos == device_model(L[y > 0]) and ce.loss_neg == device_model(L[y < 0])
            assert (ce.correct_pos, ce.correct_neg, ce.n_pos, ce.n_neg) == (
                int(ok[y > 0].sum()), int(ok[y < 0].sum()), int((y > 0).sum()), int((y < 0).sum()))
            sums_ref, _ = M.eval_class(orc, model, w, ids)
            np.testing.assert_allclose([ce.loss_pos, ce.loss_neg], sums_ref, rtol=1e-12)
            assert ce == ctx.eval_samples_class(np.random.default_rng(1).permutation(ids), w)
        else:
            c = _row_weights(data.label, ids, w_pos, w_neg, sw, weighting)
            we = ctx.eval_weighted(0, n, w)
            assert we.loss_sum == device_model(c * L)
            assert we.correct_weight == device_model(np.where(ok, c, 0.0)) and we.weight_sum == device_model(c)
            assert (we.n, we.correct) == (n, int(ok.sum()))
            sums_ref, counts_ref = M.eval_weighted(orc, model, w, ids, w_pos, w_neg, sw)
            np.testing.assert_allclose(we.loss_sum, sums_ref[0], rtol=1e-12)
            assert we == ctx.eval_samples_weighted(np.random.default_rng(2).permutation(ids), w)
    finally:
        _clear_weighting(ctx)


# ---- batch gradients ----------------------------------------------------------------------------------------------------

def _bound(model, data, w, idx, c, cw):
    b = np.zeros(data.dim)
    for k, r in enumerate(idx):
        lo, hi = data.row_ptr[r], data.row_ptr[r + 1]
        cols, vals = data.col[lo:hi], data.val[lo:hi].astype(np.float64)
        z = float(data.label[r]) * float(np.dot(vals, w[cols]))
        b[cols] += np.abs(vals) * M.row(model, z)[1] * (1.0 if cw is None else cw[k])
    return b + abs(c)


@pytest.mark.parametrize("weighting", WEIGHTINGS)
@pytest.mark.parametrize("batch", [1, 64, 4096])
def test_batch_gradient(setup, weighting, batch):
    model, data, n_train, ctx, orc, d = setup
    rng = np.random.default_rng(batch)
    idx = rng.choice(n_train, size=batch, replace=False).astype(np.int32)
    w = _weights(data.dim, 9)
    w_pos, w_neg, sw = _set_weighting(ctx, weighting, data.n_rows, seed=10)
    try:
        g = ctx.gradient(idx, w)
    finally:
        _clear_weighting(ctx)
    g_ref, _, _ = M.gradient(orc, model, w, idx, w_pos, w_neg, sw)
    c = LAM * 2.0 * float(np.sum(filt(w * d)))
    assert ((g == 0) == (g_ref == 0)).all(), "gradient support differs"
    bound = _bound(model, data, w, idx, c, _row_weights(data.label, idx, w_pos, w_neg, sw, weighting))
    assert (np.abs(g - g_ref) <= 1e-12 * bound).all()


def disjoint_problem(seed, n_rows=400, dim=1024):
    """Dyadic rows of one or two entries, row r on columns 2r and 2r + 1 only.  With lambda = 0 the device and the checker
    then do the same correctly rounded operations in the same order: a two-entry dot is p0 + p1 in the row fold and in the
    checker's serial sum, and in a batch of distinct rows every gradient column takes at most one contribution.  So their
    trajectories agree bit for bit for as many steps as they run, although the quadratic scales lengthen the weights' bits
    every step (an exact dyadic run of these models lasts only a few steps)."""
    rng = np.random.default_rng(seed)
    k = rng.integers(1, 3, size=n_rows)
    rp = np.concatenate([[0], np.cumsum(k)]).astype(np.int64)
    col = np.concatenate([2 * r + np.arange(k[r]) for r in range(n_rows)]).astype(np.int32)
    val = (rng.integers(1, 17, size=col.size) / 8.0 * rng.choice([-1.0, 1.0], size=col.size)).astype(np.float32)
    lab = rng.choice(np.array([-1, 1], dtype=np.int8), size=n_rows)
    orc = Oracle(rp, col, val, lab, dim, 0.0)
    d = np.zeros(dim)
    d[::3] = 0.25
    orc.set_dim_sparsity(d)
    w0 = rng.integers(-8, 9, size=dim) / 16.0
    return orc, (rp, col, val, lab, d), w0


@pytest.fixture(scope="module", params=MODELS)
def dyadic(request):
    from distributed_sgd_b200.native import NativeCtx
    orc, (rp, col, val, lab, d), w0 = disjoint_problem(60)
    ctx = NativeCtx(0, orc.dim, 0.0, model=request.param)
    ctx.load_csr(rp, col, val, lab)
    ctx.set_dim_sparsity(d)
    yield request.param, orc, ctx, w0, lab
    ctx.close()


@pytest.mark.parametrize("weighting", WEIGHTINGS)
def test_dyadic_gradient_bit_for_bit(dyadic, weighting):
    model, orc, ctx, w0, lab = dyadic
    idx = np.random.default_rng(11).choice(len(lab), size=300, replace=False).astype(np.int32)
    w_pos, w_neg, sw = {"none": (1.0, 1.0, None), "class": (4.0, 0.25, None),
                        "sample": (2.0, 0.5, dyadic_weights(np.random.default_rng(12), len(lab)))}[weighting]
    if weighting != "none":
        ctx.set_class_weights(w_pos, w_neg)
    if sw is not None:
        ctx.set_sample_weights(sw)
    try:
        g, loss = ctx.gradient(idx, w0, want_loss=True)
    finally:
        _clear_weighting(ctx)
    g_ref, loss_ref, _ = M.gradient(orc, model, w0, idx, w_pos, w_neg, sw)
    assert np.array_equal(g, g_ref) and loss == loss_ref


# ---- trajectories of the per-step path ---------------------------------------------------------------------------------

CASES = {   # name: (worker counts, weighting, lambda1, averaging, rate table)
    "one_worker": ([64], "none", 0.0, False, False),
    "three_workers": ([40, 24, 17], "none", 0.0, False, False),
    "l1": ([64], "none", 1e-4, False, False),
    "class_weights": ([64], "class", 0.0, False, False),
    "sample_weights": ([48, 16], "sample", 0.0, False, False),
    "averaging": ([64], "none", 0.0, True, False),
    "rate_table": ([64], "none", 0.0, False, True),
}


def _run(ctx, orc, model, w0, idx, counts, weighting, lambda1, avg, table, n_rows, steps, lr, dyadic_weights_rng=None):
    if dyadic_weights_rng is not None:
        w_pos, w_neg, sw = {"none": (1.0, 1.0, None), "class": (4.0, 0.25, None),
                            "sample": (2.0, 0.5, dyadic_weights(dyadic_weights_rng, n_rows))}[weighting]
        if weighting != "none":
            ctx.set_class_weights(w_pos, w_neg)
        if sw is not None:
            ctx.set_sample_weights(sw)
    else:
        w_pos, w_neg, sw = _set_weighting(ctx, weighting, n_rows, seed=13)
    lrs = lr / (1.0 + 0.5 * np.arange(steps)) if table else np.full(steps, lr)
    if dyadic_weights_rng is not None and table:
        lrs = lr * 2.0 ** -(np.arange(steps) % 4)
    tot = sum(counts)
    ctx.set_weights(w0)
    ctx.set_l1(lambda1)
    ctx.set_workers(counts, len(counts))
    try:
        if avg:
            ctx.average_begin()
        n0 = ctx.launch_count()
        losses = ctx.sync_steps_lr(idx, tot, lrs) if table else ctx.sync_steps(idx, tot, steps, lr)
        launches = ctx.launch_count() - n0
        w = ctx.get_weights()
        mean = ctx.average_weights()[0] if avg else None
    finally:
        if avg:
            ctx.average_end()
        ctx.set_l1(0.0)
        _clear_weighting(ctx)
    avg_sum = np.zeros(orc.dim) if avg else None
    w_ref, l_ref = M.sync_steps(orc, model, w0, idx, counts, lrs, w_pos, w_neg, sw, lambda1=lambda1, avg_sum=avg_sum)
    mean_ref = filt(avg_sum / steps) if avg else None
    return w, losses, mean, launches, w_ref, l_ref, mean_ref


@pytest.mark.parametrize("case", list(CASES))
def test_trajectory_50_steps(setup, case):
    model, data, n_train, ctx, orc, _ = setup
    counts, weighting, lambda1, avg, table = CASES[case]
    steps, lr = 50, 0.1
    rng = np.random.default_rng(len(case))
    idx = np.concatenate([rng.choice(n_train, size=sum(counts), replace=False) for _ in range(steps)]).astype(np.int32)
    w0 = _weights(data.dim, 14, scale=0.05)
    w, losses, mean, launches, w_ref, l_ref, mean_ref = _run(ctx, orc, model, w0, idx, counts, weighting, lambda1, avg,
                                                             table, data.n_rows, steps, lr)
    assert np.abs(w - w_ref).max() <= 1e-11 * np.abs(w_ref).max()
    np.testing.assert_allclose(losses, l_ref, rtol=1e-12)
    if avg:
        assert np.abs(mean - mean_ref).max() <= 1e-11 * np.abs(mean_ref).max()
    if case == "one_worker":
        assert launches == 2 * steps   # the row kernel and k_update per step: never the persistent kernel


@pytest.mark.parametrize("case", list(CASES))
def test_trajectory_bit_for_bit_on_dyadic_data(dyadic, case):
    model, orc, ctx, w0, lab = dyadic
    counts, weighting, lambda1, avg, table = CASES[case]
    lambda1 = 2.0 ** -10 if lambda1 else 0.0
    steps = 50
    rng = np.random.default_rng(len(case) + 20)
    idx = np.concatenate([rng.choice(len(lab), size=k, replace=False) for _ in range(steps) for k in counts]).astype(np.int32)
    w, losses, mean, _, w_ref, l_ref, mean_ref = _run(ctx, orc, model, w0, idx, counts, weighting, lambda1, avg, table,
                                                      len(lab), steps, 2.0 ** -6,
                                                      dyadic_weights_rng=np.random.default_rng(21))
    assert np.array_equal(w, w_ref)
    assert np.array_equal(losses, l_ref)
    if avg:
        assert np.array_equal(mean, mean_ref)


# ---- refusals ------------------------------------------------------------------------------------------------------------

def test_counts_calls_are_refused(setup):
    from distributed_sgd_b200.native import DsgdState
    model, data, n_train, ctx, _, _ = setup
    n0 = ctx.launch_count()
    for call in (lambda: ctx.eval_counts(0, 10), lambda: ctx.eval_sampled_counts(0, 10, 1, 0, 5),
                 lambda: ctx.eval_samples_counts([1, 2, 3])):
        with pytest.raises(DsgdState, match=f"the {model} model's loss sum is not an integer"):
            call()
    assert ctx.launch_count() == n0


@pytest.mark.parametrize("model", MODELS)
def test_peer_exchange_only_rank_is_refused_before_any_launch(model):
    from distributed_sgd_b200.native import DsgdState, NativeCtx
    rp = np.array([0, 1, 2], dtype=np.int64)
    ctxs = [NativeCtx(0, 4, LAM, rank=r, world=2, model=model) for r in range(2)]
    try:
        for c in ctxs:
            c.load_csr(rp, np.array([0, 1], np.int32), np.array([1.0, 1.0], np.float32), np.array([1, -1], np.int8))
            c.set_dim_sparsity(np.ones(4))
        ctxs[0].xchg_attach(1, ctxs[1])
        ctxs[1].xchg_attach(0, ctxs[0])
        n0 = ctxs[0].launch_count()
        with pytest.raises(DsgdState, match=f"the {model} model takes the NCCL allreduce path"):
            ctxs[0].sync_steps(np.array([0], np.int32), 1, 1, 0.5)
        assert ctxs[0].launch_count() == n0
    finally:
        for c in ctxs:
            c.close()


# ---- two GPUs over NCCL -------------------------------------------------------------------------------------------------

def _free_port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def _worker(rank, world, port, model, q):
    sys.path.insert(0, ROOT)
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    import torch
    import torch.distributed as dist
    from distributed_sgd_b200.core import Group
    from distributed_sgd_b200.native import NativeCtx
    from distributed_sgd_b200.utils import synthetic_rcv1
    from oracle import margin as Mw
    from oracle.oracle import Oracle as O

    torch.cuda.set_device(rank)
    dist.init_process_group("gloo", init_method=f"tcp://127.0.0.1:{port}", rank=rank, world_size=world)
    group = Group()
    data = synthetic_rcv1(n_rows=6000, seed=3)
    n_train, lam, lr, batch, steps = 4800, 0.01, 0.1, 48, 20
    ctx = NativeCtx(rank, data.dim, lam, rank=rank, world=world, model=model)
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
    orc = O(data.row_ptr, data.col, data.val, data.label, data.dim, lam)
    orc.set_dim_sparsity(d)
    w_ref, losses_ref = Mw.sync_steps(orc, model, np.zeros(data.dim), idx.reshape(-1), [batch] * world, [lr] * steps)
    ok = bool(np.allclose(losses, losses_ref, rtol=1e-12, atol=0) and np.abs(w - w_ref).max() <= 1e-11 * np.abs(w_ref).max())
    blobs = group.all_gather_bytes(w.tobytes())
    q.put((rank, ok, all(b == blobs[0] for b in blobs)))
    ctx.close()
    dist.destroy_process_group()


@pytest.mark.parametrize("model", MODELS)
def test_two_gpu_nccl(model):
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    import torch.multiprocessing as mp
    ctxmp = mp.get_context("spawn")
    q = ctxmp.Queue()
    port = _free_port()
    procs = [ctxmp.Process(target=_worker, args=(r, 2, port, model, q)) for r in range(2)]
    for p in procs:
        p.start()
    res = [q.get(timeout=300) for _ in procs]
    for p in procs:
        p.join(timeout=60)
    for rank, ok, same in res:
        assert ok, f"rank {rank}: trajectory differs from the checker"
        assert same, "weight replicas differ across GPUs"
