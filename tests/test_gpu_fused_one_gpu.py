"""The fused K-rank sync kernel (sparse LL exchange through peer memory, dsgd_persistent.cuh kMulti) exercised on ONE GPU:
K device contexts share the GPU (each limited to 1/K of the SMs with dsgd_set_grid_limit, attached to each other with
dsgd_xchg_attach), one host thread per context like one JVM thread per Slave.  The ranks' kernels run concurrently and
exchange exactly as they do over NVLink -- the receive areas just live in the same HBM -- so a single-GPU
machine runs the multi-rank path for real: trajectories against the oracle's K-worker master step (core/Master.scala:184-197),
bit-identical replicas, several launches in a row (global step counter, receive parities), short last batches.
K stops at 3 here: four spinning kernels sharing one GPU hit the device-side watchdog in 2 of 9 sessions (CUDA does not
promise co-scheduling of independent kernels; cooperative launch is per kernel) -- four and eight ranks are checked on real
GPUs by bench.py's parity record and whole-run replays.  A watchdog time-out is retried once.
"""
import numpy as np
import pytest

from helpers import make_pair, retry_once_if_not_coscheduled, run_ranks, xchg_model

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("K,batch,dim", [(2, 48, 20000), (2, 7, 3000), (3, 33, 9000), (3, 64, 11000)])
def test_fused_k_ranks_on_one_gpu_match_oracle(K, batch, dim):
    retry_once_if_not_coscheduled(lambda: _fused_k_ranks(K, batch, dim))


def _fused_k_ranks(K, batch, dim):
    import torch
    from distributed_sgd_b200.utils import synthetic_rcv1
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    data = synthetic_rcv1(n_rows=4000, dim=dim, seed=11, mean_nnz=40.0)
    n_train, lam, lr, steps = 3600, 0.01, 0.5, 24
    ctxs, orc = [], None
    for r in range(K):
        ctx, orc = make_pair(data, lam, n_train=n_train, device=0, rank=r, world=K)
        ctx.set_grid_limit(sms // K - (4 if K > 2 else 0))   # K > 2: leave SMs for the ranks' small kernels
        ctx.reserve(steps * batch, steps)      # no cudaMalloc (a device-wide sync) once the ranks wait for each other
        ctxs.append(ctx)
    for r in range(K):
        for q in range(K):
            if q != r:
                ctxs[r].xchg_attach(q, ctxs[q])
    rng = np.random.default_rng(5)
    per = n_train // K
    idx = np.stack([np.concatenate([k * per + rng.choice(per, size=batch, replace=False) for k in range(K)])
                    for _ in range(steps)]).astype(np.int32)                        # [steps, K * batch]
    w0 = rng.standard_normal(dim) * (rng.random(dim) < 0.3) * 0.1
    w_ref, losses_ref = orc.sync_steps(w0, idx.reshape(-1), [batch] * K, lr, n_steps=steps)
    out = [None] * K
    cuts = [0, 1, 9, steps]                                                          # three launches in a row

    def rank_fn(r):
        def run():
            ctx = ctxs[r]
            ctx.set_weights(w0)
            mine = idx.reshape(steps, K, batch)[:, r, :]
            ls = [ctx.sync_steps(mine[a:b].reshape(-1), batch, b - a, lr) for a, b in zip(cuts[:-1], cuts[1:])]
            out[r] = (np.concatenate(ls), ctx.get_weights())
        return run

    # contexts are closed on every way out: one left to the garbage collector would be destroyed (a device-wide sync) on
    # whatever thread collects it, possibly a rank thread of a later test whose peers are spinning
    try:
        run_ranks([rank_fn(r) for r in range(K)])
        stats = [c.xchg_stats() for c in ctxs]
    finally:
        for c in ctxs:
            c.close()
    for r in range(K):
        losses, w = out[r]
        np.testing.assert_allclose(losses, losses_ref, rtol=1e-12, atol=0)
        assert np.array_equal(w != 0, w_ref != 0)
        np.testing.assert_allclose(w, w_ref, rtol=1e-11, atol=1e-15)
        assert np.array_equal(w, out[0][1]), "weight replicas differ across ranks"
    # the words each rank pushed to each peer: its filtered raw reply's support + the counter column, one bitmap word per
    # 32 columns, every step (helpers.xchg_model)
    per_rank = idx.reshape(steps, K, batch)
    calls = [([per_rank[a:b, r, :] for r in range(K)], None) for a, b in zip(cuts[:-1], cuts[1:])]
    model = xchg_model(orc, w0, calls, lr)
    for r in range(K):
        assert stats[r] == model[r], (r, stats[r], model[r])
        assert model[r][0] < steps * (dim + 1), "the exchange is expected to be sparse"


def test_fused_ranks_exact_cancellation_and_empty_support():
    """KA5/KA9 across ranks: a column whose entries cancel inside one worker's batch is absent from that worker's reply
    (no +c for it), a column present in two replies gets +c twice; one worker whose rows all fail the gate sends an empty
    reply (bitmap words only)."""
    from helpers import data_from_csr
    import torch
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    dim = 64
    # rows 0,1: worker 0 (x on cols 3 and 5 with opposite labels -> col 3 cancels exactly); rows 2,3: worker 1
    rp = [0, 2, 4, 6, 7]
    col = [3, 5, 3, 9, 5, 9, 20]
    val = [0.5, 0.25, 0.5, 0.75, 0.125, 0.5, 1.0]
    lab = [1, -1, 1, -1]
    data = data_from_csr(rp, col, val, lab, dim)
    lam, lr = 0.05, 0.5
    ctxs, orc = [], None
    for r in range(2):
        ctx, orc = make_pair(data, lam, n_train=4, device=0, rank=r, world=2)
        ctx.set_grid_limit(sms // 2)
        ctx.reserve(64, 16)
        ctxs.append(ctx)
    ctxs[0].xchg_attach(1, ctxs[1]); ctxs[1].xchg_attach(0, ctxs[0])
    w0 = np.zeros(dim); w0[[3, 5, 9, 20]] = [0.3, -0.2, 0.1, -0.4]
    idx = np.array([[0, 1, 2, 3]] * 6, dtype=np.int32)                               # worker 0: rows 0,1; worker 1: rows 2,3
    w_ref, losses_ref = orc.sync_steps(w0, idx.reshape(-1), [2, 2], lr, n_steps=6)
    out = [None, None]

    def rank_fn(r):
        def run():
            ctxs[r].set_weights(w0)
            ls = ctxs[r].sync_steps(idx[:, 2 * r:2 * r + 2].reshape(-1), 2, 6, lr)
            out[r] = (ls, ctxs[r].get_weights())
        return run

    try:
        run_ranks([rank_fn(0), rank_fn(1)])
        stats = [c.xchg_stats() for c in ctxs]
    finally:
        for c in ctxs:
            c.close()
    for r in range(2):
        np.testing.assert_allclose(out[r][0], losses_ref, rtol=1e-13, atol=0)
        np.testing.assert_allclose(out[r][1], w_ref, rtol=1e-13, atol=1e-300)
    assert np.array_equal(out[0][1], out[1][1])
    model = xchg_model(orc, w0, [([idx[:, 0:2], idx[:, 2:4]], None)], lr)
    for r in range(2):
        assert stats[r] == model[r], (r, stats[r], model[r])
