"""Shared helpers for the GPU parity tests (oracle side lives in oracle/, test infrastructure only)."""
import threading

import numpy as np

from oracle.oracle import Oracle


def make_pair(data, lam, n_train=None, device=0, rank=0, world=1, is_async=False):
    """(NativeCtx with `data` loaded and dimSparsity installed, Oracle with the same)."""
    from distributed_sgd_b200.native import NativeCtx
    n_train = data.n_rows if n_train is None else n_train
    ctx = NativeCtx(device, data.dim, lam, rank=rank, world=world, is_async=is_async)
    ctx.load_csr(data.row_ptr, data.col, data.val, data.label)
    orc = Oracle(data.row_ptr, data.col, data.val, data.label, data.dim, lam)
    d = orc.dim_sparsity(n_train)
    orc.set_dim_sparsity(d)
    ctx.set_dim_sparsity(d)
    return ctx, orc


def data_from_csr(rp, col, val, lab, dim):
    from distributed_sgd_b200.utils.dataset import Data
    return Data(np.asarray(rp, np.int64), np.asarray(col, np.int32), np.asarray(val, np.float32),
                np.asarray(lab, np.int8), dim)


# ---- K ranks of the fused peer-exchange sync step sharing one GPU ----------------------------------------------------

def run_ranks(fns):
    """Runs fns[r]() on one host thread per rank (one JVM thread per Slave) and re-raises the first failure."""
    errs = [None] * len(fns)

    def wrap(i):
        try:
            fns[i]()
        except BaseException as e:  # noqa: BLE001 -- reported below
            errs[i] = e

    th = [threading.Thread(target=wrap, args=(i,)) for i in range(len(fns))]
    for t in th:
        t.start()
    for t in th:
        t.join(timeout=120)
    for e in errs:
        if e is not None:
            raise e
    assert not any(t.is_alive() for t in th), "a rank hangs"


def retry_once_if_not_coscheduled(attempt):
    """K spinning kernels sharing ONE GPU need all their CTAs resident at once; CUDA does not promise that for independent
    plain launches (on real multi-GPU boxes every rank has its own GPU and a cooperative launch).  A run that ends in the
    device-side watchdog is repeated once with fresh contexts; a second time-out fails the test."""
    from distributed_sgd_b200.native import DsgdError, ERR_TIMEOUT
    try:
        return attempt()
    except DsgdError as e:
        if getattr(e, "code", None) == ERR_TIMEOUT:
            import warnings
            warnings.warn("fused ranks were not co-scheduled on the shared GPU (watchdog); retrying once")
            return attempt()
        raise


def fused_ranks(data, lam, d, grid_limits, w0, calls, lr, n_train=None, after=None, before=None):
    """Runs K = len(grid_limits) ranks of the fused sync step on one GPU: rank r limited to grid_limits[r] CTAs, every rank
    attached to every other with dsgd_xchg_attach, one host thread each.  d: dimSparsity for every rank (None: computed
    from the first n_train rows).  Every rank starts from w0; calls[i] = (ids, w) is one launch: ids[r] is rank r's int32
    [steps, batch_r] sample ids (steps the same on every rank, batches may differ), w (or None) new weights installed with
    set_weights on every rank just before the launch.  before(r, ctx), if given, runs on every rank's context once the ranks
    are attached, before the first launch; after(r, ctx) runs on every rank's context once all launches are done, before
    the contexts are closed.

    Checks that the replicas, the losses and the exchange's step counts are identical across ranks, and returns
    dict(losses=[K arrays over all steps], w=[K weights], xstats=[K (value words, bitmap words, steps)], after=[K results])."""
    K = len(grid_limits)
    calls = [(list(ids), w) for ids, w in calls]
    for ids, _ in calls:
        assert len(ids) == K and len({a.shape[0] for a in ids}) == 1, "every rank runs the same steps in a launch"

    def attempt():
        ctxs = []
        try:
            for r in range(K):
                ctx, _ = make_pair(data, lam, n_train=n_train, rank=r, world=K)
                if d is not None:
                    ctx.set_dim_sparsity(d)
                ctx.set_grid_limit(grid_limits[r])
                # no cudaMalloc (a device-wide sync) once the ranks wait for each other
                ctx.reserve(max(ids[r].size for ids, _ in calls), max(ids[r].shape[0] for ids, _ in calls))
                ctxs.append(ctx)
            for r in range(K):
                for q in range(K):
                    if q != r:
                        ctxs[r].xchg_attach(q, ctxs[q])
            if before is not None:
                for r in range(K):
                    before(r, ctxs[r])
            out = [None] * K

            def rank_fn(r):
                def run():
                    ctx = ctxs[r]
                    ctx.set_weights(w0)
                    ls = []
                    for ids, w in calls:
                        if w is not None:
                            ctx.set_weights(w)
                        a = np.ascontiguousarray(ids[r], dtype=np.int32)
                        ls.append(ctx.sync_steps(a.reshape(-1), a.shape[1], a.shape[0], lr))
                    out[r] = (np.concatenate(ls), ctx.get_weights(), ctx.xchg_stats())
                return run

            run_ranks([rank_fn(r) for r in range(K)])
            post = [after(r, ctxs[r]) if after is not None else None for r in range(K)]
        finally:
            for c in ctxs:
                c.close()
        return out, post

    out, post = retry_once_if_not_coscheduled(attempt)
    for r in range(1, K):
        assert np.array_equal(out[r][1], out[0][1]), f"weight replicas of ranks 0 and {r} differ"
        np.testing.assert_array_equal(out[r][0], out[0][0], err_msg=f"losses of ranks 0 and {r} differ")
        assert out[r][2][2] == out[0][2][2], "ranks count different exchange steps"
    return dict(losses=[o[0] for o in out], w=[o[1] for o in out], xstats=[o[2] for o in out], after=post)


def xchg_model(orc, w0, calls, lr):
    """What dsgd_xchg_stats reports for every rank after the launches `calls` (as for fused_ranks): per step a rank pushes to
    each peer one value word per non-zero entry of its filtered raw reply (its batch sum of y x, before + c) plus one for
    the counter column, and one bitmap word per 32 columns of dim + 1.  The raw supports come from replaying the oracle one
    step at a time: the batch gradient at lambda = 0 (c = 0) is the raw reply.  Returns [K (value words, bitmap words,
    steps)]."""
    raw = Oracle(orc.row_ptr, orc.col, orc.val, orc.label, orc.dim, 0.0)
    K = len(calls[0][0])
    vals, steps, w = [0] * K, 0, np.asarray(w0, np.float64)
    for ids, w_new in calls:
        if w_new is not None:
            w = np.asarray(w_new, np.float64)
        for s in range(ids[0].shape[0]):
            step = [np.asarray(ids[r][s], np.int32) for r in range(K)]
            for r in range(K):
                g, _ = raw.gradient(w, step[r])
                vals[r] += int(np.count_nonzero(g)) + 1
            w, _ = orc.sync_steps(w, np.concatenate(step), [len(a) for a in step], lr, n_steps=1)
            steps += 1
    return [(vals[r], steps * ((orc.dim + 1 + 31) // 32), steps) for r in range(K)]
