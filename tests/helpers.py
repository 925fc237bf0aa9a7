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


# ---- async (Hogwild) test data ----------------------------------------------------------------------------------------

LENGTHS = [0, 1, 2, 127, 128, 129, 130, 255, 256, 257, 2000]   # pairs: odd lengths get one padding pair


def csr(rows, labels, dim):
    """rows: list of (cols, vals) in storage order."""
    rp = np.zeros(len(rows) + 1, np.int64)
    rp[1:] = np.cumsum([len(c) for c, _ in rows])
    col = np.concatenate([np.asarray(c, np.int32) for c, _ in rows]) if rp[-1] else np.zeros(0, np.int32)
    val = np.concatenate([np.asarray(v, np.float32) for _, v in rows]) if rp[-1] else np.zeros(0, np.float32)
    return data_from_csr(rp, col, val, labels, dim)


def dyadic(rng, n):
    return rng.integers(1, 1025, size=n) / 256.0                 # multiples of 2^-8 in [2^-8, 4]


def edge_rows(seed, dim=4099, n_rows=330):
    """Every length of LENGTHS in sorted, descending and random column order; short rows draw their columns from a
    512-column pool (so the rows of a batch share most of their columns), 2000-long rows from the whole range; every
    fifth row holds columns 0 and dim - 1."""
    rng = np.random.default_rng(seed)
    pool = np.concatenate([[0, dim - 1], rng.choice(np.arange(1, dim - 1), size=510, replace=False)])
    rows = []
    for i in range(n_rows):
        n = LENGTHS[i % len(LENGTHS)]
        src = pool if n <= len(pool) else np.arange(dim)
        cols = rng.choice(src, size=n, replace=False)
        if i % 5 == 0 and n >= 2:
            rest = cols[(cols != 0) & (cols != dim - 1)][:n - 2]
            cols = np.concatenate([[0, dim - 1], rest])
        order = (i // len(LENGTHS)) % 3
        cols = np.sort(cols) if order == 0 else (np.sort(cols)[::-1] if order == 1 else rng.permutation(cols))
        rows.append((cols, dyadic(rng, n)))
    labels = rng.choice(np.array([-1, 1], np.int8), size=n_rows)
    w0 = np.where(rng.random(dim) < 0.5, rng.integers(-256, 257, size=dim) / 64.0, 0.0)
    return csr(rows, labels, dim), w0


EPS = 1e-20


def filter_case(name):
    """One edge of the reference's 1e-20 filter: (rows, labels, dim, d, lam, lr, w0); a replay makes one update per row,
    in row order."""
    dim = 8
    d = np.zeros(dim)
    w0 = np.zeros(dim)
    if name == "residual":            # w - delta = 2^-72 ~ 2.1e-22: the entry must leave the map
        w0[3] = 2.0 ** -20 + 2.0 ** -72
        return [([3], [2.0 ** -20])], [1], dim, d, 0.0, 1.0, w0
    if name == "tiny_product":        # x . w = 2^-80 <= 1e-20 is dropped: dot 0, y = -1 passes the gate
        w0[2] = 2.0 ** -40
        return [([2, 5], [2.0 ** -40, 0.5])], [-1], dim, d, 0.0, 1.0, w0
    if name in ("c_at_eps", "c_above_eps"):   # S = 1, lambda = 1e-20 / 2: c = 1e-20 exactly (not added), or one ulp above
        w0[0], d[0] = 1.0, 1.0
        lam = EPS / 2 if name == "c_at_eps" else np.nextafter(EPS / 2, 1.0)
        return [([4], [2.0 ** -66])], [1], dim, d, lam, 1.0, w0
    if name == "cancel":              # m + c == 0 on column 1: the key leaves the delta; column 6 moves S for update 2
        w0[0], d[0], d[1], d[6] = -1.0, 1.0, 0.5, 0.5
        return [([1, 6], [0.5, 0.25]), ([6, 1], [0.25, 0.5])], [1, 1], dim, d, 0.25, 0.5, w0
    if name == "tiny_delta":          # (m + c) * lr = 2^-69 <= 1e-20 on column 1: no delta, and S must not move (d = 2^40)
        w0[0], d[0], d[1] = 2.0 ** -20, 1.0, 2.0 ** 40
        return [([1, 2], [2.0 ** -40, 1.0]), ([3], [1.0])], [1, 1], dim, d, 2.0 ** -21, 2.0 ** -30, w0
    raise KeyError(name)


FILTER_CASES = ["residual", "tiny_product", "c_at_eps", "c_above_eps", "cancel", "tiny_delta"]


def filter_expect(name):
    """{column: exact weight} after the replay of filter_case(name)."""
    return {
        "residual": {3: 0.0},
        "tiny_product": {2: 2.0 ** -39, 5: 0.5},
        "c_at_eps": {4: -(2.0 ** -66)},
        "c_above_eps": {4: -(2.0 ** -66 + np.nextafter(EPS, 1.0))},
        # update 1: column 1 cancels, column 6 -> 0.125 and S -> -0.9375; update 2 reads that S: c = -0.46875
        "cancel": {1: -0.015625, 6: 0.234375},
        "tiny_delta": {1: 0.0, 2: -(1.0 + 2.0 ** -40) * 2.0 ** -30, 3: -(1.0 + 2.0 ** -40) * 2.0 ** -30},
    }[name]


def conservation_rows():
    """4096 rows of 8 entries 2^-4 over 4096 columns, y = +1: from w0 = 2^10 with lr = 2^-6 the gate always passes and every
    partial sum of deltas is exact in any order.  Returns (data, entries per row)."""
    rng = np.random.default_rng(77)
    dim, n, k = 4096, 4096, 8
    rows = [(np.sort(rng.choice(dim, size=k, replace=False)), np.full(k, 2.0 ** -4)) for _ in range(n)]
    return csr(rows, np.ones(n, np.int8), dim), k


def async_workers(data, lam, d, K, w0=None, master=True, outbox=False):
    """K async contexts on device 0 (rank r of world K), `data` loaded and dimSparsity d installed, every context attached
    to every other's replica with dsgd_peer_attach.  master: rank 0 hosts the master replica and ranks 1..K-1 attach it at
    peer_rank K.  Every replica, the master's included, starts from w0 (None: zeros); outbox: every worker's outbox is
    enabled (and empty).  The caller closes the contexts."""
    from distributed_sgd_b200.native import REPLICA_MASTER, REPLICA_SELF, NativeCtx
    w0 = np.zeros(data.dim) if w0 is None else np.asarray(w0, np.float64)
    ctxs = []
    try:
        for r in range(K):
            ctx = NativeCtx(0, data.dim, lam, rank=r, world=K, is_async=True)
            ctxs.append(ctx)
            ctx.load_csr(data.row_ptr, data.col, data.val, data.label)
            ctx.set_dim_sparsity(d)
            ctx.set_weights(w0)
        if master:
            ctxs[0].async_host_master(w0)
        for r in range(K):
            for q in range(K):
                if q != r:
                    ctxs[r].peer_attach(q, ctxs[q], REPLICA_SELF)
            if master and r != 0:
                ctxs[r].peer_attach(K, ctxs[0], REPLICA_MASTER)
            if outbox:
                ctxs[r].async_outbox_enable()
    except BaseException:
        for c in ctxs:
            c.close()
        raise
    return ctxs


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
    set_weights on every rank just before the launch.  lr: one rate, or an array of one rate per step of every launch (a
    rate table: dsgd_sync_steps_lr).  before(r, ctx), if given, runs on every rank's context once the ranks
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
                        if np.ndim(lr):
                            ls.append(ctx.sync_steps_lr(a.reshape(-1), a.shape[1], lr))
                        else:
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
