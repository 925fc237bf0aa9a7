"""Per-step learning rates on the device (dsgd_sync_steps_lr, MasterSync.fit(learning_rate_decay=...)).

The reference replays the oracle one step at a time, step s with its own rate lrs[s].  Checked:

1. Against the oracle on every path: grids 1, 2, 7 and S (plain and cooperative launch), dims U - 1, 2 U + 1 and 47 237,
   batches 32 G (persistent kernel) and 32 G + 1 (k_rows + k_update), two virtual workers, the logistic single- and
   two-worker paths, fused K = 2 and K = 3 on one GPU; averaging on, so the sum and the count are checked too.  A table whose
   every entry differs: RCV1-shaped fp32 rows rtol 1e-11, logistic max |diff| <= 1e-11 max |w|, dyadic rows and a dyadic
   table bit for bit.
2. The defining property, bit for bit: one table call equals the chain of one-step scalar calls (weights, losses, the
   average), and a table of equal values equals one scalar call.  Dyadic rows; the logistic paths on rows of disjoint
   columns (every gradient entry is one addend, so every run gives the same bits).
3. Indexing: tables that alternate lr and 0, or are 0 except at one step (the first, the second, the ninth -- one full
   turn of the producer's 8-stage ring --, the last), through the persistent kernel (register and extra columns), the
   fallback and the fused kernel.
4. The 1e-20 filter at mean * lr_t, at exactly 1e-20 and one ulp above, in the second step.
5. The resident state after a table call: evaluations with w = NULL equal those given get_weights().
6. Errors: a NULL table, an async ctx, zero steps, exchange-only ranks.
7. End to end: MasterSync.fit(learning_rate_decay=..., average_from=1) equals a hand-driven chain of sync_steps_lr calls
   with the tables of learning_rates.
"""
import numpy as np
import pytest

from helpers import data_from_csr, make_pair, retry_once_if_not_coscheduled, run_ranks

pytestmark = pytest.mark.gpu

UPD_THREADS = 6 * 32            # update threads per CTA; U = UPD_THREADS * G register columns of the persistent kernel
EPS = 1e-20
STEPS = 20


@pytest.fixture(scope="module")
def S():
    from distributed_sgd_b200.native import NativeCtx
    ctx = NativeCtx(0, 8, 0.0)
    s = int(ctx.info()["sm_count"])
    ctx.close()
    return s


# ---- tables and the reference ------------------------------------------------------------------------------------------

def table(lr0, n):
    """lr0 (1 + 0.1 t)^-0.75: every entry differs."""
    return lr0 * np.power(1.0 + 0.1 * np.arange(n, dtype=np.float64), -0.75)


def dyadic_table(n, e0=6):
    """Powers of two that change from every step to the next: 2^-e0, 2^-(e0+1), 2^-(e0+2), 2^-e0, ..."""
    return 2.0 ** -(e0 + np.arange(n) % 3)


def readout(A, n):
    v = A / n
    return np.where(np.abs(v) > EPS, v, 0.0)


def ref_chain(orc, w0, steps_ids, counts, lrs, A=None):
    """The oracle one step at a time, step s with lrs[s]; A += the weights after every step.  (weights, A, losses)."""
    w = np.asarray(w0, np.float64)
    A, losses = (np.zeros_like(w) if A is None else A.copy()), []
    for ids, lr in zip(steps_ids, lrs):
        w, ls = orc.sync_steps(w, np.ascontiguousarray(ids, np.int32), counts, float(lr), n_steps=1)
        A = A + w
        losses.append(ls)
    return w, A, np.concatenate(losses)


# ---- data -------------------------------------------------------------------------------------------------------------

def _synth(dim, n_rows, seed):
    from distributed_sgd_b200.utils import synthetic_rcv1
    return synthetic_rcv1(n_rows=n_rows, dim=dim, seed=seed, mean_nnz=min(94.5, dim / 8.0), max_nnz=min(2000, dim // 2))


def _dyadic(dim, n_rows, seed):
    """Rows of 1 to 40 distinct columns with values k / 16, weights k / 8 on 30 % of the columns: with lambda = 0 and a
    dyadic learning rate every gradient sum and every weight is exact, so the trajectories are the oracle's bit for bit."""
    rng = np.random.default_rng(seed)
    nnz = rng.integers(1, 41, size=n_rows)
    rp = np.concatenate([[0], np.cumsum(nnz)])
    col = np.concatenate([rng.choice(dim, size=k, replace=False) for k in nnz])
    val = rng.integers(1, 33, size=int(rp[-1])) / 16.0
    lab = rng.choice([-1, 1], size=n_rows)
    w0 = rng.integers(-32, 33, size=dim) / 8.0 * (rng.random(dim) < 0.3)
    return data_from_csr(rp, col, val, lab, dim), w0


def _disjoint(n_rows, per_row, seed):
    """Row i holds columns [per_row i, per_row (i + 1)), random fp32 values: every gradient entry of a step is ONE addend."""
    rng = np.random.default_rng(seed)
    dim = n_rows * per_row
    rp = np.arange(n_rows + 1, dtype=np.int64) * per_row
    col = np.arange(dim, dtype=np.int32)
    val = (rng.random(dim) * 2.0 + 1e-3).astype(np.float32)
    lab = rng.choice([-1, 1], size=n_rows)
    w0 = rng.standard_normal(dim) * (rng.random(dim) < 0.3) * 0.1
    return data_from_csr(rp, col, val, lab, dim), w0


def _ids(rng, n_rows, steps, batch):
    return np.stack([rng.choice(n_rows, size=batch, replace=False) for _ in range(steps)]).astype(np.int32)


def _logistic_pair(data, lam):
    from distributed_sgd_b200.native import NativeCtx
    from oracle.logistic import LogisticOracle
    ctx = NativeCtx(0, data.dim, lam, logistic=True)
    ctx.load_csr(data.row_ptr, data.col, data.val, data.label)
    orc = LogisticOracle(data.row_ptr, data.col, data.val, data.label, data.dim, lam)
    d = orc.dim_sparsity(data.n_rows)
    orc.set_dim_sparsity(d)
    ctx.set_dim_sparsity(d)
    return ctx, orc


def _call(ctx, ids, lr):
    """One call over ids [steps, batch]: a table call if lr is an array, a scalar call otherwise."""
    ids = np.ascontiguousarray(ids, np.int32)
    if np.ndim(lr):
        return ctx.sync_steps_lr(ids.reshape(-1), ids.shape[1], np.asarray(lr, np.float64))
    return ctx.sync_steps(ids.reshape(-1), ids.shape[1], ids.shape[0], float(lr))


# ---- K ranks of the fused step on one GPU ------------------------------------------------------------------------------

def fused_run(data, lam, grids, w0, calls, average=False, after=None):
    """K = len(grids) ranks on one GPU (rank r limited to grids[r] CTAs, attached to each other), one host thread each.
    calls: list of (per-rank ids [steps, batch_r], lr) with lr a scalar (dsgd_sync_steps) or a table (dsgd_sync_steps_lr).
    Every rank reserves -- and begins averaging -- BEFORE the threads start: no cudaMalloc while the ranks wait for each
    other.  Returns [K (weights, losses, (average, n) or None, after(ctx) or None)]; the replicas must be identical."""
    K = len(grids)

    def attempt():
        ctxs = []
        try:
            for r in range(K):
                ctx, _ = make_pair(data, lam, rank=r, world=K)
                ctx.set_grid_limit(grids[r])
                ctx.reserve(max(c[r].size for c, _ in calls), max(c[r].shape[0] for c, _ in calls))
                if average:
                    ctx.average_begin()
                ctxs.append(ctx)
            for r in range(K):
                for q in range(K):
                    if q != r:
                        ctxs[r].xchg_attach(q, ctxs[q])
            out = [None] * K

            def rank_fn(r):
                def run():
                    ctx = ctxs[r]
                    ctx.set_weights(w0)
                    ls = [_call(ctx, c[r], lr) for c, lr in calls]
                    out[r] = (ctx.get_weights(), np.concatenate(ls), ctx.average_weights() if average else None,
                              after(ctx) if after else None)
                return run

            run_ranks([rank_fn(r) for r in range(K)])
        finally:
            for c in ctxs:
                c.close()
        return out

    out = retry_once_if_not_coscheduled(attempt)
    for r in range(1, K):
        assert np.array_equal(out[r][0], out[0][0]), f"weight replicas of ranks 0 and {r} differ"
        np.testing.assert_array_equal(out[r][1], out[0][1], err_msg=f"losses of ranks 0 and {r} differ")
    return out


def _fused_steps(calls):
    """The oracle's view of fused launches: per step the ranks' slices side by side; and the per-rank batch sizes."""
    steps = np.concatenate([np.concatenate(c, axis=1) for c in calls], axis=0)
    return steps, [a.shape[1] for a in calls[0]]


def _check_avg(avg, n, A_ref, steps, what, exact=False):
    assert n == steps, f"{what}: {n} steps averaged, expected {steps}"
    ref = readout(A_ref, steps)
    if exact:
        np.testing.assert_array_equal(avg, ref, err_msg=what)
    else:
        np.testing.assert_allclose(avg, ref, rtol=1e-11, atol=1e-15, err_msg=what)


# ---- 1. against the oracle ----------------------------------------------------------------------------------------------

def _grid(S, name):
    limit = {"G1": 1, "G2": 2, "G7": 7, "S_plain": S, "S_coop": 0}[name]
    return limit, (limit or S)


GRID_CASES = ([("G1", k) for k in ("U-1", "2U+1", "rcv1")] + [("G2", "U-1"), ("G2", "2U+1")]
              + [("G7", k) for k in ("U-1", "2U+1", "rcv1")] + [("S_plain", "2U+1"), ("S_coop", "U-1"), ("S_coop", "rcv1")])


@pytest.mark.parametrize("grid,dim_kind", GRID_CASES)
def test_grid_sweep_against_oracle(S, grid, dim_kind):
    limit, G = _grid(S, grid)
    U = UPD_THREADS * G
    dim = {"U-1": U - 1, "2U+1": 2 * U + 1, "rcv1": 47237}[dim_kind]
    n_rows = 32 * G + 64
    data = _synth(dim, n_rows, seed=1000 * G + dim + 1)
    ctx, orc = make_pair(data, lam=1e-2)
    ctx.set_grid_limit(limit)
    rng = np.random.default_rng(dim + G + 1)
    try:
        for b in (32 * G, 32 * G + 1):      # the persistent kernel's largest batch, and the fallback's smallest
            lrs = table(0.5 / b, STEPS)
            idx = _ids(rng, n_rows, STEPS, b)
            w0 = rng.standard_normal(dim) * (rng.random(dim) < 0.3) * 0.1
            ctx.set_weights(w0)
            ctx.average_begin()
            losses = ctx.sync_steps_lr(idx.reshape(-1), b, lrs)
            ctx.average_end()
            avg, n = ctx.average_weights()
            w_ref, A_ref, losses_ref = ref_chain(orc, w0, idx, [b], lrs)
            what = f"G {G} ({grid}), dim {dim}, batch {b}"
            np.testing.assert_allclose(losses, losses_ref, rtol=1e-12, atol=0, err_msg=what)
            np.testing.assert_allclose(ctx.get_weights(), w_ref, rtol=1e-11, atol=1e-15, err_msg=what)
            _check_avg(avg, n, A_ref, STEPS, what)
    finally:
        ctx.close()


def test_two_virtual_workers_against_oracle():
    dim, n_rows, b = 47237, 4096, 256
    data = _synth(dim, n_rows, seed=7)
    ctx, orc = make_pair(data, lam=1e-2)
    rng = np.random.default_rng(8)
    idx = _ids(rng, n_rows, STEPS, 2 * b)
    w0 = rng.standard_normal(dim) * (rng.random(dim) < 0.3) * 0.1
    lrs = table(0.5 / b, STEPS)
    try:
        ctx.set_workers([b, b], 2)
        ctx.set_weights(w0)
        ctx.average_begin()
        losses = ctx.sync_steps_lr(idx.reshape(-1), 2 * b, lrs)
        avg, n = ctx.average_weights()
        w_ref, A_ref, losses_ref = ref_chain(orc, w0, idx, [b, b], lrs)
        np.testing.assert_allclose(losses, losses_ref, rtol=1e-12, atol=0)
        np.testing.assert_allclose(ctx.get_weights(), w_ref, rtol=1e-11, atol=1e-15)
        _check_avg(avg, n, A_ref, STEPS, "two virtual workers")
    finally:
        ctx.close()


@pytest.mark.parametrize("counts", [[256], [128, 128]])
def test_logistic_against_oracle(counts):
    dim, n_rows = 47237, 4096
    data = _synth(dim, n_rows, seed=9)
    ctx, orc = _logistic_pair(data, 1e-3)
    rng = np.random.default_rng(10)
    tot = sum(counts)
    idx = _ids(rng, n_rows, STEPS, tot)
    w0 = rng.standard_normal(dim) * (rng.random(dim) < 0.3) * 0.1
    lrs = table(0.5 / tot, STEPS)
    try:
        ctx.set_workers(counts, len(counts))
        ctx.set_weights(w0)
        ctx.average_begin()
        losses = ctx.sync_steps_lr(idx.reshape(-1), tot, lrs)
        avg, n = ctx.average_weights()
        w_ref, A_ref, losses_ref = ref_chain(orc, w0, idx, counts, lrs)
        w = ctx.get_weights()
        assert np.max(np.abs(w - w_ref)) <= 1e-11 * np.max(np.abs(w_ref))
        np.testing.assert_allclose(losses, losses_ref, rtol=1e-11, atol=0)
        ref = readout(A_ref, STEPS)
        assert n == STEPS
        assert np.max(np.abs(avg - ref)) <= 1e-11 * np.max(np.abs(ref)), f"logistic {counts}"
    finally:
        ctx.close()


@pytest.mark.parametrize("K", [2, 3])
def test_fused_ranks_against_oracle_bit_for_bit(K):
    """Fused K-rank steps on one GPU, dyadic rows and table, two launches with different rank batches and tables."""
    G, dim, n_rows = 5, 2047, 600
    data, w0 = _dyadic(dim, n_rows, seed=20 + K)
    rng = np.random.default_rng(K)
    c1 = [_ids(rng, n_rows, 12, 32 * G - r) for r in range(K)]
    c2 = [_ids(rng, n_rows, 8, 7 + r) for r in range(K)]
    lrs1, lrs2 = dyadic_table(12), dyadic_table(8, e0=7)
    res = fused_run(data, 0.0, [G] * K, w0, [(c1, lrs1), (c2, lrs2)], average=True)
    _, orc = make_pair(data, 0.0)
    w, A, losses = w0, None, []
    for c, lrs in ((c1, lrs1), (c2, lrs2)):   # the launches' steps in order, onto one sum
        steps, counts = _fused_steps([c])
        w, A, ls = ref_chain(orc, w, steps, counts, lrs, A)
        losses.append(ls)
    for r in range(K):
        np.testing.assert_array_equal(res[r][0], w, err_msg=f"rank {r}: weights")
        np.testing.assert_array_equal(res[r][1], np.concatenate(losses), err_msg=f"rank {r}: losses")
        avg, n = res[r][2]
        _check_avg(avg, n, A, 20, f"fused K = {K}, rank {r}", exact=True)


# ---- 2. the defining property: one table call == the chain of one-step scalar calls --------------------------------------

PATHS = ["persistent_G7", "persistent_S", "fallback_G1", "two_workers", "logistic", "logistic_two_workers", "fused_K2",
         "fused_K3"]


def _single_setup(S, path, seed):
    """(ctx, data, w0, batch, counts) for a one-ctx path.  persistent_G7 has dim 2U + 1: register and extra columns."""
    if path.startswith("logistic"):
        n_rows = 1024
        data, w0 = _disjoint(n_rows, 4, seed=seed)
        ctx = _logistic_pair(data, 1e-3)[0]
        b = 256
    else:
        G = 7 if path == "persistent_G7" else (S if path == "persistent_S" else 1)
        dim = 2 * UPD_THREADS * 7 + 1 if path == "persistent_G7" else 2047
        n_rows = 32 * S + 64
        data, w0 = _dyadic(dim, n_rows, seed=seed)
        ctx = make_pair(data, 0.0)[0]
        ctx.set_grid_limit({"persistent_G7": 7, "persistent_S": 0, "fallback_G1": 1, "two_workers": 0}[path])
        b = {"persistent_G7": 32 * 7, "persistent_S": 32 * G, "fallback_G1": 33, "two_workers": 64}[path]
    counts = [b // 2, b // 2] if path.endswith("two_workers") else [b]
    if len(counts) > 1:
        ctx.set_workers(counts, len(counts))
    return ctx, data, w0, b, counts


@pytest.mark.parametrize("path", PATHS)
def test_table_call_equals_chain_of_scalar_steps(S, path):
    lrs = dyadic_table(STEPS) if not path.startswith("logistic") else table(0.5 / 256, STEPS)
    if path.startswith("fused"):
        K = int(path[-1])
        G = 5
        data, w0 = _dyadic(2047, 600, seed=90 + K)
        rng = np.random.default_rng(91)
        ids = [_ids(rng, 600, STEPS, 32 * G - r) for r in range(K)]
        one = fused_run(data, 0.0, [G] * K, w0, [(ids, lrs)], average=True)
        chain = fused_run(data, 0.0, [G] * K, w0, [([a[s:s + 1] for a in ids], lrs[s:s + 1]) for s in range(STEPS)],
                          average=True)
        scal = fused_run(data, 0.0, [G] * K, w0, [(ids, 2.0 ** -6)])
        flat = fused_run(data, 0.0, [G] * K, w0, [(ids, np.full(STEPS, 2.0 ** -6))])
        np.testing.assert_array_equal(one[0][0], chain[0][0])
        np.testing.assert_array_equal(one[0][1], chain[0][1])
        assert one[0][2][1] == chain[0][2][1] == STEPS
        np.testing.assert_array_equal(one[0][2][0], chain[0][2][0])
        np.testing.assert_array_equal(flat[0][0], scal[0][0])
        np.testing.assert_array_equal(flat[0][1], scal[0][1])
        return
    ctx, data, w0, b, counts = _single_setup(S, path, seed=92)
    idx = _ids(np.random.default_rng(93), data.n_rows, STEPS, b)
    try:
        ctx.set_weights(w0)
        ctx.average_begin()
        l_one = ctx.sync_steps_lr(idx.reshape(-1), b, lrs)
        w_one, (a_one, n_one) = ctx.get_weights(), ctx.average_weights()
        ctx.set_weights(w0)
        ctx.average_begin()
        l_chain = np.concatenate([ctx.sync_steps(idx[s], b, 1, float(lrs[s])) for s in range(STEPS)])
        w_chain, (a_chain, n_chain) = ctx.get_weights(), ctx.average_weights()
        ctx.average_end()
        np.testing.assert_array_equal(w_one, w_chain, err_msg=f"{path}: weights")
        np.testing.assert_array_equal(l_one, l_chain, err_msg=f"{path}: losses")
        assert n_one == n_chain == STEPS
        np.testing.assert_array_equal(a_one, a_chain, err_msg=f"{path}: average")
        lr = float(lrs[0])                       # a table of equal values == one scalar call
        ctx.set_weights(w0)
        l_flat = ctx.sync_steps_lr(idx.reshape(-1), b, np.full(STEPS, lr))
        w_flat = ctx.get_weights()
        ctx.set_weights(w0)
        l_scal = ctx.sync_steps(idx.reshape(-1), b, STEPS, lr)
        np.testing.assert_array_equal(w_flat, ctx.get_weights(), err_msg=f"{path}: equal table, weights")
        np.testing.assert_array_equal(l_flat, l_scal, err_msg=f"{path}: equal table, losses")
    finally:
        ctx.close()


# ---- 3. indexing ---------------------------------------------------------------------------------------------------------

INDEX_PATHS = ["persistent_G7", "persistent_S", "fallback_G1", "fused_K2"]
PATTERNS = ["alternate", "only_0", "only_1", "only_8", "only_last"]


def _pattern(name, n, lr=2.0 ** -5):
    t = np.zeros(n)
    if name == "alternate":
        t[0::2] = lr
    else:
        t[{"only_0": 0, "only_1": 1, "only_8": 8, "only_last": n - 1}[name]] = lr
    return t


@pytest.mark.parametrize("pattern", PATTERNS)
@pytest.mark.parametrize("path", INDEX_PATHS)
def test_indexing(S, path, pattern):
    """Bit for bit against the oracle replayed with the same table; with the alternating table, the weights after the
    last (zero) step equal the weights after the step before it."""
    lrs = _pattern(pattern, STEPS)
    if path == "fused_K2":
        G = 5
        data, w0 = _dyadic(2 * UPD_THREADS * 2 + 1, 600, seed=100)
        rng = np.random.default_rng(101)
        ids = [_ids(rng, 600, STEPS, 32 * G - r) for r in range(2)]
        runs = [fused_run(data, 0.0, [G, G], w0, [(ids, lrs)])]
        if pattern == "alternate":
            runs.append(fused_run(data, 0.0, [G, G], w0, [([a[:-1] for a in ids], lrs[:-1])]))
        _, orc = make_pair(data, 0.0)
        steps, counts = _fused_steps([ids])
        w_ref, _, l_ref = ref_chain(orc, w0, steps, counts, lrs)
        np.testing.assert_array_equal(runs[0][0][0], w_ref, err_msg="fused: weights")
        np.testing.assert_array_equal(runs[0][0][1], l_ref, err_msg="fused: losses")
        if pattern == "alternate":
            np.testing.assert_array_equal(runs[1][0][0], runs[0][0][0])
        return
    ctx, data, w0, b, counts = _single_setup(S, path, seed=102)
    _, orc = make_pair(data, 0.0)
    idx = _ids(np.random.default_rng(103), data.n_rows, STEPS, b)
    try:
        ctx.set_weights(w0)
        losses = ctx.sync_steps_lr(idx.reshape(-1), b, lrs)
        w = ctx.get_weights()
        w_ref, _, l_ref = ref_chain(orc, w0, idx, counts, lrs)
        np.testing.assert_array_equal(w, w_ref, err_msg=f"{path}: weights")
        np.testing.assert_array_equal(losses, l_ref, err_msg=f"{path}: losses")
        assert not np.array_equal(w, w0)
        if pattern == "alternate":
            ctx.set_weights(w0)
            ctx.sync_steps_lr(idx[:-1].reshape(-1), b, lrs[:-1])
            np.testing.assert_array_equal(ctx.get_weights(), w, err_msg=f"{path}: a zero step moved the weights")
    finally:
        ctx.close()


# ---- 4. the 1e-20 filter at mean * lr_t -----------------------------------------------------------------------------------

def _filter_data(n_rows):
    """Rows 0 and 1 hold column 0 (value 1, label +1); row i >= 2 holds column i alone.  At w = 0 every row's gradient
    passes the gate, so a step that holds rows 0 and 1 has the gradient sum 2 on column 0 (mean 2 for one worker, 1 for
    two ranks with one row each)."""
    col = np.concatenate([[0, 0], np.arange(2, n_rows)]).astype(np.int32)
    rp = np.arange(n_rows + 1, dtype=np.int64)
    return data_from_csr(rp, col, np.ones(n_rows), np.ones(n_rows), n_rows)


@pytest.mark.parametrize("side", ["at", "above"])
@pytest.mark.parametrize("path", ["persistent", "fallback", "fused_K2"])
def test_filter_at_mean_times_lr(path, side):
    """Step 1 (not the first) puts mean * lr_t on column 0 at exactly 1e-20 (dropped: no update) or one ulp above."""
    n_rows = 128
    data = _filter_data(n_rows)
    w0 = np.zeros(n_rows)
    mean = 1.0 if path == "fused_K2" else 2.0
    lr_t = EPS / mean if side == "at" else float(np.nextafter(EPS / mean, 1.0))
    assert mean * lr_t == (EPS if side == "at" else np.nextafter(EPS, 1.0))
    lrs = np.array([2.0 ** -4, lr_t, 2.0 ** -4])
    if path == "fused_K2":
        ids = [np.array([[2, 3], [0, 4], [5, 6]], np.int32), np.array([[7, 8], [1, 9], [10, 11]], np.int32)]
        w = fused_run(data, 0.0, [2, 2], w0, [(ids, lrs)])[0][0]
        steps, counts = _fused_steps([ids])
    else:
        b = 4 if path == "persistent" else 33
        rng = np.random.default_rng(110)
        others = rng.permutation(np.arange(2, n_rows))
        steps = np.stack([others[:b], np.concatenate([[0, 1], others[b:2 * b - 2]]), others[2 * b:3 * b]]).astype(np.int32)
        counts = [b]
        ctx = make_pair(data, 0.0)[0]
        try:
            ctx.set_grid_limit(1 if path == "fallback" else 0)
            ctx.set_weights(w0)
            ctx.sync_steps_lr(steps.reshape(-1), b, lrs)
            w = ctx.get_weights()
        finally:
            ctx.close()
    _, orc = make_pair(data, 0.0)
    w_ref, _, _ = ref_chain(orc, w0, steps, counts, lrs)
    assert abs(w_ref[0]) == (0.0 if side == "at" else np.nextafter(EPS, 1.0))   # dropped, or a step of exactly that
    np.testing.assert_array_equal(w, w_ref)


# ---- 5. resident state after a table call ----------------------------------------------------------------------------

@pytest.mark.parametrize("path", ["persistent_S", "fallback_G1", "logistic", "fused_K2"])
def test_resident_state_after_a_table_call(S, path):
    def reads(ctx, n):
        w = ctx.get_weights()
        return [(ctx.eval_sums(0, n), ctx.eval_sums(0, n, w)), (ctx.eval(0, n), ctx.eval(0, n, w))]

    if path == "fused_K2":
        data, w0 = _dyadic(2047, 600, seed=120)
        rng = np.random.default_rng(121)
        ids = [_ids(rng, 600, STEPS, 150) for _ in range(2)]
        res = fused_run(data, 0.0, [5, 5], w0, [(ids, dyadic_table(STEPS))], after=lambda c: reads(c, 600))
        pairs = res[0][3] + res[1][3]
    else:
        ctx, data, w0, b, _ = _single_setup(S, path, seed=122)
        idx = _ids(np.random.default_rng(123), data.n_rows, STEPS, b)
        try:
            ctx.set_weights(w0)
            # dyadic rows and table: every weight and ||w||^2 is exact, so the resident reduction order cannot show
            ctx.sync_steps_lr(idx.reshape(-1), b, table(0.5 / b, STEPS) if path == "logistic" else dyadic_table(STEPS))
            pairs = reads(ctx, data.n_rows)
        finally:
            ctx.close()
    for resident, explicit in pairs:
        assert resident == explicit, (path, resident, explicit)


# ---- 6. errors ---------------------------------------------------------------------------------------------------------

def test_errors(S):
    from distributed_sgd_b200.native import ERR_INVALID, ERR_STATE, DsgdError, DsgdState, NativeCtx
    data, w0 = _dyadic(64, 40, seed=130)
    ctx, _ = make_pair(data, 0.0)
    try:
        ctx.set_weights(w0)
        ids = np.arange(8, dtype=np.int32)
        rc = ctx._l.dsgd_sync_steps_lr(ctx._h, ids.ctypes.data, 8, 1, None, None)      # NULL table
        assert rc == ERR_INVALID
        before = ctx.launch_count()
        assert ctx.sync_steps_lr(np.zeros(0, np.int32), 8, np.zeros(0)).size == 0      # zero steps: nothing happens
        assert ctx.launch_count() == before
        rc = ctx._l.dsgd_sync_steps_lr(ctx._h, ids.ctypes.data, 8, 0, None, None)      # ... a NULL table included
        assert rc == 0 and ctx.launch_count() == before
        np.testing.assert_array_equal(ctx.get_weights(), w0)
    finally:
        ctx.close()
    actx = NativeCtx(0, 64, 0.0, is_async=True)
    try:
        with pytest.raises(DsgdError) as e:
            actx.sync_steps_lr(np.zeros(8, np.int32), 8, [0.5])
        assert e.value.code == ERR_STATE
    finally:
        actx.close()
    # exchange-only ranks: a batch above 32 G per rank is refused before anything is launched, as with a scalar rate
    G = S // 2
    batch = 32 * G + 1
    data = _synth(2000, batch + 8, seed=131)
    ctxs = []
    try:
        for r in range(2):
            c, _ = make_pair(data, 1e-3, rank=r, world=2)
            c.set_grid_limit(G)
            c.reserve(batch, 1)
            ctxs.append(c)
        ctxs[0].xchg_attach(1, ctxs[1])
        ctxs[1].xchg_attach(0, ctxs[0])
        for c in ctxs:
            c.set_weights(np.zeros(2000))
            before = c.launch_count()
            with pytest.raises(DsgdState, match="fused peer-exchange kernel cannot take this step"):
                c.sync_steps_lr(np.arange(batch, dtype=np.int32), batch, [0.5])
            assert c.launch_count() == before
    finally:
        for c in ctxs:
            c.close()


# ---- 7. end to end ------------------------------------------------------------------------------------------------------

def test_master_fit_equals_a_chain_of_table_calls():
    """fit(learning_rate_decay, learning_rate_power, average_from=1) on dyadic rows, batch 100 over 1 250 rows (12 full
    steps and a short one per epoch, so each epoch is two calls): its calls, replayed by hand with the tables of
    learning_rates on a fresh context, give the same weights and the same average bit for bit."""
    from distributed_sgd_b200 import MasterSync, Slave, SparseSVM
    from distributed_sgd_b200.ml import EarlyStopping, learning_rates
    data, _ = _dyadic(3000, 1600, seed=140)
    train, test = data.split_at(1250)
    model = SparseSVM(0.0)
    slave = Slave(0, 0, train, model, world=1, device=0, test_data=test)
    master = MasterSync(0, train, test, model, 1, slave=slave, seed=0)
    calls = []
    ctx = master.ctx
    real_lr, real_begin = ctx.sync_steps_lr, ctx.average_begin

    def rec_lr(samples, n_per_step, lrs, want_losses=True):
        calls.append(("steps", np.array(samples), n_per_step, np.array(lrs)))
        return real_lr(samples, n_per_step, lrs, want_losses=want_losses)

    def rec_begin():
        calls.append(("begin",))
        return real_begin()

    ctx.sync_steps_lr, ctx.average_begin = rec_lr, rec_begin
    lr0, a, p = 0.5, 0.05, 0.75
    try:
        state = master.fit(np.zeros(data.dim), max_epochs=3, batch_size=100, learning_rate=lr0,
                           stopping_criterion=EarlyStopping.no_improvement(patience=5, min_delta=0.01), average_from=1,
                           learning_rate_decay=a, learning_rate_power=p)
        w_fit = ctx.get_weights()
    finally:
        slave.stop()
    steps = [c for c in calls if c[0] == "steps"]
    assert len(steps) == 6 and sum(len(c[3]) for c in steps) == 39
    np.testing.assert_array_equal(np.concatenate([c[3] for c in steps]), learning_rates(lr0, a, p, 0, 39))
    hand, _ = make_pair(train, 0.0)
    try:
        hand.set_weights(np.zeros(data.dim))
        t = 0
        for c in calls:
            if c[0] == "begin":
                hand.average_begin()
                continue
            n = len(c[3])
            hand.sync_steps_lr(c[1], c[2], learning_rates(lr0, a, p, t, n))
            t += n
        np.testing.assert_array_equal(hand.get_weights(), w_fit)
        avg, n_avg = hand.average_weights()
        assert n_avg == 26 and master.history["averaged_steps"] == 26
        np.testing.assert_array_equal(state.grad, avg)
    finally:
        hand.close()
