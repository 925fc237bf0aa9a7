"""Class weights on the device (dsgd_set_class_weights, dsgd_eval*_class) against their checker (oracle/cw.py):

* (1, 1), set or never set, is the unweighted library: same weights, losses, gradients and launch counts; so is (1, 1) set
  again after other weights.
* Dyadic rows and dyadic weights, rates, lambda and dimSparsity: weights bit for bit and per-step losses to the rounding of
  ||w||^2, one worker and virtual workers,
  combined with averaging, a rate table and L1; a weight of 0 for one class.
* RCV1-shaped fp32 rows: 20-step trajectories of both models within the tolerances of the unweighted tests; dsgd_gradient
  at 1, 2 047, 2 048 and 262 144 ids.
* The per-class evaluations in all three forms: integers equal the checker's and add up to dsgd_eval_counts and
  dsgd_eval_metrics of the same rows; logistic sums have the same bits in any row order.
* Errors: invalid weights, an async context, a rank wired with the peer exchange only, and the *_class calls' codes.
"""
import numpy as np
import pytest

from helpers import csr, make_pair
from oracle import cw as CW
from oracle.logistic import LogisticOracle
from oracle.oracle import Oracle

pytestmark = pytest.mark.gpu


def dyadic_data(seed, n_rows=3000, dim=512, pos_share=0.3):
    """Rows of dyadic values (multiples of 1/8 up to 2, either sign) of 0 to 160 non-zeros (several 128-pair chunks)."""
    rng = np.random.default_rng(seed)
    rows = []
    for i in range(n_rows):
        k = int(rng.choice([0, 1, 3, 8, 40, 130, 160], p=[0.05, 0.1, 0.3, 0.3, 0.15, 0.05, 0.05]))
        c = np.sort(rng.choice(dim, size=min(k, dim), replace=False))
        k = len(c)
        rows.append((c, rng.integers(1, 17, size=k) / 8.0 * rng.choice([-1.0, 1.0], size=k)))
    lab = np.where(rng.random(n_rows) < pos_share, 1, -1).astype(np.int8)
    return csr(rows, lab, dim), rng


def pair(data, lam, logistic=False, n_train=None):
    """(NativeCtx, checker) with the rows loaded and dimSparsity installed."""
    from distributed_sgd_b200.native import NativeCtx
    if not logistic:
        return make_pair(data, lam, n_train=n_train)
    ctx = NativeCtx(0, data.dim, lam, logistic=True)
    ctx.load_csr(data.row_ptr, data.col, data.val, data.label)
    orc = LogisticOracle(data.row_ptr, data.col, data.val, data.label, data.dim, lam)
    d = orc.dim_sparsity(data.n_rows if n_train is None else n_train)
    orc.set_dim_sparsity(d)
    ctx.set_dim_sparsity(d)
    return ctx, orc


def dyadic_w0(rng, dim):
    return rng.integers(-8, 9, size=dim) / 16.0


def dyadic_pair(data, lam, logistic=False):
    """pair() with a dyadic dimSparsity (every third column 1/4) instead of the rows' 1 / (df + 1): with dyadic rows, weights,
    rates and lambda every sum of a step is then exact, so it has the same bits in any order."""
    ctx, orc = pair(data, lam, logistic)
    d = np.zeros(data.dim)
    d[::3] = 0.25
    orc.set_dim_sparsity(d)
    ctx.set_dim_sparsity(d)
    return ctx, orc


# ---- the default is the unweighted library -------------------------------------------------------------------------------

@pytest.mark.parametrize("logistic,batch,workers", [(False, 64, None), (False, 32 * 132 + 1, None), (False, 64, [40, 24]),
                                                    (True, 64, None)])
def test_unit_weights_are_the_unweighted_library(logistic, batch, workers):
    from distributed_sgd_b200.utils import synthetic_rcv1
    data = synthetic_rcv1(n_rows=6000, seed=3)
    rng = np.random.default_rng(1)
    idx = rng.integers(0, 6000, size=batch * 3).astype(np.int32)
    runs = []
    for mode in ("never", "explicit", "back"):
        ctx, _ = pair(data, 1e-5, logistic)
        try:
            if workers:
                ctx.set_workers(workers, len(workers))
            if mode == "explicit":
                ctx.set_class_weights(1.0, 1.0)
            if mode == "back":
                ctx.set_class_weights(2.0, 0.5)
                ctx.sync_steps(idx[:batch], batch, 1, 0.5)
                ctx.set_class_weights(1.0, 1.0)
            assert ctx.get_class_weights() == (1.0, 1.0) and ctx.info()["class_weights"] == [1.0, 1.0]
            ctx.set_weights(np.zeros(data.dim))
            n0 = ctx.launch_count()
            losses = ctx.sync_steps(idx, batch, 3, 0.5)
            g, gl = ctx.gradient(idx[:100], want_loss=True)
            runs.append((losses, ctx.get_weights(), g, gl, ctx.launch_count() - n0))
        finally:
            ctx.close()
    for r in runs[1:]:
        assert r[4] == runs[0][4]
        if logistic:   # its fp64 scatter adds in the order of arrival: equal to rounding from run to run
            for a, b in zip(r[:4], runs[0][:4]):
                np.testing.assert_allclose(a, b, rtol=1e-11, atol=1e-15)
        else:
            assert np.array_equal(r[0], runs[0][0]) and np.array_equal(r[1], runs[0][1]) and np.array_equal(r[2], runs[0][2])
            assert r[3] == runs[0][3]


# ---- bit for bit on dyadic rows ------------------------------------------------------------------------------------------

@pytest.mark.parametrize("lam", [2.0 ** -6, 0.0])
@pytest.mark.parametrize("wp,wn", [(4.0, 0.25), (0.0, 2.0), (0.5, 0.0)])
@pytest.mark.parametrize("batch,workers", [(1, None), (64, None), (132, None), (32 * 132 + 1, None), (64, [40, 24]),
                                           (88, [50, 31, 7])])
def test_dyadic_steps_bit_for_bit(wp, wn, batch, workers, lam):
    """lam = 0 keeps the loss path bit for bit at every step: the loss is then the weighted per-class sum over the batch alone
    (counters -> weighted double -> the update kernel, or the persistent kernel's packed hinge word)."""
    data, rng = dyadic_data(11)
    ctx, orc = dyadic_pair(data, lam)
    try:
        counts = workers or [batch]
        if workers:
            ctx.set_workers(workers, len(workers))
        ctx.set_class_weights(wp, wn)
        w0 = dyadic_w0(rng, data.dim)
        lrs = [0.5, 0.25, 0.125, 0.0625]
        idx = rng.integers(0, data.n_rows, size=batch * len(lrs)).astype(np.int32)
        ctx.set_weights(w0)
        # two calls in a row without set_weights; the second with a rate table
        l0 = ctx.sync_steps(idx[:batch * 2], batch, 2, 0.5)
        l1 = ctx.sync_steps_lr(idx[batch * 2:], batch, lrs[2:])
        w_ref, l_ref = CW.sync_steps(orc, w0, idx, counts, [0.5, 0.5] + lrs[2:], wp, wn)
        if len(counts) == 3:   # the mean over three workers leaves the dyadic grid: sums depend on their order in the last bits
            np.testing.assert_allclose(ctx.get_weights(), w_ref, rtol=1e-12, atol=1e-15)
            np.testing.assert_allclose(np.concatenate([l0, l1]), l_ref, rtol=1e-12)
        else:
            assert np.array_equal(ctx.get_weights(), w_ref)
            # the first loss is exact; later weights carry more bits than a sum of their squares holds, so ||w||^2 rounds
            # by the order of the sum
            assert l0[0] == l_ref[0]
            if lam == 0.0:
                assert np.array_equal(np.concatenate([l0, l1]), l_ref)
            np.testing.assert_allclose(np.concatenate([l0, l1]), l_ref, rtol=1e-13)
    finally:
        ctx.close()


@pytest.mark.parametrize("label", [1, -1])
def test_one_cta_holds_32_rows_of_one_class_at_hinge_2(label):
    """One CTA (grid limit 1) takes all 32 rows of a step, every one of one class and mispredicted (hinge 2 each): that
    class's 16-bit half of the CTA's hinge word holds its maximum, 64, and the other half 0."""
    rows = [(np.array([0]), np.array([1.0]))] * 32
    data = csr(rows, np.full(32, label, np.int8), 4)
    ctx, orc = make_pair(data, 0.0)
    try:
        ctx.set_grid_limit(1)
        w0 = np.array([float(label), 0.0, 0.0, 0.0])   # y * dot > 0 -> the prediction is -y
        ctx.set_weights(w0)
        ce = ctx.eval_class(0, 32)
        assert (ce.loss_pos + ce.loss_neg, ce.correct_pos + ce.correct_neg, ce.n_pos + ce.n_neg) == (64.0, 0, 32)
        ctx.set_class_weights(0.25, 8.0)
        n0 = ctx.launch_count()
        loss = ctx.sync_steps(np.tile(np.arange(32, dtype=np.int32), 2), 32, 2, 2.0 ** -8)
        assert ctx.launch_count() - n0 == 2   # the persistent kernel and its record initialisation
        w_ref, l_ref = CW.sync_steps(orc, w0, np.tile(np.arange(32), 2), [32], [2.0 ** -8] * 2, 0.25, 8.0)
        assert loss[0] == (0.25 if label > 0 else 8.0) * 64 / 32
        assert np.array_equal(loss, l_ref) and np.array_equal(ctx.get_weights(), w_ref)
    finally:
        ctx.close()


def long_dyadic_data(seed, n_rows=400, dim=512):
    """Dyadic rows of 0, 128, 160 or 300 non-zeros: several chunks each, and 32 of them per CTA pass what a stage holds, so
    rows are left out of the chunk list and taken whole from global memory."""
    rng = np.random.default_rng(seed)
    rows = []
    for i in range(n_rows):
        k = int(rng.choice([0, 128, 160, 300]))
        c = np.sort(rng.choice(dim, size=k, replace=False))
        rows.append((c, rng.integers(1, 17, size=k) / 8.0 * rng.choice([-1.0, 1.0], size=k)))
    return csr(rows, rng.choice(np.array([-1, 1], np.int8), size=n_rows), dim), rng


@pytest.mark.parametrize("lam", [2.0 ** -6, 0.0])
@pytest.mark.parametrize("grid", [1, 2, 7, 0])
@pytest.mark.parametrize("long_rows", [False, True])
def test_persistent_kernel_at_every_grid_size(grid, long_rows, lam):
    """The persistent kernel's weighted form at 1, 2, 7 and one CTA per SM, batches of 1, G, 32 G rows (persistent) and
    32 G + 1 (the per-step path), alternating, in calls that follow each other without set_weights; stages with empty rows,
    rows of several chunks and rows outside the chunk list.  At lambda = 0 weights and losses (the weighted hinge sum
    alone) bit for bit; with lambda > 0 to rounding, each call continued from the device's weights."""
    data, rng = long_dyadic_data(15) if long_rows else dyadic_data(14)
    ctx, orc = dyadic_pair(data, lam)
    try:
        G = grid or ctx.info()["sm_count"]
        ctx.set_grid_limit(grid)
        ctx.set_class_weights(4.0, 0.25)
        w = dyadic_w0(rng, data.dim)
        ctx.set_weights(w)
        for batch, persistent in ((1, True), (32 * G + 1, False), (G, True), (32 * G, True), (32 * G + 1, False), (32 * G, True)):
            lrs = [2.0 ** -3, 2.0 ** -4, 2.0 ** -5]
            idx = rng.integers(0, data.n_rows, size=batch * len(lrs)).astype(np.int32)
            n0 = ctx.launch_count()
            losses = ctx.sync_steps_lr(idx, batch, lrs)
            assert (ctx.launch_count() - n0 == 2) == persistent
            w, l_ref = CW.sync_steps(orc, w, idx, [batch], lrs, 4.0, 0.25)
            if lam == 0.0:
                assert np.array_equal(ctx.get_weights(), w) and np.array_equal(losses, l_ref)
            else:   # over these 18 steps the weights outgrow the dyadic grid: c = 2 lambda (w . d) rounds by the sum's order
                np.testing.assert_allclose(ctx.get_weights(), w, rtol=1e-12, atol=1e-15)
                np.testing.assert_allclose(losses, l_ref, rtol=1e-12)
                w = ctx.get_weights()
    finally:
        ctx.close()


@pytest.mark.parametrize("avg,table,l1", [(a, t, l) for a in (False, True) for t in (False, True) for l in (False, True)])
def test_persistent_kernel_every_combination(avg, table, l1):
    data, rng = dyadic_data(16)
    ctx, orc = dyadic_pair(data, 2.0 ** -6)
    try:
        ctx.set_class_weights(0.5, 2.0)
        lam1 = 2.0 ** -7 if l1 else 0.0
        if l1:
            ctx.set_l1(lam1)
        w0 = dyadic_w0(rng, data.dim)
        lrs = [0.25, 0.125, 0.0, 0.0625] if table else [0.125] * 4
        idx = rng.integers(0, data.n_rows, size=256 * 4).astype(np.int32)
        ctx.set_weights(w0)
        if avg:
            ctx.average_begin()
        n0 = ctx.launch_count()
        losses = ctx.sync_steps_lr(idx, 256, lrs) if table else ctx.sync_steps(idx, 256, 4, 0.125)
        assert ctx.launch_count() - n0 == 2
        avg_ref = np.zeros(data.dim)
        w_ref, l_ref = CW.sync_steps(orc, w0, idx, [256], lrs, 0.5, 2.0, lambda1=lam1, avg_sum=avg_ref)
        assert np.array_equal(ctx.get_weights(), w_ref) and losses[0] == l_ref[0]
        np.testing.assert_allclose(losses, l_ref, rtol=1e-13)
        if avg:
            a, n_avg = ctx.average_weights()
            assert n_avg == 4
            np.testing.assert_allclose(a, avg_ref / 4, rtol=1e-15, atol=0)
    finally:
        ctx.close()


@pytest.mark.parametrize("logistic", [False, True])
def test_dyadic_steps_with_averaging_rate_table_and_l1(logistic):
    data, rng = dyadic_data(12)
    ctx, orc = dyadic_pair(data, 2.0 ** -6, logistic)
    try:
        ctx.set_class_weights(4.0, 0.25)
        ctx.set_l1(2.0 ** -7)
        w0 = dyadic_w0(rng, data.dim)
        lrs = [0.5, 0.25, 0.0, 0.125]
        idx = rng.integers(0, data.n_rows, size=64 * len(lrs)).astype(np.int32)
        ctx.set_weights(w0)
        ctx.average_begin()
        losses = ctx.sync_steps_lr(idx, 64, lrs)
        avg, n_avg = ctx.average_weights()
        avg_ref = np.zeros(data.dim)
        w_ref, l_ref = CW.sync_steps(orc, w0, idx, [64], lrs, 4.0, 0.25, logistic=logistic, lambda1=2.0 ** -7, avg_sum=avg_ref)
        assert n_avg == len(lrs)
        if logistic:
            np.testing.assert_allclose(ctx.get_weights(), w_ref, rtol=1e-11, atol=1e-15)
            np.testing.assert_allclose(losses, l_ref, rtol=1e-11)
        else:
            assert np.array_equal(ctx.get_weights(), w_ref) and losses[0] == l_ref[0]
            np.testing.assert_allclose(losses, l_ref, rtol=1e-13)
            assert np.array_equal(avg * n_avg, avg_ref) or np.allclose(avg, avg_ref / n_avg, rtol=1e-15, atol=0)
    finally:
        ctx.close()


# ---- RCV1-shaped fp32 rows -----------------------------------------------------------------------------------------------

@pytest.mark.parametrize("logistic", [False, True])
@pytest.mark.parametrize("workers", [None, [40, 24]])
def test_rcv1_shaped_trajectory(logistic, workers):
    from distributed_sgd_b200.utils import synthetic_rcv1
    data = synthetic_rcv1(n_rows=8000, seed=21)
    ctx, orc = pair(data, 1e-5, logistic)
    try:
        if workers:
            ctx.set_workers(workers, len(workers))
        ctx.set_class_weights(2.0, 0.5)
        rng = np.random.default_rng(2)
        steps, batch = 20, 64
        idx = rng.integers(0, data.n_rows, size=batch * steps).astype(np.int32)
        ctx.set_weights(np.zeros(data.dim))
        losses = ctx.sync_steps(idx, batch, steps, 0.5)
        w = ctx.get_weights()
        w_ref, l_ref = CW.sync_steps(orc, np.zeros(data.dim), idx, workers or [batch], [0.5] * steps, 2.0, 0.5,
                                     logistic=logistic)
        np.testing.assert_allclose(losses, l_ref, rtol=1e-11)
        assert np.array_equal(w != 0, w_ref != 0)
        if logistic:
            assert np.max(np.abs(w - w_ref)) <= 1e-11 * np.max(np.abs(w_ref))
        else:
            np.testing.assert_allclose(w, w_ref, rtol=1e-11, atol=1e-15)
    finally:
        ctx.close()


@pytest.mark.parametrize("logistic", [False, True])
@pytest.mark.parametrize("n", [1, 2047, 2048, 262144])
def test_weighted_gradient_request(logistic, n):
    from distributed_sgd_b200.utils import synthetic_rcv1
    data = synthetic_rcv1(n_rows=20000, seed=22)
    ctx, orc = pair(data, 1e-5, logistic)
    try:
        ctx.set_class_weights(2.0, 0.5)
        rng = np.random.default_rng(3)
        w = rng.standard_normal(data.dim) * 0.05
        idx = rng.integers(0, data.n_rows, size=n).astype(np.int32)
        g, loss = ctx.gradient(idx, w, want_loss=True)
        g_ref, loss_ref, _ = CW.gradient(orc, w, idx, 2.0, 0.5, logistic=logistic)
        assert abs(loss - loss_ref) <= 1e-11 * abs(loss_ref)
        assert np.array_equal(g != 0, g_ref != 0)
        # per entry: a sum of the rows' terms in another order, against the sum of the terms' magnitudes in that column
        # (every term is at most max(w_pos, w_neg) |x_j| = 2 |x_j|)
        mag = np.zeros(data.dim)
        for r, m in zip(*np.unique(idx, return_counts=True)):
            sl = slice(data.row_ptr[r], data.row_ptr[r + 1])
            mag[data.col[sl]] += 2.0 * m * np.abs(data.val[sl].astype(np.float64))
        assert np.all(np.abs(g - g_ref) <= 1e-13 * mag + 1e-15 * np.abs(g_ref))
        # the unweighted calls are untouched by the weights
        assert ctx.eval_sums(0, 3000, w)[0] == pytest.approx(sum(CW.eval_class(orc, w, np.arange(3000), logistic)[0]), rel=1e-12)
    finally:
        ctx.close()


# ---- the per-class evaluations -------------------------------------------------------------------------------------------

@pytest.mark.parametrize("logistic", [False, True])
def test_eval_class_against_the_checker_and_the_unweighted_calls(logistic):
    from distributed_sgd_b200.utils import synthetic_rcv1
    data = synthetic_rcv1(n_rows=120000, seed=23)
    ctx, orc = pair(data, 1e-5, logistic)
    try:
        rng = np.random.default_rng(4)
        w = rng.standard_normal(data.dim) * 0.05
        ctx.set_class_weights(3.0, 0.5)   # the evaluations do not read them
        for n in (1, 31, 32, 33, 2047, 2048, 100000):
            b = int(rng.integers(0, data.n_rows - n + 1))
            ids = np.arange(b, b + n, dtype=np.int32)
            ce = ctx.eval_class(b, b + n, w)
            sums_ref, counts_ref = CW.eval_class(orc, w, ids, logistic)
            assert [ce.correct_pos, ce.correct_neg, ce.n_pos, ce.n_neg] == list(counts_ref)
            assert ce.n_pos == int(np.count_nonzero(data.label[ids] > 0)) and ce.n_pos + ce.n_neg == n
            loss_sum, correct, n2 = ctx.eval_sums(b, b + n, w)
            assert correct == ce.correct_pos + ce.correct_neg and n2 == ce.norm_squared
            m = ctx.eval_metrics(b, b + n, w)
            assert (ce.n_pos, ce.n_neg) == (m[0] + m[1] + m[2], m[3] + m[4] + m[5])
            assert (ce.correct_pos, ce.correct_neg) == (m[0], m[4])
            if logistic:
                np.testing.assert_allclose([ce.loss_pos, ce.loss_neg], sums_ref, rtol=1e-12)
                assert abs(ce.loss_pos + ce.loss_neg - loss_sum) <= 2 * np.spacing(loss_sum)
            else:
                assert [ce.loss_pos, ce.loss_neg] == list(sums_ref) and ce.loss_pos + ce.loss_neg == loss_sum
                assert ctx.eval_counts(b, b + n, w)[0] == int(ce.loss_pos + ce.loss_neg)
            # the same rows as a list, reversed and shuffled, and as a drawn sample of all of them: the same bits
            for order in (ids, ids[::-1], rng.permutation(ids)):
                assert ctx.eval_samples_class(order, w) == ce
            if n > 1:
                assert ctx.eval_sampled_class(b, b + n, 12345, 0, n, w) == ce
                lo, hi = ctx.eval_sampled_class(b, b + n, 12345, 0, n // 2, w), ctx.eval_sampled_class(b, b + n, 12345, n // 2, n, w)
                assert tuple(x + y for x, y in zip(lo[3:], hi[3:])) == ce[3:]
        one = np.flatnonzero(data.label > 0)[:500].astype(np.int32)
        ce = ctx.eval_samples_class(one, w)
        assert ce.n_neg == 0 and ce.loss_neg == 0.0 and ce.correct_neg == 0 and ce.n_pos == 500
    finally:
        ctx.close()


# ---- errors --------------------------------------------------------------------------------------------------------------

def test_invalid_weights_and_async_context():
    from distributed_sgd_b200.native import DsgdInvalid, DsgdState, NativeCtx
    ctx = NativeCtx(0, 16, 0.1)
    try:
        for bad in ((-1.0, 1.0), (1.0, -0.5), (float("nan"), 1.0), (1.0, float("inf"))):
            with pytest.raises(DsgdInvalid):
                ctx.set_class_weights(*bad)
        assert ctx.get_class_weights() == (1.0, 1.0)
        ctx.set_class_weights(0.0, 0.0)
        assert ctx.get_class_weights() == (0.0, 0.0)
    finally:
        ctx.close()
    a = NativeCtx(0, 16, 0.1, is_async=True)
    try:
        with pytest.raises(DsgdState):
            a.set_class_weights(2.0, 1.0)
        assert a.get_class_weights() == (1.0, 1.0)
    finally:
        a.close()


def test_eval_class_error_codes():
    from distributed_sgd_b200.native import DsgdEmpty, DsgdRange, DsgdState, NativeCtx
    ctx = NativeCtx(0, 16, 0.1)
    try:
        with pytest.raises(DsgdState):
            ctx.eval_class(0, 1)
        data, _ = dyadic_data(13, n_rows=50, dim=16)
        ctx.load_csr(data.row_ptr, data.col, data.val, data.label)
        with pytest.raises(DsgdRange):
            ctx.eval_class(0, 51)
        with pytest.raises(DsgdEmpty):
            ctx.eval_class(5, 5)
        with pytest.raises(DsgdEmpty):
            ctx.eval_samples_class(np.zeros(0, np.int32))
        with pytest.raises(DsgdRange):
            ctx.eval_samples_class(np.array([50], np.int32))
        with pytest.raises(DsgdEmpty):
            ctx.eval_sampled_class(0, 50, 1, 3, 3)
    finally:
        ctx.close()


def test_exchange_only_ranks_refuse_before_launching():
    """Two ranks on one GPU wired with the peer exchange only: with class weights the call fails before anything is launched."""
    from distributed_sgd_b200.native import DsgdState
    from distributed_sgd_b200.utils import synthetic_rcv1
    data = synthetic_rcv1(n_rows=2000, seed=5)
    ctxs = [make_pair(data, 1e-5, rank=r, world=2)[0] for r in range(2)]
    try:
        ctxs[0].xchg_attach(1, ctxs[1])
        ctxs[1].xchg_attach(0, ctxs[0])
        ctxs[0].set_class_weights(2.0, 0.5)
        n0 = ctxs[0].launch_count()
        with pytest.raises(DsgdState, match="class weights"):
            ctxs[0].sync_steps(np.arange(32, dtype=np.int32), 32, 1, 0.5)
        assert ctxs[0].launch_count() == n0
    finally:
        for c in ctxs:
            c.close()


# ---- MasterSync.fit on an unbalanced set ---------------------------------------------------------------------------------

def test_master_sync_fit_balanced_matches_the_checker_replay():
    from distributed_sgd_b200 import EarlyStopping, Master, Slave, SparseSVM
    from distributed_sgd_b200.core import Group
    from distributed_sgd_b200.core.master import EpochDraw
    from distributed_sgd_b200.ml import SplitStrategy
    from distributed_sgd_b200.utils import synthetic_rcv1
    from distributed_sgd_b200.utils.dataset import Data
    full = synthetic_rcv1(n_rows=12000, seed=31)
    rng = np.random.default_rng(5)
    pos, neg = np.flatnonzero(full.label > 0), np.flatnonzero(full.label < 0)
    keep = np.sort(np.concatenate([neg, rng.choice(pos, size=len(neg) // 9, replace=False)]))   # about 10 % positives
    lens = np.diff(full.row_ptr)[keep]
    rp = np.concatenate([[0], np.cumsum(lens)]).astype(np.int64)
    take = np.concatenate([np.arange(full.row_ptr[r], full.row_ptr[r + 1]) for r in keep])
    data = Data(rp, full.col[take], full.val[take], full.label[keep], full.dim)
    train, test = data.split_at(int(data.n_rows * 0.8))
    model = SparseSVM(1e-5, class_weight="balanced")
    slave = Slave(0, 0, train, model, False, test_data=test)
    try:
        n_pos = int(np.count_nonzero(train.label > 0))
        wp, wn = train.n_rows / (2.0 * n_pos), train.n_rows / (2.0 * (train.n_rows - n_pos))
        assert slave.class_weight == (wp, wn) == slave.ctx.get_class_weights()
        master = Master.create(0, train, test, model, False, 1, slave=slave, group=Group(), seed=7)
        state = master.fit(np.zeros(data.dim), 2, 64, 0.5, EarlyStopping.no_improvement(patience=5, min_delta=0.0))
        orc = Oracle(data.row_ptr, data.col, data.val, data.label, data.dim, 1e-5)
        orc.set_dim_sparsity(model.dim_sparsity)
        w = np.zeros(data.dim)
        for epoch in range(2):
            for st in EpochDraw.draw(7, epoch, SplitStrategy.vanilla(train.n_rows, 1), 64):
                w, _ = CW.sync_steps(orc, w, st[0], [len(st[0])], [0.5], wp, wn)
        np.testing.assert_allclose(state.grad, w, rtol=1e-10, atol=1e-14)
        rep = master.local_class_report(state.grad, test_data=True)
        sums, counts = CW.eval_class(orc, state.grad, np.arange(train.n_rows, data.n_rows))
        assert [rep["correct_pos"], rep["correct_neg"], rep["n_pos"], rep["n_neg"]] == list(counts)
        assert master.local_loss(state.grad, test_data=True) == pytest.approx(rep["weighted_loss"], rel=1e-14)
    finally:
        slave.stop()
