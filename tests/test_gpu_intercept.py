"""The intercept (DSGD_FLAG_INTERCEPT, fit_intercept) on the device.

The independent check is the augmented context: with lambda = 0 and no L1 penalty an intercept ctx of dimension dim is a
plain ctx of dimension dim + 1 whose rows all carry one more pair (dim, 1.0), the intercept being that column's weight.  On
dyadic rows and weights every partial sum is exact, so the SVM agrees bit for bit in every reader and training step (the
plain side's SVM steps run on the persistent kernel, the intercept's on the per-step path); the smooth models' gradients
are sums of non-dyadic values that the plain side adds with fp64 reductions in arrival order, so their gradients and
trajectories are compared at rtol 1e-12 and 1e-11 (a cancelling gradient column against the largest entry).  With beta = 0 an intercept ctx is the plain library bit for bit."""
import numpy as np
import pytest

from helpers import data_from_csr

pytestmark = pytest.mark.gpu

MODELS = ["svm", "logistic", "squared_hinge", "modified_huber"]
DIM = 700
N_ROWS = 100_003   # > 2^16 and not a multiple of any block: range sets of 1, 2 047, 2 048 and all rows below


def _rows(seed, n=N_ROWS, dim=DIM):
    """Dyadic rows: 1..12 distinct sorted columns of [0, dim), values k / 256 with k in [-512, 512] \\ {0}, labels +-1."""
    rng = np.random.default_rng(seed)
    lens = rng.integers(1, 13, size=n)
    rp = np.zeros(n + 1, np.int64)
    rp[1:] = np.cumsum(lens)
    col = np.concatenate([np.sort(rng.choice(dim, size=k, replace=False)) for k in lens]).astype(np.int32)
    val = rng.integers(1, 513, size=rp[-1]) * rng.choice([-1, 1], size=rp[-1]) / 256.0
    lab = rng.choice(np.array([-1, 1], np.int8), size=n, p=[0.7, 0.3])
    return rp, col, val.astype(np.float32), lab


def _augment(rp, col, val, dim):
    """Every row with one more pair (dim, 1.0) at its end."""
    n = rp.size - 1
    lens = np.diff(rp)
    rp2 = rp + np.arange(n + 1)
    col2 = np.empty(rp2[-1], np.int32)
    val2 = np.empty(rp2[-1], np.float32)
    last = rp2[1:] - 1
    mask = np.ones(rp2[-1], bool)
    mask[last] = False
    col2[mask], val2[mask] = col, val
    col2[last], val2[last] = dim, 1.0
    assert (np.diff(rp2) == lens + 1).all()
    return rp2, col2, val2


@pytest.fixture(scope="module")
def rows():
    return _rows(7)


def _ctx(model, data, lam, d, intercept=False):
    from distributed_sgd_b200.native import NativeCtx
    ctx = NativeCtx(0, data.dim, lam, model=model, intercept=intercept)
    ctx.load_csr(data.row_ptr, data.col, data.val, data.label)
    ctx.set_dim_sparsity(d)
    return ctx


def _trio(model, rows, lam=0.0, n=None):
    """(intercept ctx, augmented plain ctx of dim + 1, plain ctx of dim) over the first n rows."""
    rp, col, val, lab = rows
    if n is not None:
        rp, col, val, lab = rp[:n + 1], col[:rp[n]], val[:rp[n]], lab[:n]
    rng = np.random.default_rng(3)
    d = rng.integers(0, 65, size=DIM) / 64.0
    base = data_from_csr(rp, col, val, lab, DIM)
    aug = data_from_csr(*_augment(rp, col, val, DIM), lab, DIM + 1)
    return (_ctx(model, base, lam, d, True), _ctx(model, aug, lam, np.append(d, 0.0)), _ctx(model, base, lam, d))


def _weights(seed, beta):
    rng = np.random.default_rng(seed)
    w = rng.integers(-64, 65, size=DIM) / 512.0
    return np.append(w, beta)


def _close(a, b):
    """Gradients of the smooth models: fp64 reductions in arrival order, so a column whose terms cancel is compared to the
    size of the largest entry"""
    np.testing.assert_allclose(a, b, rtol=1e-12, atol=1e-12 * np.abs(b).max())


def _same(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    assert a.shape == b.shape and (a.view(np.int64) == b.view(np.int64)).all(), (a, b)


def _readers(ctx, w, n_rows, model, cls, sw):
    """Every reader an intercept ctx serves, as one list of values, over range, drawn and listed row sets."""
    ids = np.arange(0, n_rows, 3, dtype=np.int32)[:5000]
    out = {}
    for b, e in ((0, 1), (0, 2047), (5, 2053), (0, n_rows)):
        if e > n_rows:
            continue
        out[f"eval_sums{b},{e}"] = ctx.eval_sums(b, e, w)
        out[f"eval_sampled_sums{b},{e}"] = ctx.eval_sampled_sums(b, e, 11, 0, min(e - b, 1500), w)
        if model == "svm":
            out[f"eval_counts{b},{e}"] = ctx.eval_counts(b, e, w)
        if cls:
            out[f"eval_class{b},{e}"] = ctx.eval_class(b, e, w)
        if sw:
            out[f"eval_weighted{b},{e}"] = ctx.eval_weighted(b, e, w)
    out["eval_samples_sums"] = ctx.eval_samples_sums(ids, w)
    out["forward"] = ctx.forward(ids, w)
    out["margins"] = ctx.margins(ids, w)
    if model in ("logistic", "modified_huber"):
        out["probabilities"] = ctx.probabilities(ids, w)
    if cls:
        out["eval_samples_class"] = ctx.eval_samples_class(ids, w)
    if sw:
        out["eval_samples_weighted"] = ctx.eval_samples_weighted(ids, w)
    return out


def _weighting(ctxs, cls, sw, n_rows, seed=5):
    rng = np.random.default_rng(seed)
    s = rng.integers(0, 9, size=n_rows) / 4.0
    for c in ctxs:
        if cls:
            c.set_class_weights(2.0, 0.5)
        if sw:
            c.set_sample_weights(s)


@pytest.mark.parametrize("model", MODELS)
@pytest.mark.parametrize("weighting", ["none", "class", "sample"])
def test_readers_equal_the_augmented_context_and_beta_zero_the_plain_one(model, weighting, rows):
    cls, sw = weighting == "class", weighting == "sample"
    ic, aug, plain = _trio(model, rows)
    _weighting((ic, aug, plain), cls, sw, N_ROWS)
    for beta in (0.0, 0.375, -1.25):
        w = _weights(1, beta)
        a = _readers(ic, w, N_ROWS, model, cls, sw)
        b = _readers(aug, w, N_ROWS, model, cls, sw)
        for k in a:
            va, vb = a[k], b[k]
            if isinstance(va, tuple) and hasattr(va, "_fields") and "norm_squared" in va._fields:
                va, vb = va._replace(norm_squared=0.0), vb._replace(norm_squared=0.0)
            elif isinstance(va, tuple) and len(va) == 3:
                va, vb = va[:2], vb[:2]
            _same(np.asarray(va, np.float64), np.asarray(vb, np.float64))
        if beta == 0.0:   # the plain library, ||w||^2 included
            c = _readers(plain, w[:DIM], N_ROWS, model, cls, sw)
            for k in a:
                _same(np.asarray(a[k], np.float64), np.asarray(c[k], np.float64))
        else:             # beta is not in ||w||^2
            assert ic.eval_sums(0, 10, w)[2] == plain.eval_sums(0, 10, w[:DIM])[2]


def _flat(v):
    """A reader's result (arrays, tuples of them, scalars) as one float64 vector"""
    if isinstance(v, np.ndarray):
        return v.astype(np.float64).ravel()
    if isinstance(v, (tuple, list)):
        return np.concatenate([_flat(x) for x in v]) if len(v) else np.zeros(0)
    return np.array([float(v)])


def _scoring(ctx, w, sw):
    """The metrics, curve, calibration and isotonic readers over range, drawn and listed row sets"""
    ids = np.arange(1, 30_000, 7, dtype=np.int32)
    out = {"metrics": ctx.eval_metrics(0, N_ROWS, w), "metrics_2048": ctx.eval_metrics(5, 2053, w),
           "sampled_metrics": ctx.eval_sampled_metrics(0, 50_000, 13, 0, 4000, w),
           "samples_metrics": ctx.eval_samples_metrics(ids, w),
           "curve": ctx.eval_curve(0, 20_000, w), "samples_curve": ctx.eval_samples_curve(ids, w),
           "sampled_curve": ctx.eval_sampled_curve(0, 50_000, 13, 0, 4000, w)}
    a, b, _, _ = cal = ctx.calibrate(0, 20_000, w)
    out["platt"] = cal
    out["platt_samples"] = ctx.calibrate_samples(ids, w)
    out["platt_prob"] = ctx.calibrated_probabilities(ids, a, b, w)
    out["platt_quality"] = ctx.eval_calibration(20_000, 40_000, a, b, 10, w)
    iso = ctx.calibrate_isotonic(0, 20_000, w)
    out["isotonic"] = iso
    out["isotonic_prob"] = ctx.isotonic_probabilities(ids, iso[0], iso[1], w)
    out["isotonic_quality"] = ctx.eval_isotonic_calibration(20_000, 40_000, iso[0], iso[1], 10, w)
    if sw:
        out["weighted_curve"] = ctx.eval_weighted_curve(0, 20_000, w)
        wa, wb = ctx.calibrate_weighted(0, 20_000, w)[:2]
        out["weighted_platt"] = ctx.calibrate_weighted(0, 20_000, w)
        out["weighted_platt_quality"] = ctx.eval_weighted_calibration(20_000, 40_000, wa, wb, 10, w)
        wiso = ctx.calibrate_isotonic_weighted(0, 20_000, w)
        out["weighted_isotonic"] = wiso
        out["weighted_isotonic_quality"] = ctx.eval_weighted_isotonic_calibration(20_000, 40_000, wiso[0], wiso[1], 10, w)
    return out


@pytest.mark.parametrize("model", ["svm", "logistic", "modified_huber"])
@pytest.mark.parametrize("weighting", ["none", "sample"])
def test_metrics_curves_and_calibration_score_with_the_intercept(model, weighting, rows):
    """Every ranking and calibration reader ranks the scores x . w + beta: equal to the augmented context bit for bit, and
    at beta = 0 to the plain library"""
    sw = weighting == "sample"
    ic, aug, plain = _trio(model, rows)
    _weighting((ic, aug, plain), False, sw, N_ROWS)
    for beta in (0.0, 0.375):
        w = _weights(1, beta)
        a = _scoring(ic, w, sw)
        b = _scoring(aug, w, sw)
        for k in a:
            _same(_flat(a[k]), _flat(b[k]))
        if beta == 0.0:
            c = _scoring(plain, w[:DIM], sw)
            for k in a:
                _same(_flat(a[k]), _flat(c[k]))
    # the intercept moves the scores: the confusion counts at beta = 0 and at beta = 4 differ
    assert not np.array_equal(ic.eval_metrics(0, N_ROWS, _weights(1, 0.0)), ic.eval_metrics(0, N_ROWS, _weights(1, 4.0)))


@pytest.mark.parametrize("model", MODELS)
@pytest.mark.parametrize("weighting", ["none", "class", "sample"])
def test_gradient_carries_the_intercept_last(model, weighting, rows):
    cls, sw = weighting == "class", weighting == "sample"
    ic, aug, plain = _trio(model, rows)
    _weighting((ic, aug, plain), cls, sw, N_ROWS)
    ids = np.random.default_rng(2).integers(0, N_ROWS, size=3000).astype(np.int32)
    for beta in (0.0, 0.625):
        w = _weights(4, beta)
        gi, li = ic.gradient(ids, w, want_loss=True)
        ga, la = aug.gradient(ids, w, want_loss=True)
        assert gi.shape == (DIM + 1,) and li == la
        if model == "svm":
            _same(gi, ga)
        else:
            _close(gi, ga)
        if beta == 0.0:
            gp, lp = plain.gradient(ids, w[:DIM], want_loss=True)
            assert lp == li
            if model == "svm":
                _same(gi[:DIM], gp)
            else:
                _close(gi[:DIM], gp)


def _train(ctx, ids, n_per, n_steps, lr, table, avg, workers):
    if workers:
        ctx.set_workers(workers, len(workers))
    if avg:
        ctx.average_begin()
    if table:
        lrs = lr * 0.5 ** (np.arange(n_steps) % 3)   # dyadic rates keep every sum exact
        losses = ctx.sync_steps_lr(ids, n_per, lrs)
    else:
        losses = ctx.sync_steps(ids, n_per, n_steps, lr)
    out = [losses, ctx.get_weights()]
    if avg:
        out.append(ctx.average_weights()[0])
        ctx.average_end()
    return out


@pytest.mark.parametrize("model", MODELS)
@pytest.mark.parametrize("case", ["plain", "class", "sample", "table_avg", "workers", "workers_class"])
def test_training_equals_the_augmented_context(model, case, rows):
    cls, sw = "class" in case, case == "sample"
    n = 20_000
    ic, aug, _ = _trio(model, rows, n=n)
    _weighting((ic, aug), cls, sw, n)
    w0 = _weights(9, 0.25)
    ic.set_weights(w0)
    aug.set_weights(w0)
    n_per, n_steps = 96, 12
    ids = np.random.default_rng(8).integers(0, n, size=n_per * n_steps).astype(np.int32)
    workers = [40, 56] if case.startswith("workers") else None
    a = _train(ic, ids, n_per, n_steps, 0.0625, case == "table_avg", case == "table_avg", workers)
    b = _train(aug, ids, n_per, n_steps, 0.0625, case == "table_avg", case == "table_avg", workers)
    assert a[1][DIM] != 0.25   # the intercept moved
    for x, y in zip(a, b):
        if model == "svm":
            _same(x, y)
        else:
            np.testing.assert_allclose(x, y, rtol=1e-11, atol=1e-300)
    # the resident weights after the steps are what every reader with w = None reads
    ids_e = np.arange(0, n, 7, dtype=np.int32)
    _same(ic.margins(ids_e), ic.margins(ids_e, a[1]))
    # ||w||^2 of the resident weights is k_update's block sum, of explicit ones k_prepare's: the same value in another order
    res, req = ic.eval_sums(0, n), ic.eval_sums(0, n, a[1])
    _same(res[:2], req[:2])
    assert res[2] == pytest.approx(req[2], rel=1e-14)
    if model == "svm":
        _same(ic.gradient(ids_e[:500]), ic.gradient(ids_e[:500], a[1]))
    else:
        _close(ic.gradient(ids_e[:500]), ic.gradient(ids_e[:500], a[1]))


@pytest.mark.parametrize("model", ["svm", "logistic"])
def test_the_intercept_is_left_out_of_every_penalty(model, rows):
    """At lambda > 0 and with an L1 penalty: beta's gradient has no c, beta's step has no soft threshold, and neither
    ||w||^2, ||w||_1 nor the non-zero count sees beta.  One step from w0 against the step restated here."""
    n = 5000
    ic = _trio(model, rows, lam=0.125, n=n)[0]
    w0 = _weights(6, 0.5)
    ic.set_weights(w0)
    ids = np.arange(0, 200, dtype=np.int32)
    g = ic.gradient(ids)
    ic_l1 = _trio(model, rows, lam=0.125, n=n)[0]
    ic_l1.set_weights(w0)
    ic_l1.set_l1(10.0)   # a threshold of lr * 10 = 0.625 would zero beta = 0.5 if it applied
    for c in (ic, ic_l1):
        c.sync_steps(ids, ids.size, 1, 0.0625)
    filt = (lambda v: v if abs(v) > 1e-20 else 0.0)
    beta1 = filt(0.5 - filt(filt(g[DIM] / 1.0) * 0.0625))
    assert ic.get_weights()[DIM] == beta1 and ic_l1.get_weights()[DIM] == beta1
    ic0 = _trio(model, rows, lam=0.0, n=n)[0]   # lambda = 0: c = 0
    ic0.set_weights(w0)
    g0 = ic0.gradient(ids)
    assert g[DIM] == g0[DIM] != 0.0                   # c is not added to beta's entry ...
    assert (g[:DIM][g0[:DIM] != 0.0] != g0[:DIM][g0[:DIM] != 0.0]).any()   # ... but to the weights' entries
    wl = ic_l1.get_weights()
    l1, nnz = ic_l1.weights_l1()
    assert nnz == np.count_nonzero(wl[:DIM]) and l1 == pytest.approx(np.abs(wl[:DIM]).sum(), rel=1e-15)
    assert ic.eval_sums(0, 10)[2] == pytest.approx(float(np.dot(ic.get_weights()[:DIM], ic.get_weights()[:DIM])), rel=1e-14)


def test_device_lengths(rows):
    from distributed_sgd_b200.native import DsgdInvalid
    ic, _, _ = _trio("svm", rows, n=3000)
    with pytest.raises(DsgdInvalid, match=f"expected {DIM + 1}"):
        ic.set_weights(np.zeros(DIM))
    ic.set_weights(_weights(1, 0.5))
    assert ic.get_weights()[DIM] == 0.5


def test_a_peer_exchange_only_rank_is_refused_before_any_launch(rows):
    """Two ranks on one GPU wired with the peer exchange only (no dsgd_comm_init): a plain ctx would take the fused kernel,
    an intercept ctx has no fused form and is refused naming the intercept, its weights untouched."""
    from distributed_sgd_b200.native import DsgdState, NativeCtx
    rp, col, val, lab = rows
    data = data_from_csr(rp[:1001], col[:rp[1000]], val[:rp[1000]], lab[:1000], DIM)
    ctxs = []
    for r in range(2):
        ctx = NativeCtx(0, DIM, 0.0, rank=r, world=2, intercept=True)
        ctx.load_csr(data.row_ptr, data.col, data.val, data.label)
        ctx.set_dim_sparsity(np.zeros(DIM))
        ctx.set_grid_limit(8)
        ctxs.append(ctx)
    ctxs[0].xchg_attach(1, ctxs[1])
    ctxs[1].xchg_attach(0, ctxs[0])
    w0 = _weights(1, 0.5)
    ctxs[0].set_weights(w0)
    with pytest.raises(DsgdState, match="the intercept takes the NCCL allreduce path"):
        ctxs[0].sync_steps(np.arange(32, dtype=np.int32), 32, 1, 0.1)
    _same(ctxs[0].get_weights(), w0)
    assert ctxs[0].xchg_stats()[2] == 0   # the fused kernel never ran


def test_master_sync_fit_with_an_intercept():
    """Thinned positives (about 10 %): MasterSync.fit returns dim + 1 weights with a non-zero intercept, and every epoch's
    loss is a separate evaluation of the weights it reports."""
    from distributed_sgd_b200.core.master import Master
    from distributed_sgd_b200.core.slave import Slave
    from distributed_sgd_b200.ml import SparseLogistic
    from distributed_sgd_b200.ml.early_stopping import no_improvement
    rp, col, val, lab = _rows(11, n=6000, dim=300)
    rng = np.random.default_rng(1)
    lab = np.where(rng.random(lab.size) < 0.1, 1, -1).astype(np.int8)
    train = data_from_csr(rp[:5001], col[:rp[5000]], val[:rp[5000]], lab[:5000], 300)
    test = data_from_csr(rp[5000:] - rp[5000], col[rp[5000]:], val[rp[5000]:], lab[5000:], 300)
    model = SparseLogistic(1e-4, fit_intercept=True)
    slave = Slave(0, 0, train, model, False, test_data=test)
    master = Master.create(0, train, test, model, False, 1, slave=slave)
    seen = []
    state = master.fit(np.zeros(301), 3, 64, 0.05, no_improvement(patience=10, min_delta=0.0),
                       on_epoch=lambda e, h: seen.append((h["loss"], slave.ctx.get_weights())))
    w = state.grad
    assert w.shape == (301,) and w[300] != 0.0
    for loss, we in seen:
        assert master.local_loss(we) == pytest.approx(loss, rel=1e-13)
    slave.stop()


@pytest.mark.parametrize("model", MODELS)
@pytest.mark.parametrize("l1", [0.0, 1e-4])
def test_training_at_lambda_against_the_restatement(model, l1):
    """RCV1-shaped fp32 rows, lambda > 0, with and without L1, a decaying rate table: 10 steps against the literal
    restatement of the intercept's step (oracle/scala_semantics_intercept.py), losses at rtol 1e-12 and the weights at rtol
    1e-11 against the largest entry (the device sums a row's terms in its fold order, the restatement in column order)."""
    from distributed_sgd_b200.native import NativeCtx
    from distributed_sgd_b200.utils import synthetic_rcv1
    from oracle import scala_semantics_intercept as si
    data = synthetic_rcv1(n_rows=3000, seed=12)
    lam, batch, n_steps = 1e-3, 32, 10
    ctx = NativeCtx(0, data.dim, lam, model=model, intercept=True)
    ctx.load_csr(data.row_ptr, data.col, data.val, data.label)
    d = ctx.compute_dim_sparsity(2400)
    if l1:
        ctx.set_l1(l1)
    rng = np.random.default_rng(3)
    w0 = np.append(rng.normal(0.0, 0.01, size=data.dim), -0.25)
    ctx.set_weights(w0)
    ids = rng.integers(0, 2400, size=batch * n_steps).astype(np.int32)
    lrs = 0.05 / (1.0 + 0.1 * np.arange(n_steps))   # small enough that no squared-hinge loss reaches 2^52
    losses = ctx.sync_steps_lr(ids, batch, lrs)
    w = ctx.get_weights()
    rws = si.csr_rows(data.row_ptr, data.col, data.val)
    w_ref, l_ref = si.steps(rws, data.label, d, w0, ids, batch, model, lam, lrs, l1)
    np.testing.assert_allclose(losses, l_ref, rtol=1e-12)
    np.testing.assert_allclose(w, w_ref, rtol=1e-11, atol=1e-11 * np.abs(w_ref).max())
    assert w[data.dim] != -0.25
