"""Isotonic calibration on the device (dsgd_calibrate_isotonic*, dsgd_isotonic_probabilities,
dsgd_eval_isotonic_calibration*; DESIGN.md §4.16) against the checker of oracle/iso.py run over the device's own margins.

The property the design rests on: the fit is the upper concave hull of integer points, built with exact int64 cross products,
and every block value is one IEEE division of two exact counts -- so X, Y, the block counts and the info words are ONE bit
pattern per (weights, row multiset), whatever the row form, the row order, the tile size, the grid or the model flag."""
import os

import numpy as np
import pytest

from helpers import csr
from oracle import iso

pytestmark = pytest.mark.gpu

LAM = 1e-4
N_ROWS, N_TRAIN = 100_000, 80_000
SIZES = [1, 2, 31, 32, 33, 2047, 2048, 100_000]


def trained(ctx, n_train, steps=300, batch=64, lr=0.5, seed=0):
    rng = np.random.default_rng(seed)
    ctx.set_weights(np.zeros(ctx.dim))
    ctx.sync_steps(rng.integers(0, n_train, size=steps * batch).astype(np.int32), batch, steps, lr, want_losses=False)
    return ctx.get_weights()


def bits(a):
    a = np.asarray(a)
    return a.view(np.int64) if a.dtype == np.float64 else a


def assert_same_fit(dev, ref, what=""):
    """A NativeCtx.calibrate_isotonic* result against an iso.Fit, bit for bit."""
    x, y, br, bp, info = dev
    assert np.array_equal(info, ref.info), (what, info, ref.info)
    assert np.array_equal(bits(x), bits(ref.x)), what
    assert np.array_equal(bits(y), bits(ref.y)), what
    assert np.array_equal(br, ref.block_rows) and np.array_equal(bp, ref.block_pos), what


@pytest.fixture(scope="module")
def rcv():
    """(SVM, SparseLogistic and SparseModifiedHuber contexts on the same rows, data, weights trained on the SVM context)"""
    from distributed_sgd_b200.native import NativeCtx
    from distributed_sgd_b200.utils import synthetic_rcv1
    data = synthetic_rcv1(n_rows=N_ROWS, seed=21)
    ctxs = []
    for model in ("svm", "logistic", "modified_huber"):
        c = NativeCtx(0, data.dim, LAM, model=model)
        c.load_csr(data.row_ptr, data.col, data.val, data.label)
        c.compute_dim_sparsity(N_TRAIN)
        ctxs.append(c)
    w = trained(ctxs[0], N_TRAIN)
    yield ctxs, data, w
    for c in ctxs:
        c.close()


@pytest.fixture
def tile():
    """Sets DSGD_ISOTONIC_TILE for one test and restores it."""
    old = os.environ.get("DSGD_ISOTONIC_TILE")

    def set_tile(t):
        if t is None:
            os.environ.pop("DSGD_ISOTONIC_TILE", None)
        else:
            os.environ["DSGD_ISOTONIC_TILE"] = str(t)
    yield set_tile
    set_tile(old)


# ---- the fit over trained margins -------------------------------------------------------------------------------------

def test_fit_equals_the_checker_in_every_row_form_and_model(rcv):
    (svm, logi, hub), data, w = rcv
    rng = np.random.default_rng(5)
    for n in SIZES:
        b = 0 if n == N_ROWS else 777
        ids = np.arange(b, b + n, dtype=np.int32)
        ref = iso.fit(svm.margins(ids, w), data.label[ids])
        assert ref.info[2] == n and ref.info[3] == 0
        assert_same_fit(svm.calibrate_isotonic(b, b + n, w), ref, f"range {n}")
        assert_same_fit(svm.calibrate_isotonic_samples(ids[::-1].copy(), w), ref, f"reversed {n}")
        assert_same_fit(svm.calibrate_isotonic_samples(rng.permutation(ids).astype(np.int32), w), ref, f"shuffled {n}")
        assert_same_fit(svm.calibrate_isotonic_sampled(b, b + n, 0x1234 + n, 0, n, w), ref, f"drawn {n}")
        assert_same_fit(logi.calibrate_isotonic(b, b + n, w), ref, f"logistic {n}")
        assert_same_fit(hub.calibrate_isotonic(b, b + n, w), ref, f"modified huber {n}")
        print(f"n = {n}: {ref.info[0]} blocks, {ref.info[1]} points over {ref.info[4]} distinct scores")


def test_fit_is_one_bit_pattern_for_every_tile_and_grid_limit(rcv, tile):
    (svm, _, _), data, w = rcv
    ref = iso.fit(svm.margins(np.arange(N_ROWS, dtype=np.int32), w), data.label)
    try:
        for t in (1, 2, 3, 64, 1000, 2048):
            tile(t)
            for limit in (1, 2, 0):
                svm.set_grid_limit(limit)
                assert_same_fit(svm.calibrate_isotonic(0, N_ROWS, w), ref, f"tile {t}, grid limit {limit}")
    finally:
        svm.set_grid_limit(0)


def test_w_none_reads_the_resident_weights(rcv):
    (svm, _, _), data, w = rcv
    svm.set_weights(w)
    a, b = svm.calibrate_isotonic(N_TRAIN, N_ROWS), svm.calibrate_isotonic(N_TRAIN, N_ROWS, w)
    for u, v in zip(a, b):
        assert np.array_equal(bits(u), bits(v))
    ids = np.arange(N_TRAIN, N_ROWS, dtype=np.int32)
    fit = iso.fit(svm.margins(ids, w), data.label[ids])
    assert np.array_equal(bits(svm.isotonic_probabilities(ids, fit.x, fit.y)),
                          bits(svm.isotonic_probabilities(ids, fit.x, fit.y, w)))


def test_launches_are_counted(rcv, tile):
    (svm, _, _), _, w = rcv
    tile(1000)
    before = svm.launch_count()
    svm.calibrate_isotonic(0, N_ROWS, w)
    # the curve pass (score, count, sum, emit), one tile launch, at least 7 merge rounds over >= 100 tiles, one emit
    assert svm.launch_count() - before >= 4 + 1 + 7 + 1


# ---- planted margins: one column, w = 1, so x . w is the row's value --------------------------------------------------

# the weights of a planted context: column 0 carries the margins, columns 1 and 2 (+inf and -inf) make a row's margin NaN,
# column 3 adds 0
W_PLANT = np.array([1.0, np.inf, -np.inf, 0.0])


def planted(values, labels):
    """A context whose row i holds values[i] in column 0 and 1.0 in column 3, or 1.0 in columns 1 and 2 where values[i] is
    NaN: with W_PLANT its margin is values[i] (float32-rounded), or inf - inf = NaN.  Every row has two entries."""
    from distributed_sgd_b200.native import NativeCtx
    rows = [([1, 2], [1.0, 1.0]) if np.isnan(v) else ([0, 3], [v, 1.0]) for v in values]
    data = csr(rows, np.where(np.asarray(labels) > 0, 1, -1).astype(np.int8), 4)
    ctx = NativeCtx(0, 4, LAM)
    ctx.load_csr(data.row_ptr, data.col, data.val, data.label)
    return ctx, data


PLANTS = {
    # every point on the hull: score k (margin k) has k + 2 rows, one positive -- rates 1/(k+2) strictly decrease
    "every point a vertex": lambda: (np.repeat(np.arange(400.0), np.arange(2, 402)),
                                     np.concatenate([[1] + [-1] * (k + 1) for k in range(400)])),
    # two rows per score, one positive: every point collinear, one block
    "collinear": lambda: (np.repeat(np.arange(3000.0), 2), np.tile([1, -1], 3000)),
    # collinear runs between vertices
    "collinear runs": lambda: (np.repeat(np.arange(900.0), 2),
                               np.concatenate([[1, 1]] * 300 + [[1, -1]] * 300 + [[-1, -1]] * 300)),
    # mass ties: a handful of scores shared by thousands of rows
    "mass ties": lambda: (np.random.default_rng(3).integers(-2, 3, size=20_000).astype(np.float64),
                          np.random.default_rng(4).choice([-1, 1], size=20_000)),
    # one class only
    "positives only": lambda: (np.random.default_rng(5).normal(size=5000), np.ones(5000)),
    "negatives only": lambda: (np.random.default_rng(6).normal(size=5000), -np.ones(5000)),
    # NaN margins left out, and +-0 as one score
    "nan and signed zeros": lambda: (np.array([np.nan, 0.0, -0.0, 1.0, -1.0, np.nan, 0.0, 2.0] * 500),
                                     np.array([1, 1, -1, -1, 1, -1, 1, -1] * 500)),
}


@pytest.mark.parametrize("name", sorted(PLANTS))
def test_planted_fits_equal_the_checker_at_every_tile(name, tile):
    values, labels = PLANTS[name]()
    ctx, data = planted(values, labels)
    try:
        w = W_PLANT
        ids = np.arange(data.n_rows, dtype=np.int32)
        f = ctx.margins(ids, w)
        assert np.array_equal(np.isnan(f), np.isnan(values))
        ref = iso.fit(f, data.label)
        lit = iso.fit_literal(f, data.label)
        assert np.array_equal(bits(ref.x), bits(lit.x)) and np.array_equal(bits(ref.y), bits(lit.y))
        for t in (1, 2, 7, 64, 2048):
            tile(t)
            for limit in (1, 0):
                ctx.set_grid_limit(limit)
                assert_same_fit(ctx.calibrate_isotonic(0, data.n_rows, w), ref, f"{name}: tile {t}, limit {limit}")
        ctx.set_grid_limit(0)
        assert_same_fit(ctx.calibrate_isotonic_samples(ids[::-1].copy(), w), ref, f"{name}: reversed")
        if name == "every point a vertex":
            assert ref.info[0] == 400 == ref.info[4]
        if name == "collinear":
            assert ref.info[0] == 1 and list(ref.y) == [0.5, 0.5]
    finally:
        ctx.close()


def test_all_nan_is_empty():
    from distributed_sgd_b200.native import DsgdEmpty
    ctx, data = planted([np.nan] * 40, [1, -1] * 20)
    try:
        with pytest.raises(DsgdEmpty):
            ctx.calibrate_isotonic(0, data.n_rows, W_PLANT)
    finally:
        ctx.close()


# ---- apply ------------------------------------------------------------------------------------------------------------

def test_probabilities_are_numpy_interp_bit_for_bit():
    X = np.array([-3.0, -1.5, -0.25, 0.0, 0.75, 2.0, 2.5])
    Y = np.array([0.0, 0.1, 0.1, 0.4, 0.7, 0.9, 1.0])
    between = (X[:-1] + X[1:]) / 2
    s = np.concatenate([X, between, between + 1e-3, [-10.0, 10.0, -3.5, 2.75, 0.0, -0.0, 1e-300, -1e-300], [np.nan]])
    ctx, data = planted(-s, np.ones(s.size))       # margin -s: score s
    try:
        ids = np.arange(data.n_rows, dtype=np.int32)
        w = W_PLANT
        f = ctx.margins(ids, w)
        for k in (7, 2):
            p = ctx.isotonic_probabilities(ids, X[:k], Y[:k], w)
            want = np.interp(-f, X[:k], Y[:k])
            assert np.array_equal(np.isnan(p), np.isnan(f))
            ok = ~np.isnan(f)
            assert np.array_equal(bits(p[ok]), bits(want[ok]))
            assert np.array_equal(bits(p[ok]), bits(iso.probs(f, X[:k], Y[:k])[ok]))   # NaN payloads are the device's
        p1 = ctx.isotonic_probabilities(ids, X[:1], Y[:1], w)             # one point: Y_0 everywhere, NaN for NaN
        assert np.all(p1[~np.isnan(f)] == Y[0]) and np.all(np.isnan(p1[np.isnan(f)]))
        big = np.linspace(-5.0, 5.0, 10_000)                               # past the shared-memory map: read through L2
        bigy = np.linspace(0.0, 1.0, 10_000)
        assert np.array_equal(bits(ctx.isotonic_probabilities(ids, big, bigy, w)[ok]), bits(np.interp(-f, big, bigy)[ok]))
    finally:
        ctx.close()


def test_bad_maps_are_invalid():
    from distributed_sgd_b200.native import DsgdInvalid
    ctx, data = planted([1.0, 2.0], [1, -1])
    try:
        ids = np.arange(2, dtype=np.int32)
        for X, Y in (([0.0, 0.0], [0.1, 0.2]), ([1.0, 0.0], [0.1, 0.2]), ([0.0, np.inf], [0.1, 0.2]),
                     ([0.0, 1.0], [0.1, 1.5]), ([0.0, 1.0], [np.nan, 0.5]), ([], []), ([0.0, 1.0], [0.5])):
            with pytest.raises(DsgdInvalid):
                ctx.isotonic_probabilities(ids, X, Y, W_PLANT)
            with pytest.raises(DsgdInvalid):
                ctx.eval_isotonic_calibration(0, 2, X, Y, 10, W_PLANT)
    finally:
        ctx.close()


def test_trained_probabilities_equal_the_checker(rcv):
    (svm, _, hub), data, w = rcv
    fit = svm.calibrate_isotonic(0, N_TRAIN, w)
    ids = np.arange(N_TRAIN, N_ROWS, dtype=np.int32)
    f = svm.margins(ids, w)
    for c in (svm, hub):
        p = c.isotonic_probabilities(ids, fit[0], fit[1], w)
        assert np.array_equal(bits(p), bits(np.interp(-f, fit[0], fit[1])))


# ---- quality ----------------------------------------------------------------------------------------------------------

def assert_quality(dev, ref):
    sums, rows, pos, psum, words = dev
    assert list(words) == [ref.rows, ref.left_out, ref.infinite]
    assert np.array_equal(rows, ref.bin_rows) and np.array_equal(pos, ref.bin_pos)
    assert bits(sums[:1])[0] == bits(np.array([ref.brier_sum]))[0]
    assert np.array_equal(bits(psum), bits(ref.bin_psum))
    np.testing.assert_allclose(sums[1], ref.log_loss_sum, rtol=1e-12)


def test_quality_equals_the_checker(rcv):
    (svm, _, _), data, w = rcv
    fit = svm.calibrate_isotonic(0, N_TRAIN, w)
    ids = np.arange(N_TRAIN, N_ROWS, dtype=np.int32)
    f = svm.margins(ids, w)
    for n_bins in (1, 10, 64):
        ref = iso.quality(f, data.label[ids], fit[0], fit[1], n_bins)
        assert_quality(svm.eval_isotonic_calibration(N_TRAIN, N_ROWS, fit[0], fit[1], n_bins, w), ref)
        assert_quality(svm.eval_samples_isotonic_calibration(ids[::-1].copy(), fit[0], fit[1], n_bins, w), ref)
        assert_quality(svm.eval_sampled_isotonic_calibration(N_TRAIN, N_ROWS, 99, 0, N_ROWS - N_TRAIN, fit[0], fit[1],
                                                             n_bins, w), ref)
    # on its own train rows an isotonic map puts p = 0 or 1 only where the block is pure: no infinite term
    tr = np.arange(N_TRAIN, dtype=np.int32)
    q = svm.eval_isotonic_calibration(0, N_TRAIN, fit[0], fit[1], 10, w)
    assert q[4][2] == 0
    assert_quality(q, iso.quality(svm.margins(tr, w), data.label[tr], fit[0], fit[1], 10))


def test_quality_counts_infinite_log_loss_terms():
    ctx, data = planted([1.0, 2.0, 3.0, 4.0, np.nan], [-1, -1, 1, 1, 1])
    try:
        w = W_PLANT
        X, Y = np.array([-3.5, -1.5]), np.array([0.0, 1.0])     # s = -1 -> 1 (a negative row), s = -4 -> 0 (a positive row)
        f = ctx.margins(np.arange(5, dtype=np.int32), w)
        ref = iso.quality(f, data.label, X, Y, 10)
        assert ref.infinite == 2 and ref.left_out == 1
        assert_quality(ctx.eval_isotonic_calibration(0, 5, X, Y, 10, w), ref)
    finally:
        ctx.close()


def test_isotonic_brier_is_no_larger_than_platts_when_a_is_positive(rcv):
    (svm, _, hub), data, w = rcv
    for c in (svm, hub):
        a, b, _, _ = c.calibrate(0, N_TRAIN, w)
        if not a > 0:
            continue
        fit = c.calibrate_isotonic(0, N_TRAIN, w)
        q_iso = c.eval_isotonic_calibration(0, N_TRAIN, fit[0], fit[1], 10, w)
        q_pl = c.eval_calibration(0, N_TRAIN, a, b, 10, w)
        assert q_iso[0][0] <= q_pl[0][0] * (1 + 8 * np.finfo(float).eps), (q_iso[0][0], q_pl[0][0])


def test_full_size_test_rows():
    """The full-size set's 140 000 test rows, fitted and applied against the checker."""
    from distributed_sgd_b200.native import NativeCtx
    from distributed_sgd_b200.utils import synthetic_rcv1
    data = synthetic_rcv1(n_rows=700_000, seed=0)
    n_train = 560_000
    ctx = NativeCtx(0, data.dim, LAM)
    try:
        ctx.load_csr(data.row_ptr, data.col, data.val, data.label)
        ctx.compute_dim_sparsity(n_train)
        w = trained(ctx, n_train, steps=200)
        ids = np.arange(n_train, data.n_rows, dtype=np.int32)
        f = ctx.margins(ids, w)
        ref = iso.fit(f, data.label[ids])
        assert_same_fit(ctx.calibrate_isotonic(n_train, data.n_rows, w), ref, "full-size test rows")
        p = ctx.isotonic_probabilities(ids, ref.x, ref.y, w)
        assert np.array_equal(bits(p), bits(np.interp(-f, ref.x, ref.y)))
    finally:
        ctx.close()
