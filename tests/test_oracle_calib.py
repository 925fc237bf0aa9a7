"""The calibration checker (oracle/calib.py, oracle/dsgd_oracle_calib.c) against its literal restatement, scipy's optimiser,
scikit-learn's quality numbers and hand-worked cases.  No GPU."""
import math

import numpy as np
import pytest

from oracle import calib


def scores(seed, n, sep=1.0, noise=1.5, p_pos=0.4):
    rng = np.random.default_rng(seed)
    y = np.where(rng.random(n) < p_pos, 1, -1)
    return -y * sep + rng.normal(size=n) * noise, y                  # a positive row has a negative score


@pytest.mark.parametrize("seed,n", [(0, 2), (1, 33), (2, 2048), (3, 20_000)])
def test_c_checker_against_the_literal_one(seed, n):
    f, y = scores(seed, n)
    if n == 2:
        y = np.array([1, -1])
    a, b = calib.fit(f, y), calib.fit_literal(f, y)
    assert (a.iterations, a.status, a.rows, a.nan_rows, a.evaluations) == (b.iterations, b.status, b.rows, b.nan_rows, b.evaluations)
    # long double Neumaier sums and math.fsum both round an almost exact sum: the same double but for a rare last bit
    np.testing.assert_allclose([a.a, a.b, a.objective], [b.a, b.b, b.objective], rtol=1e-13)
    t_pos, t_neg = calib.targets(f, y)[:2]
    for pt in ((0.0, 0.3), (a.a, a.b), (-0.7, 2.0)):
        np.testing.assert_allclose(calib.sums(f, y, t_pos, t_neg, *pt), calib.sums_literal(f, y, t_pos, t_neg, *pt), rtol=1e-13,
                                   atol=1e-13)


def test_optimum_against_scipy():
    from scipy.optimize import minimize
    f, y = scores(5, 5000)
    t_pos, t_neg = calib.targets(f, y)[:2]
    fit = calib.fit(f, y)
    assert fit.status == calib.CONVERGED
    res = minimize(lambda ab: calib.sums(f, y, t_pos, t_neg, ab[0], ab[1])[0], [0.0, 0.0],
                   jac=lambda ab: calib.sums(f, y, t_pos, t_neg, ab[0], ab[1])[1:3], method="BFGS", options={"gtol": 1e-9})
    assert abs(res.x[0] - fit.a) <= 1e-6 and abs(res.x[1] - fit.b) <= 1e-6
    assert fit.a > 0


def test_nan_rows_are_left_out_and_one_class_is_refused():
    f, y = scores(6, 500)
    g = f.copy()
    g[::7] = np.nan
    keep = ~np.isnan(g)
    a, b = calib.fit(g, y), calib.fit(f[keep], y[keep])
    assert (a.a, a.b, a.objective, a.iterations) == (b.a, b.b, b.objective, b.iterations)
    assert a.nan_rows == int((~keep).sum()) and a.rows == int(keep.sum())
    with pytest.raises(ValueError):
        calib.fit(f, np.ones(500))
    with pytest.raises(ValueError):
        calib.fit(np.full(4, np.nan), [1, -1, 1, -1])


def test_quality_against_scikit_learn():
    skm = pytest.importorskip("sklearn.metrics")
    skc = pytest.importorskip("sklearn.calibration")
    f, y = scores(7, 8000)
    fit = calib.fit(f, y)
    for n_bins in (1, 10, 64):
        q = calib.quality(f, y, fit.a, fit.b, n_bins)
        p, o = calib.probs(f, fit.a, fit.b), (y > 0).astype(int)
        assert q.rows == 8000 and q.left_out == 0 and q.bin_rows.sum() == 8000
        assert q.brier_sum / q.rows == pytest.approx(skm.brier_score_loss(o, p), rel=1e-12)
        assert q.log_loss_sum / q.rows == pytest.approx(skm.log_loss(o, p), rel=1e-10)
        freq, mean_p = skc.calibration_curve(o, p, n_bins=n_bins, strategy="uniform")
        s = calib.summary(q)
        filled = q.bin_rows > 0
        np.testing.assert_allclose(s["observed"][filled], freq, rtol=1e-12)
        np.testing.assert_allclose(s["mean_predicted"][filled], mean_p, rtol=1e-12)
        assert 0 <= s["ece"] <= s["mce"] <= 1


def test_two_rows_by_hand():
    """N+ = N- = 1: both targets are 2/3 and 1/3, B starts at log(1) = 0, and the first point's sums are those of p = 1/2."""
    f, y = np.array([-1.5, 2.0]), np.array([1, -1])
    t_pos, t_neg, b0, n_pos, n_neg, n_nan = calib.targets(f, y)
    assert (t_pos, t_neg, b0, n_pos, n_neg, n_nan) == (2 / 3, 1 / 3, 0.0, 1, 1, 0)
    s = calib.sums(f, y, t_pos, t_neg, 0.0, 0.0)
    assert s[0] == pytest.approx(2 * math.log(2), rel=1e-15)
    assert s[1] == pytest.approx(-1.5 * (2 / 3 - 0.5) + 2.0 * (1 / 3 - 0.5), rel=1e-14) and abs(s[2]) < 1e-16
    assert s[3:].tolist() == pytest.approx([(2.25 + 4.0) / 4, 0.5 / 4, 0.5], rel=1e-15)
    fit = calib.fit(f, y)
    assert fit.status == calib.CONVERGED and fit.a > 0


def test_separable_scores_stop_at_the_targets():
    """Without the smoothed targets A would grow without bound; with them the fitted probabilities of the outermost rows
    approach the targets and the fit converges."""
    f = np.array([-3.0, -2.0, -1.0, 1.0, 2.0, 4.0])
    y = np.array([1, 1, 1, -1, -1, -1])
    fit = calib.fit(f, y)
    assert fit.status == calib.CONVERGED and 0 < fit.a < 10
    p = calib.probs(f, fit.a, fit.b)
    assert (p[:3] > 0.5).all() and (p[3:] < 0.5).all()


def test_equal_scores_rest_on_the_ridge():
    f, y = np.full(8, 0.75), np.array([1, -1, 1, -1, -1, -1, 1, -1])
    t_pos, t_neg = calib.targets(f, y)[:2]
    s = calib.sums(f, y, t_pos, t_neg, 0.0, 0.2)
    assert abs(s[3] * s[5] - s[4] * s[4]) < 1e-15                     # singular without the ridge
    fit = calib.fit(f, y)
    assert fit.status == calib.CONVERGED and math.isfinite(fit.a) and math.isfinite(fit.b)
    # every row gets one probability: the mean target
    p = calib.probs(f, fit.a, fit.b)[0]
    assert p == pytest.approx((3 * t_pos + 5 * t_neg) / 8, abs=1e-5)


@pytest.mark.parametrize("big", [700.0, 800.0, 1e6])
def test_scores_beyond_exp(big):
    """exp(big) overflows in the unstable form; here every term stays finite and the two checkers agree."""
    f = np.array([-big, -big * 1.01, big, big * 1.02, -1.0, 1.0])
    y = np.array([1, 1, -1, -1, -1, 1])
    t_pos, t_neg = calib.targets(f, y)[:2]
    s = calib.sums(f, y, t_pos, t_neg, 1.0, 0.0)
    assert np.isfinite(s).all()
    assert s[0] == pytest.approx(sum(calib.sums_literal(f, y, t_pos, t_neg, 1.0, 0.0)[:1]), rel=1e-14)
    a, b = calib.fit(f, y), calib.fit_literal(f, y)
    assert a.status == b.status == calib.CONVERGED and a.iterations == b.iterations
    assert a.a == pytest.approx(b.a, rel=1e-12)


def test_a_term_of_2_to_the_52_makes_the_sum_nan():
    f, y = np.array([-1e9, 1e9, 3.0, -3.0]), np.array([1, -1, 1, -1])
    t_pos, t_neg = calib.targets(f, y)[:2]
    s = calib.sums(f, y, t_pos, t_neg, 0.0, 0.0)                     # f^2 p q = 2.5e17 >= 2^52
    assert math.isnan(s[3]) and np.isfinite(s[[0, 1, 2, 4, 5]]).all()
    fit, lit = calib.fit(f, y), calib.fit_literal(f, y)
    assert fit.status == lit.status == calib.NON_FINITE and math.isnan(fit.a) and math.isnan(fit.b)


def test_p_of_exactly_one_lands_in_the_last_bin():
    q = calib.quality([-1000.0, 1000.0], [1, -1], 1.0, 0.0, 4)
    assert q.bin_rows.tolist() == [1, 0, 0, 1] and q.bin_pos.tolist() == [0, 0, 0, 1] and q.bin_psum.tolist() == [0.0, 0.0, 0.0, 1.0]
