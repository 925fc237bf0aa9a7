"""The weighted calibration checker (oracle/dsgd_oracle_wcalib.c) against its literal restatement (oracle/wcalib.py), the
unweighted calibration checker at c = 1, the repeated-row identity of integer weights, and scikit-learn's weighted Platt
fit.  CPU only."""
import math

import numpy as np
import pytest

from oracle import calib as oc
from oracle import wcalib as ow


def scores(seed, n, p_pos=0.4):
    rng = np.random.default_rng(seed)
    y = np.where(rng.random(n) < p_pos, 1, -1)
    f = -y * 1.0 + rng.normal(0.0, 1.5, n)
    return f, y


def weight_sets(n, seed):
    rng = np.random.default_rng(seed)
    rand = rng.random(n) * 3.0
    ints = rng.integers(0, 5, n).astype(np.float64)
    zeros = np.where(rng.random(n) < 0.3, 0.0, rand)
    tiny = np.where(rng.random(n) < 0.5, 2.0 ** -165, rand)
    big = np.where(rng.random(n) < 0.1, 2.0 ** 40, rand)
    return {"random": rand, "integer": ints, "zeros": zeros, "tiny": tiny, "big": big}


def bits(a):
    return np.asarray(a, dtype=np.float64).view(np.int64)


@pytest.mark.parametrize("seed,n", [(1, 1), (2, 37), (3, 500), (4, 3000)])
def test_quality_and_targets_equal_the_literal_restatement(seed, n):
    f, y = scores(seed, n)
    f[::17] = np.nan
    for name, c in weight_sets(n, seed).items():
        for a, b in ((1.3, -0.2), (0.0, 0.0), (4.0, 1.0)):
            q = ow.quality(f, y, c, a, b, 10)
            s, bw, bp, bs, rows, out = ow.quality_literal(f, y, c, a, b, 10)
            assert np.array_equal(bits(q.sums), bits(s)), name
            for got, want in ((q.bin_weight, bw), (q.bin_pos_weight, bp), (q.bin_psum, bs)):
                assert np.array_equal(bits(got), bits(want)), name
            assert (q.rows, q.left_out) == (rows, out)
        ws, tg = ow.targets(f, y, c)
        ws_l, tg_l = ow.targets_literal(f, y, c)
        assert np.array_equal(bits(ws), bits(ws_l)) and np.array_equal(bits(tg), bits(tg_l)), name


@pytest.mark.parametrize("seed,n", [(5, 40), (6, 700), (7, 4000)])
def test_unit_weights_equal_the_unweighted_checker(seed, n):
    f, y = scores(seed, n)
    f[::23] = np.nan
    c = np.ones(n)
    wf, uf = ow.fit(f, y, c), oc.fit(f, y)
    assert bits([wf.a, wf.b, wf.objective]).tolist() == bits([uf.a, uf.b, uf.objective]).tolist()
    assert (wf.iterations, wf.status, wf.rows, wf.nan_rows, wf.evaluations) == \
        (uf.iterations, uf.status, uf.rows, uf.nan_rows, uf.evaluations)
    t = oc.targets(f, y)
    assert (wf.w_pos, wf.w_neg, wf.nan_weight) == (t[3], t[4], float(t[5]))
    wq, uq = ow.quality(f, y, c, wf.a, wf.b, 10), oc.quality(f, y, wf.a, wf.b, 10)
    assert np.array_equal(wq.bin_weight, uq.bin_rows) and np.array_equal(wq.bin_pos_weight, uq.bin_pos)
    assert wq.sums[2] == uq.rows and (wq.rows, wq.left_out) == (uq.rows, uq.left_out)
    # the unweighted checker sums in long double, this one exactly: they agree to the last bits
    np.testing.assert_allclose(wq.sums[:2], [uq.brier_sum, uq.log_loss_sum], rtol=1e-14)
    np.testing.assert_allclose(wq.bin_psum, uq.bin_psum, rtol=1e-14)


@pytest.mark.parametrize("seed", [8, 9])
def test_integer_weights_equal_repeated_rows(seed):
    n = 600
    f, y = scores(seed, n)
    c = np.random.default_rng(seed).integers(0, 4, n).astype(np.float64)
    rep = np.repeat(np.arange(n), c.astype(int))
    wf, uf = ow.fit(f, y, c), oc.fit(f[rep], y[rep])
    ws, tg = ow.targets(f, y, c)
    t = oc.targets(f[rep], y[rep])
    assert bits(tg).tolist() == bits(t[:3]).tolist()
    assert abs(wf.a - uf.a) <= 1e-8 * max(1.0, abs(uf.a)) and abs(wf.b - uf.b) <= 1e-8 * max(1.0, abs(uf.b))
    assert wf.objective == pytest.approx(uf.objective, rel=1e-10)
    wq, uq = ow.quality(f, y, c, wf.a, wf.b, 10), oc.quality(f[rep], y[rep], wf.a, wf.b, 10)
    assert np.array_equal(wq.bin_weight, uq.bin_rows) and np.array_equal(wq.bin_pos_weight, uq.bin_pos)


def test_zero_weight_rows_form_no_terms_and_an_empty_class_is_refused():
    f, y = scores(10, 300)
    c = np.random.default_rng(10).random(300) + 0.5
    c[::3] = 0.0
    keep = c > 0
    wf, sub = ow.fit(f, y, c), ow.fit(f[keep], y[keep], c[keep])
    assert bits([wf.a, wf.b, wf.objective]).tolist() == bits([sub.a, sub.b, sub.objective]).tolist()
    f2 = f.copy()
    f2[~keep] = np.inf      # a zero-weight row's term is never formed, so its score cannot spoil a sum
    assert ow.fit(f2, y, c).status == oc.CONVERGED
    c_pos_zero = np.where(y > 0, 2.0 ** -162, c)
    with pytest.raises(ValueError):
        ow.fit(f, y, c_pos_zero)
    assert ow.targets(f, y, c_pos_zero)[0][0] == 0.0


def test_a_weighted_term_of_2_to_the_52_is_non_finite():
    f, y = scores(11, 50)
    c = np.ones(50)
    c[0] = 2.0 ** 53
    assert ow.fit(f, y, c).status == oc.NON_FINITE
    q = ow.quality(f, y, c, 1.0, 0.0, 10)
    assert math.isnan(q.sums[2])


def _objective(f, y, c, a, b):
    ws, tg = ow.targets(f, y, c)
    return ow.sums(f, y, c, tg[0], tg[1], a, b)[0]


@pytest.mark.parametrize("seed", [12, 13, 14])
def test_objective_no_worse_than_scikit_learn(seed):
    skc = pytest.importorskip("sklearn.calibration")
    n = 2000
    f, y = scores(seed, n)
    c = np.random.default_rng(seed).random(n) * 3.0
    fit = ow.fit(f, y, c)
    assert fit.status == oc.CONVERGED
    # scikit-learn's sigmoid is 1 / (1 + exp(A f + B)) over the decision values with y in {0, 1}
    a_sk, b_sk = skc._sigmoid_calibration(f, (y > 0).astype(int), sample_weight=c)
    F_sk = _objective(f, y, c, float(a_sk), float(b_sk))
    assert fit.objective <= F_sk + 1e-9 * abs(F_sk)


# ---- the weighted isotonic fit -----------------------------------------------------------------------------------------

from oracle import iso as oi  # noqa: E402


def iso_sets():
    rng = np.random.default_rng(20)
    n = 400
    f, y = scores(21, n)
    c = rng.random(n) * 3.0
    ties = np.round(f * 4) / 4
    yield "random", f, y, c
    yield "ties", ties, y, c
    yield "one class", f, np.ones(n), c
    yield "nan", np.where(rng.random(n) < 0.1, np.nan, f), y, c
    s = np.arange(40, dtype=np.float64)                      # every point a vertex: strictly concave counts
    yield "vertices", -s, np.ones(40), 1.0 / (s + 1.0)
    yield "collinear", -np.arange(30.0), np.where(np.arange(30) % 2 == 0, 1, -1), np.ones(30)
    z = c.copy()
    z[np.argmax(-f)] = 0.0
    z[np.argmin(-f)] = 0.0
    yield "zero weight at the extremes", f, y, z
    yield "tiny and big", f, y, np.where(rng.random(n) < 0.3, 2.0 ** -165, np.where(rng.random(n) < 0.1, 2.0 ** 40, c))


@pytest.mark.parametrize("name,f,y,c", list(iso_sets()), ids=lambda v: v if isinstance(v, str) else "")
def test_isotonic_checker_equals_the_pav_restatement(name, f, y, c):
    fit = ow.fit_isotonic(f, y, c)
    x, yv, bw, bp = ow.fit_isotonic_pav(f, y, c)
    for a, b in ((fit.x, x), (fit.y, yv), (fit.block_weight, bw), (fit.block_pos_weight, bp)):
        assert np.asarray(a).tobytes() == np.asarray(b).tobytes(), name
    if name == "zero weight at the extremes":
        keep = c > 0
        assert -f[~keep].max() not in fit.x and -f[~keep].min() not in fit.x


def test_isotonic_at_unit_weights_equals_the_unweighted_checker():
    f, y = scores(22, 800)
    f[::31] = np.nan
    w, u = ow.fit_isotonic(f, y, np.ones(f.size)), oi.fit(f, y)
    assert w.x.tobytes() == u.x.tobytes() and w.y.tobytes() == u.y.tobytes()
    assert np.array_equal(w.block_weight, u.block_rows) and np.array_equal(w.block_pos_weight, u.block_pos)
    assert list(w.info) == [int(v) for v in u.info]


def test_isotonic_integer_weights_equal_repeated_rows():
    f, y = scores(23, 500)
    c = np.random.default_rng(23).integers(0, 4, 500).astype(np.float64)
    rep = np.repeat(np.arange(500), c.astype(int))
    w, u = ow.fit_isotonic(f, y, c), oi.fit(f[rep], y[rep])
    assert w.x.tobytes() == u.x.tobytes() and w.y.tobytes() == u.y.tobytes()
    assert np.array_equal(w.block_weight, u.block_rows)


def test_isotonic_errors():
    f, y = scores(24, 50)
    with pytest.raises(ValueError):
        ow.fit_isotonic(f, y, np.zeros(50))
    with pytest.raises(ow.RangeError):
        ow.fit_isotonic(f, y, np.where(np.arange(50) == 0, 2.0 ** 52, 1.0))      # a weight of 2^52
    big = np.full(50, 2.0 ** 51)
    ow.fit_isotonic(f, y, big)                                # 50 * 2^51 < 2^96: accepted, and 2^64 is too


def test_isotonic_against_scikit_learn():
    isr = pytest.importorskip("sklearn.isotonic")
    for name, f, y, c in iso_sets():
        if name in ("one class", "nan", "tiny and big"):
            continue
        fit = ow.fit_isotonic(f, y, c)
        m = isr.IsotonicRegression(increasing=True, out_of_bounds="clip").fit(-f, (y > 0).astype(float), sample_weight=c)
        if m.X_thresholds_.size != fit.x.size or not np.array_equal(m.X_thresholds_, fit.x):
            continue   # scikit-learn pools running float means: a near-tie can pool differently (as test_oracle_isotonic)
        np.testing.assert_allclose(m.y_thresholds_, fit.y, rtol=0, atol=8 * np.finfo(float).eps)
