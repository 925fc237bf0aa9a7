"""The isotonic checker (oracle/dsgd_oracle_iso.c) against its literal restatement (pool-adjacent-violators over
fractions.Fraction, oracle/iso.py) and against scikit-learn's IsotonicRegression; CPU only."""
import math
from fractions import Fraction

import numpy as np
import pytest

from oracle import iso


def bits(a):
    return np.asarray(a, dtype=np.float64).view(np.int64)


def same(a, b):
    assert np.array_equal(a.info, b.info), (a.info, b.info)
    assert np.array_equal(bits(a.x), bits(b.x)) and np.array_equal(bits(a.y), bits(b.y))
    assert np.array_equal(a.block_rows, b.block_rows) and np.array_equal(a.block_pos, b.block_pos)


def random_set(rng, n, levels=None, nan=0.0):
    f = rng.normal(size=n) if levels is None else rng.integers(0, levels, size=n).astype(np.float64)
    p = 1.0 / (1.0 + np.exp(f))                                     # positives more likely at low margins
    y = np.where(rng.random(n) < p, 1, -1)
    if nan:
        f[rng.random(n) < nan] = np.nan
    return f, y


HAND = {
    "ties": (np.array([0.0, 0.0, 1.0, 1.0, 1.0, 2.0]), np.array([1, -1, 1, 1, -1, -1])),
    "positives only": (np.array([3.0, 1.0, 2.0, 2.0]), np.array([1, 1, 1, 1])),
    "negatives only": (np.array([3.0, 1.0, 2.0]), np.array([-1, -1, -1])),
    "every point a vertex": (np.repeat(np.arange(50.0), np.arange(2, 52)),
                             np.concatenate([[1] + [-1] * (k + 1) for k in range(50)])),
    "collinear": (np.repeat(np.arange(20.0), 2), np.tile([1, -1], 20)),
    "collinear runs": (np.repeat(np.arange(30.0), 2), np.concatenate([[1, 1]] * 10 + [[1, -1]] * 10 + [[-1, -1]] * 10)),
    "nan scores": (np.array([np.nan, 1.0, np.nan, -1.0, 0.0, -0.0]), np.array([1, 1, -1, -1, 1, -1])),
    "one row": (np.array([0.5]), np.array([1])),
}


@pytest.mark.parametrize("name", sorted(HAND))
def test_checker_equals_the_fraction_pav_on_hand_built_sets(name):
    f, y = HAND[name]
    same(iso.fit(f, y), iso.fit_literal(f, y))


def test_hand_built_answers():
    fit = iso.fit(*HAND["every point a vertex"])
    assert fit.info[0] == 50 and fit.info[4] == 50 and fit.info[1] == 50
    fit = iso.fit(*HAND["collinear"])
    assert fit.info[0] == 1 and list(fit.y) == [0.5, 0.5] and list(fit.x) == [-19.0, 0.0]
    fit = iso.fit(*HAND["positives only"])
    assert list(fit.y) == [1.0, 1.0] and list(fit.block_rows) == [4]
    fit = iso.fit(*HAND["nan scores"])
    assert fit.info[3] == 2 and fit.info[2] == 4 and fit.info[4] == 3          # -0 and +0 are one score
    assert all(math.copysign(1.0, v) > 0 for v in fit.x if v == 0.0)
    with pytest.raises(ValueError):
        iso.fit(np.array([np.nan, np.nan]), np.array([1, -1]))


@pytest.mark.parametrize("seed", range(12))
def test_checker_equals_the_fraction_pav_on_random_sets(seed):
    rng = np.random.default_rng(seed)
    n = int(rng.integers(1, 3000))
    f, y = random_set(rng, n, levels=None if seed % 3 else int(rng.integers(1, 40)), nan=0.05 if seed % 4 == 0 else 0.0)
    if np.all(np.isnan(f)):
        return
    a, b = iso.fit(f, y), iso.fit_literal(f, y)
    same(a, b)
    # the hull property, exactly: block values strictly decrease with the score, each is fl(pos / rows)
    vals = [Fraction(int(p), int(r)) for p, r in zip(a.block_pos, a.block_rows)]
    assert all(u < v for u, v in zip(vals, vals[1:]))
    assert sorted(set(a.y.tolist())) == sorted({float(np.float64(p) / np.float64(r)) for p, r in zip(a.block_pos, a.block_rows)})
    assert int(np.sum(a.block_rows)) == a.info[2]


@pytest.mark.parametrize("seed", range(8))
def test_random_sets_agree_with_scikit_learn(seed):
    sk = pytest.importorskip("sklearn.isotonic")
    rng = np.random.default_rng(100 + seed)
    n = int(rng.integers(50, 5000))
    f, y = random_set(rng, n, levels=None if seed % 2 else 25)
    fit = iso.fit(f, y)
    s, o = -f, (y > 0).astype(np.float64)
    reg = sk.IsotonicRegression(increasing=True, out_of_bounds="clip").fit(s, o)
    if not np.array_equal(reg.X_thresholds_, fit.x):
        pytest.skip("scikit-learn's rounded pooling merged differently here (see DESIGN.md §4.16)")
    # scikit-learn pools running float means, so a pooled value can be off the exact fl(pos / rows) by more than one
    # rounding: 2 ulp has been seen on these sets
    ulp = np.spacing(np.maximum(np.abs(fit.y), np.abs(reg.y_thresholds_)))
    assert np.all(np.abs(reg.y_thresholds_ - fit.y) <= 4 * ulp)
    probe = np.concatenate([fit.x, (fit.x[:-1] + fit.x[1:]) / 2, [fit.x[0] - 1, fit.x[-1] + 1]])
    equal = reg.y_thresholds_ == fit.y
    if np.all(equal):
        want = np.interp(probe, fit.x, fit.y)
        assert np.array_equal(bits(iso.probs(-probe, fit.x, fit.y)), bits(want))


def test_scikit_learn_merges_blocks_the_exact_hull_keeps_apart():
    """Two adjacent blocks whose exact values differ by less than their rounding: 1/3 against 33333333/100000000 are
    distinct rationals, so the hull keeps both blocks, but scikit-learn's floating-point means may compare them as it
    likes; the probabilities agree to an ulp either way."""
    sk = pytest.importorskip("sklearn.isotonic")
    f = np.concatenate([np.full(3, 1.0), np.full(30, 0.0)])
    y = np.concatenate([[1, -1, -1], [1] * 10 + [-1] * 20])
    fit = iso.fit(f, y)
    assert fit.info[0] == 1                                              # 1/3 == 10/30: collinear, one block
    reg = sk.IsotonicRegression(increasing=True, out_of_bounds="clip").fit(-f, (y > 0).astype(float))
    assert np.allclose(reg.predict(-f), iso.probs(f, fit.x, fit.y), rtol=0, atol=1e-15)


def test_interp_is_numpy_interp_bit_for_bit():
    rng = np.random.default_rng(7)
    X = np.sort(rng.normal(size=40))
    Y = np.sort(rng.random(40))
    s = np.concatenate([X, rng.normal(size=2000) * 2, [0.0, -0.0, X[0] - 1, X[-1] + 1, np.inf, -np.inf]])
    got = iso.probs(-s, X, Y)
    assert np.array_equal(bits(got), bits(np.interp(s, X, Y)))
    assert np.isnan(iso.probs(np.array([np.nan]), X, Y)[0])


def test_quality_sums():
    rng = np.random.default_rng(9)
    f, y = random_set(rng, 3000, nan=0.01)
    fit = iso.fit(f[:2000], y[:2000])
    q = iso.quality(f[2000:], y[2000:], fit.x, fit.y, 10)
    ok = ~np.isnan(f[2000:])
    p = iso.probs(f[2000:], fit.x, fit.y)[ok]
    o = (y[2000:][ok] > 0).astype(float)
    assert q.rows == int(ok.sum()) and q.left_out == int((~ok).sum())
    exact = sum(Fraction(v) for v in (p - o) ** 2)
    assert abs(Fraction(q.brier_sum) - exact) <= Fraction(np.spacing(q.brier_sum))
    with np.errstate(divide="ignore"):
        terms = np.where(o > 0, -np.log(p), -np.log1p(-p))
    assert q.infinite == int(np.sum(np.isinf(terms)))
    assert math.isclose(q.log_loss_sum, math.fsum(terms[np.isfinite(terms)]), rel_tol=1e-12)
    assert int(q.bin_rows.sum()) == q.rows
