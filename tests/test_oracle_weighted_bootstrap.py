"""The grouped restatement of a weighted bootstrap replicate (tests/weighted_bootstrap_model.py) against the weighted-curve
checker over the expanded list, bit for bit, on planted cases: ties, +-0, NaN scores, zero and huge weights, one class, n = 1
and one tie group longer than several of the device's 256-element tiles."""
import math

import numpy as np
import pytest

from oracle import bootstrap as ob
from oracle import wcurve as owc
from weighted_bootstrap_model import XSum, grouped


def _bits(x):
    return np.asarray(x, np.float64).view(np.int64)


def _same(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return np.array_equal(np.isnan(a), np.isnan(b)) and np.array_equal(_bits(np.where(np.isnan(a), 0.0, a)),
                                                                     _bits(np.where(np.isnan(b), 0.0, b)))


def _check(margins, labels, c, m, model="svm"):
    margins, labels, c, m = (np.asarray(margins, np.float64), np.asarray(labels), np.asarray(c, np.float64),
                             np.asarray(m, np.int64))
    cl = c * ob.row_losses(model, margins, labels)
    r = grouped(margins, labels, c, cl, m)
    ex = np.repeat(np.arange(margins.size), m)
    assert r.size == ex.size
    if ex.size == 0:
        assert r.nan_rows == 0 and not _bits(r.wsums).any() and _bits(r.loss) == 0
        return r
    ref = owc.wcurve(margins[ex], labels[ex], c[ex], points=False)
    assert r.nan_rows == int(ref.words[7])
    assert _same(r.wsums, ref.wsums), (r.wsums, ref.wsums)
    assert _same(r.loss, owc.read(cl[ex])), (r.loss, owc.read(cl[ex]))
    return r


def _case(rng, n, levels=5, nan=0.0, zero_w=0.0):
    margins = rng.integers(-levels, levels + 1, size=n) / 4.0
    margins[rng.random(n) < nan] = np.nan
    labels = np.where(rng.random(n) < 0.4, 1, -1)
    c = rng.integers(1, 9, size=n) / 4.0
    c[rng.random(n) < zero_w] = 0.0
    return margins, labels, c


@pytest.mark.parametrize("model", ["svm", "logistic", "squared_hinge", "modified_huber"])
@pytest.mark.parametrize("seed", range(4))
def test_planted_ties_zero_weights_and_nan_scores(model, seed):
    rng = np.random.default_rng(seed)
    margins, labels, c = _case(rng, 300, nan=0.02 if seed % 2 else 0.0, zero_w=0.2)
    margins[:6] = [0.0, -0.0, 0.0, -0.0, 0.25, -0.25]       # +-0 are one score
    for b in range(3):
        _check(margins, labels, c, ob.multiplicities(0x77 + seed, b, margins.size), model)


def test_random_fp64_weights_and_class_weights():
    rng = np.random.default_rng(11)
    margins = rng.standard_normal(400)
    margins[0:392:7] = margins[1:393:7]                     # ties between otherwise distinct scores
    labels = np.where(rng.random(400) < 0.3, 1, -1)
    for c in (owc.weights(labels, 2.0, 0.5), owc.weights(labels, 1.0, 1.0, rng.random(400) * 3.0),
              owc.weights(labels, 1.0, 1.0)):
        _check(margins, labels, c, ob.multiplicities(5, 1, 400), "logistic")


def test_one_class_one_row_and_empty_replicates():
    rng = np.random.default_rng(2)
    margins, _, c = _case(rng, 50)
    _check(margins, np.ones(50), c, ob.multiplicities(1, 0, 50))
    _check(margins, -np.ones(50), c, ob.multiplicities(1, 0, 50))
    for m in ([1], [3], [0]):
        for y in (1, -1):
            _check([0.5], [y], [1.5], m)
    r = _check([np.nan], [1], [0.0], [2])                   # a NaN row of weight 0: only the row count shows it
    assert r.nan_rows == 2 and r.wsums[7] == 0.0


def test_one_group_over_several_tiles():
    rng = np.random.default_rng(4)
    n = 1500
    labels = np.where(rng.random(n) < 0.5, 1, -1)
    c = rng.integers(0, 5, size=n) / 2.0
    r = _check(np.zeros(n), labels, c, ob.multiplicities(9, 0, n))
    assert not math.isnan(r.wsums[6]) and not math.isnan(r.wsums[8])
    margins = np.zeros(n)
    margins[:10] = -1.0                                      # ten rows above the long group, ten below it
    margins[-10:] = 1.0
    _check(margins, labels, c, ob.multiplicities(9, 1, n))


def test_weights_too_large_for_the_sums_read_nan():
    rng = np.random.default_rng(6)
    margins, labels, c = _case(rng, 200)
    c[np.flatnonzero(labels < 0)[0]] = 2.0 ** 52
    r = _check(margins, labels, c, np.ones(200, np.int64))
    assert math.isnan(r.wsums[12]) and math.isnan(r.wsums[6])
    c[np.flatnonzero(labels < 0)[0]] = np.inf
    _check(margins, labels, c, np.full(200, 2))


def test_read_is_the_checker_read():
    rng = np.random.default_rng(8)
    v = rng.random(100) * 1e6
    s = XSum()
    for x in v:
        s = s.add(float(x))
    assert _bits(s.read()) == _bits(owc.read(v))
    assert math.isnan(XSum().add(2.0 ** 52).read())
