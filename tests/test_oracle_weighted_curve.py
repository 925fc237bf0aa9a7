"""The weighted-curve checker (oracle/dsgd_oracle_wcurve.c, the checker of dsgd_eval_*weighted_curve) against a literal
restatement in exact fractions, scikit-learn's weighted ROC AUC, average precision and roc_curve, the unweighted curve
checker at c = 1, the expanded-list identity for integer weights and zero-weight rows left out.  Its read() is pinned to
the model of the device's fixed-point reader (tests/loss_sum_model.py).  No GPU."""
import math
from fractions import Fraction

import numpy as np
import pytest
from sklearn.metrics import average_precision_score, roc_auc_score, roc_curve

from oracle import curve as oc
from oracle import wcurve as ow
from oracle.oracle import Oracle
from loss_sum_model import device_model


def empty_rows(labels, dim=8):
    """An oracle over len(labels) empty rows: the margins come from the caller."""
    n = len(labels)
    return Oracle(np.zeros(n + 1, np.int64), np.zeros(0, np.int32), np.zeros(0, np.float32), np.asarray(labels, np.int8),
                  dim, 0.0)


def tied_margins(rng, n, levels=6):
    vals = np.concatenate([[0.0, -0.0], rng.integers(-4, 5, size=levels) / 4.0])
    return vals[rng.integers(0, len(vals), size=n)]


def within_ulps(x, exact, k):
    return abs(Fraction(x) - exact) <= k * Fraction(math.ulp(float(exact)))


def test_read_is_the_device_reader():
    rng = np.random.default_rng(0)
    for _ in range(50):
        v = np.concatenate([rng.random(40) * 10.0 ** rng.integers(-50, 15), [0.0, 2.0 ** -161, 2.0 ** -160, 3.0 * 2 ** -162],
                            rng.integers(0, 1000, 5).astype(float)])
        assert ow.read(v) == device_model(v)
    assert math.isnan(ow.read([1.0, 2.0 ** 52])) and math.isnan(device_model([1.0, 2.0 ** 52]))
    assert ow.read([2.0 ** 52 - 1, 0.5]) == device_model([2.0 ** 52 - 1, 0.5])


@pytest.mark.parametrize("seed", range(12))
def test_auc_and_ap_within_four_ulps_of_the_exact_values(seed):
    """Each of AUC and AP rounds several times between the exact sums and the result: every read() within one ulp, every
    product and ratio within half an ulp.  Four ulps bounds what those steps reach together (2.5 seen over 300 draws)."""
    rng = np.random.default_rng(seed)
    n = int(rng.integers(2, 60))
    m = tied_margins(rng, n) if seed % 2 else rng.standard_normal(n)
    y = np.where(rng.random(n) < 0.4, 1, -1)
    c = rng.random(n) * 3.0
    c[rng.random(n) < 0.2] = 0.0
    got = ow.wcurve(m, y, c)
    auc, ap = ow.literal(m, y, c)
    for x, ex in ((got.auc, auc), (got.ap, ap)):
        if isinstance(ex, float) and math.isnan(ex):
            assert math.isnan(x)
        else:
            assert within_ulps(x, Fraction(ex), 4), (x, float(ex))


@pytest.mark.parametrize("seed", range(8))
def test_against_scikit_learn_with_positive_weights(seed):
    rng = np.random.default_rng(100 + seed)
    n = 300
    m = tied_margins(rng, n, 20) if seed % 2 else rng.standard_normal(n)
    y = np.where(rng.random(n) < 0.3, 1, -1)
    c = rng.random(n) * 4.0 + 0.01
    got = ow.wcurve(m, y, c)
    s = -m + 0.0
    assert got.auc == pytest.approx(roc_auc_score(y > 0, s, sample_weight=c), rel=1e-12)
    assert got.ap == pytest.approx(average_precision_score(y > 0, s, sample_weight=c), rel=1e-12)
    fpr, tpr, thr = roc_curve(y > 0, s, sample_weight=c, drop_intermediate=False)
    assert np.array_equal(thr[1:], got.thr)
    np.testing.assert_allclose(tpr[1:], got.tpw / got.wsums[11], rtol=1e-12)
    np.testing.assert_allclose(fpr[1:], got.fpw / got.wsums[12], rtol=1e-12)


@pytest.mark.parametrize("seed", range(6))
def test_at_unit_weights_it_is_the_curve_checker(seed):
    rng = np.random.default_rng(200 + seed)
    n = 500
    m = tied_margins(rng, n) if seed % 2 else rng.standard_normal(n)
    if seed == 4:
        m[rng.integers(0, n, 3)] = np.nan
    y = np.where(rng.random(n) < 0.5, 1, -1)
    got = ow.wcurve(m, y, np.ones(n))
    ref = oc.curve(empty_rows(y), np.zeros(8), margins=m)
    assert np.array_equal(got.thr, ref.thr) and np.array_equal(got.tpw, ref.tp) and np.array_equal(got.fpw, ref.fp)
    assert np.array_equal(got.wsums[:8], got.words.astype(np.float64))
    assert got.wsums[8] == ow.read(ref.v)   # S_ap has the limbs of the unweighted S
    if seed == 4:
        assert math.isnan(got.ap) and math.isnan(got.auc) and got.wsums[7] == 3.0
    else:
        assert got.ap == ow.read(ref.v) / len(ref.v)
        assert abs(got.ap - ref.ap) <= math.ulp(ref.ap)


@pytest.mark.parametrize("seed", range(6))
def test_integer_weights_are_the_expanded_list(seed):
    rng = np.random.default_rng(300 + seed)
    n = 200
    m = tied_margins(rng, n)
    y = np.where(rng.random(n) < 0.5, 1, -1)
    c = rng.integers(0, 5, n).astype(np.float64)
    got = ow.wcurve(m, y, c)
    rep = np.repeat(np.arange(n), c.astype(int))
    ex = ow.wcurve(m[rep], y[rep], np.ones(rep.size))
    assert got.wsums[6] == float(ex.words[6])          # U2w = U2 of the expanded list
    assert np.array_equal(got.wsums[[0, 1, 2, 3, 4, 5, 9, 10, 11, 12]], ex.wsums[[0, 1, 2, 3, 4, 5, 9, 10, 11, 12]])
    assert got.auc == ex.auc and got.ap == pytest.approx(ex.ap, rel=1e-15)
    keep = np.isin(got.thr, ex.thr)                    # zero-weight rows' scores are points of their own
    assert np.array_equal(got.thr[keep], ex.thr) and np.array_equal(got.tpw[keep], ex.tpw)


@pytest.mark.parametrize("seed", range(6))
def test_zero_weight_rows_count_as_rows_left_out(seed):
    rng = np.random.default_rng(400 + seed)
    n = 250
    m = tied_margins(rng, n) if seed % 2 else rng.standard_normal(n)
    y = np.where(rng.random(n) < 0.4, 1, -1)
    c = rng.random(n) * 2.0
    zero = rng.random(n) < 0.3
    c[zero] = 0.0
    a = ow.wcurve(m, y, c)
    b = ow.wcurve(m[~zero], y[~zero], c[~zero])
    assert np.array_equal(a.wsums, b.wsums) and a.auc == b.auc and a.ap == b.ap


def test_one_class_sets_and_nan_scores():
    m = np.array([-1.0, 0.5, 0.0, -2.0])
    c = np.array([1.0, 2.0, 0.5, 0.25])
    pos = ow.wcurve(m, np.ones(4), c)
    assert pos.ap == 1.0 and math.isnan(pos.auc) and pos.wsums[12] == 0.0 and pos.wsums[11] == 3.75
    neg = ow.wcurve(m, -np.ones(4), c)
    assert math.isnan(neg.ap) and math.isnan(neg.auc)
    m[1] = np.nan
    y = np.array([1, 1, -1, -1])
    r = ow.wcurve(m, y, c)
    assert math.isnan(r.auc) and math.isnan(r.ap) and r.wsums[7] == 2.0 and r.wsums[2] == 2.0 and r.wsums[11] == 3.0
