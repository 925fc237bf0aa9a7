"""The C oracle's curves and average precision (dsgd_oracle_curve, the checker of dsgd_eval_*curve) against a brute-force
pure-Python restatement (exact fractions for AP) and scikit-learn's roc_curve / average_precision_score.  No GPU."""
import math
from fractions import Fraction

import numpy as np
import pytest
from sklearn.metrics import average_precision_score, roc_curve

from oracle import curve as oc
from oracle import metrics as om
from oracle.oracle import Oracle, OracleError


def empty_rows(labels, dim=8):
    """An oracle over len(labels) empty rows: the margins come from the caller."""
    n = len(labels)
    return Oracle(np.zeros(n + 1, np.int64), np.zeros(0, np.int32), np.zeros(0, np.float32), np.asarray(labels, np.int8),
                  dim, 0.0)


def tied_scores(rng, n, levels):
    """Margins from a few levels, so that many rows tie; +0 and -0 both among them."""
    vals = np.concatenate([[0.0, -0.0], rng.integers(-4, 5, size=levels) / 4.0])
    return vals[rng.integers(0, len(vals), size=n)]


def brute(margins, labels):
    """(thr, tp, fp, v, exact AP or None) from the definitions: every distinct non-NaN score, and every row counted against
    it; v and AP from the counts at each positive row's own score."""
    rows = [(-m + 0.0, y > 0) for m, y in zip(margins, labels) if not math.isnan(m)]   # -0 + 0.0 == +0
    thr = sorted({s for s, _ in rows}, reverse=True)
    tp = [sum(1 for s, p in rows if p and s >= t) for t in thr]
    fp = [sum(1 for s, p in rows if not p and s >= t) for t in thr]
    at = dict(zip(thr, zip(tp, fp)))
    v = [Fraction(at[s][0], at[s][0] + at[s][1]) for s, p in rows if p]
    P = len(v)
    nan = any(math.isnan(m) for m in margins)
    ap = None if nan or P == 0 else sum(v, Fraction(0)) / P
    return np.array(thr), np.array(tp, np.int64), np.array(fp, np.int64), v, ap


def check(margins, labels, idx=None):
    margins = np.asarray(margins, dtype=np.float64)
    labels = np.asarray(labels)
    orc = empty_rows(labels)
    ids = np.arange(len(labels)) if idx is None else np.asarray(idx)
    m = margins[ids]
    got = oc.curve(orc, np.zeros(8), idx=ids, margins=m)
    thr, tp, fp, v, ap = brute(m, labels[ids])
    assert np.array_equal(got.thr, thr) and not np.signbit(got.thr[got.thr == 0]).any()   # a zero score is +0
    assert np.array_equal(got.tp, tp) and np.array_equal(got.fp, fp)
    assert sorted(got.v) == sorted(float(x) for x in v)              # each v_i is one IEEE division of exact counts
    assert got.nan == int(np.isnan(m).sum())
    if ap is None:
        assert math.isnan(got.ap)
    else:
        assert got.ap == float(ap) or abs(got.ap - float(ap)) <= 2 * math.ulp(float(ap))
    # U2 of the metrics checker from the curve: sum_k (fp[k] - fp[k-1]) (tp[k] + tp[k-1])
    words = om.metrics(orc, np.zeros(8), idx=ids, margins=m)
    tp0, fp0 = np.concatenate([[0], got.tp]), np.concatenate([[0], got.fp])
    assert int(np.sum(np.diff(fp0) * (tp0[1:] + tp0[:-1]))) == words[6]
    assert (got.tp[-1] if len(got.tp) else 0) == len(got.v)
    return got


@pytest.mark.parametrize("seed", range(12))
def test_random_sets_against_brute_force_and_scikit_learn(seed):
    rng = np.random.default_rng(seed)
    n = int(rng.integers(2, 300))
    labels = np.where(rng.random(n) < rng.uniform(0.1, 0.9), 1, -1)
    labels[0], labels[1] = 1, -1                              # both classes present
    m = tied_scores(rng, n, levels=3) if seed % 2 else rng.standard_normal(n)
    got = check(m, labels)
    # scikit-learn: roc_curve without drop_intermediate has one point per distinct score after its prepended (0, 0)
    y = (labels > 0).astype(int)
    fpr, tpr, thr = roc_curve(y, -m, drop_intermediate=False)
    P, N = int(y.sum()), int((1 - y).sum())
    assert np.array_equal(thr[1:], got.thr)
    assert np.array_equal(np.rint(tpr[1:] * P).astype(np.int64), got.tp)
    assert np.array_equal(np.rint(fpr[1:] * N).astype(np.int64), got.fp)
    np.testing.assert_allclose(got.ap, average_precision_score(y, -m), rtol=1e-12)


def test_heavy_ties_and_signed_zeros():
    rng = np.random.default_rng(7)
    n = 1000
    labels = np.where(rng.random(n) < 0.4, 1, -1)
    m = np.where(rng.random(n) < 0.5, 0.0, -0.0)              # every score is +-0: one point
    got = check(m, labels)
    P = int((labels > 0).sum())
    assert list(got.thr) == [0.0] and list(got.tp) == [P] and list(got.fp) == [n - P]
    assert abs(got.ap - P / n) <= math.ulp(P / n)             # every v_i is fl(P / n)
    check(tied_scores(rng, 5000, levels=2), labels=np.where(rng.random(5000) < 0.3, 1, -1))


def test_nan_rows_one_class_single_rows_and_repeats():
    rng = np.random.default_rng(3)
    n = 200
    labels = np.where(rng.random(n) < 0.5, 1, -1)
    m = rng.standard_normal(n)
    m[::17] = np.nan
    got = check(m, labels)
    assert got.nan == len(m[::17]) and math.isnan(got.ap)
    pos, neg = np.flatnonzero(labels > 0), np.flatnonzero(labels < 0)
    m = tied_scores(rng, n, levels=4)
    got = check(m, labels, idx=pos)                           # no negative: every v_i is 1
    assert got.ap == 1.0 and (got.fp == 0).all()
    got = check(m, labels, idx=neg)                           # no positive: AP undefined, tp all 0
    assert math.isnan(got.ap) and (got.tp == 0).all()
    for i in (pos[:1], neg[:1]):
        got = check(m, labels, idx=i)
        assert len(got.thr) == 1
    got = check(m, labels, idx=np.repeat(np.concatenate([pos[:3], neg[:2]]), 40))   # repeated ids count every time
    assert got.tp[-1] == 120 and got.fp[-1] == 80
    # every positive ranked above every negative: S = P exactly, AP = 1
    m2 = np.where(labels > 0, -1.0 - rng.random(n), 1.0 + rng.random(n))
    assert check(m2, labels).ap == 1.0


def test_own_dots_equal_passed_margins_and_errors():
    rng = np.random.default_rng(5)
    n, dim = 300, 16
    lens = rng.integers(0, 6, size=n)
    rp = np.concatenate([[0], np.cumsum(lens)]).astype(np.int64)
    col = np.concatenate([rng.choice(dim, size=k, replace=False) for k in lens]).astype(np.int32)
    val = (rng.integers(-8, 9, size=int(rp[-1])) / 8.0).astype(np.float32)
    lab = np.where(rng.random(n) < 0.4, 1, -1).astype(np.int8)
    orc = Oracle(rp, col, val, lab, dim, 0.0)
    w = rng.integers(-2, 3, size=dim) / 4.0
    ids = rng.integers(0, n, size=500).astype(np.int32)
    a = oc.curve(orc, w, idx=ids)
    b = oc.curve(orc, w, idx=ids, margins=om.margins(orc, w, idx=ids))
    for x, y in zip(a[:4], b[:4]):
        assert np.array_equal(x, y)
    assert a.ap == b.ap
    c = oc.curve(orc, w, begin=20, n=100)
    d = oc.curve(orc, w, idx=np.arange(20, 120))
    assert np.array_equal(c.thr, d.thr) and np.array_equal(c.tp, d.tp) and c.ap == d.ap
    with pytest.raises(OracleError):
        oc.curve(orc, w, idx=[0, n])
    with pytest.raises(OracleError):
        oc.curve(orc, w, begin=0, n=0)
