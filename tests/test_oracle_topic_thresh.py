"""The topic threshold checker (oracle/dsgd_oracle_topic_thresh.c) against the literal numpy restatement
(tests/topic_thresholds_model.py), bit for bit: random margins, tie-heavy margins from a few values (+-0 among them), NaN
and +-inf margins, adjacent doubles and subnormal pairs (the midpoint falls back to c_(j+1)), topics without a positive
row, all-positive topics, no rows, fbr equal to a best F1, at T = 1, 103 and 1024; listed rows with repeats and the
checker's own dots.  In every case the thresholded rule at the returned tau counts words 4 and 5, and candidate j's counts
unless its margin is +inf."""
import numpy as np
import pytest

from oracle import metrics as metrics_oracle
from oracle import topic_thresh as thresh_oracle
from oracle.oracle import Oracle
from topic_thresholds_model import (BELOW_FBR, NO_MARGIN, NO_POSITIVE, TUNED, candidate_counts, counts_at, midpoint, tune,
                                    tune_topic)


def _case(seed, T, n_rows=40, dim=30):
    rng = np.random.default_rng(seed)
    lens = rng.integers(0, 6, size=n_rows)
    row_ptr = np.concatenate([[0], np.cumsum(lens)]).astype(np.int64)
    col = np.concatenate([np.sort(rng.choice(dim, size=k, replace=False)) for k in lens]).astype(np.int32)
    val = rng.standard_normal(col.size).astype(np.float32)
    label = np.where(rng.random(n_rows) < 0.5, 1, -1).astype(np.int8)
    orc = Oracle(row_ptr, col, val, label, dim, 1e-4)
    has = rng.random((n_rows, T)) < min(0.5, 4.0 / T)
    return orc, has, rng


def _csr(has):
    tptr = np.concatenate([[0], np.cumsum(has.sum(axis=1))]).astype(np.int64)
    return tptr, np.nonzero(has)[1].astype(np.int32)


def _margins(kind, rng, T, n):
    if kind == "random":
        return rng.standard_normal((T, n))
    if kind == "ties":                                        # a few values: many ties, +0 and -0 among them
        m = rng.integers(-2, 3, size=(T, n)).astype(np.float64)
        m[rng.random((T, n)) < 0.2] = -0.0
        return m
    if kind == "nan_inf":
        m = rng.standard_normal((T, n))
        r = rng.random((T, n))
        m[r < 0.1] = np.nan
        m[(r >= 0.1) & (r < 0.2)] = np.inf
        m[(r >= 0.2) & (r < 0.3)] = -np.inf
        return m
    if kind == "adjacent":                                    # adjacent doubles and subnormal pairs
        base = np.array([1.0, -3.5, 5e-324, -5e-324, 2.2250738585072014e-308, 0.0, 1e300])
        m = rng.choice(base, size=(T, n))
        nxt = np.nextafter(m, np.inf)
        pick = rng.random((T, n)) < 0.5
        return np.where(pick, nxt, m)
    raise ValueError(kind)


def _check_case(orc, has, m, fbr=0.0, idx=None):
    T = m.shape[0]
    tptr, tids = _csr(has)
    if idx is None:
        thr, words = thresh_oracle.topic_thresh(orc, tptr, tids, T, fbr, begin=0, n=m.shape[1], margins=m)
        h = has
    else:
        thr, words = thresh_oracle.topic_thresh(orc, tptr, tids, T, fbr, idx=idx, margins=m)
        h = has[idx]
    ref_thr, ref_words = tune(m, h, fbr)
    assert np.array_equal(thr.view(np.int64), ref_thr.view(np.int64)), (thr, ref_thr)
    assert np.array_equal(words, ref_words)
    for t in range(T):
        w = words[8 * t:8 * t + 8]
        assert counts_at(m[t], h[:, t], thr[t]) == (w[4], w[5])
        assert w[0] == m.shape[1] and w[1] == h[:, t].sum() and w[2] == np.isnan(m[t]).sum()
        if w[7] >= 0:
            c = sorted({float(v) + 0.0 for v in m[t][~np.isnan(m[t])]})
            if c[w[7]] != np.inf:
                assert candidate_counts(m[t], h[:, t], w[7]) == (w[4], w[5])
    return thr, words


@pytest.mark.parametrize("kind", ["random", "ties", "nan_inf", "adjacent"])
@pytest.mark.parametrize("T", [1, 103, 1024])
def test_checker_equals_numpy(T, kind):
    for seed in range(1 if T == 1024 else 3):
        orc, has, rng = _case(1000 * T + seed, T, n_rows=12 if T == 1024 else 40)
        _check_case(orc, has, _margins(kind, rng, T, has.shape[0]))


def test_midpoint_falls_back_on_adjacent_doubles_and_subnormals():
    for c in (1.0, -3.5, 5e-324, -5e-324, 0.0, 1e300, -np.inf):
        c1 = float(np.nextafter(c, np.inf))
        assert midpoint(c, c1) == c1 or c < midpoint(c, c1) <= c1
    assert midpoint(1.0, float(np.nextafter(1.0, 2.0))) == float(np.nextafter(1.0, 2.0))
    assert midpoint(5e-324, 1e-323) == 1e-323                  # 2.5e-324 + 5e-324 rounds to 5e-324 = c_j
    assert midpoint(-5e-324, 5e-324) == 0.0
    assert midpoint(1.0, 3.0) == 2.0
    assert midpoint(-np.inf, 0.0) == 0.0 and midpoint(0.0, np.inf) == np.inf and midpoint(-np.inf, np.inf) == np.inf


def test_statuses_no_positive_all_positive_and_no_rows():
    orc, has, rng = _case(5, 3)
    n = has.shape[0]
    m = rng.standard_normal((3, n))
    has[:, 0] = False                                          # no positive row
    has[:, 1] = True                                           # every row positive
    m[1, :3] = np.inf                                          # the best candidate is the last, at +inf
    m[2, :] = np.nan                                           # no non-NaN margin
    thr, words = _check_case(orc, has, m)
    w = words.reshape(3, 8)
    assert w[0, 6] == NO_POSITIVE and thr[0] == 0.0 and w[0, 7] == -1 and w[0, 4] == 0 and w[0, 5] == np.sum(m[0] < 0)
    assert w[1, 6] == TUNED and thr[1] == np.inf and w[1, 7] == w[1, 3] - 1 and w[1, 4] == w[1, 5] == n - 3
    assert w[2, 6] == NO_MARGIN and thr[2] == 0.0 and w[2, 7] == -1 and list(w[2, 4:6]) == [0, 0] and w[2, 2] == n
    # no rows at all: every topic has no margin
    thr, words = thresh_oracle.topic_thresh(orc, *_csr(has), 3, 0.0, begin=0, n=0, margins=np.zeros((3, 0)))
    assert list(thr) == [0.0] * 3 and words.reshape(3, 8).tolist() == [[0, 0, 0, 0, 0, 0, NO_MARGIN, -1]] * 3
    assert np.array_equal(words, tune(np.zeros((3, 0)), np.zeros((0, 3), dtype=bool))[1])


def test_fbr_is_a_strict_bound():
    orc, has, rng = _case(9, 4)
    m = rng.standard_normal((4, has.shape[0]))
    _, words = _check_case(orc, has, m)
    for t in range(4):
        w = words[8 * t:8 * t + 8]
        if w[6] != TUNED:
            continue
        f1 = (2 * int(w[4])) / (int(w[1]) + int(w[5]))
        # fbr equal to the best F1: not below it, still tuned; the next double up: below it, tau_0
        _, at = tune_topic(m[t], has[:, t], f1)
        assert at[6] == TUNED and at[7] == w[7]
        if f1 < 1.0:
            thr_up, up = tune_topic(m[t], has[:, t], float(np.nextafter(f1, 2.0)))
            assert up[6] == BELOW_FBR and up[7] == 0
        _check_case(orc, has, m, fbr=f1)
    _check_case(orc, has, m, fbr=1.0)


def test_listed_rows_with_repeats_and_own_dots():
    orc, has, rng = _case(7, 9)
    idx = np.array([5, 5, 0, 39, 17, 3, 5, 20, 20], dtype=np.int32)
    m = _margins("ties", rng, 9, idx.size)
    _check_case(orc, has, m, idx=idx)
    W = rng.standard_normal((9, orc.dim))
    mm = np.stack([metrics_oracle.margins(orc, W[t]) for t in range(9)])
    thr, words = thresh_oracle.topic_thresh(orc, *_csr(has), 9, 0.0, W=W)
    ref = tune(mm, has)
    assert np.array_equal(thr, ref[0]) and np.array_equal(words, ref[1])
