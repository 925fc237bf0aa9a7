"""The C oracle's ranking metrics (dsgd_oracle_metrics, the checker of dsgd_eval_*metrics) against two independent counts: a
brute-force O(P N) pair count in numpy, and scipy's Mann-Whitney U (2 U = U2).  No GPU."""
import numpy as np
import pytest
from scipy.stats import mannwhitneyu

from oracle import metrics as om
from oracle.oracle import Oracle, OracleError


def brute(margins, labels):
    """The eight words from margins and labels: confusion counts by -signum(margin), U2 over every (positive, negative) pair."""
    m = np.asarray(margins, dtype=np.float64)
    y = np.asarray(labels)
    nan = np.isnan(m)
    p = np.where(m > 0, -1, np.where(m < 0, 1, 0))          # -signum; NaN compares false both ways: 0
    pos, neg = y > 0, y < 0
    words = [np.sum(pos & (p == 1)), np.sum(pos & (p == -1)), np.sum(pos & (p == 0)),
             np.sum(neg & (p == 1)), np.sum(neg & (p == -1)), np.sum(neg & (p == 0)), 0, np.sum(nan)]
    s = -m
    sp, sn = s[pos & ~nan], s[neg & ~nan]
    words[6] = int(np.sum(2 * (sp[:, None] > sn[None, :]) + (sp[:, None] == sn[None, :])))
    return np.array(words, dtype=np.int64)


def empty_rows(labels, dim=8):
    """An oracle over len(labels) empty rows: the margins come from the caller."""
    n = len(labels)
    return Oracle(np.zeros(n + 1, np.int64), np.zeros(0, np.int32), np.zeros(0, np.float32), np.asarray(labels, np.int8),
                  dim, 0.0)


def tied_scores(rng, n, levels):
    """Margins from a few levels, so that many rows tie; +0 and -0 both among them."""
    vals = np.concatenate([[0.0, -0.0], rng.integers(-4, 5, size=levels) / 4.0])
    return vals[rng.integers(0, len(vals), size=n)]


@pytest.mark.parametrize("seed", range(12))
def test_random_sets_against_brute_force_and_mann_whitney(seed):
    rng = np.random.default_rng(seed)
    n = int(rng.integers(2, 400))
    labels = np.where(rng.random(n) < rng.uniform(0.1, 0.9), 1, -1)
    labels[0], labels[1] = 1, -1                              # both classes present
    m = tied_scores(rng, n, levels=3) if seed % 2 else rng.standard_normal(n)
    orc = empty_rows(labels)
    got = om.metrics(orc, np.zeros(8), idx=np.arange(n), margins=m)
    assert np.array_equal(got, brute(m, labels))
    s = -m
    u = mannwhitneyu(s[labels > 0], s[labels < 0], alternative="two-sided", method="asymptotic").statistic
    assert 2 * u == got[6]
    assert got[:6].sum() == n and got[7] == 0


def test_heavy_ties_and_signed_zeros():
    rng = np.random.default_rng(7)
    n = 1000
    labels = np.where(rng.random(n) < 0.4, 1, -1)
    m = np.where(rng.random(n) < 0.5, 0.0, -0.0)              # every score is +-0: one score, every pair ties
    orc = empty_rows(labels)
    got = om.metrics(orc, np.zeros(8), idx=np.arange(n), margins=m)
    P, N = int((labels > 0).sum()), int((labels < 0).sum())
    assert got[6] == P * N                                    # U2 = 1 per pair: AUC 1/2
    assert got[2] == P and got[5] == N and got[0] == got[1] == got[3] == got[4] == 0
    m = tied_scores(rng, n, levels=2)
    assert np.array_equal(om.metrics(orc, np.zeros(8), idx=np.arange(n), margins=m), brute(m, labels))


def test_one_class_and_single_row():
    for labels in ([1] * 9, [-1] * 9, [1], [-1]):
        n = len(labels)
        m = np.linspace(-1.0, 1.0, n)
        got = om.metrics(empty_rows(labels), np.zeros(8), idx=np.arange(n), margins=m)
        assert got[6] == 0 and np.array_equal(got, brute(m, labels))


def test_nan_scores_are_counted_and_left_out_of_the_pairs():
    labels = np.array([1, 1, -1, -1, 1, -1])
    m = np.array([np.nan, -1.0, 1.0, np.nan, 0.5, -2.0])
    got = om.metrics(empty_rows(labels), np.zeros(8), idx=np.arange(6), margins=m)
    assert got[7] == 2
    assert got[2] == 1 and got[5] == 1                        # the NaN rows have no prediction
    # pairs without NaN: positives s = {1.0, -0.5}, negatives s = {-1.0, 2.0}: (1 > -1) (-0.5 > -1) -> U2 = 4
    assert got[6] == 4 and np.array_equal(got, brute(m, labels))


def test_repeated_ids_count_every_time():
    rng = np.random.default_rng(3)
    labels = np.where(rng.random(50) < 0.5, 1, -1)
    labels[:2] = (1, -1)
    base = tied_scores(rng, 50, levels=4)
    idx = rng.integers(0, 50, size=300).astype(np.int32)
    got = om.metrics(empty_rows(labels), np.zeros(8), idx=idx, margins=base[idx])
    assert np.array_equal(got, brute(base[idx], labels[idx]))


def test_own_dots_on_dyadic_rows():
    """margins == NULL ranks the oracle's left-fold dots; on dyadic rows and weights every dot is exact."""
    rng = np.random.default_rng(11)
    n, dim = 600, 64
    lens = rng.integers(0, 12, size=n)
    rp = np.concatenate([[0], np.cumsum(lens)]).astype(np.int64)
    col = np.concatenate([rng.choice(dim, size=k, replace=False) for k in lens]).astype(np.int32)
    val = (rng.integers(-8, 9, size=rp[-1]) / 8.0).astype(np.float32)
    labels = np.where(rng.random(n) < 0.5, 1, -1).astype(np.int8)
    orc = Oracle(rp, col, val, labels, dim, 0.0)
    w = rng.integers(-2, 3, size=dim) / 4.0                  # few distinct dots: many ties, zero rows among them
    m = om.margins(orc, w, begin=0, n=n)
    exact = np.array([sum(float(val[k]) * w[col[k]] for k in range(rp[r], rp[r + 1])) for r in range(n)])
    assert np.array_equal(m, exact)
    ids = np.arange(n, dtype=np.int32)
    want = brute(m, labels)
    assert np.array_equal(om.metrics(orc, w, idx=ids), want)
    assert np.array_equal(om.metrics(orc, w, begin=0, n=n), want)
    assert np.array_equal(om.metrics(orc, w, begin=100, n=200), brute(m[100:300], labels[100:300]))
    assert np.array_equal(orc.forward(w, ids), np.where(m > 0, -1.0, np.where(m < 0, 1.0, 0.0)))


def test_errors():
    orc = empty_rows([1, -1, 1])
    with pytest.raises(OracleError):
        om.metrics(orc, np.zeros(8), idx=np.zeros(0, np.int32))
    with pytest.raises(OracleError):
        om.metrics(orc, np.zeros(8), idx=[0, 3])
    with pytest.raises(OracleError):
        om.metrics(orc, np.zeros(8), begin=2, n=2)
