"""The topic-ranking checker (oracle/dsgd_oracle_topic_rank.c) against the literal numpy restatement
(tests/topic_ranking_model.py): random margins, tie-heavy integer-valued margins (+-0 among them), NaN margins, rows without
topics and rows with every topic, at T = 1, 2, 103 and 1024; listed rows with repeats; the checker's own dots; and the model's
ranks against scipy's "max" ranks."""
import numpy as np
import pytest
from scipy.stats import rankdata

from oracle import metrics as metrics_oracle
from oracle import topic_rank as rank_oracle
from oracle.oracle import Oracle
from topic_ranking_model import order, ranks, topic_ranking, topk


def _case(seed, T, n_rows=40, dim=30, ties=False, nan=True):
    rng = np.random.default_rng(seed)
    lens = rng.integers(0, 6, size=n_rows)
    row_ptr = np.concatenate([[0], np.cumsum(lens)]).astype(np.int64)
    col = np.concatenate([np.sort(rng.choice(dim, size=k, replace=False)) for k in lens]).astype(np.int32)
    val = rng.standard_normal(col.size).astype(np.float32)
    label = np.where(rng.random(n_rows) < 0.5, 1, -1).astype(np.int8)
    orc = Oracle(row_ptr, col, val, label, dim, 1e-4)
    has = rng.random((n_rows, T)) < min(0.5, 4.0 / T)
    has[:3] = False                                           # rows without a topic
    has[3:5] = True                                           # rows with every topic
    tptr = np.concatenate([[0], np.cumsum(has.sum(axis=1))]).astype(np.int64)
    tids = np.nonzero(has)[1].astype(np.int32)
    if ties:                                                  # integer-valued: many scores tie, +0 and -0 among them
        m = rng.integers(-2, 3, size=(T, n_rows)).astype(np.float64)
        m[rng.random((T, n_rows)) < 0.2] = -0.0
    else:
        m = rng.standard_normal((T, n_rows))
    if nan:
        m[:, 5] = np.nan
        m[T - 1, 6:9] = np.nan                                # one NaN score in a row is enough
    return orc, has, tptr, tids, m


@pytest.mark.parametrize("ties", [False, True])
@pytest.mark.parametrize("T,k", [(1, 1), (2, 1), (2, 2), (103, 5), (103, 32), (1024, 32)])
def test_checker_equals_numpy_on_planted_margins(T, k, ties):
    for seed in range(2 if T == 1024 else 4):
        orc, has, tptr, tids, m = _case(100 * T + seed, T, n_rows=12 if T == 1024 else 40, ties=ties)
        words, sums = rank_oracle.topic_rank(orc, tptr, tids, T, k, margins=m)
        ref_w, ref_s = topic_ranking(m, has, k)
        assert np.array_equal(words, ref_w), (seed, words[:8 + k], ref_w[:8 + k])
        assert np.array_equal(sums, ref_s), (seed, sums, ref_s)
        n = m.shape[1]
        assert words[0] == n and words[0] == words[1] + words[2] + words[3] and words[7] == 0
        assert words[2] >= 4 and words[3] >= 1                # the planted NaN rows and rows without a topic
        if T > 1 and not ties:
            assert words[4] >= 1                              # a ranked row with every topic


def test_a_row_with_every_topic_has_no_ranking_loss_term_and_perfect_scores():
    T, k = 6, 3
    m = np.random.default_rng(0).standard_normal((T, 1))
    has = np.ones((1, T), dtype=bool)
    words, sums = topic_ranking(m, has, k)
    assert list(words[:8]) == [1, 1, 0, 0, 1, T, 0, 0] and list(words[8:8 + k]) == [1, 2, 3]
    assert sums[0] == 1.0 and sums[1] == 0.0 and list(sums[2:]) == [1 / T, 2 / T, 3 / T]


def test_listed_rows_with_repeats_and_a_range():
    orc, has, tptr, tids, m = _case(7, 9, ties=True)
    idx = np.array([5, 5, 0, 39, 17, 3, 5, 20], dtype=np.int32)
    got = rank_oracle.topic_rank(orc, tptr, tids, 9, 4, idx=idx, margins=m[:, idx])
    ref = topic_ranking(m[:, idx], has[idx], 4)
    assert np.array_equal(got[0], ref[0]) and np.array_equal(got[1], ref[1])
    got = rank_oracle.topic_rank(orc, tptr, tids, 9, 4, begin=10, n=25, margins=m[:, 10:35])
    ref = topic_ranking(m[:, 10:35], has[10:35], 4)
    assert np.array_equal(got[0], ref[0]) and np.array_equal(got[1], ref[1])


def test_checker_own_dots_equal_the_metrics_checker_margins():
    orc, has, tptr, tids, _ = _case(11, 5)
    W = np.random.default_rng(3).standard_normal((5, orc.dim))
    m = np.stack([metrics_oracle.margins(orc, W[t]) for t in range(5)])
    got = rank_oracle.topic_rank(orc, tptr, tids, 5, 3, W=W)
    ref = topic_ranking(m, has, 3)
    assert np.array_equal(got[0], ref[0]) and np.array_equal(got[1], ref[1])


def test_halves_add_up_to_the_whole():
    orc, has, tptr, tids, m = _case(13, 17, n_rows=60)
    k = 5
    whole = topic_ranking(m, has, k)[0]
    a = rank_oracle.topic_rank(orc, tptr, tids, 17, k, begin=0, n=25, margins=m[:, :25])[0]
    b = rank_oracle.topic_rank(orc, tptr, tids, 17, k, begin=25, n=35, margins=m[:, 25:])[0]
    both = a + b
    for s in range(2 + k):                                   # propagate the carries of the merged limbs
        q = both[8 + k + 7 * s:8 + k + 7 * s + 6]
        for i in range(5):
            q[i + 1] += q[i] >> 40
            q[i] &= (1 << 40) - 1
    assert np.array_equal(both, whole)


@pytest.mark.parametrize("seed", range(6))
def test_ranks_are_scipys_max_ranks(seed):
    rng = np.random.default_rng(seed)
    T = [1, 2, 5, 103, 1024, 40][seed]
    s = rng.integers(-3, 4, size=T).astype(np.float64) if seed % 2 else rng.standard_normal(T)
    s[rng.random(T) < 0.1] = -0.0
    assert np.array_equal(ranks(s), rankdata(-s, method="max").astype(np.int64))


def test_order_and_topk_follow_the_tie_rule():
    m = np.array([[1.0, np.nan], [-0.0, np.nan], [0.0, 2.0], [-1.0, np.nan], [0.0, np.nan]])   # [T = 5, n = 2]
    assert order(m[:, 0]) == [3, 1, 2, 4, 0]                  # -0 and +0 are one score: the lower t first
    ids, top = topk(m, 3)
    assert ids.tolist() == [[3, 1, 2], [2, -1, -1]]
    assert top[0].tolist() == [-1.0, -0.0, 0.0] and np.signbit(top[0, 1]) and not np.signbit(top[0, 2])
    assert top[1, 0] == 2.0 and np.isnan(top[1, 1:]).all()
