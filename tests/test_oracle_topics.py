"""The topic-evaluation checker (oracle/dsgd_oracle_topics.c) against the literal numpy restatement (tests/topics_model.py):
random margins, tie-heavy margins (few distinct values, +-0, NaN), rows without topics, T = 1, listed rows with repeats,
and the checker's own dots."""
import numpy as np
import pytest

from oracle import metrics as metrics_oracle
from oracle import topics as topics_oracle
from oracle.oracle import Oracle
from topics_model import topic_words


def _case(seed, n_rows=60, dim=40, T=5, ties=False):
    rng = np.random.default_rng(seed)
    lens = rng.integers(0, 6, size=n_rows)
    row_ptr = np.concatenate([[0], np.cumsum(lens)]).astype(np.int64)
    col = np.concatenate([np.sort(rng.choice(dim, size=k, replace=False)) for k in lens]).astype(np.int32)
    val = rng.standard_normal(col.size).astype(np.float32)
    label = np.where(rng.random(n_rows) < 0.5, 1, -1).astype(np.int8)
    orc = Oracle(row_ptr, col, val, label, dim, 1e-4)
    has = rng.random((n_rows, T)) < 0.3
    has[:3] = False                                          # rows without a topic
    tptr = np.concatenate([[0], np.cumsum(has.sum(axis=1))]).astype(np.int64)
    tids = np.nonzero(has)[1].astype(np.int32)
    if ties:
        m = rng.choice([-1.0, -0.0, 0.0, 1.0, 2.0, np.nan], size=(T, n_rows))
    else:
        m = rng.standard_normal((T, n_rows))
        m[rng.random((T, n_rows)) < 0.05] = np.nan
    return orc, has, tptr, tids, m


@pytest.mark.parametrize("ties", [False, True])
@pytest.mark.parametrize("T", [1, 5, 17])
def test_checker_equals_numpy_on_planted_margins(T, ties):
    for seed in range(4):
        orc, has, tptr, tids, m = _case(1000 * T + seed, T=T, ties=ties)
        got = topics_oracle.topics(orc, tptr, tids, T, margins=m)
        assert np.array_equal(got, topic_words(m, has)), (seed, got)


def test_checker_listed_rows_with_repeats_and_a_range():
    orc, has, tptr, tids, m = _case(7, T=4, ties=True)
    idx = np.array([5, 5, 0, 59, 17, 3, 5], dtype=np.int32)
    got = topics_oracle.topics(orc, tptr, tids, 4, idx=idx, margins=m[:, idx])
    assert np.array_equal(got, topic_words(m[:, idx], has[idx]))
    got = topics_oracle.topics(orc, tptr, tids, 4, begin=10, n=30, margins=m[:, 10:40])
    assert np.array_equal(got, topic_words(m[:, 10:40], has[10:40]))


def test_checker_own_dots_equal_the_metrics_checker_margins():
    orc, has, tptr, tids, _ = _case(11, T=3)
    W = np.random.default_rng(3).standard_normal((3, orc.dim))
    m = np.stack([metrics_oracle.margins(orc, W[t]) for t in range(3)])
    got = topics_oracle.topics(orc, tptr, tids, 3, W=W)
    assert np.array_equal(got, topic_words(m, has))
    assert got[8 * 3] == orc.n_rows and got[8 * 3 + 3] >= 3      # rows; the three rows planted without a topic


def test_per_topic_words_are_the_metrics_checker_over_topic_labels():
    orc, has, tptr, tids, m = _case(13, T=4, ties=True)
    got = topics_oracle.topics(orc, tptr, tids, 4, margins=m)
    for t in range(4):
        o = Oracle(orc.row_ptr, orc.col, orc.val, np.where(has[:, t], 1, -1).astype(np.int8), orc.dim, orc.lam)
        ref = metrics_oracle.metrics(o, np.zeros(orc.dim), margins=m[t])
        ref[6] = 0
        assert np.array_equal(got[8 * t:8 * t + 8], ref)
