"""The bootstrap draw of dsgd_eval_*bootstrap (distributed_sgd_b200/csrc/dsgd_bootstrap.h) and its checkers.  No GPU.

* The thresholds T_k committed in the header are floor(F(k) 2^64) rebuilt exactly with fractions.
* The Python restatement of the draw (oracle/bootstrap.py) equals the host library's, compiled from the same header.
* Over 2^20 draws at one key, the frequencies of m = 0..6 and the lag-1 correlations across positions and across replicates
  are those of independent Poisson(1) draws, to within 5 sigma.  The draws are a fixed function of the key: deterministic.
* The replicate as k_boot_rep forms it from tie groups (oracle.bootstrap.grouped) equals the literal evaluation of the
  expanded list by the metrics, curve and loss checkers on planted cases: ties, +0 and -0, NaN, one class, n = 1.
"""
import math

import numpy as np
import pytest

from distributed_sgd_b200 import native
from oracle import bootstrap as ob
from oracle.oracle import Oracle

MODELS = ["svm", "logistic", "squared_hinge", "modified_huber"]


def test_thresholds_equal_the_header():
    t = ob.thresholds()
    assert ob.header_thresholds() == t
    assert len(t) == 20 and t == sorted(t) and t[-1] < 2 ** 64
    assert abs(t[0] / 2 ** 64 - math.exp(-1)) < 1e-15
    assert 1 - t[-1] / 2 ** 64 < 1e-18                     # the tail beyond 19 draws, given to 20, is about 1.6e-19


def test_python_draw_equals_the_host_library():
    h = native.host_lib()
    rng = np.random.default_rng(7)
    keys = rng.integers(0, 2 ** 63, size=100_000, dtype=np.uint64) * np.uint64(2) + rng.integers(0, 2, size=100_000,
                                                                                                   dtype=np.uint64)
    bs = rng.integers(0, 5000, size=100_000)
    ii = rng.integers(0, 1 << 26, size=100_000)
    seen = set()
    for k, b, i in zip(keys.tolist(), bs.tolist(), ii.tolist()):
        m = h.dsgd_bootstrap_draw(k, b, i)
        assert m == ob.multiplicity(k, b, i)
        seen.add(m)
    assert {0, 1, 2, 3, 4} <= seen
    # the vectorised form too
    for b in (0, 3, 4999):
        assert [h.dsgd_bootstrap_draw(12345, b, i) for i in range(300)] == ob.multiplicities(12345, b, 300).tolist()


def test_draws_are_poisson_and_uncorrelated():
    B, n = 16, 1 << 16
    m = np.stack([ob.multiplicities(0xC0FFEE, b, n) for b in range(B)])   # 2^20 draws
    N = m.size
    for k in range(7):
        p = math.exp(-1) / math.factorial(k)
        cnt = int((m == k).sum())
        assert abs(cnt - N * p) <= 5 * math.sqrt(N * p * (1 - p)), (k, cnt, N * p)
    assert m.max() <= 20
    z = (m - 1.0)                                           # mean 1, variance 1

    def corr(a, b):
        return float((a * b).mean())

    lag_i = corr(z[:, :-1], z[:, 1:])
    lag_b = corr(z[:-1, :], z[1:, :])
    assert abs(lag_i) <= 5 / math.sqrt(B * (n - 1)), lag_i
    assert abs(lag_b) <= 5 / math.sqrt((B - 1) * n), lag_b


def empty_rows(labels, dim=8):
    n = len(labels)
    return Oracle(np.zeros(n + 1, np.int64), np.zeros(0, np.int32), np.zeros(0, np.float32), np.asarray(labels, np.int8),
                  dim, 0.0)


def planted(rng, n, one_class=False, nan=False):
    vals = np.concatenate([[0.0, -0.0, 0.5, -0.5, 3.0, -2.0], rng.integers(-8, 9, size=4) / 8.0])
    margins = vals[rng.integers(0, len(vals), size=n)]
    if nan:
        margins[rng.integers(0, n)] = np.nan
    labels = np.ones(n, np.int8) if one_class else np.where(rng.random(n) < 0.4, 1, -1).astype(np.int8)
    return margins, labels


def same(a, b):
    assert np.array_equal(a.words, b.words)
    assert (math.isnan(a.ap) and math.isnan(b.ap)) or a.ap == b.ap
    assert (math.isnan(a.loss) and math.isnan(b.loss)) or a.loss == b.loss


@pytest.mark.parametrize("model", MODELS)
@pytest.mark.parametrize("case", ["ties", "nan", "one_class", "n1", "negatives"])
def test_grouped_replicate_equals_the_expanded_list(model, case):
    rng = np.random.default_rng(hash(case) % 1000)
    n = 1 if case == "n1" else 60
    margins, labels = planted(rng, n, one_class=case == "one_class", nan=case == "nan")
    if case == "negatives":
        labels[:] = -1
    orc = empty_rows(labels)
    ids = rng.integers(0, n, size=n) if n > 1 else np.zeros(1, np.int64)   # a list with repeats
    mg = margins[ids]
    for b in range(6):
        m = ob.multiplicities(99, b, n)
        if case == "n1" and b == 0:
            m = np.array([2])
        same(ob.grouped(model, mg, labels[ids], m), ob.replicate(orc, model, np.zeros(8), ids, m, mg))
