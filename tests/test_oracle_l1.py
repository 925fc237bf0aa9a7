"""The checker of the sync step with an L1 penalty (oracle/l1.py, the L1 step of oracle/dsgd_oracle_margin.c), without a GPU:

1. The proximal step on hand-worked values: shrinking by tau, |u| = tau -> 0, u - tau at exactly 1e-20 (filtered) and one ulp
   above (kept), tau = 0 -> u itself (also for values the filter would drop and for -0), the C form equal to the literal one.
2. The C checker against the literal restatement, both models, one and several workers, scalar rates and tables with zero
   entries: weights bit for bit, losses bit for bit on dyadic data and within 1e-14 on random data.
3. lambda1 = 0 gives the plain step bit for bit: dsgd_oracle_sync_steps for the SVM, the literal restatement of
   scala_semantics_margin.py for the logistic model.
"""
import math

import numpy as np
import pytest

from conftest import random_csr
from oracle import cw as CW
from oracle import l1 as L1
from oracle.logistic import LogisticOracle
from oracle.oracle import Oracle
from oracle.scala_semantics_margin import literal_sync_steps
from test_oracle_class_weight import literal_model

TINY = np.nextafter(1e-20, 1.0)   # the smallest double the 1e-20 filter keeps


@pytest.mark.parametrize("u,tau,expect", [
    (3.0, 1.0, 2.0), (-3.0, 1.0, -2.0), (0.75, 0.25, 0.5), (-0.75, 0.25, -0.5),
    (1.0, 1.0, 0.0), (-1.0, 1.0, 0.0), (0.5, 1.0, 0.0), (-0.5, 1.0, 0.0), (0.0, 1.0, 0.0), (-0.0, 1.0, 0.0),
    (0.25 + 1e-20, 0.25, 0.0),                       # fl(0.25 + 1e-20) is 0.25: |u| = tau
    (2.0 ** -60 + 1e-20, 2.0 ** -60, 0.0),           # u - tau is exactly fl(1e-20) or below: filtered
    (5.0, 0.0, 5.0), (-5.0, 0.0, -5.0), (1e-25, 0.0, 1e-25), (0.0, 0.0, 0.0),
])
def test_prox_known_answers(u, tau, expect):
    for f in (L1.prox, L1.literal_prox):
        got = f(u, tau)
        assert got == expect and math.copysign(1.0, got) == math.copysign(1.0, expect) or (got == 0.0 and expect == 0.0), \
            (f, u, tau, got)


def test_prox_filter_edge():
    """u - tau exactly 1e-20 is dropped, one ulp above 1e-20 is kept, on both sides of 0.  tau = 2^-70 is a multiple of the ulp
    of 1e-20 (2^-119) and u stays below 2^-66, so u = v + tau and u - tau = v are exact."""
    tau = 2.0 ** -70
    for v, kept in ((1e-20, False), (TINY, True)):
        u = v + tau
        assert u - tau == v
        for f in (L1.prox, L1.literal_prox):
            assert f(u, tau) == (v if kept else 0.0)
            assert f(-u, tau) == (-v if kept else 0.0)


def test_prox_tau_zero_is_identity_on_every_value():
    vals = [0.0, -0.0, 1e-300, -1e-25, 1e-20, 3.5, -7.25, float(np.nextafter(0.0, 1.0))]
    for v in vals:
        for f in (L1.prox, L1.literal_prox):
            r = f(v, 0.0)
            assert r == v and math.copysign(1.0, r) == math.copysign(1.0, v)


def test_prox_c_equals_literal_on_random_values():
    rng = np.random.default_rng(5)
    u = np.concatenate([rng.standard_normal(2000) * 10.0 ** rng.integers(-22, 3, size=2000), [0.0, -0.0]])
    tau = np.abs(rng.standard_normal(u.size)) * 10.0 ** rng.integers(-22, 1, size=u.size)
    tau[::7] = 0.0
    for a, t in zip(u.tolist(), tau.tolist()):
        assert L1.prox(a, t) == L1.literal_prox(a, t)


def test_l1_norm_exact_and_count():
    w = np.array([0.5, -0.25, 0.0, -0.0, 3.0, -1e-3])
    assert L1.l1_norm(w) == math.fsum(abs(x) for x in w)
    rng = np.random.default_rng(2)
    w = rng.standard_normal(10000) * 10.0 ** rng.integers(-12, 6, size=10000)
    assert abs(L1.l1_norm(w) - math.fsum(np.abs(w))) <= 2.0 ** -52 * math.fsum(np.abs(w))


def _dyadic_csr(rng, n_rows, dim):
    nnz = rng.integers(1, 9, size=n_rows)
    rp = np.concatenate([[0], np.cumsum(nnz)]).astype(np.int64)
    col = np.concatenate([rng.choice(dim, size=k, replace=False) for k in nnz]).astype(np.int32)
    val = (rng.integers(1, 17, size=int(rp[-1])) / 8.0 * rng.choice([-1, 1], size=int(rp[-1]))).astype(np.float32)
    lab = rng.choice([-1, 1], size=n_rows).astype(np.int8)
    return rp, col, val, lab


def _case(seed, dyadic, logistic, counts, steps, table):
    rng = np.random.default_rng(seed)
    dim, n = 48, 80
    if dyadic:
        rp, col, val, lab = _dyadic_csr(rng, n, dim)
        lam, lam1 = 2.0 ** -6, 2.0 ** -5
        w0 = rng.integers(-16, 17, size=dim) / 8.0 * (rng.random(dim) < 0.6)
        lrs = 2.0 ** -(2 + np.arange(steps) % 3)
    else:
        rp, col, val, lab = random_csr(rng, n, dim, max_nnz=8)
        lam, lam1 = 0.01, 0.003
        w0 = rng.standard_normal(dim) * (rng.random(dim) < 0.6) * 0.3
        lrs = 0.3 * (1.0 + 0.1 * np.arange(steps)) ** -0.75
    if table:
        lrs = lrs.copy()
        lrs[1::3] = 0.0
    orc = (LogisticOracle if logistic else Oracle)(rp, col, val, lab, dim, lam)
    d = orc.dim_sparsity(n)
    orc.set_dim_sparsity(d)
    per = sum(counts)
    idx = np.concatenate([rng.choice(n, size=per, replace=False) for _ in range(steps)]).astype(np.int32)
    return (rp, col, val, lab, dim, lam, lam1, d, w0, idx, lrs), orc


@pytest.mark.parametrize("logistic", [False, True])
@pytest.mark.parametrize("counts", [[6], [3, 4, 2]])
@pytest.mark.parametrize("dyadic", [True, False])
@pytest.mark.parametrize("table", [False, True])
def test_c_checker_matches_literal(logistic, counts, dyadic, table):
    (rp, col, val, lab, dim, lam, lam1, d, w0, idx, lrs), orc = _case(11 + len(counts), dyadic, logistic, counts, 12, table)
    w_c, l_c = L1.sync_steps(orc, w0, idx, counts, lrs, lam1, logistic=logistic)
    w_l, l_l = L1.literal_sync_steps(rp, col, val, lab, dim, lam, lam1, d, w0, idx, counts, lrs, logistic=logistic)
    assert np.array_equal(w_c, np.array(w_l)), np.flatnonzero(w_c != np.array(w_l))
    if dyadic and not logistic:
        assert np.array_equal(l_c, np.array(l_l))
    else:
        np.testing.assert_allclose(l_c, l_l, rtol=1e-14, atol=0)


@pytest.mark.parametrize("logistic", [False, True])
@pytest.mark.parametrize("counts", [[6], [3, 4, 2]])
def test_lambda1_zero_is_the_plain_step(logistic, counts):
    """lambda1 = 0 gives the step without the penalty: dsgd_oracle.c's for the SVM; for the logistic model the literal
    restatement over Sparse vectors (scala_semantics_margin.py), whose loss sums are the checker's fixed-point sums."""
    (rp, col, val, lab, dim, lam, lam1, d, w0, idx, lrs), orc = _case(3, False, logistic, counts, 10, False)
    lr = 0.25
    w_c, l_c = L1.sync_steps(orc, w0, idx, counts, np.full(10, lr), 0.0, logistic=logistic)
    if logistic:
        w_r, l_r = literal_sync_steps(literal_model(True, lam), CW.literal_rows(rp, col, val, dim), lab, dim, lam, d, w0, idx,
                                      counts, np.full(10, lr))
    else:
        w_r, l_r = orc.sync_steps(w0, idx, counts, lr, n_steps=10)
    assert np.array_equal(w_c, w_r)
    assert np.array_equal(l_c, l_r)


def test_zero_rate_entries_leave_the_weights_of_the_plain_step():
    """A table entry of 0 makes tau 0: the step is the step without the penalty (here: no update at all)."""
    (rp, col, val, lab, dim, lam, lam1, d, w0, idx, lrs), orc = _case(4, True, False, [6], 3, False)
    w_c, _ = L1.sync_steps(orc, w0, idx, [6], np.zeros(3), lam1)
    assert np.array_equal(w_c, w0)


def test_averaging_sum():
    (rp, col, val, lab, dim, lam, lam1, d, w0, idx, lrs), orc = _case(8, True, False, [6], 5, False)
    A = np.zeros(dim)
    w_all, _ = L1.sync_steps(orc, w0, idx, [6], lrs, lam1, avg_sum=A)
    w, B = np.asarray(w0, np.float64), np.zeros(dim)
    for t in range(5):
        w, _ = L1.sync_steps(orc, w, idx[6 * t:6 * (t + 1)], [6], lrs[t:t + 1], lam1)
        B += w
    assert np.array_equal(A, B) and np.array_equal(w, w_all)
