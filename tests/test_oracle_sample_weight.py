"""The sample-weight checker (oracle/sw.py, the sample weighting of oracle/dsgd_oracle_margin.c), without a GPU:

1. The C checker against the literal restatement over Sparse vectors on dyadic data with dyadic sample weights (some zero):
   SVM weights and losses bit for bit, logistic to rounding; one and several workers, rate tables; the weighted evaluation.
2. At sample weights 1 it gives the class-weighted steps and gradients of the literal restatements: weights bit for bit,
   losses bit for bit for the SVM.
3. Hand-worked cases: a weight of 0, a product x_j * c_i at exactly 1e-20 and one ulp above, and an integer weight k on a row
   equal to that row listed k times.
"""
import numpy as np
import pytest

from oracle import cw as CW
from oracle import sw as SW
from oracle.logistic import LogisticOracle
from oracle.oracle import Oracle
from oracle.scala_semantics_margin import literal_sync_steps
from test_oracle_class_weight import TINY, dyadic_problem, literal_model


def dyadic_weights(rng, n):
    """Multiples of 1/4 in [0, 4], about one in five of them 0."""
    s = rng.integers(1, 17, size=n) / 4.0
    s[rng.random(n) < 0.2] = 0.0
    return s


@pytest.mark.parametrize("counts", [[8], [5, 3], [4, 3, 2]])
@pytest.mark.parametrize("wp,wn", [(1.0, 1.0), (2.0, 0.5)])
def test_svm_c_equals_literal_bit_for_bit_on_dyadic_data(counts, wp, wn):
    orc, (rp, col, val, lab, dim, d), w0, rng = dyadic_problem(3)
    sw = dyadic_weights(rng, len(lab))
    lrs = [0.5, 0.25, 0.0, 0.125]
    idx = rng.integers(0, len(lab), size=sum(counts) * len(lrs)).astype(np.int32)
    w_c, l_c = SW.sync_steps(orc, w0, idx, counts, lrs, sw, wp, wn)
    rows = CW.literal_rows(rp, col, val, dim)
    w_l, l_l = SW.literal_sync_steps(rows, lab, dim, orc.lam, d, w0, idx, counts, lrs, sw, wp, wn)
    assert np.array_equal(w_c, np.asarray(w_l))
    assert list(l_c) == l_l


@pytest.mark.parametrize("counts", [[8], [5, 3]])
def test_logistic_c_equals_literal(counts):
    orc, (rp, col, val, lab, dim, d), w0, rng = dyadic_problem(4, cls=LogisticOracle)
    sw = dyadic_weights(rng, len(lab))
    lrs = [0.5, 0.25, 0.125]
    idx = rng.integers(0, len(lab), size=sum(counts) * len(lrs)).astype(np.int32)
    w_c, l_c = SW.sync_steps(orc, w0, idx, counts, lrs, sw, 2.0, 0.5, logistic=True)
    rows = CW.literal_rows(rp, col, val, dim)
    w_l, l_l = SW.literal_sync_steps(rows, lab, dim, orc.lam, d, w0, idx, counts, lrs, sw, 2.0, 0.5, logistic=True)
    np.testing.assert_allclose(w_c, w_l, rtol=1e-13, atol=1e-15)
    np.testing.assert_allclose(l_c, l_l, rtol=1e-14)


@pytest.mark.parametrize("logistic", [False, True])
@pytest.mark.parametrize("wp,wn", [(1.0, 1.0), (2.0, 0.5)])
def test_eval_c_equals_literal(logistic, wp, wn):
    orc, (rp, col, val, lab, dim, d), w0, rng = dyadic_problem(6, cls=LogisticOracle if logistic else Oracle)
    sw = dyadic_weights(rng, len(lab))
    idx = rng.integers(0, len(lab), size=40).astype(np.int32)
    sums, counts = SW.eval_weighted(orc, w0, idx, wp, wn, sw, logistic=logistic)
    rows = CW.literal_rows(rp, col, val, dim)
    sums_l, counts_l = SW.literal_eval(SW.Sparse({j: float(v) for j, v in enumerate(w0)}, dim), rows, lab,
                                       [int(i) for i in idx], sw, wp, wn, logistic)
    assert list(sums) == sums_l   # both the device's limb sum of the same terms
    assert list(counts) == counts_l


@pytest.mark.parametrize("logistic", [False, True])
def test_unit_sample_weights_are_the_class_weighted_step(logistic):
    """At sample weights 1 the steps and the gradient are the class-weighted ones of the literal restatements: oracle/cw.py's
    without the L1 penalty, scala_semantics_margin.py's with it."""
    orc, (rp, col, val, lab, dim, d), w0, rng = dyadic_problem(5, n_rows=64)
    counts, lrs = [6, 4], [0.5, 0.25, 0.125]
    idx = rng.integers(0, 64, size=10 * 3).astype(np.int32)
    ones = np.ones(64)
    rows = CW.literal_rows(rp, col, val, dim)
    w = SW.Sparse({j: float(v) for j, v in enumerate(w0)}, dim)
    ids = [int(i) for i in idx[:10]]
    for wp, wn in ((1.0, 1.0), (2.0, 0.5)):
        for lambda1 in (0.0, 2.0 ** -5):
            w_sw, l_sw = SW.sync_steps(orc, w0, idx, counts, lrs, ones, wp, wn, logistic=logistic, lambda1=lambda1)
            if lambda1 == 0.0:
                w_cw, l_cw = CW.literal_sync_steps(rows, lab, dim, orc.lam, d, w0, idx, counts, lrs, wp, wn, logistic=logistic)
            else:
                w_cw, l_cw = literal_sync_steps(literal_model(logistic, orc.lam), rows, lab, dim, orc.lam, d, w0, idx, counts,
                                                lrs, wp, wn, None, 1 if (wp, wn) != (1.0, 1.0) else 0, lambda1)
            assert np.array_equal(w_sw, w_cw)
            if not logistic:   # dyadic hinge terms: both loss sums exact
                assert np.array_equal(l_sw, l_cw)
            else:              # the fixed-point sum against the literal sums: to rounding
                np.testing.assert_allclose(l_sw, l_cw, rtol=1e-15)
        g_sw, loss_sw, _ = SW.gradient(orc, w0, idx[:10], None, wp, wn, logistic=logistic)
        g_cw = SW.vec_sum([CW.literal_backward(w, rows[r], int(lab[r]), wp if lab[r] > 0 else wn, logistic) for r in ids])
        g_cw = g_cw + g_cw.value_like(orc.lam * 2.0 * w.dot(SW.Sparse({j: float(v) for j, v in enumerate(d)}, dim)))
        sums, _ = CW.literal_loss_sums(w, rows, lab, ids, logistic)
        assert np.array_equal(g_sw, [g_cw.get(j) for j in range(dim)])
        np.testing.assert_allclose(loss_sw, orc.lam * w.norm_squared() + (wp * sums[0] + wn * sums[1]) / 10,
                                   rtol=0 if not logistic else 1e-15)


def test_zero_weight_scatters_nothing_and_still_counts():
    # two rows over one column: row 0 (y = +1) at weight 0, row 1 (y = -1) at weight 1; w = 0: hinge 1 each, gate passes
    rp, col, val, lab = (np.array([0, 1, 2], np.int64), np.array([0, 0], np.int32), np.array([0.5, 0.25], np.float32),
                         np.array([1, -1], np.int8))
    orc = Oracle(rp, col, val, lab, 2, 0.0)
    orc.set_dim_sparsity(np.zeros(2))
    g, loss, s = SW.gradient(orc, np.zeros(2), [0, 1], np.array([0.0, 1.0]))
    assert list(g) == [-0.25, 0.0] and s == 1.0 and loss == 0.5   # S / n with n = 2 rows, the zero-weight one included
    sums, counts = SW.eval_weighted(orc, np.zeros(2), [0, 1], sw=np.array([0.0, 1.0]))
    assert list(sums) == [1.0, 0.0, 1.0] and list(counts) == [2, 0]


@pytest.mark.parametrize("above", [False, True])
def test_filter_edge_of_x_times_c(above):
    # x = 2^-10, c = s = 1e-20 * 2^10 (one ulp more when `above`): the product is exactly 1e-20 (filtered) or the next double
    s = float(np.float64(1e-20) * 1024.0)
    if above:
        s = float(np.nextafter(s, 1.0))
    x = 2.0 ** -10
    rp, col, val, lab = np.array([0, 1], np.int64), np.array([3], np.int32), np.array([x], np.float32), np.array([1], np.int8)
    orc = Oracle(rp, col, val, lab, 4, 0.0)
    orc.set_dim_sparsity(np.zeros(4))
    g, _, _ = SW.gradient(orc, np.zeros(4), [0], np.array([s]))
    expect = x * s
    assert (expect > 1e-20) == above
    assert g[3] == (expect if above else 0.0)
    if above:
        assert g[3] == TINY or g[3] > 1e-20


@pytest.mark.parametrize("logistic", [False, True])
def test_integer_weight_equals_the_row_listed_k_times(logistic):
    orc, _, w0, rng = dyadic_problem(8, n_rows=32, cls=LogisticOracle if logistic else Oracle)
    ids = np.arange(12, dtype=np.int32)
    k = rng.choice([0.0, 2.0, 4.0], size=32)
    sw = np.ones(32)
    sw[:12] = k[:12]
    rep = np.concatenate([np.repeat(ids[i:i + 1], int(sw[i])) for i in range(12)]).astype(np.int32)
    g_w, _, s_w = SW.gradient(orc, w0, ids, sw, logistic=logistic, regularize=False)
    g_r, _, s_r = SW.gradient(orc, w0, rep, None, logistic=logistic, regularize=False)
    if logistic:   # the scatter adds k copies of a product against one product times k: to rounding
        np.testing.assert_allclose(g_w, g_r, rtol=1e-14, atol=1e-300)
    else:
        assert np.array_equal(g_w, g_r)
    # k * L is exact (k a power of two or 0) and so is every term's rounding to 2^-160: the loss sums have the same bits
    assert s_w == s_r
    sums_w, _ = SW.eval_weighted(orc, w0, ids, sw=sw, logistic=logistic)
    sums_r, _ = SW.eval_weighted(orc, w0, rep, logistic=logistic)
    assert list(sums_w) == list(sums_r)
