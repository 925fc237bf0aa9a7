"""The class-weight checker (oracle/cw.py, the class weighting of oracle/dsgd_oracle_margin.c), without a GPU:

1. The C checker against the literal restatement over Sparse vectors on dyadic data, both models' paths that are exact there
   (SVM weights and losses bit for bit; logistic weights and losses to rounding), one and several workers, rate tables.
2. At weights (1, 1) it gives the unweighted steps, gradients and evaluations: against dsgd_oracle.c for the SVM's gradient
   and evaluation and against the literal restatements otherwise, weights bit for bit.
3. Hand-worked cases: a weight of 0 for one class, a product x_j * w_y at exactly 1e-20 and one ulp above, a batch whose
   weighted contributions cancel exactly in a column.
4. A structural known answer on dyadic data: with (w_pos, w_neg) = (2, 1) the raw gradient sum of a batch equals the unweighted
   sum over the same batch with every positive row taken twice, and the weighted hinge total equals that batch's hinge total.
"""
import numpy as np
import pytest

from oracle import cw as CW
from oracle import l1 as L1
from oracle import scala_semantics as S
from oracle.logistic import LogisticOracle
from oracle.oracle import Oracle
from oracle.scala_semantics_logistic import SparseLogistic
from oracle.scala_semantics_margin import literal_correct

TINY = np.nextafter(1e-20, 1.0)   # the smallest double the 1e-20 filter keeps


def dyadic_problem(seed, n_rows=48, dim=24, cls=Oracle, lam=2.0 ** -6):
    rng = np.random.default_rng(seed)
    rp, col, val = [0], [], []
    for _ in range(n_rows):
        k = int(rng.integers(0, 7))
        c = np.sort(rng.choice(dim, size=k, replace=False))
        col += c.tolist()
        val += (rng.integers(1, 17, size=k) / 8.0 * rng.choice([-1.0, 1.0], size=k)).tolist()
        rp.append(len(col))
    lab = rng.choice(np.array([-1, 1], dtype=np.int8), size=n_rows)
    rp, col, val = np.asarray(rp, np.int64), np.asarray(col, np.int32), np.asarray(val, np.float32)
    orc = cls(rp, col, val, lab, dim, lam)
    d = np.zeros(dim)
    d[::3] = 0.25
    orc.set_dim_sparsity(d)
    w0 = rng.integers(-8, 9, size=dim) / 16.0
    return orc, (rp, col, val, lab, dim, d), w0, rng


def literal_model(logistic: bool, lam: float):
    """The literal SparseSVM or SparseLogistic with the weighted backward of CW.literal_backward (c None: unweighted), as
    scala_semantics_margin.literal_sync_steps takes a model."""
    class Weighted(SparseLogistic if logistic else S.SparseSVM):
        def backward(self, w, x, y, c=None):
            return CW.literal_backward(w, x, y, 1.0 if c is None else c, logistic)
    return Weighted(lam, None)


@pytest.mark.parametrize("counts", [[8], [5, 3], [4, 3, 2]])
@pytest.mark.parametrize("wp,wn", [(4.0, 0.25), (0.0, 1.0), (2.0, 0.0), (1.0, 1.0)])
def test_svm_c_equals_literal_bit_for_bit_on_dyadic_data(counts, wp, wn):
    orc, (rp, col, val, lab, dim, d), w0, rng = dyadic_problem(3)
    lrs = [0.5, 0.25, 0.0, 0.125]
    idx = rng.integers(0, len(lab), size=sum(counts) * len(lrs)).astype(np.int32)
    w_c, l_c = CW.sync_steps(orc, w0, idx, counts, lrs, wp, wn)
    rows = CW.literal_rows(rp, col, val, dim)
    w_l, l_l = CW.literal_sync_steps(rows, lab, dim, orc.lam, d, w0, idx, counts, lrs, wp, wn)
    assert np.array_equal(w_c, np.asarray(w_l))
    assert list(l_c) == l_l


@pytest.mark.parametrize("counts", [[8], [5, 3]])
def test_logistic_c_equals_literal(counts):
    orc, (rp, col, val, lab, dim, d), w0, rng = dyadic_problem(4, cls=LogisticOracle)
    lrs = [0.5, 0.25, 0.125]
    idx = rng.integers(0, len(lab), size=sum(counts) * len(lrs)).astype(np.int32)
    w_c, l_c = CW.sync_steps(orc, w0, idx, counts, lrs, 4.0, 0.25, logistic=True)
    rows = CW.literal_rows(rp, col, val, dim)
    w_l, l_l = CW.literal_sync_steps(rows, lab, dim, orc.lam, d, w0, idx, counts, lrs, 4.0, 0.25, logistic=True)
    np.testing.assert_allclose(w_c, w_l, rtol=1e-13, atol=1e-15)
    np.testing.assert_allclose(l_c, l_l, rtol=1e-14)
    sums, cnt = CW.eval_class(orc, w0, idx, logistic=True)
    sums_l, cnt_l = CW.literal_loss_sums(CW.Sparse({j: float(v) for j, v in enumerate(w0)}, dim), rows, lab,
                                         [int(i) for i in idx], True)
    np.testing.assert_allclose(sums, sums_l, rtol=1e-15)
    assert list(cnt) == cnt_l


@pytest.mark.parametrize("logistic", [False, True])
def test_unit_weights_are_the_unweighted_step(logistic):
    """At weights (1, 1): the steps against oracle/l1.py's literal restatement, with and without the L1 penalty; the gradient
    and the evaluation against dsgd_oracle.c for the SVM and against scala_semantics_logistic.py for the logistic model."""
    orc, (rp, col, val, lab, dim, d), w0, rng = dyadic_problem(5, n_rows=64)
    counts, lrs = [6, 4], [0.5, 0.25, 0.125]
    idx = rng.integers(0, 64, size=10 * 3).astype(np.int32)
    for lambda1 in (0.0, 2.0 ** -5):
        w_cw, l_cw = CW.sync_steps(orc, w0, idx, counts, lrs, 1.0, 1.0, logistic=logistic, lambda1=lambda1)
        w_ref, l_ref = L1.literal_sync_steps(rp, col, val, lab, dim, orc.lam, lambda1, d, w0, idx, counts, lrs, logistic=logistic)
        assert np.array_equal(w_cw, w_ref)
        np.testing.assert_allclose(l_cw, l_ref, rtol=0 if not logistic else 1e-15)
    g, loss, sums = CW.gradient(orc, w0, idx[:10], 1.0, 1.0, logistic=logistic)
    if logistic:
        rows, ids = CW.literal_rows(rp, col, val, dim), [int(i) for i in idx[:10]]
        w = S.Sparse({j: float(v) for j, v in enumerate(w0)}, dim)
        model = SparseLogistic(orc.lam, S.Sparse({j: float(v) for j, v in enumerate(d)}, dim))
        data = [(rows[r], int(lab[r])) for r in range(len(lab))]
        g_ref = S.slave_gradient(model, data, w, ids)
        g_ref = [g_ref.get(j) for j in range(dim)]
        loss_ref, acc_ref = model.loss(w, [data[r] for r in ids]), literal_correct(w, rows, lab, ids) / 10
    else:
        g_ref, _ = orc.gradient(w0, idx[:10])
        loss_ref, acc_ref = orc.loss_acc(w0, idx=idx[:10])
    assert np.array_equal(g, g_ref)
    np.testing.assert_allclose(loss, loss_ref, rtol=0 if not logistic else 1e-15)
    s, c = CW.eval_class(orc, w0, idx[:10], logistic=logistic)
    assert (c[0] + c[1]) / 10 == acc_ref and c[2] + c[3] == 10


def one_row(vals, label, dim=4):
    rp = np.array([0, len(vals)], np.int64)
    orc = Oracle(rp, np.arange(len(vals), dtype=np.int32), np.asarray(vals, np.float32), np.array([label], np.int8), dim, 0.0)
    orc.set_dim_sparsity(np.zeros(dim))
    return orc


def test_zero_weight_class_adds_nothing_and_costs_nothing():
    orc, _, w0, rng = dyadic_problem(6)
    idx = np.arange(20, dtype=np.int32)
    g, loss, sums = CW.gradient(orc, w0, idx, 0.0, 1.0, regularize=False)
    neg = idx[orc.label[idx] < 0]
    g_neg, _, sums_neg = CW.gradient(orc, w0, neg, 1.0, 1.0, regularize=False)
    assert np.array_equal(g, g_neg) and sums[1] == sums_neg[1]
    assert loss == orc.lam * float(np.dot(w0, w0)) + sums[1] / 20


def test_filter_edge_of_the_weighted_product():
    """x_j * w_y at exactly 1e-20 is dropped, one ulp above is kept: x = 2^-10 (exact in fp32), w_y = v * 2^10."""
    orc = one_row([2.0 ** -10], +1)
    for v, kept in ((1e-20, False), (TINY, True)):
        g, _, _ = CW.gradient(orc, np.zeros(4), [0], v * 1024.0, 1.0, regularize=False)
        assert g[0] == (v if kept else 0.0)
    orc = one_row([2.0 ** -10], -1)
    g, _, _ = CW.gradient(orc, np.zeros(4), [0], 1.0, TINY * 1024.0, regularize=False)
    assert g[0] == -TINY


def test_weighted_contributions_cancel_exactly_in_a_column():
    """Rows (+1: x_0 = 1, x_1 = 1) and (-1: x_0 = 4, x_1 = 1) with weights (4, 1): column 0 gets 4 - 4 = 0 and is absent from
    the reply (no c added), column 1 gets 4 - 1 = 3 (+ c)."""
    rp = np.array([0, 2, 4], np.int64)
    col = np.array([0, 1, 0, 1], np.int32)
    orc = Oracle(rp, col, np.array([1, 1, 4, 1], np.float32), np.array([1, -1], np.int8), 3, 0.5)
    d = np.array([0.0, 0.0, 1.0])
    orc.set_dim_sparsity(d)
    w = np.array([0.0, 0.0, 0.25])   # c = 2 * 0.5 * 0.25 = 0.25, every dot 0
    g, loss, sums = CW.gradient(orc, w, [0, 1], 4.0, 1.0)
    assert list(g) == [0.0, 3.25, 0.0]
    assert list(sums) == [1.0, 1.0] and loss == 0.5 * 0.0625 + (4.0 + 1.0) / 2


def test_weight_two_is_the_positive_rows_taken_twice():
    orc, _, w0, rng = dyadic_problem(7, n_rows=80)
    idx = rng.integers(0, 80, size=32).astype(np.int32)
    doubled = np.concatenate([idx, idx[orc.label[idx] > 0]]).astype(np.int32)
    g, _, sums = CW.gradient(orc, w0, idx, 2.0, 1.0, regularize=False)
    g2, _, sums2 = CW.gradient(orc, w0, doubled, 1.0, 1.0, regularize=False)
    assert np.array_equal(g, g2)
    assert 2.0 * sums[0] + sums[1] == sums2[0] + sums2[1]
