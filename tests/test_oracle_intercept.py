"""The intercept's restatement (oracle/scala_semantics_intercept.py) on the CPU: without beta it is the checker of record's
plain step (oracle/margin.py) for every model, at lambda > 0 and with L1; at lambda = 0 without L1 its intercept step is
the plain step of the dim + 1 problem whose rows end in (dim, 1.0), bit for bit on dyadic rows; and planted cases where
counting beta in c, in ||w||^2 or in the L1 step would change the result."""
import numpy as np
import pytest

from oracle import scala_semantics_intercept as si

MODELS = ["svm", "logistic", "squared_hinge", "modified_huber"]


def _problem(seed, n=60, dim=24):
    rng = np.random.default_rng(seed)
    rows, rp, col, val = [], [0], [], []
    for _ in range(n):
        k = int(rng.integers(1, 7))
        cols = np.sort(rng.choice(dim, size=k, replace=False)).astype(np.int32)
        vals = (rng.integers(1, 257, size=k) * rng.choice([-1, 1], size=k) / 64.0).astype(np.float32)
        rows.append((cols, vals))
        col.extend(cols)
        val.extend(vals)
        rp.append(len(col))
    lab = rng.choice(np.array([-1, 1], np.int8), size=n)
    d = rng.integers(0, 17, size=dim) / 16.0
    return rows, np.array(rp, np.int64), np.array(col, np.int32), np.array(val, np.float32), lab, d


@pytest.mark.parametrize("model", MODELS)
@pytest.mark.parametrize("lam,l1", [(0.0, 0.0), (0.0625, 0.0), (0.0625, 0.25)])
def test_without_beta_it_is_the_checker_of_record(model, lam, l1):
    from oracle import margin
    from oracle.oracle import Oracle
    rows, rp, col, val, lab, d = _problem(1)
    dim = len(d)
    orc = Oracle(rp, col, val, lab, dim, lam)
    orc.set_dim_sparsity(d)
    rng = np.random.default_rng(2)
    ids = rng.integers(0, len(rows), size=8 * 5).astype(np.int32)
    w0 = rng.integers(-32, 33, size=dim) / 128.0
    lrs = [0.25, 0.125, 0.25, 0.0625, 0.25]
    w_ref, l_ref = margin.sync_steps(orc, model, w0, ids, [8], lrs, lambda1=l1)
    w, l = si.steps(rows, lab, d, w0, ids, 8, model, lam, lrs, l1, intercept=False)
    np.testing.assert_allclose(w, w_ref, rtol=1e-12, atol=1e-300)
    np.testing.assert_allclose(l, l_ref, rtol=1e-12)


@pytest.mark.parametrize("model", MODELS)
def test_the_intercept_is_the_augmented_column_at_lambda_zero(model):
    rows, rp, col, val, lab, d = _problem(3)
    dim = len(d)
    aug = [(np.append(c, dim).astype(np.int32), np.append(v, 1.0).astype(np.float32)) for c, v in rows]
    rng = np.random.default_rng(4)
    ids = rng.integers(0, len(rows), size=8 * 6).astype(np.int32)
    w0 = np.append(rng.integers(-32, 33, size=dim) / 128.0, 0.375)
    lrs = [0.25] * 6
    wi, li = si.steps(rows, lab, d, w0, ids, 8, model, 0.0, lrs)
    wa, la = si.steps(aug, lab, np.append(d, 0.0), w0, ids, 8, model, 0.0, lrs, intercept=False)
    if model == "svm":   # dyadic sums: exact in any order
        assert (wi.view(np.int64) == wa.view(np.int64)).all() and (li.view(np.int64) == la.view(np.int64)).all()
    else:                # beta is added after the row's dot, the augmented column inside it
        np.testing.assert_allclose(wi, wa, rtol=1e-13, atol=1e-300)
        np.testing.assert_allclose(li, la, rtol=1e-13)
    assert wi[dim] != 0.375


def test_beta_is_in_no_penalty():
    """One row x = (1 at column 0), y = +1, SVM, w = (0.5), beta = 0.5, d = (1): z = 1 >= 0 scatters s = 1."""
    rows = [(np.array([0], np.int32), np.array([1.0], np.float32))]
    lab, d = np.array([1], np.int8), np.array([1.0])
    w0 = np.array([0.5, 0.5])
    lam, lr = 0.25, 0.5
    w, loss = si.step(rows, lab, d, w0, [0], "svm", lam, lr)
    c = lam * 2.0 * 0.5                                  # 2 lambda (w . d) over the weight alone: 0.25
    assert w[0] == 0.5 - (1.0 + c) * lr                  # the weight's entry gets c
    assert w[1] == 0.5 - 1.0 * lr                        # beta's does not (with beta in c it would be 0.5 - 1.5 lr)
    assert loss == lam * 0.25 + 2.0                      # ||w||^2 = 0.25 without beta; hinge 1 - y p = 2 (score 1 > 0)
    w1, loss1 = si.step(rows, lab, d, w0, [0], "svm", 0.0, lr, lambda1=2.0)   # threshold lr * 2 = 1 >= |every value|
    assert w1[0] == 0.0 and w1[1] == 0.5 - 1.0 * lr      # beta is never thresholded
    assert loss1 == 2.0 * 0.5 + 2.0                      # ||w||_1 = 0.5 without beta
