"""The checker of the margin models (oracle/dsgd_oracle_margin.c), without a GPU:
1. hand-computed known answers of L(z) and s(z) for both models, both branch points included;
2. the C checker against the literal restatement over Sparse vectors (oracle/scala_semantics_margin.py) bit for bit on
   random dyadic problems, in every weighting, with L1, the averaging sum and rate tables;
3. its SVM (0) and logistic (1) forms against the same literal restatement with those models' backward (oracle/cw.py), bit
   for bit in the class and sample weightings with L1 and the averaging sum."""
import numpy as np
import pytest

from oracle import cw as CW
from oracle import margin as M
from oracle.scala_semantics_margin import MODEL_CLASSES, literal_correct, literal_pass_loss, literal_sync_steps
from oracle.scala_semantics import Sparse
from test_oracle_class_weight import dyadic_problem, literal_model
from test_oracle_sample_weight import dyadic_weights

MARGIN = ("squared_hinge", "modified_huber")
# z -> (L, s) by hand: t = 1 + z; squared hinge t^2, 2t above z = -1; modified Huber t^2, 2t on (-1, 1], 4z, 4 above
KNOWN = {
    "squared_hinge": {-1.5: (0.0, 0.0), -1.0: (0.0, 0.0), -0.5: (0.25, 1.0), 0.0: (1.0, 2.0), 1.0: (4.0, 4.0),
                      1.5: (6.25, 5.0)},
    "modified_huber": {-1.5: (0.0, 0.0), -1.0: (0.0, 0.0), -0.5: (0.25, 1.0), 0.0: (1.0, 2.0), 1.0: (4.0, 4.0),
                       1.5: (6.0, 4.0)},
}


@pytest.mark.parametrize("model", MARGIN)
@pytest.mark.parametrize("z", [-1.5, -1.0, -0.5, 0.0, 1.0, 1.5])
def test_known_answers(model, z):
    assert M.row(model, z) == KNOWN[model][z]
    lit = MODEL_CLASSES[model]
    assert (lit.loss_z(z), lit.scale_z(z)) == KNOWN[model][z]


@pytest.mark.parametrize("model", MARGIN)
def test_branch_points(model):
    """Just past z = -1 the row has a loss and a gradient; modified Huber is continuous at z = 1 in value and slope."""
    above = np.nextafter(-1.0, 0.0)
    l, s = M.row(model, above)
    assert 0.0 < l < 1e-30 and 0.0 < s < 1e-15
    if model == "modified_huber":
        below_one, above_one = np.nextafter(1.0, 0.0), np.nextafter(1.0, 2.0)
        # fl(1 + z) rounds 2 - 2^-53 to 2 (ties to even): just below 1 the quadratic branch already reaches 4
        assert M.row(model, below_one) == (4.0, 4.0) and M.row(model, 0.75) == (3.0625, 3.5)
        assert M.row(model, above_one) == (4.0 * above_one, 4.0) and 4.0 * above_one > 4.0


def test_models_differ_only_above_one():
    for z in (-3.0, -1.0, -0.75, 0.5, 1.0):
        assert M.row("squared_hinge", z) == M.row("modified_huber", z)
    assert M.row("squared_hinge", 3.0) == (16.0, 8.0) and M.row("modified_huber", 3.0) == (12.0, 4.0)


def _weights(weighting, rng, n):
    if weighting == "none":
        return 1.0, 1.0, None
    if weighting == "class":
        return 4.0, 0.25, None
    return 2.0, 0.5, dyadic_weights(rng, n)


def _code(wp, wn, sw):
    return 2 if sw is not None else (1 if (wp, wn) != (1.0, 1.0) else 0)


@pytest.mark.parametrize("model", MARGIN)
@pytest.mark.parametrize("weighting", ["none", "class", "sample"])
@pytest.mark.parametrize("counts,lambda1,avg", [([8], 0.0, False), ([5, 3], 0.0, True), ([4, 3, 2], 2.0 ** -7, False),
                                                ([6], 2.0 ** -8, True)])
def test_c_equals_literal_bit_for_bit_on_dyadic_data(model, weighting, counts, lambda1, avg):
    orc, (rp, col, val, lab, dim, d), w0, rng = dyadic_problem(40 + len(counts))
    wp, wn, sw = _weights(weighting, rng, len(lab))
    lrs = [0.25, 0.125, 0.0, 0.0625]
    idx = rng.integers(0, len(lab), size=sum(counts) * len(lrs)).astype(np.int32)
    avg_c = np.zeros(dim) if avg else None
    avg_l = [0.0] * dim if avg else None
    w_c, l_c = M.sync_steps(orc, model, w0, idx, counts, lrs, wp, wn, sw, lambda1=lambda1, avg_sum=avg_c)
    rows = CW.literal_rows(rp, col, val, dim)
    w_l, l_l = literal_sync_steps(MODEL_CLASSES[model](orc.lam, None), rows, lab, dim, orc.lam, d, w0, idx, counts, lrs,
                                  wp, wn, sw, _code(wp, wn, sw), lambda1, avg_l)
    assert np.array_equal(w_c, np.asarray(w_l))
    assert list(l_c) == l_l
    if avg:
        assert np.array_equal(avg_c, np.asarray(avg_l))


@pytest.mark.parametrize("model", MARGIN)
@pytest.mark.parametrize("weighting", ["none", "class", "sample"])
def test_gradient_and_evaluations_equal_literal(model, weighting):
    orc, (rp, col, val, lab, dim, d), w0, rng = dyadic_problem(50)
    wp, wn, sw = _weights(weighting, rng, len(lab))
    rows = CW.literal_rows(rp, col, val, dim)
    lit = MODEL_CLASSES[model](orc.lam, None)
    w = Sparse({j: float(v) for j, v in enumerate(w0)}, dim)
    ids = rng.integers(0, len(lab), size=20).tolist()
    code = _code(wp, wn, sw)
    g, loss, s = M.gradient(orc, model, w0, ids, wp, wn, sw, regularize=False)
    g_l = Sparse({}, dim)
    for r in ids:
        c = None if code == 0 else ((wp if lab[r] > 0 else wn) * (1.0 if sw is None else float(sw[r])) if code == 2
                                    else (wp if lab[r] > 0 else wn))
        g_l = g_l + lit.backward(w, rows[r], int(lab[r]), c)
    assert np.array_equal(g, np.asarray([g_l.get(j) for j in range(dim)]))
    assert s == literal_pass_loss(lit, w, rows, lab, ids, wp, wn, sw, code)
    _, _, s0, correct = M.loss_acc(orc, model, w0, ids)
    assert s0 == literal_pass_loss(lit, w, rows, lab, ids) and correct == literal_correct(w, rows, lab, ids)
    sums, counts = M.eval_class(orc, model, w0, ids)
    pos = [r for r in ids if lab[r] > 0]
    neg = [r for r in ids if lab[r] <= 0]
    assert list(sums) == [literal_pass_loss(lit, w, rows, lab, pos), literal_pass_loss(lit, w, rows, lab, neg)]
    assert list(counts) == [literal_correct(w, rows, lab, pos), literal_correct(w, rows, lab, neg), len(pos), len(neg)]
    wsums, wcounts = M.eval_weighted(orc, model, w0, ids, wp, wn, sw)
    assert wsums[0] == literal_pass_loss(lit, w, rows, lab, ids, wp, wn, sw, 2)
    assert list(wcounts) == [len(ids), correct]


def test_sample_losses_match_rows():
    orc, _, w0, rng = dyadic_problem(51)
    for model in MARGIN:
        ls = M.sample_losses(orc, model, w0, begin=0, n=orc.n_rows)
        z = orc.label * np.array([M.loss_acc(orc, model, w0, [r])[2] for r in range(orc.n_rows)])
        assert np.array_equal(ls, z / orc.label)   # one row's S is its loss


@pytest.mark.parametrize("model", [0, 1])
@pytest.mark.parametrize("weighting", ["class", "sample"])
def test_models_zero_and_one_equal_literal(model, weighting):
    """The SVM and logistic forms of the checker against the literal restatement of the weighted, L1 and averaged steps
    (scala_semantics_margin.py) with the literal SparseSVM / SparseLogistic: weights, averaging sums and losses bit for
    bit."""
    orc, (rp, col, val, lab, dim, d), w0, rng = dyadic_problem(52)
    wp, wn, sw = _weights(weighting, rng, orc.n_rows)
    counts, lrs = [6, 4], [0.25, 0.125, 0.0625]
    idx = rng.integers(0, orc.n_rows, size=sum(counts) * len(lrs)).astype(np.int32)
    avg_m, avg_l = np.zeros(orc.dim), [0.0] * dim
    w_m, l_m = M.sync_steps(orc, model, w0, idx, counts, lrs, wp, wn, sw, lambda1=2.0 ** -8, avg_sum=avg_m)
    w_l, l_l = literal_sync_steps(literal_model(model == 1, orc.lam), CW.literal_rows(rp, col, val, dim), lab, dim, orc.lam, d,
                                  w0, idx, counts, lrs, wp, wn, sw, _code(wp, wn, sw), 2.0 ** -8, avg_l)
    assert np.array_equal(w_m, np.asarray(w_l)) and np.array_equal(avg_m, np.asarray(avg_l))
    assert list(l_m) == l_l
