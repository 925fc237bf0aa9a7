"""Planted margins of the squared-hinge and modified-Huber models, without a GPU: the known-answer table that
tests/test_gpu_margin_exact.py checks the device against, checked here against the margin checker
(oracle/dsgd_oracle_margin.c).

Every planted row has x = 1 (fp32) on columns of its own and the weight y * z there, so that its dot is exactly y * z and
its margin exactly z (a NaN margin: two columns at +inf and -inf).  KNOWN lists (L, s) by hand; the tests derive the same
values from fractions.Fraction, in the order of operations the models state (t = fl(1 + z), then t * t, 2 * t or 4 * z, each
correctly rounded), and every per-row value an evaluation, a gradient or a probability reports from the sum model of
tests/loss_sum_model.py.  Nothing here calls the code it checks to make an expected value.

The planted margins cover both branch points and the ulps beside them, fl(1 + z) = 2 just below z = 1, the 2^52 limit of
the fixed-point loss sum (the squared hinge reaches it at z = 2^26 - 1, where t * t = 2^52, modified Huber at z = 2^50,
where 4 z = 2^52), a loss in [2^51, 2^52), a squared hinge whose t * t overflows to inf, and NaN."""
import math
from fractions import Fraction

import numpy as np
import pytest

from loss_sum_model import MAX_VALUE, R
from oracle import margin as M
from oracle.oracle import Oracle

MODELS = ("squared_hinge", "modified_huber")
WEIGHTINGS = ("none", "class", "sample")
W_POS, W_NEG = 2.0, 0.5
SAMPLE_CYCLE = (0.75, 3.0, 0.1, 0.0, 1.0 / 3.0)   # sample weights of the planted rows, in turn
NAN = math.nan
SH_HALF = 47453132.0    # squared hinge: t = 47453133, t * t = 2251799831515689 in [2^51, 2^52)
MH_HALF = 3.0 * 2.0 ** 48   # modified Huber: 4 z = 3 * 2^50 in [2^51, 2^52)
HUGE = 2.0 ** 600       # squared hinge: t * t overflows to inf

# z -> (L, s), by hand
KNOWN = {
    "squared_hinge": {
        -1.0 - 2.0 ** -52: (0.0, 0.0),
        -1.0: (0.0, 0.0),
        -1.0 + 2.0 ** -53: (2.0 ** -106, 2.0 ** -52),       # t = 2^-53 exactly
        -0.5: (0.25, 1.0),
        0.0: (1.0, 2.0),
        1.0 - 2.0 ** -53: (4.0, 4.0),                        # fl(2 - 2^-53) = 2 (ties to even)
        1.0: (4.0, 4.0),
        1.0 + 2.0 ** -52: (4.0, 4.0),                        # fl(2 + 2^-52) = 2 (ties to even)
        2.0 ** 26 - 2.0: (2.0 ** 52 - 2.0 ** 27 + 1.0, 2.0 ** 27 - 2.0),   # the largest loss that is summed
        2.0 ** 26 - 1.0: (2.0 ** 52, 2.0 ** 27),             # t * t = 2^52: not summed
        SH_HALF: (2251799831515689.0, 94906266.0),
        HUGE: (math.inf, 2.0 ** 601),
        NAN: (NAN, NAN),                                     # the filter drops a NaN scale: no gradient
    },
    "modified_huber": {
        -1.0 - 2.0 ** -52: (0.0, 0.0),
        -1.0: (0.0, 0.0),
        -1.0 + 2.0 ** -53: (2.0 ** -106, 2.0 ** -52),
        -0.5: (0.25, 1.0),
        0.0: (1.0, 2.0),
        1.0 - 2.0 ** -53: (4.0, 4.0),
        1.0: (4.0, 4.0),
        1.0 + 2.0 ** -52: (4.0 + 2.0 ** -50, 4.0),          # the linear branch: 4 z exactly
        2.0 ** 50 - 1.0: (2.0 ** 52 - 4.0, 4.0),             # the largest loss that is summed
        2.0 ** 50: (2.0 ** 52, 4.0),                          # 4 z = 2^52: not summed
        MH_HALF: (3.0 * 2.0 ** 50, 4.0),
        HUGE: (2.0 ** 602, 4.0),
        NAN: (NAN, 4.0),                                      # both comparisons false: the linear branch's scale
    },
}


def same(a, b) -> bool:
    """a == b, NaN equal to NaN"""
    return a == b or (math.isnan(a) and math.isnan(b))


def _fl(q: Fraction) -> float:
    """q correctly rounded to a double (inf past the largest one)"""
    try:
        return float(q)
    except OverflowError:
        return math.inf if q > 0 else -math.inf


def exact_row(model, z):
    """(L, s) from Fraction: t = fl(1 + z), then fl(t * t) and fl(2 t) (or fl(4 z) and 4 above z = 1 for modified Huber)."""
    if math.isnan(z):   # z <= -1 and z <= 1 are false: t * t, 2 t and 4 z are NaN, the linear branch's scale is 4
        return NAN, (NAN if model == "squared_hinge" else 4.0)
    if z <= -1.0:
        return 0.0, 0.0
    if model == "modified_huber" and z > 1.0:
        return _fl(4 * Fraction(z)), 4.0
    t = _fl(1 + Fraction(z))
    return _fl(Fraction(t) ** 2), _fl(2 * Fraction(t))


def r_value(v) -> float:
    """What one summed value reports: R(v), NaN if it is not summed (NaN, inf, >= 2^52)"""
    r = R(v)
    return NAN if r is None else float(r)


def planted_rows(model):
    """[(z, y, sample weight)] of a model's planted table, the labels alternating"""
    return [(z, 1 if k % 2 == 0 else -1, SAMPLE_CYCLE[k % len(SAMPLE_CYCLE)]) for k, z in enumerate(KNOWN[model])]


def planted_csr(rows, extra=()):
    """CSR of planted rows [(z, y, ...)] with x = 1 on columns of their own, and the weights per row: row r's dot is y * z
    at ws[r] (a NaN margin: columns at +inf and -inf).  `extra`: (row, value) entries on further columns of their own,
    at weight 0.  Returns (rp, col, val, lab, dim, ws, cols): ws[r] the dense weights of row r alone, cols[r] its
    planted columns."""
    rp, col, val, cols, wv = [0], [], [], [], []
    extra = list(extra)
    for r, (z, y, *_) in enumerate(rows):
        mine = []
        if math.isnan(z):
            mine = [(len(wv), 1.0, math.inf), (len(wv) + 1, 1.0, -math.inf)]
        else:
            mine = [(len(wv), 1.0, y * z)]
        wv += [m[2] for m in mine]
        for e_row, e_val in extra:
            if e_row == r:
                mine.append((len(wv), e_val, 0.0))
                wv.append(0.0)
        col += [m[0] for m in mine]
        val += [m[1] for m in mine]
        cols.append([m[0] for m in mine[:2 if math.isnan(z) else 1]])
        rp.append(len(col))
    dim = max(len(wv), 2)
    ws = []
    for r in range(len(rows)):
        w = np.zeros(dim)
        for c in cols[r]:
            w[c] = wv[c]
        ws.append(w)
    lab = np.array([y for _, y, *_ in rows], np.int8)
    return (np.array(rp, np.int64), np.array(col, np.int32), np.array(val, np.float32), lab, dim, ws, cols)


def row_weight(weighting, y, s_i):
    """c_i of a row: 1, w_y or fl(w_y * s_i)"""
    wy = W_POS if y > 0 else W_NEG
    return 1.0 if weighting == "none" else (wy if weighting == "class" else wy * s_i)


def expected_row(model, weighting, z, y, s_i):
    """Every per-row value the device reports for one planted row, from the table:
    S (unweighted evaluation), (S+, S-) (per-class evaluation), the weighted evaluation's (S, sum c [correct], sum c),
    the one-row gradient's loss at lambda = 0 and its entry on the row's column, the prediction and the modified-Huber
    probability."""
    L, s = KNOWN[model][z]
    dot = y * z
    pred = 0.0 if (math.isnan(dot) or dot == 0.0) else (-1.0 if dot > 0.0 else 1.0)
    c = row_weight(weighting, y, s_i)   # also the weighted evaluation's c_i: w = (1, 1) and s_i = 1 when unset
    sums = r_value(L)
    cls = (sums, 0.0) if y > 0 else (0.0, sums)
    weighted = (r_value(c * L), r_value(c) if pred == y else 0.0, r_value(c))
    if weighting == "class":
        loss = W_POS * cls[0] + W_NEG * cls[1]
    elif weighting == "sample":
        loss = r_value(c * L)
    else:
        loss = sums
    v = y * s if weighting == "none" else (y * s) * c
    g = v if abs(v) > 1e-20 else 0.0
    m = -dot
    m = NAN if math.isnan(m) else min(max(m, -1.0), 1.0)
    prob = (m + 1.0) / 2.0
    return dict(sums=sums, cls=cls, weighted=weighted, loss=loss, g=g, pred=pred, prob=prob)


# ---- the table --------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("model", MODELS)
def test_table_is_the_exact_arithmetic(model):
    for z, (L, s) in KNOWN[model].items():
        el, es = exact_row(model, z)
        assert same(el, L) and same(es, s), (z, (el, es), (L, s))


@pytest.mark.parametrize("model", MODELS)
def test_table_covers_the_edges(model):
    """The 2^52 limit is met exactly: the last summed loss is below it, the next one is it."""
    ls = {z: L for z, (L, _) in KNOWN[model].items()}
    last, first_out = (2.0 ** 26 - 2.0, 2.0 ** 26 - 1.0) if model == "squared_hinge" else (2.0 ** 50 - 1.0, 2.0 ** 50)
    assert ls[last] < MAX_VALUE and R(ls[last]) == ls[last]
    assert ls[first_out] == MAX_VALUE and R(ls[first_out]) is None
    half = SH_HALF if model == "squared_hinge" else MH_HALF
    assert 2.0 ** 51 <= ls[half] < 2.0 ** 52
    if model == "squared_hinge":
        assert ls[HUGE] == math.inf


@pytest.mark.parametrize("model", MODELS)
def test_table_matches_the_checker_row(model):
    for z, (L, s) in KNOWN[model].items():
        l, sc = M.row(model, z)
        assert same(l, L) and same(sc, s), (z, (l, sc), (L, s))


def _checker(model, rows, extra=()):
    rp, col, val, lab, dim, ws, cols = planted_csr(rows, extra)
    orc = Oracle(rp, col, val, lab, dim, 0.0)
    orc.set_dim_sparsity(np.zeros(dim))
    return orc, ws, cols


@pytest.mark.parametrize("model", MODELS)
@pytest.mark.parametrize("weighting", WEIGHTINGS)
def test_one_row_values_match_the_checker(model, weighting):
    """Every one-row value of expected_row against the checker's gradient, evaluations and prediction."""
    rows = planted_rows(model)
    orc, ws, cols = _checker(model, rows)
    sw = np.array([s for _, _, s in rows]) if weighting == "sample" else None
    wp, wn = (W_POS, W_NEG) if weighting != "none" else (1.0, 1.0)
    for r, (z, y, s_i) in enumerate(rows):
        e = expected_row(model, weighting, z, y, s_i)
        w = ws[r]
        _, _, s0, _ = M.loss_acc(orc, model, w, [r])
        assert same(s0, e["sums"]), (z, s0, e["sums"])
        sums, counts = M.eval_class(orc, model, w, [r])
        assert same(sums[0], e["cls"][0]) and same(sums[1], e["cls"][1]), (z, sums, e["cls"])
        wsums, _ = M.eval_weighted(orc, model, w, [r], wp, wn, sw)
        assert all(same(a, b) for a, b in zip(wsums, e["weighted"])), (z, wsums, e["weighted"])
        g, loss, _ = M.gradient(orc, model, w, [r], wp, wn, sw)
        assert same(loss, e["loss"]), (z, loss, e["loss"])
        assert (g[cols[r]] == e["g"]).all() and np.count_nonzero(g) == len(cols[r]) * (e["g"] != 0.0), (z, g[cols[r]], e["g"])
        assert same(orc.forward(w, [r])[0], e["pred"]), z
