"""SparseSquaredHinge and SparseModifiedHuber on the GPU, checked exactly, each model in each weighting (none, class,
sample):

a. Planted margins (tests/test_oracle_margin_planted.py: x = 1 on columns of their own, the weight y * z there): every
   one-row evaluation, gradient, prediction and modified-Huber probability against the known-answer table, at both
   branch points and the ulps beside them, at the 2^52 limit of the fixed-point loss sum, at an overflowing t * t and at NaN.
b. The 2^52 rule and the recovery from it: a pass or a step with one row whose loss is not summed reads NaN, exactly as
   the checker does, and the next pass or step at the same weights without that row reads its finite value, in every
   evaluation form and in the steps of one and of several virtual workers.  The class-weighted forms sum the unweighted
   losses per class and scale the sums (fl(w_pos S+) + fl(w_neg S-)); the sample-weighted forms sum R(fl(c_i L_i)).  So a
   class weight of 2 with L in [2^51, 2^52) is finite in the first and NaN in the second, and a class weight of 0 with
   L >= 2^52 is NaN (0 * NaN) in the first and an exact 0 in the second.
c. The 1e-20 filter under scales above 1: the scatter is filt(filt(x) * ((y * s) * c)), so an entry at or below 1e-20
   adds nothing even where x * s is above it (k_repack stores it as 0 when the rows are loaded), and an entry above it adds
   nothing where x * (y * s) * c falls below it.
d. Pass sums of every size and form against the exact sum of the per-row values, per class and sample-weighted too.
e. A step's loss is lambda ||w||^2 (+ lambda1 ||w||_1) + S / n for the S an evaluation of the same ids reports at the
   pre-step weights, folded over virtual workers in fp64, bit for bit.
f. Dyadic rows sharing columns, hot columns included: gradients and sync runs bit for bit against the checker, for as many
   steps as a witness proves every sum exact in any order (so that the order of the device's REDs cannot matter).
g. (Two GPUs) the part f trajectory over NCCL."""
import math
import os
import socket
import sys
from fractions import Fraction

import numpy as np
import pytest

from loss_sum_model import R, describe, exact_sum, r_units, within_one_ulp
from oracle import margin as M
from oracle.oracle import Oracle
from test_oracle_margin_planted import (KNOWN, MH_HALF, MODELS, SH_HALF, W_NEG, W_POS, WEIGHTINGS, exact_row,
                                        expected_row, planted_csr, planted_rows, r_value, same)
from test_oracle_sample_weight import dyadic_weights

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LAM = 1e-5
OVER = {"squared_hinge": 2.0 ** 26 - 1.0, "modified_huber": 2.0 ** 50}   # L = 2^52: the first loss not summed
HALF = {"squared_hinge": SH_HALF, "modified_huber": MH_HALF}             # L in [2^51, 2^52)


@pytest.fixture(scope="module")
def sm():
    from distributed_sgd_b200.native import NativeCtx
    with NativeCtx(0, 16, 0.1) as c:
        return int(c.info()["sm_count"])


def _ctx(model, rp, col, val, lab, dim, lam=0.0, d=None):
    from distributed_sgd_b200.native import NativeCtx
    ctx = NativeCtx(0, dim, lam, model=model)
    ctx.load_csr(rp, col, val, lab)
    ctx.set_dim_sparsity(np.zeros(dim) if d is None else d)
    return ctx


def _set_weighting(ctx, weighting, sw, w_pos=W_POS, w_neg=W_NEG):
    """Installs a weighting; returns (w_pos, w_neg, sw) for the checker."""
    if weighting == "none":
        return 1.0, 1.0, None
    ctx.set_class_weights(w_pos, w_neg)
    if weighting == "class":
        return w_pos, w_neg, None
    ctx.set_sample_weights(sw)
    return w_pos, w_neg, sw


def _clear_weighting(ctx):
    ctx.set_class_weights(1.0, 1.0)
    ctx.set_sample_weights(None)


# ---- a. planted margins ------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("weighting", WEIGHTINGS)
@pytest.mark.parametrize("model", MODELS)
def test_planted_margins_bit_for_bit(model, weighting):
    rows = planted_rows(model)
    rp, col, val, lab, dim, ws, cols = planted_csr(rows)
    ctx = _ctx(model, rp, col, val, lab, dim)
    try:
        _set_weighting(ctx, weighting, np.array([s for *_, s in rows]))
        for r, (z, y, s_i) in enumerate(rows):
            e = expected_row(model, weighting, z, y, s_i)
            w = ws[r]
            what = f"row {r}, z = {z!r}"
            assert same(ctx.eval_samples_sums([r], w)[0], e["sums"]), what
            ce = ctx.eval_samples_class([r], w)
            assert same(ce.loss_pos, e["cls"][0]) and same(ce.loss_neg, e["cls"][1]), (what, ce)
            we = ctx.eval_samples_weighted([r], w)
            assert all(same(a, b) for a, b in zip((we.loss_sum, we.correct_weight, we.weight_sum), e["weighted"])), (what, we)
            g, loss = ctx.gradient([r], w, want_loss=True)
            with np.errstate(over="ignore"):
                want = e["loss"] if np.isfinite(np.dot(w, w)) else math.nan   # lambda ||w||^2 = 0 * inf
            assert same(loss, want), (what, loss, want)
            assert (g[cols[r]] == e["g"]).all() and np.count_nonzero(g) == len(cols[r]) * (e["g"] != 0.0), (what, g[cols[r]])
            assert ctx.forward([r], w)[0] == e["pred"], what
            if model == "modified_huber":
                p = ctx.probabilities([r], w)[0]
                assert same(p, e["prob"]) and (math.isnan(p) or np.signbit(p) == np.signbit(e["prob"])), (what, p, e["prob"])
        if model == "modified_huber":
            # both clip ends and the -0.0 margin of a zero dot are planted
            probs = {expected_row(model, "none", z, y, s)["prob"] for z, y, s in rows}
            assert {0.0, 0.5, 1.0} <= probs
    finally:
        ctx.close()


# ---- b. the 2^52 rule and the recovery ---------------------------------------------------------------------------------

ORDINARY = [(-0.5, 1), (0.25, -1), (1.5, 1), (-2.0, -1), (0.75, 1), (3.0, -1), (-1.0 + 2.0 ** -53, 1), (1.0, -1)]
SW_B = (0.75, 3.0, 0.1, 1.0 / 3.0, 2.5)


def _rule_problem(model, head):
    """Rows head + ORDINARY (each (z, y)) with their sample weights, the checker, the ctx and the weights of every row."""
    rows = [(z, y, SW_B[k % len(SW_B)]) for k, (z, y) in enumerate(list(head) + ORDINARY)]
    rp, col, val, lab, dim, ws, _ = planted_csr(rows)
    w = np.sum(ws, axis=0)
    orc = Oracle(rp, col, val, lab, dim, 0.0)
    orc.set_dim_sparsity(np.zeros(dim))
    ctx = _ctx(model, rp, col, val, lab, dim)
    ctx.set_weights(w)
    return rows, orc, ctx, w, np.array([s for *_, s in rows])


def _loss(model, z):
    return exact_row(model, z)[0]


@pytest.mark.parametrize("model", MODELS)
def test_over_limit_evaluations_read_nan_then_recover(model):
    """Rows 0 (y = +1) and 1 (y = -1) have L = 2^52.  Every NaN pass is followed by a finite pass of another form."""
    from distributed_sgd_b200.native import host_lib
    rows, orc, ctx, w, _ = _rule_problem(model, [(OVER[model], 1), (OVER[model], -1)])
    try:
        n = len(rows)
        ids = np.arange(n, dtype=np.int32)
        ok = ids[2:]
        ex = exact_sum([_loss(model, z) for z, *_ in rows[2:]])
        want = orc_s = M.loss_acc(orc, model, w, ok)[2]
        assert within_one_ulp(want, ex), describe(want, ex)
        assert math.isnan(M.loss_acc(orc, model, w, ids)[2])
        key = 0xB52
        drawn_ok = np.array([2 + host_lib().dsgd_feistel_pos(p, n - 2, key) for p in range(n - 2)], np.int32)
        passes = [
            ("range", lambda: ctx.eval_sums(0, n)[0], lambda: ctx.eval_sums(2, n)[0]),
            ("list", lambda: ctx.eval_samples_sums(ids[::-1].copy())[0], lambda: ctx.eval_samples_sums(ok)[0]),
            ("drawn", lambda: ctx.eval_sampled_sums(0, n, key, 0, n)[0], lambda: ctx.eval_sampled_sums(2, n, key, 0, n - 2)[0]),
            ("drawn list", lambda: ctx.eval_samples_sums(np.concatenate([[1], drawn_ok]))[0],
             lambda: ctx.eval_samples_sums(drawn_ok)[0]),
            ("weighted", lambda: ctx.eval_weighted(0, n).loss_sum, lambda: ctx.eval_weighted(2, n).loss_sum),
        ]
        g_want = orc_s / (n - 2)   # lambda = 0
        passes.append(("gradient", lambda: ctx.gradient(ids, want_loss=True)[1], lambda: ctx.gradient(ok, want_loss=True)[1]))
        for name, bad, good in passes + passes[::-1]:
            assert math.isnan(bad()), name
            got, want = good(), g_want if name == "gradient" else orc_s
            assert got == want, f"{name} after a NaN pass: {got!r}, want {want!r}"
        # per class: only the class of the over-limit row is NaN
        pos = [r for r in range(2, n) if rows[r][1] > 0]
        neg = [r for r in range(2, n) if rows[r][1] < 0]
        s_pos, s_neg = (M.eval_class(orc, model, w, rr)[0][k] for k, rr in ((0, pos), (1, neg)))
        for rng_begin, nan_pos, nan_neg in ((0, True, True), (1, False, True), (2, False, False)):
            ce = ctx.eval_class(rng_begin, n, w)
            assert math.isnan(ce.loss_pos) == nan_pos and math.isnan(ce.loss_neg) == nan_neg, (rng_begin, ce)
            assert nan_pos or ce.loss_pos == s_pos
            assert nan_neg or ce.loss_neg == s_neg
            ref, _ = M.eval_class(orc, model, w, np.arange(rng_begin, n))
            assert same(ce.loss_pos, ref[0]) and same(ce.loss_neg, ref[1])
        ce = ctx.eval_samples_class(np.array([0] + pos + neg, np.int32))
        assert math.isnan(ce.loss_pos) and ce.loss_neg == s_neg
        ce = ctx.eval_sampled_class(2, n, key, 0, n - 2)
        assert (ce.loss_pos, ce.loss_neg) == (s_pos, s_neg)
    finally:
        ctx.close()


@pytest.mark.parametrize("counts", [[9], [4, 5]])
@pytest.mark.parametrize("weighting", WEIGHTINGS)
@pytest.mark.parametrize("model", MODELS)
def test_over_limit_step_loss_reads_nan_then_recovers(model, weighting, counts):
    rows, orc, ctx, w, sw = _rule_problem(model, [(OVER[model], 1)])
    lr = 2.0 ** -10
    bad = np.array([0] + list(range(1, 9)), np.int32)    # the over-limit row and 8 others
    good = np.array(list(range(1, 9)) + [3], np.int32)   # 9 ordinary ids, one twice
    try:
        wp, wn, swc = _set_weighting(ctx, weighting, sw)
        ctx.set_workers(counts, len(counts))
        for ids, nan in ((bad, True), (good, False), (bad, True), (good, False)):
            ctx.set_weights(w)
            loss = ctx.sync_steps(ids, 9, 1, lr)[0]
            w_ref, l_ref = M.sync_steps(orc, model, w, ids, counts, [lr], wp, wn, swc)
            assert math.isnan(loss) == nan and same(loss, l_ref[0]), (list(ids), loss, l_ref[0])
            assert np.array_equal(ctx.get_weights(), w_ref)
    finally:
        ctx.set_workers([], 0)
        ctx.close()


@pytest.mark.parametrize("counts", [[5], [2, 3]])
@pytest.mark.parametrize("model", MODELS)
def test_class_and_sample_forms_apply_the_limit_differently(model, counts):
    """Class weights (2, 1/2) and a loss in [2^51, 2^52): the class form is finite (fl(2 S+) >= 2^52 is a double), the
    sample form is NaN (c_i L_i >= 2^52 is not summed).  Class weights (0, 1) and a loss of 2^52: the class form is NaN
    (0 * NaN), the sample form adds an exact 0."""
    rows, orc, ctx, w, _ = _rule_problem(model, [(HALF[model], 1), (OVER[model], 1)])
    lr = 2.0 ** -10
    ones = np.ones(len(rows))
    try:
        ctx.set_workers(counts, len(counts))
        for (wp, wn), head in (((2.0, 0.5), 0), ((0.0, 1.0), 1)):
            ids = np.array([head, 2, 3, 4, 5], np.int32)
            class_nan = head == 1
            ctx.set_class_weights(wp, wn)
            ctx.set_sample_weights(None)
            # the class form: the per-class sums, the class-weighted gradient's loss and step loss
            ce = ctx.eval_samples_class(ids, w)
            assert math.isnan(ce.loss_pos) == class_nan
            assert math.isnan(ce.weighted_loss_sum(wp, wn)) == class_nan
            g_loss = ctx.gradient(ids, w, want_loss=True)[1]
            _, l_ref, _ = M.gradient(orc, model, w, ids, wp, wn)
            assert math.isnan(g_loss) == class_nan and same(g_loss, l_ref), (g_loss, l_ref)
            if not class_nan:
                assert g_loss * 5 >= 2.0 ** 52
            ctx.set_weights(w)
            loss = ctx.sync_steps(ids, 5, 1, lr)[0]
            _, l_ref = M.sync_steps(orc, model, w, ids, counts, [lr], wp, wn)
            assert math.isnan(loss) == class_nan and same(loss, l_ref[0]), (loss, l_ref)
            # the sample form: the weighted evaluation (c_i = w_y without sample weights) and the sample-weighted step
            we = ctx.eval_samples_weighted(ids, w)
            sums, _ = M.eval_weighted(orc, model, w, ids, wp, wn)
            assert math.isnan(we.loss_sum) == (not class_nan) and same(we.loss_sum, sums[0]), (we, sums)
            ctx.set_sample_weights(ones)
            ctx.set_weights(w)
            loss = ctx.sync_steps(ids, 5, 1, lr)[0]
            _, l_ref = M.sync_steps(orc, model, w, ids, counts, [lr], wp, wn, ones)
            assert math.isnan(loss) == (not class_nan) and same(loss, l_ref[0]), (loss, l_ref)
    finally:
        ctx.set_workers([], 0)
        ctx.close()


# ---- c. the filter under scales above 1 ---------------------------------------------------------------------------------

def _f32_around(v):
    """(largest fp32 <= v, smallest fp32 > v) as doubles"""
    f = np.float32(v)
    if float(f) > v:
        return float(np.nextafter(f, np.float32(0))), float(f)
    return float(f), float(np.nextafter(f, np.float32(np.inf)))


BELOW, ABOVE = _f32_around(1e-20)
TINY = (BELOW, ABOVE, -BELOW, -ABOVE, float(np.float32(2e-20)), float(np.float32(-3e-20)))
ANCHORS = {"squared_hinge": (1.0, 2.0 ** 26 - 1.0), "modified_huber": (2.0, 7.5)}   # s = 4, 2^27; s = 4, 4
SW_C = (0.1, 3.0, 0.3, 1.0 / 3.0, 0.05, 0.7)


def _filter_problem(model):
    rows, extra = [], []
    for a in ANCHORS[model]:
        for x in TINY:
            for y in (1, -1):
                extra.append((len(rows), x))
                rows.append((a, y, SW_C[len(rows) % len(SW_C)]))
    return rows, extra


@pytest.mark.parametrize("weighting", WEIGHTINGS)
@pytest.mark.parametrize("model", MODELS)
def test_filter_under_scales_above_one(model, weighting):
    rows, extra = _filter_problem(model)
    rp, col, val, lab, dim, ws, cols = planted_csr(rows, extra)
    w = np.sum(ws, axis=0)
    sw = np.array([s for *_, s in rows])
    orc = Oracle(rp, col, val, lab, dim, 0.0)
    orc.set_dim_sparsity(np.zeros(dim))
    ctx = _ctx(model, rp, col, val, lab, dim)
    try:
        wp, wn, swc = _set_weighting(ctx, weighting, sw)
        ids = np.arange(len(rows), dtype=np.int32)
        g = ctx.gradient(ids, w)
        g_ref, _, _ = M.gradient(orc, model, w, ids, wp, wn, swc)
        assert np.array_equal(g == 0, g_ref == 0), "gradient support differs from the checker"
        assert np.array_equal(g, g_ref)
        # the same bits from the stated order: filt(filt(x) * ((y * s) * c)) on the tiny entry's own column
        lifted = straddled = 0
        for r, (z, y, s_i) in enumerate(rows):
            x = float(val[rp[r] + 1])
            s = exact_row(model, z)[1]
            c = 1.0 if weighting == "none" else ((wp if y > 0 else wn) * (s_i if weighting == "sample" else 1.0))
            v = y * s if weighting == "none" else (y * s) * c
            fx = x if abs(x) > 1e-20 else 0.0
            want = fx * v if abs(fx * v) > 1e-20 else 0.0
            assert g[col[rp[r] + 1]] == want, (r, x, s, c, g[col[rp[r] + 1]], want)
            lifted += abs(x) <= 1e-20 < abs(x * s)
            straddled += abs(x * s) > 1e-20 >= abs(x * v)
        assert lifted >= 4, "no entry below the filter that the scale would lift above it"
        if weighting == "sample":
            assert straddled >= 1, "no entry whose x * s and x * (y * s) * c straddle the filter"
        # one sync step scatters the same way
        ctx.set_weights(w)
        ctx.sync_steps(ids, len(ids), 1, 2.0 ** -4)
        w_ref, _ = M.sync_steps(orc, model, w, ids, [len(ids)], [2.0 ** -4], wp, wn, swc)
        assert np.array_equal(ctx.get_weights(), w_ref)
    finally:
        ctx.close()


# ---- d. pass sums in every form ------------------------------------------------------------------------------------------

N_BIG = 100_000


def _np_row(model, z):
    """L(z) elementwise, in the models' order of operations (numpy float64 is correctly rounded)"""
    t = 1.0 + z
    if model == "squared_hinge":
        return np.where(z <= -1.0, 0.0, t * t)
    return np.where(z <= -1.0, 0.0, np.where(z <= 1.0, t * t, 4.0 * z))


# Rows of the big set with x = 1 on a column of their own, planted at these positions, and their margins: losses with bits
# in limb 1 (t a few multiples of 2^-53) and in limb 5 (above 2^40), which random weights do not reach
PLANT_AT = [0, 3, 8, 700, 2046, 8447, 8448, 50000, 99999]
PLANT_Z = {"squared_hinge": [-1.0 + 3 * 2.0 ** -53, 2.0 ** 22 + 0.5, -1.0 + 2.0 ** -30],
           "modified_huber": [-1.0 + 3 * 2.0 ** -53, 2.0 ** 40 + 0.75, -1.0 + 2.0 ** -30]}


def _planted_big(model, rng):
    """N_BIG rows: RCV1-shaped rows with planted rows at PLANT_AT, and weights (unit normal scaled by 10^U(-2, 5), the
    planted rows' at y * z)."""
    from distributed_sgd_b200.utils import synthetic_rcv1
    from helpers import data_from_csr
    base = synthetic_rcv1(n_rows=N_BIG - len(PLANT_AT), seed=31)
    k = len(PLANT_AT)
    planted = np.zeros(N_BIG, bool)
    planted[PLANT_AT] = True
    lens = np.ones(N_BIG, np.int64)
    lens[~planted] = np.diff(base.row_ptr)
    rp = np.concatenate([[0], np.cumsum(lens)])
    at = np.zeros(int(rp[-1]), bool)
    at[rp[PLANT_AT]] = True
    col = np.empty(int(rp[-1]), np.int32)
    val = np.empty(int(rp[-1]), np.float32)
    col[~at], val[~at] = base.col, base.val
    col[at], val[at] = base.dim + np.arange(k), 1.0
    lab = np.empty(N_BIG, np.int8)
    lab[~planted] = base.label
    lab[planted] = [1 if j % 2 == 0 else -1 for j in range(k)]
    w = rng.standard_normal(base.dim + k) * 10.0 ** rng.uniform(-2.0, 5.0, base.dim + k)
    zs = PLANT_Z[model]
    w[base.dim:] = [float(lab[p]) * zs[j % len(zs)] for j, p in enumerate(PLANT_AT)]
    return data_from_csr(rp, col, val, lab, base.dim + k), w


@pytest.fixture(scope="module", params=MODELS)
def big(request):
    """100 000 rows, weights whose losses reach from 2^-106 to above 2^40, the per-row losses and sample weights."""
    model = request.param
    rng = np.random.default_rng(5)
    data, w = _planted_big(model, rng)
    ctx = _ctx(model, data.row_ptr, data.col, data.val, data.label, data.dim, lam=LAM)
    d = ctx.compute_dim_sparsity(N_BIG)
    ctx.set_dim_sparsity(d)
    ctx.set_weights(w)
    z = data.label * ctx.margins(np.arange(N_BIG, dtype=np.int32))
    L = _np_row(model, z)
    sw = rng.uniform(0.0, 3.0, N_BIG) * (rng.random(N_BIG) < 0.9)
    sw[PLANT_AT[::3]] = 2.0 ** -20   # c_i L_i of the planted 9 * 2^-106 losses: bits in limb 0 (below 2^-120)
    yield dict(model=model, data=data, ctx=ctx, w=w, z=z, L=L, sw=sw)
    ctx.close()


def _units(vals):
    return np.array([r_units(v) for v in vals], dtype=object)


def _exact(units, ids):
    return Fraction(int(units[np.asarray(ids)].sum()), 1 << 160)


def test_per_row_values_are_one_row_evaluations(big):
    """The per-row values of the pass sums are what one-row evaluations report; they cover limbs 1 to 5 (limb 0, below
    2^-120, cannot be reached: t = fl(1 + z) is a multiple of 2^-53, so every loss is a multiple of 2^-106)."""
    ctx, L, model = big["ctx"], big["L"], big["model"]
    assert np.isfinite(L).all() and (L < 2.0 ** 52).all()
    probe = np.concatenate([np.arange(1024), np.argsort(L)[:512], np.argsort(L)[-512:]])
    for r in probe:
        assert ctx.eval_samples_sums([int(r)])[0] == r_value(L[r]), (r, L[r])
    assert (L == 0).any() and L.max() > 2.0 ** 40
    u = _units(L)
    for k in range(1, 6):
        assert any((int(x) >> (40 * k)) & ((1 << 40) - 1) for x in u), f"no value has bits in limb {k}"
    assert not any(int(x) & ((1 << 54) - 1) for x in u)   # multiples of 2^-106


def _sizes(sm):
    return [1, 2, 7, 8, 9, 64 * sm - 1, 64 * sm, 64 * sm + 1, 2047, 2048, N_BIG]


@pytest.mark.parametrize("weighting", WEIGHTINGS)
def test_pass_sums_are_exact_in_every_form(big, sm, weighting):
    from distributed_sgd_b200.native import host_lib
    ctx, data, L = big["ctx"], big["data"], big["L"]
    y = data.label.astype(np.float64)
    sw = big["sw"]
    c = np.where(y > 0, W_POS, W_NEG) * sw
    vals = c * L if weighting == "sample" else L
    units = _units(vals)
    limbs = range(0 if weighting == "sample" else 1, 6)   # unweighted losses are multiples of 2^-106: no limb 0
    for k in limbs:
        assert any(int(x) >> (40 * k) & ((1 << 40) - 1) for x in units), f"no value has bits in limb {k}"
    pos_units = np.where(y > 0, units, 0)
    neg_units = np.where(y > 0, 0, units)
    rng = np.random.default_rng(17)

    def read(kind, rows):
        """rows: ("range", b, e) | ("list", ids) | ("drawn", b, e, key, k)"""
        if weighting == "none":
            f = {"range": ctx.eval_sums, "list": ctx.eval_samples_sums, "drawn": ctx.eval_sampled_sums}[kind]
            return f(*rows)[0]
        if weighting == "class":
            f = {"range": ctx.eval_class, "list": ctx.eval_samples_class, "drawn": ctx.eval_sampled_class}[kind]
            ce = f(*rows)
            return ce.loss_pos, ce.loss_neg
        f = {"range": ctx.eval_weighted, "list": ctx.eval_samples_weighted, "drawn": ctx.eval_sampled_weighted}[kind]
        return f(*rows).loss_sum

    def check(got, ids, what):
        if weighting == "class":
            for s, u in zip(got, (pos_units, neg_units)):
                ex = _exact(u, ids)
                assert within_one_ulp(s, ex), f"{what}: " + describe(s, ex)
        else:
            ex = _exact(units, ids)
            assert within_one_ulp(got, ex), f"{what}: " + describe(got, ex)

    try:
        _set_weighting(ctx, "class" if weighting == "class" else ("sample" if weighting == "sample" else "none"), sw)
        for n in _sizes(sm):
            ids = np.arange(n, dtype=np.int32)
            key = 0x5EED0000 + n
            drawn = np.fromiter((host_lib().dsgd_feistel_pos(p, n, key) for p in range(n)), dtype=np.int32, count=n)
            forms = {
                "range": read("range", (0, n)),
                "list": read("list", (ids,)),
                "reversed": read("list", (ids[::-1].copy(),)),
                "shuffled": read("list", (rng.permutation(ids),)),
                "drawn": read("drawn", (0, n, key, 0, n)),
                "drawn list": read("list", (drawn,)),
            }
            check(forms["range"], ids, f"n={n}")
            for form, s in forms.items():
                assert np.array_equal(s, forms["range"]), f"n={n}, {form}: {s!r} against the range's {forms['range']!r}"
            rep = rng.integers(0, n, size=n + 5).astype(np.int32)
            s_rep = read("list", (rep,))
            check(s_rep, rep, f"n={n} with repeats")
            assert np.array_equal(read("list", (rng.permutation(rep),)), s_rep)
    finally:
        _clear_weighting(ctx)


# ---- e. step losses are evaluations --------------------------------------------------------------------------------------

@pytest.mark.parametrize("lambda1", [0.0, 1e-4])
@pytest.mark.parametrize("counts", [[64], [40, 24, 17]])
@pytest.mark.parametrize("weighting", WEIGHTINGS)
def test_step_loss_is_the_evaluation(big, weighting, counts, lambda1):
    ctx, w = big["ctx"], big["w"]
    tot = sum(counts)
    rng = np.random.default_rng(tot + len(counts))
    try:
        _set_weighting(ctx, weighting, big["sw"])
        ctx.set_weights(w * 1e-4)
        ctx.set_l1(lambda1)
        ctx.set_workers(counts, len(counts))
        for _ in range(3):
            ids = rng.choice(N_BIG, size=tot, replace=False).astype(np.int32)
            fold, off = 0.0, 0
            for k, nk in enumerate(counts):
                part = ids[off:off + nk]
                if weighting == "none":
                    s, _, n2 = ctx.eval_samples_sums(part)
                elif weighting == "class":
                    ce = ctx.eval_samples_class(part)
                    s, n2 = ce.weighted_loss_sum(W_POS, W_NEG), ce.norm_squared
                else:
                    we = ctx.eval_samples_weighted(part)
                    s, n2 = we.loss_sum, we.norm_squared
                fold = s if k == 0 else fold + s
                off += nk
            want = LAM * n2 + lambda1 * ctx.weights_l1()[0] + fold / tot if lambda1 else LAM * n2 + fold / tot
            got = ctx.sync_steps(ids, tot, 1, 0.25)[0]
            assert got == want, f"{got!r} against {want!r}"
    finally:
        ctx.set_workers([], 0)
        ctx.set_l1(0.0)
        _clear_weighting(ctx)


# ---- f. shared-column dyadic runs ----------------------------------------------------------------------------------------

LAM_D, LAM1_D, LR_D = 2.0 ** -8, 2.0 ** -10, 2.0 ** -5
HOT = 4


def _dyadic_shared(n_rows=6000, dim=256, seed=7):
    """Rows with values in +-{1/2, 1, 3/2, 2}: each takes each of the HOT hot columns with probability 0.8 and 2 to 6 other
    columns.  Weights on a 2^-5 grid in [-1/4, 1/4], d = 2^-2 on every fourth column."""
    from helpers import data_from_csr
    rng = np.random.default_rng(seed)
    rp, col, val = [0], [], []
    for _ in range(n_rows):
        cs = {c for c in range(HOT) if rng.random() < 0.8} | set(rng.integers(HOT, dim, size=int(rng.integers(2, 7))).tolist())
        for c in sorted(cs):
            col.append(c)
            val.append(float(rng.choice([-2.0, -1.5, -1.0, -0.5, 0.5, 1.0, 1.5, 2.0])))
        rp.append(len(col))
    lab = rng.choice(np.array([-1, 1], np.int8), size=n_rows)
    w0 = rng.integers(-8, 9, size=dim) / 32.0
    d = np.zeros(dim)
    d[::4] = 0.25
    return data_from_csr(rp, col, val, lab, dim), w0, d


def _grid(a):
    """K such that every entry of a is a multiple of 2^-K (0 for an empty or all-zero a)"""
    a = np.abs(np.asarray(a, np.float64))
    a = a[a != 0]
    if a.size == 0:
        return 0
    m, e = np.frexp(a)
    mi = (m * 2.0 ** 53).astype(np.int64)
    low = e.astype(np.int64) - 53 + np.log2((mi & -mi).astype(np.float64)).astype(np.int64)
    return int(max(0, -low.min()))


def _sums_exact(terms, groups):
    """Whether every group sum of terms (np.add.at by groups) is exact in any order: sum |term| < 2^(53 - K)"""
    if terms.size == 0:
        return True
    K = _grid(terms)
    acc = np.zeros(int(groups.max()) + 1)
    np.add.at(acc, groups, np.abs(terms))
    return bool((acc < 2.0 ** (53 - K)).all())


def _witness(model, data, w, d, ids_by_worker, w_pos, w_neg, sw):
    """Whether one step (or one gradient) at weights w is exact in any summation order: the row dots, every gradient
    column of every worker, c = 2 lambda (w . d) and ||w||^2."""
    if not (_sums_exact(w * w, np.zeros(w.size, np.int64)) and
            _sums_exact(np.where(np.abs(w * d) > 1e-20, w * d, 0.0), np.zeros(w.size, np.int64))):
        return False
    for ids in ids_by_worker:
        lo, hi = data.row_ptr[ids], data.row_ptr[ids + 1]
        ent = np.concatenate([np.arange(a, b) for a, b in zip(lo, hi)])
        rowof = np.repeat(np.arange(len(ids)), hi - lo)
        x = data.val[ent].astype(np.float64)
        cols = data.col[ent]
        prod = x * w[cols]
        if not _sums_exact(prod, rowof):
            return False
        dots = np.zeros(len(ids))
        np.add.at(dots, rowof, prod)
        y = data.label[ids].astype(np.float64)
        s = np.array([M.row(model, float(v))[1] for v in y * dots])
        c = np.where(y > 0, w_pos, w_neg) * (sw[ids] if sw is not None else 1.0)
        v = (y * s) * c
        if not _sums_exact(x * v[rowof], cols):
            return False
    return True


@pytest.fixture(scope="module")
def shared():
    data, w0, d = _dyadic_shared()
    orc = Oracle(data.row_ptr, data.col, data.val, data.label, data.dim, LAM_D)
    orc.set_dim_sparsity(d)
    sw = dyadic_weights(np.random.default_rng(8), data.n_rows)
    return data, w0, d, orc, sw


def _dyadic_weighting(weighting, sw):
    return {"none": (1.0, 1.0, None), "class": (4.0, 0.25, None), "sample": (2.0, 0.5, sw)}[weighting]


@pytest.mark.parametrize("resident", [False, True])
@pytest.mark.parametrize("weighting", WEIGHTINGS)
@pytest.mark.parametrize("model", MODELS)
def test_shared_column_gradient_bit_for_bit(shared, sm, model, weighting, resident):
    data, w0, d, orc, sw_all = shared
    wp, wn, sw = _dyadic_weighting(weighting, sw_all)
    ctx = _ctx(model, data.row_ptr, data.col, data.val, data.label, data.dim, lam=LAM_D, d=d)
    try:
        if weighting != "none":
            ctx.set_class_weights(wp, wn)
        if sw is not None:
            ctx.set_sample_weights(sw)
        for n in (1, 64, 4096, 32 * sm + 1):
            idx = np.random.default_rng(n).choice(data.n_rows, size=n, replace=False).astype(np.int32)
            assert _witness(model, data, w0, d, [idx], wp, wn, sw), f"batch {n}: the sums are not provably exact"
            if resident:
                ctx.set_weights(w0)
                g, loss = ctx.gradient(idx, want_loss=True)
            else:
                g, loss = ctx.gradient(idx, w0, want_loss=True)
            g_ref, loss_ref, _ = M.gradient(orc, model, w0, idx, wp, wn, sw)
            assert n == 1 or (np.abs(g[:HOT]) > 0).all(), "the hot columns take no gradient"
            diff = np.flatnonzero(g != g_ref)
            assert diff.size == 0, f"batch {n}, column {diff[0]}: {g[diff[0]]!r} against {g_ref[diff[0]]!r}"
            assert loss == loss_ref, (n, loss, loss_ref)
    finally:
        ctx.close()


OPTIONS = {   # name: (lambda1, averaging, rate table)
    "plain": (0.0, False, False),
    "l1": (LAM1_D, False, False),
    "avg": (0.0, True, False),
    "table": (0.0, False, True),
    "all": (LAM1_D, True, True),
}
RUNS = [(o, c) for o in OPTIONS for c in (("sync_steps_lr",) if OPTIONS[o][2] else ("sync_steps", "sync_step", "staged"))]
MAX_STEPS = 8


def _witnessed_run(model, data, w0, d, orc, counts, lrs, wp, wn, sw, lambda1, rng):
    """Step ids and checker weights for as many steps (up to len(lrs)) as the witness holds before each; returns (idx,
    number of steps, checker weights, losses, averaging sum)."""
    tot = sum(counts)
    w = w0.copy()
    idx, losses, avg_sum = [], [], np.zeros(data.dim)
    for t in range(len(lrs)):
        step = rng.choice(data.n_rows, size=tot, replace=False).astype(np.int32)
        parts = np.split(step, np.cumsum(counts)[:-1])
        if not _witness(model, data, w, d, parts, wp, wn, sw):
            break
        w, l = M.sync_steps(orc, model, w, step, counts, lrs[t:t + 1], wp, wn, sw, lambda1=lambda1, avg_sum=avg_sum)
        idx.append(step)
        losses.append(l[0])
    return np.concatenate(idx) if idx else np.zeros(0, np.int32), len(idx), w, np.array(losses), avg_sum


@pytest.mark.parametrize("option,call", RUNS)
@pytest.mark.parametrize("counts", [[64], [40, 24, 17, 47]])
@pytest.mark.parametrize("weighting", WEIGHTINGS)
@pytest.mark.parametrize("model", MODELS)
def test_shared_column_run_bit_for_bit(shared, model, weighting, counts, option, call):
    """Four virtual workers rather than three: the mean over three workers leaves the dyadic grid after one step."""
    data, w0, d, orc, sw_all = shared
    wp, wn, sw = _dyadic_weighting(weighting, sw_all)
    lambda1, avg, table = OPTIONS[option]
    lrs = LR_D * 2.0 ** -(np.arange(MAX_STEPS) % 3) if table else np.full(MAX_STEPS, LR_D)
    idx, steps, w_ref, l_ref, avg_sum = _witnessed_run(model, data, w0, d, orc, counts, lrs, wp, wn, sw, lambda1,
                                                       np.random.default_rng(len(counts) * 10 + len(option)))
    assert steps >= 2, f"the witness allows only {steps} exact step(s)"
    lrs = lrs[:steps]
    tot = sum(counts)
    ctx = _ctx(model, data.row_ptr, data.col, data.val, data.label, data.dim, lam=LAM_D, d=d)
    try:
        if weighting != "none":
            ctx.set_class_weights(wp, wn)
        if sw is not None:
            ctx.set_sample_weights(sw)
        ctx.set_weights(w0)
        ctx.set_l1(lambda1)
        ctx.set_workers(counts, len(counts))
        if avg:
            ctx.average_begin()
        if call == "sync_steps_lr":
            losses = ctx.sync_steps_lr(idx, tot, lrs)
        elif call == "sync_steps":
            losses = ctx.sync_steps(idx, tot, steps, LR_D)
        elif call == "sync_step":
            losses = np.array([ctx.sync_step(idx[t * tot:(t + 1) * tot], LR_D) for t in range(steps)])
        else:
            ctx.stage_samples(idx)
            ctx.sync_steps_staged(0, tot, steps, LR_D, want_losses=True)
            losses = ctx.read_losses(steps)
        w = ctx.get_weights()
        diff = np.flatnonzero(w != w_ref)
        assert diff.size == 0, f"{steps} steps, column {diff[0]}: {w[diff[0]]!r} against {w_ref[diff[0]]!r}"
        assert np.array_equal(losses, l_ref), (losses, l_ref)
        if avg:
            mean, n = ctx.average_weights()
            mean_ref = avg_sum / steps
            assert n == steps and np.array_equal(mean, np.where(np.abs(mean_ref) > 1e-20, mean_ref, 0.0))
    finally:
        ctx.close()


# ---- g. two GPUs ---------------------------------------------------------------------------------------------------------

def _free_port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def _nccl_worker(rank, world, port, model, q):
    sys.path.insert(0, ROOT)
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    import torch
    import torch.distributed as dist
    from distributed_sgd_b200.core import Group
    from distributed_sgd_b200.native import NativeCtx

    torch.cuda.set_device(rank)
    dist.init_process_group("gloo", init_method=f"tcp://127.0.0.1:{port}", rank=rank, world_size=world)
    group = Group()
    data, w0, d = _dyadic_shared()
    orc = Oracle(data.row_ptr, data.col, data.val, data.label, data.dim, LAM_D)
    orc.set_dim_sparsity(d)
    batch = 48
    idx, steps, w_ref, l_ref, _ = _witnessed_run(model, data, w0, d, orc, [batch] * world, np.full(MAX_STEPS, LR_D),
                                                 1.0, 1.0, None, 0.0, np.random.default_rng(9))
    ctx = NativeCtx(rank, data.dim, LAM_D, rank=rank, world=world, model=model)
    ctx.load_csr(data.row_ptr, data.col, data.val, data.label)
    ctx.set_dim_sparsity(d)
    uid = NativeCtx.comm_unique_id() if rank == 0 else b""
    ctx.comm_init(group.broadcast_bytes(uid, 0))
    mine = idx.reshape(steps, world, batch)[:, rank, :]
    ctx.set_weights(w0)
    losses = ctx.sync_steps(mine.reshape(-1), batch, steps, LR_D)
    q.put((rank, steps, bool(np.array_equal(losses, l_ref)), bool(np.array_equal(ctx.get_weights(), w_ref))))
    ctx.close()
    dist.destroy_process_group()


@pytest.mark.parametrize("model", MODELS)
def test_two_gpu_nccl_shared_column_run_bit_for_bit(model):
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    import torch.multiprocessing as mp
    ctxmp = mp.get_context("spawn")
    q = ctxmp.Queue()
    port = _free_port()
    procs = [ctxmp.Process(target=_nccl_worker, args=(r, 2, port, model, q)) for r in range(2)]
    for p in procs:
        p.start()
    res = [q.get(timeout=300) for _ in procs]
    for p in procs:
        p.join(timeout=60)
    for rank, steps, same_losses, same_w in res:
        assert steps >= 2, f"the witness allows only {steps} exact step(s)"
        assert same_losses, f"rank {rank}: step losses differ from the checker"
        assert same_w, f"rank {rank}: weights differ from the checker"
