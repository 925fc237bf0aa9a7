"""Resident-weight reads (w == NULL) after every writer of a context with an L1 penalty, class weights or a rate table.

The reader x writer matrix of test_gpu_resident_state.py, on the options that came after it.  A request with w == NULL
reads the resident weights and what is derived from them: c, ||w||^2, the fp32 shadow w32 and, on an L1 context, ||w||_1 in
scal[kScalL1], which only the per-step L1 update reads (for the loss of its step).

Writers, each on a context left with its options on (the persistent kernel at batch 64, the per-step path at 32 G + 1):

- L1 (SVM): set_weights, the persistent kL1 form at full grid and at grid limit 2, the per-step path, two virtual workers
  [40, 24], staged steps, averaging and a rate table on both paths;  L1 (logistic, fp32 rows): steps and a rate table;
- class weights (2, 1/2) (SVM): the persistent kCw form, the per-step path, two workers, staged steps, with L1 on both
  paths, with a rate table;  class weights (logistic, fp32 rows): steps;
- a rate table alone on both paths;
- writers of state only: set_l1 turning on after set_weights with it off (a fresh context: ||w||_1 was never derived), on ->
  off -> set_weights(w1) -> on, from one lambda1 > 0 to another; set_class_weights (1, 1) -> (2, 1/2) and back;
  set_dim_sparsity and compute_dim_sparsity with lambda1 > 0;
- the fused K = 2 kernel on one GPU with a rate table (its kLrTable epilogue).

Readers: everything read_all of test_gpu_resident_state.py reads, and margins (below and above 2 048 ids), probabilities
(logistic), eval_metrics in its three forms, eval_curve with points and AP only, calibrate, calibrated_probabilities and
eval_calibration (range and list), weights_l1, and on a weighted context eval_class in its three forms and the weighted
gradient (k_rows<…, kClassWeighted, …> below 2 048 ids, the streaming pass above).  w == NULL against the weights from
get_weights: every
integer word and every value that depends on the weights alone (margins, metrics and curve words, AP, the fit, calibrated
probabilities, calibration sums and bins, weights_l1) bit for bit; the rest as in test_gpu_resident_state.py.  Those
against the checkers of oracle/: margins bit for bit on dyadic rows (else within 1e-12 of sum |x_j w_j|), metrics words and
curve points exact over the device's own margins, AP within 2 ulp, (A, B) within 1e-8 max(1, |A|) and F within rtol 1e-10,
eval_class integers exact, the weighted gradient within 1e-13 of the summed magnitudes of its terms, weights_l1 exact on
dyadic weights.

The next step after every writer, with the context's options still on, on both paths: the same weights and loss as the same
step after set_weights(w) re-derives everything, and oracle/l1.sync_steps or oracle/cw.sync_steps; on dyadic rows bit for
bit.  The per-step path is the only reader of scal[kScalL1], so every writer of it (set_l1, set_weights, the persistent
epilogue and the per-step update) is followed by a per-step step.

Dyadic constants (test_gpu_resident_state.py: values multiples of 1/2, weights of 2^-5, d = 4 on one column, lr 2 lambda d =
1): lambda1 = 2^-4 (tau = lr lambda1 = 2^-5, then 2^-3 for the change), class weights 2 and 1/2, rate tables of 2^-1, 0 and
2^-2.  Every weight stays a multiple of 2^-8 below 2^6, so ||w||^2, ||w||_1 and every gradient sum are exact in any order:
the persistent kernel's per-CTA fp64 partials of ||w||_1 and the per-step path's fixed-point limbs give the same bits.

Every case first shows, on the oracle, that a reader still using the state from before the writer would fail (at least 1 %
of the streaming pass's rows change prediction, c and ||w||^2 move, and on an L1 context ||w||_1 too); for the writers of
state only, that the next step's loss under the stale ||w||_1, lambda1 or class weights differs from the right one.

The last two tests run every list-form reader between staged calls on contexts with L1, class weights and averaging on,
and require the staged steps to give the bits of a run with no reader in between (the logistic model's to rounding).
"""
import math
import struct
import zlib

import numpy as np
import pytest

from helpers import fused_ranks
from oracle import calib as CB
from oracle import curve as OC
from oracle import cw as CW
from oracle import l1 as L1
from oracle import metrics as OM
from test_gpu_resident_state import (BATCH, DIMS, KEY, KINDS, N_ROWS, N_SMALL, N_STREAM, S, _grad_scale, _moved,  # noqa: F401
                                     _one_worker, _reset, _steps, compare, envs, oracle_all, read_all, witness)

pytestmark = pytest.mark.gpu

CLASS_W = (2.0, 0.5)
CAL_AB = (1.5, -0.25)          # the link calibrated_probabilities and eval_calibration are read at


def consts(env):
    """(lambda1, the other lambda1 of set_l1_change, the writers' rate table): powers of two on dyadic rows."""
    if env.kind == "dyadic":
        return 2.0 ** -4, 2.0 ** -3, np.array([2.0 ** -1, 0.0, 2.0 ** -2])
    return 2e-3, 5e-3, np.array([env.lr, 0.0, env.lr / 2])


def _big_step(env, S):
    """The per-step path's batch of 32 G + 1 ids (one more than the persistent kernel takes on S CTAs)."""
    return np.random.default_rng(env.dim + 5).choice(N_ROWS, size=32 * S + 1, replace=False).astype(np.int32)


def _set_options(ctx, env, options):
    lam1 = consts(env)[0]
    ctx.set_l1(lam1 if "l1" in options else 0.0)
    ctx.set_class_weights(*(CLASS_W if "cw" in options else (1.0, 1.0)))


def _bits(v):
    if isinstance(v, np.ndarray):
        return v.tobytes()
    if isinstance(v, (tuple, list)):
        return tuple(_bits(x) for x in v)
    if isinstance(v, float):
        return struct.pack("<d", v)
    return v


def _abs_oracle(env):
    """The oracle over |x| (for |w|): sum_j |x_j w_j| per row, the scale of a margin's rounding."""
    if not hasattr(env, "abs_orc"):
        from oracle.oracle import Oracle
        dt = env.data
        env.abs_orc = Oracle(dt.row_ptr, dt.col, np.abs(dt.val), dt.label, env.dim, env.lam)
    return env.abs_orc


# ---- the readers beyond read_all -----------------------------------------------------------------------------------------

def read_more(ctx, env, w, model, weighted):
    """Every reader added since read_all, once, at the weights w (None: resident).  {reader: value}."""
    ids = env.ids
    a, b = CAL_AB
    out = {}
    for name in ("fwd_rows", "fwd_stream"):
        out["margins_" + name] = ctx.margins(ids[name], w)
    if model == "logistic":
        out["probabilities"] = ctx.probabilities(ids["fwd_stream"], w)
    out["metrics_range"] = ctx.eval_metrics(0, N_STREAM, w)
    out["metrics_sampled"] = ctx.eval_sampled_metrics(0, N_ROWS, KEY, 100, 1100, w)
    out["metrics_list"] = ctx.eval_samples_metrics(ids["samples"], w)
    out["curve_range"] = ctx.eval_curve(0, N_STREAM, w)
    out["ap_range"] = ctx.eval_curve(0, N_STREAM, w, curve=False)
    out["curve_list"] = ctx.eval_samples_curve(ids["samples"], w)
    out["calibrate_range"] = ctx.calibrate(0, N_STREAM, w)
    out["calibrate_list"] = ctx.calibrate_samples(ids["samples"], w)
    out["calibrated"] = ctx.calibrated_probabilities(ids["fwd_stream"], a, b, w)
    out["calibration_range"] = ctx.eval_calibration(0, N_STREAM, a, b, 10, w)
    out["calibration_list"] = ctx.eval_samples_calibration(ids["samples"], a, b, 10, w)
    out["weights_l1"] = ctx.weights_l1(w)
    if weighted:
        out["class_range"] = ctx.eval_class(0, N_STREAM, w)
        out["class_rows"] = ctx.eval_class(N_STREAM, N_STREAM + N_SMALL, w)
        out["class_sampled"] = ctx.eval_sampled_class(0, N_ROWS, KEY, 0, 2500, w)
        out["class_list"] = ctx.eval_samples_class(ids["samples"], w)
    return out


CLASS_IDS = {"class_range": lambda env: np.arange(N_STREAM), "class_rows": lambda env: np.arange(N_STREAM, N_STREAM + N_SMALL),
             "class_sampled": lambda env: env.sampled[:2500], "class_list": lambda env: env.ids["samples"]}


def check_more(ctx, env, orc, w, got, model, exact, what):
    """The readers of read_more at the explicit weights w against the checkers."""
    ids, data = env.ids, env.data
    bad = []
    for name in ("fwd_rows", "fwd_stream"):
        m, ref = got["margins_" + name], OM.margins(orc, w, idx=ids[name])
        if exact:
            ok = np.array_equal(m, ref)
        else:
            ok = (np.abs(m - ref) <= 1e-12 * OM.margins(_abs_oracle(env), np.abs(w), idx=ids[name])).all()
        if not ok:
            bad.append(f"margins over {name}: {np.count_nonzero(m != ref)} differ from the checker's")
    if model == "logistic":
        m = ctx.margins(ids["fwd_stream"], w)
        e = np.exp(-np.abs(m))
        ref = np.where(m <= 0, 1.0 / (1.0 + e), e / (1.0 + e))     # sigmoid(-m)
        if not np.allclose(got["probabilities"], ref, rtol=1e-12, atol=0):
            bad.append("probabilities against sigmoid(-m) of the device's margins")
    rows = {"range": np.arange(N_STREAM, dtype=np.int32), "sampled": env.sampled[100:1100], "list": ids["samples"]}
    dev_m = {k: ctx.margins(v, w) for k, v in rows.items()}
    for k in ("range", "sampled", "list"):
        words = got["metrics_" + k]
        if not np.array_equal(words, OM.metrics(orc, w, idx=rows[k], margins=dev_m[k])):
            bad.append(f"metrics words ({k}) against the checker on the device's margins")
        if exact and not np.array_equal(words, OM.metrics(orc, w, idx=rows[k])):
            bad.append(f"metrics words ({k}) against the checker's own dots")
    for k in ("range", "list"):
        words, ap, thr, tp, fp = got["curve_" + k]
        ref = OC.curve(orc, w, idx=rows[k], margins=dev_m[k])
        if not (np.array_equal(thr, ref.thr) and np.array_equal(tp, ref.tp) and np.array_equal(fp, ref.fp)):
            bad.append(f"curve points ({k}) against the checker")
        if not np.array_equal(words, got["metrics_" + k]):
            bad.append(f"curve words ({k}) against eval_metrics")
        if not (ap == ref.ap or abs(ap - ref.ap) <= 2 * np.spacing(ref.ap)):
            bad.append(f"AP ({k}) {ap!r} against {ref.ap!r}")
    words, ap, n_pts = got["ap_range"]
    if not (np.array_equal(words, got["curve_range"][0]) and _bits(ap) == _bits(got["curve_range"][1])
            and n_pts == len(got["curve_range"][2])):
        bad.append("the AP-only pass against the pass with points")
    lab = np.asarray(data.label)
    # CUDA's exp and glibc's differ in the last bit of some terms: near the optimum, where the sufficient-decrease bound
    # lies within rounding of F, the device's line search may fail one Newton step before the checker converges (or after),
    # at a point within the tolerances of the checker's
    for k in ("range", "list"):
        a, b, obj, info = got["calibrate_" + k]
        ref = CB.fit(dev_m[k], lab[rows[k]])
        done = (CB.CONVERGED, CB.LINE_SEARCH_FAILED)
        if int(info[1]) not in done or ref.status not in done or abs(a - ref.a) > 1e-8 * max(1.0, abs(ref.a)) or \
                abs(b - ref.b) > 1e-8 * max(1.0, abs(ref.b)) or abs(obj - ref.objective) > 1e-10 * abs(ref.objective):
            bad.append(f"calibrate ({k}): {(a, b, obj, int(info[1]))} against {ref}")
    a, b = CAL_AB
    if not np.allclose(got["calibrated"], CB.probs(ctx.margins(ids["fwd_stream"], w), a, b), rtol=1e-12, atol=0):
        bad.append("calibrated probabilities against the checker")
    for k in ("range", "list"):
        sums, rows_b, pos_b, psum, cw_words = got["calibration_" + k]
        ref = CB.quality(dev_m[k], lab[rows[k]], a, b, 10)
        if cw_words.tolist() != [ref.rows, ref.left_out] or not np.allclose(sums, [ref.brier_sum, ref.log_loss_sum], rtol=1e-12):
            bad.append(f"eval_calibration ({k}) sums or words against the checker")
        if np.abs(rows_b - ref.bin_rows).sum() > 2 * ref.edge_rows or np.abs(pos_b - ref.bin_pos).sum() > 2 * ref.edge_rows:
            bad.append(f"eval_calibration ({k}) bins against the checker")
    l1, nnz = got["weights_l1"]
    if nnz != np.count_nonzero(w):
        bad.append(f"weights_l1: {nnz} non-zeros against {np.count_nonzero(w)}")
    want = math.fsum(np.abs(w))
    if not (l1 == want == L1.l1_norm(w) if exact else abs(l1 - want) <= 2.0 ** -52 * want):
        bad.append(f"weights_l1: {l1!r} against {want!r}")
    n2 = math.fsum(w * w)
    for k, f in CLASS_IDS.items():
        if k not in got:
            continue
        ce = got[k]
        sums, counts = CW.eval_class(orc, w, f(env), model == "logistic")
        if [ce.correct_pos, ce.correct_neg, ce.n_pos, ce.n_neg] != list(counts):
            bad.append(f"{k}: counts {ce[3:]} against {tuple(counts)}")
        if model == "logistic":
            ok = np.allclose([ce.loss_pos, ce.loss_neg], sums, rtol=1e-12, atol=0)
        else:
            ok = [ce.loss_pos, ce.loss_neg] == list(sums)
        if not ok:
            bad.append(f"{k}: loss sums {ce.loss_pos!r}, {ce.loss_neg!r} against {tuple(sums)}")
        if not (ce.norm_squared == n2 if exact else abs(ce.norm_squared - n2) <= 1e-12 * n2):
            bad.append(f"{k}: ||w||^2 {ce.norm_squared!r} against {n2!r}")
    assert not bad, f"{what}:\n" + "\n".join(bad)


def check_weighted_gradients(ctx, env, orc, w, c, got_res, got_exp, model, exact, what):
    """The class-weighted gradient requests at w == NULL and at w against oracle/cw.gradient."""
    wp, wn = ctx.get_class_weights()
    for name in ("grad_stream", "grad_rows"):
        idx = env.ids[name]
        (g_res, l_res), (g, loss) = [(d[name]["grad"], d[name]["loss"]) for d in (got_res, got_exp)]
        g_ref, loss_ref, _ = CW.gradient(orc, w, idx, wp, wn, logistic=model == "logistic")
        # the summed magnitudes of a column's terms: each row's is at most max(w_pos, w_neg) |x_j|, and c enters once
        mag = max(wp, wn) * _grad_scale(env, env.data, idx, 0.0) + abs(c)
        if exact:
            assert np.array_equal(g_res, g) and l_res == loss, f"{what}: {name} at w == NULL against the explicit weights"
            assert np.array_equal(g, g_ref) and loss == loss_ref, f"{what}: {name} against the checker"
            continue
        tol = 1e-13 * mag + 1e-15 * np.abs(g_ref)
        for a, who in ((g_res, "w == NULL"), (g, "explicit weights")):
            assert np.array_equal(a != 0, g_ref != 0), f"{what}: {name} ({who}): supports differ from the checker's"
            j = np.flatnonzero(np.abs(a - g_ref) > tol)
            assert j.size == 0, f"{what}: {name} ({who}) column {j[0]}: {a[j[0]]!r} against {g_ref[j[0]]!r}"
        for v, who in ((l_res, "w == NULL"), (loss, "explicit weights")):
            assert abs(v - loss_ref) <= 1e-11 * abs(loss_ref), f"{what}: {name} loss ({who}) {v!r} against {loss_ref!r}"


def check_all_readers(ctx, env, orc, model, exact_resident, exact_oracle, what, weighted=None, check_gradients=None):
    """Every reader at w == NULL against the explicit weights, and those against the checkers; returns (w, c).  weighted:
    the gradient is weighted (default: by class weights other than (1, 1)), and check_gradients checks it (default:
    check_weighted_gradients)."""
    w = ctx.get_weights()
    if weighted is None:
        weighted = ctx.get_class_weights() != (1.0, 1.0)
    resident, explicit = read_all(ctx, env, None, model), read_all(ctx, env, w, model)
    want, c = oracle_all(orc, env, w, model)
    scales = {n: _grad_scale(env, env.data, env.ids[n], c) for n in ("grad_stream", "grad_rows")}
    if weighted:       # the weighted gradient has its own checker; read_all's evaluations are unweighted
        (check_gradients or check_weighted_gradients)(ctx, env, orc, w, c, resident, explicit, model, exact_oracle, what)
        for d in (resident, explicit, want):
            del d["grad_stream"], d["grad_rows"]
    compare(resident, explicit, exact_resident, f"{what}, w == NULL against the explicit weights", scales)
    compare(explicit, want, exact_oracle, f"{what}, explicit weights against the oracle", scales)

    more_res, more_exp = read_more(ctx, env, None, model, weighted), read_more(ctx, env, w, model, weighted)
    bad = []
    for k, v in more_exp.items():
        r = more_res[k]
        if k.startswith("class_") and not exact_resident:     # ||w||^2: the step kernels sum it in another order
            if abs(r.norm_squared - v.norm_squared) > 1e-12 * v.norm_squared:
                bad.append(f"{k}.norm_squared: {r.norm_squared!r} against {v.norm_squared!r}")
            r, v = r._replace(norm_squared=0.0), v._replace(norm_squared=0.0)
        if _bits(r) != _bits(v):
            bad.append(k)
    assert not bad, f"{what}, w == NULL against the explicit weights: {bad}"
    check_more(ctx, env, orc, w, more_exp, model, exact_oracle, f"{what}, explicit weights against the checkers")
    return w, c


# ---- the next step from the resident state --------------------------------------------------------------------------------

def step_ref(ctx, orc, w, ids, batch, lrs, model, lam1=None, class_w=None):
    """The next step of the checker under the context's options (or those given): (w, loss)."""
    lam1 = ctx.info()["lambda1"] if lam1 is None else lam1
    wp, wn = ctx.get_class_weights() if class_w is None else class_w
    if (wp, wn) != (1.0, 1.0):
        w_ref, l_ref = CW.sync_steps(orc, w, ids, [batch], lrs, wp, wn, logistic=model == "logistic", lambda1=lam1)
    else:
        w_ref, l_ref = L1.sync_steps(orc, w, ids, [batch], lrs, lam1, logistic=model == "logistic")
    return w_ref, l_ref[0]


def check_next_step(ctx, env, orc, S, w, c, exact, path, table, model, what, ref=None, cmax=None):
    """One step with the context's options on (path "persistent": batch 64; "per_step": 32 G + 1), from the resident state
    and after set_weights(w) re-derives it: the same weights and loss, and the checker's.  ref: the checker's step, as
    step_ref takes and returns it; cmax: the largest weight of a row (else the larger class weight)."""
    _one_worker(ctx)
    ctx.set_grid_limit(0)
    ids = env.ids["step"] if path == "persistent" else _big_step(env, S)
    batch = ids.size
    lrs = np.array([env.lr])

    def step():
        loss = ctx.sync_steps_lr(ids, batch, lrs)[0] if table else ctx.sync_steps(ids, batch, 1, env.lr)[0]
        return loss, ctx.get_weights()

    loss, w1 = step()
    ctx.set_weights(w)
    loss_twin, w1_twin = step()
    w_ref, loss_ref = (ref or step_ref)(ctx, orc, w, ids, batch, lrs, model)
    what = f"{what}, next step on the {path} path"
    if exact:
        assert loss == loss_twin == loss_ref, f"{what}: loss {loss!r} / re-set {loss_twin!r} / checker {loss_ref!r}"
        for a, name in ((w1, "resident"), (w1_twin, "re-set")):
            diff = np.flatnonzero(a != w_ref)
            assert diff.size == 0, f"{what}, from the {name} state, column {diff[0]}: {a[diff[0]]!r} against " \
                                   f"{w_ref[diff[0]]!r} ({diff.size} differ)"
        return
    assert abs(loss - loss_twin) <= 1e-12 * abs(loss_twin), f"{what}: loss {loss!r} against {loss_twin!r}"
    assert abs(loss_twin - loss_ref) <= 1e-12 * abs(loss_ref), f"{what}: loss {loss_twin!r} against the checker's {loss_ref!r}"
    wmax = max(ctx.get_class_weights()) if cmax is None else cmax
    tol = 1e-12 * (np.abs(w1_twin) + env.lr * wmax * _grad_scale(env, env.data, ids, c))
    assert np.array_equal(w1 != 0, w1_twin != 0), f"{what}: supports differ"
    bad = np.flatnonzero(np.abs(w1 - w1_twin) > tol)
    assert bad.size == 0, f"{what}, column {bad[0]}: {w1[bad[0]]!r} against {w1_twin[bad[0]]!r}"
    assert np.array_equal(w1_twin != 0, w_ref != 0), f"{what}: supports differ from the checker's"
    np.testing.assert_allclose(w1_twin, w_ref, rtol=1e-11, atol=1e-15, err_msg=f"{what}: against the checker")


# ---- writers ----------------------------------------------------------------------------------------------------------------

SVM_CASES = [
    # (options at the reset, writer)
    *[("l1", wr) for wr in ("set_weights", "persistent", "persistent_grid2", "per_step", "two_workers", "staged",
                            "avg_persistent", "avg_per_step", "table_persistent", "table_per_step")],
    *[("cw", wr) for wr in ("persistent", "per_step", "two_workers", "staged", "table_persistent")],
    *[("cw+l1", wr) for wr in ("persistent", "per_step")],
    *[("", wr) for wr in ("table_persistent", "table_per_step")],
    ("", "set_l1_on"), ("l1", "set_l1_cycle"), ("l1", "set_l1_change"), ("l1", "set_dim_sparsity"),
    ("l1", "compute_dim_sparsity"), ("", "cw_on"), ("cw", "cw_off"),
]
LOGISTIC_CASES = [("l1", "steps"), ("l1", "table_steps"), ("cw", "steps")]
STATE_ONLY = ("set_l1_on", "set_l1_change", "cw_on", "cw_off")


def write(ctx, env, S, writer, rng):
    """Runs the writer on ctx (its options already set); returns the dimSparsity it leaves."""
    lam1, lam1b, lrs = consts(env)
    big = 32 * S + 1
    if writer == "set_weights":
        ctx.set_weights(env.w1)
    elif writer in ("persistent", "persistent_grid2", "avg_persistent", "steps"):
        if writer == "persistent_grid2":
            ctx.set_grid_limit(2)                     # batch 64 = 32 G: still the persistent kernel
        if writer == "avg_persistent":
            ctx.average_begin()
        ctx.sync_steps(_steps(rng, BATCH, 2), BATCH, 2, env.lr)
    elif writer in ("per_step", "avg_per_step"):
        if writer == "avg_per_step":
            ctx.average_begin()
        ctx.sync_steps(_steps(rng, big, 2), big, 2, env.lr)
    elif writer in ("table_persistent", "table_steps"):
        ctx.sync_steps_lr(_steps(rng, BATCH, lrs.size), BATCH, lrs)
    elif writer == "table_per_step":
        ctx.sync_steps_lr(_steps(rng, big, lrs.size), big, lrs)
    elif writer == "two_workers":
        ctx.set_workers([40, 24], 2)
        ctx.sync_steps(_steps(rng, BATCH, 2), BATCH, 2, env.lr)
    elif writer == "staged":
        ctx.stage_samples(_steps(rng, BATCH, 5))
        ctx.sync_steps_staged(BATCH, BATCH, 3, env.lr)
    elif writer == "set_l1_on":                     # the context's own: ||w||_1 never derived, scal[kScalL1] = 0
        ctx.set_weights(env.w1)
        ctx.set_l1(lam1)
    elif writer == "set_l1_cycle":                  # scal[kScalL1] holds ||w0||_1 while the penalty is off
        ctx.set_l1(0.0)
        ctx.set_weights(env.w1)
        ctx.set_l1(lam1)
    elif writer == "set_l1_change":
        ctx.set_l1(lam1b)
    elif writer == "set_dim_sparsity":
        ctx.set_dim_sparsity(env.d2)
        return env.d2
    elif writer == "compute_dim_sparsity":
        return ctx.compute_dim_sparsity(env.n_train2)
    elif writer == "cw_on":
        ctx.set_class_weights(*CLASS_W)
    elif writer == "cw_off":
        ctx.set_class_weights(1.0, 1.0)
    else:
        raise KeyError(writer)
    if writer.startswith("avg_"):
        ctx.average_end()
    return env.d


def state_witness(ctx, env, orc, S, writer, w_after, model):
    """The next per-step loss under the state from before a writer of state only differs from the right one."""
    lam1, lam1b, _ = consts(env)
    ids = _big_step(env, S)
    lrs = np.array([env.lr])
    _, right = step_ref(ctx, orc, w_after, ids, ids.size, lrs, model)
    if writer == "set_l1_on":                       # a stale scal[kScalL1] = 0
        stale = right - lam1 * math.fsum(np.abs(w_after))
    elif writer == "set_l1_cycle":                  # a stale ||w0||_1
        stale = right - lam1 * (math.fsum(np.abs(w_after)) - math.fsum(np.abs(env.w0)))
    elif writer == "set_l1_change":
        _, stale = step_ref(ctx, orc, w_after, ids, ids.size, lrs, model, lam1=lam1)
    else:
        _, stale = step_ref(ctx, orc, w_after, ids, ids.size, lrs, model,
                            class_w=(1.0, 1.0) if writer == "cw_on" else CLASS_W)
    assert _moved(right, stale), f"{writer}: the next loss under the stale state ({stale!r}) is the right one ({right!r})"


def run_case(ctx_of, env, S, options, writer, model):
    kind = env.kind
    what = f"{'logistic' if model == 'logistic' else 'SVM'} [{options or 'no options'}], {kind}, dim {env.dim}, {writer}"
    exact = kind == "dyadic" and writer != "compute_dim_sparsity"   # compute_dim_sparsity's d = 1 / (df + 1)
    table = "table" in writer
    for i, path in enumerate(("per_step", "persistent")):
        rng = np.random.default_rng([zlib.crc32(f"{options}/{writer}".encode()), env.dim])
        ctx, own = ctx_of(writer)
        try:
            _reset(ctx, env, env.w0)
            _set_options(ctx, env, options)
            d_after = write(ctx, env, S, writer, rng)
            w_after = ctx.get_weights()
            orc = env.oracle(d_after, model=model)
            if i == 0:
                orc_before = env.oracle(env.d, model=model)
                if writer in STATE_ONLY:
                    state_witness(ctx, env, orc, S, writer, w_after, model)
                elif writer == "set_l1_cycle":
                    witness(env, "w", env.w0, w_after, env.d, d_after, orc_before=orc_before, orc_after=orc)
                    state_witness(ctx, env, orc, S, writer, w_after, model)
                else:
                    witness(env, "d" if "dim_sparsity" in writer else "w", env.w0, w_after, env.d, d_after,
                            orc_before=orc_before, orc_after=orc)
                    if ctx.info()["lambda1"] > 0 and "dim_sparsity" not in writer:
                        assert _moved(math.fsum(np.abs(env.w0)), math.fsum(np.abs(w_after))), "||w||_1 does not move"
                w, c = check_all_readers(ctx, env, orc, model, kind == "dyadic", exact, what)
            else:
                w, c = w_after, 2.0 * env.lam * math.fsum(w_after * d_after)
            check_next_step(ctx, env, orc, S, w, c, exact, path, table, model, what)
        finally:
            if own:
                ctx.close()


def _ctx_of(env, which):
    def get(writer):
        if writer != "set_l1_on":
            return env.ctx(which), False
        from distributed_sgd_b200.native import NativeCtx
        c = NativeCtx(0, env.dim, env.lam, logistic=which == "logistic")
        c.load_csr(env.data.row_ptr, env.data.col, env.data.val, env.data.label)
        return c, True
    return get


@pytest.mark.parametrize("options,writer", SVM_CASES, ids=[f"{o or 'none'}-{w}" for o, w in SVM_CASES])
@pytest.mark.parametrize("dim", DIMS)
@pytest.mark.parametrize("kind", KINDS)
def test_svm(envs, S, kind, dim, options, writer):
    env = envs(kind, dim)
    try:
        run_case(_ctx_of(env, "sync"), env, S, options, writer, "svm")
    finally:
        _set_options(env.ctx("sync"), env, "")


@pytest.mark.parametrize("options,writer", LOGISTIC_CASES, ids=[f"{o}-{w}" for o, w in LOGISTIC_CASES])
@pytest.mark.parametrize("dim", DIMS)
def test_logistic(envs, S, dim, options, writer):
    """fp32 rows only: the logistic loss of dyadic rows is not dyadic.  The logistic model always takes the per-step path."""
    env = envs("fp32", dim)
    try:
        run_case(_ctx_of(env, "logistic"), env, S, options, writer, "logistic")
    finally:
        _set_options(env.ctx("logistic"), env, "")


# ---- fused K = 2 on one GPU with a rate table ------------------------------------------------------------------------------

@pytest.mark.parametrize("kind", KINDS)
def test_fused_two_ranks_rate_table(envs, S, kind):
    """Two ranks of the fused peer-exchange step on one GPU, one call with a rate table; every reader on both ranks."""
    env = envs(kind, 700)
    rng = np.random.default_rng(78)
    lrs = np.array([env.lr, env.lr / 2])
    per_rank = [np.stack([rng.choice(N_ROWS, size=BATCH, replace=False) for _ in range(2)]).astype(np.int32)
                for _ in range(2)]
    orc = env.oracle(env.d)

    def after(r, ctx):
        what = f"fused K = 2 with a rate table, {kind}, rank {r}"
        w = ctx.get_weights()
        witness(env, "w", env.w0, w, env.d, env.d, orc_after=orc)
        check_all_readers(ctx, env, orc, "svm", kind == "dyadic", kind == "dyadic", what)
        return w

    res = fused_ranks(env.data, env.lam, env.d, [S // 2, S // 2], env.w0, [(per_rank, None)], lrs, after=after)
    w_ref, l_ref = L1.sync_steps(orc, env.w0, np.concatenate(per_rank, axis=1).reshape(-1), [BATCH, BATCH], lrs, 0.0)
    if kind == "dyadic":
        np.testing.assert_array_equal(res["after"][0], w_ref)
        np.testing.assert_array_equal(res["losses"][0], l_ref)
    else:
        np.testing.assert_allclose(res["after"][0], w_ref, rtol=1e-11, atol=1e-15)
        np.testing.assert_allclose(res["losses"][0], l_ref, rtol=1e-12)


# ---- the staged sample stream ------------------------------------------------------------------------------------------------

def _list_readers(ctx, env, rng, logistic):
    """Every list-form reader on ids the stream does not hold, fewer and more than it does, and weights_l1."""
    w = ctx.get_weights()
    a, b = CAL_AB
    for n in (100, N_STREAM):
        other = rng.choice(N_ROWS, size=n, replace=False).astype(np.int32)
        for wx in (None, env.w1):
            ctx.forward(other, wx)
            ctx.gradient(other, wx, want_loss=True)
            ctx.margins(other, wx)
            if logistic:
                ctx.probabilities(other, wx)
            ctx.eval_samples_metrics(other, wx)
            ctx.eval_samples_curve(other, wx)
            ctx.eval_samples_curve(other, wx, curve=False)
            ctx.eval_samples_class(other, wx)
            ctx.calibrate_samples(other, wx)
            ctx.calibrated_probabilities(other, a, b, wx)
            ctx.eval_samples_calibration(other, a, b, 10, wx)
    ctx.weights_l1()
    ctx.weights_l1(env.w1)
    assert np.array_equal(ctx.get_weights(), w)


@pytest.mark.parametrize("kind,logistic", [("dyadic", False), ("fp32", True)])
def test_readers_leave_the_staged_stream(envs, kind, logistic):
    """L1, class weights and averaging on: stage 4 steps, run them as two staged calls of 2, with every list-form reader
    before the first and between the two; losses, weights, the average and its count have the bits of a run with no reader
    in between (the logistic model to rounding: its gradient scatter adds in arrival order), and the checker's."""
    env = envs(kind, 700)
    ctx = env.ctx("logistic" if logistic else "sync")
    lam1 = consts(env)[0]
    stream = _steps(np.random.default_rng(3), BATCH, 4)
    runs = []
    try:
        for readers in (False, True):
            rng = np.random.default_rng(9)
            _reset(ctx, env, env.w0)
            _set_options(ctx, env, "cw+l1")
            ctx.stage_samples(stream)
            ctx.average_begin()
            losses = []
            for first in (0, 2 * BATCH):
                if readers:
                    _list_readers(ctx, env, rng, logistic)
                ctx.sync_steps_staged(first, BATCH, 2, env.lr, want_losses=True)
                losses.append(ctx.read_losses(2))
            avg, n = ctx.average_weights()
            ctx.average_end()
            runs.append((np.concatenate(losses), ctx.get_weights(), avg, n))
    finally:
        _set_options(ctx, env, "")
    for got, want, name in zip(runs[1], runs[0], ("losses", "weights", "average", "count")):
        if logistic and name != "count":   # its fp64 scatter adds land in arrival order: runs agree to rounding
            np.testing.assert_allclose(got, want, rtol=1e-13, atol=1e-16, err_msg=f"{name} with the readers in between")
        else:
            assert _bits(got) == _bits(want), f"{name} differ with the readers in between"
    assert runs[0][3] == runs[1][3] == 4
    avg_sum = np.zeros(env.dim)
    w_ref, l_ref = CW.sync_steps(env.oracle(env.d, logistic=logistic), env.w0, stream, [BATCH], np.full(4, env.lr), *CLASS_W,
                                 logistic=logistic, lambda1=lam1, avg_sum=avg_sum)
    if kind == "dyadic":
        assert np.array_equal(runs[0][1], w_ref) and np.array_equal(runs[0][0], l_ref)
        v = avg_sum / 4
        assert np.array_equal(runs[0][2], np.where(np.abs(v) > 1e-20, v, 0.0))
    else:
        np.testing.assert_allclose(runs[0][0], l_ref, rtol=1e-11)
        assert np.abs(runs[0][1] - w_ref).max() <= 1e-11 * np.abs(w_ref).max()
