"""Resident-weight reads (w == NULL) after every writer of a context with sample weights, and the weighted readers after
every writer.

The reader x writer matrix of test_gpu_resident_state.py and test_gpu_resident_options.py, on per-row sample weights.  They
have no derived state: dsgd_set_sample_weights only stores them, and every kernel forms c_i = fl(w_y s_i) live -- the row
kernel, the persistent kernel's producer and epilogue, and k_metrics_score.  So a writer of the weights or of the class
weights is followed, with no set_weights in between, by every reader and by the next step.

Writers, each on a context left with its options on (the persistent kernel at batch 64, the per-step path at 32 G + 1):

- sample weights s (SVM): set_weights, the persistent kSampleWeighted form at full grid and at grid limit 2, the per-step
  path, sync_step, two virtual workers [40, 24], staged steps, averaging and a rate table on both paths;  s and class weights
  (2, 1/2): persistent, per-step, two workers, staged;  s and L1: persistent, per-step and a rate table on both paths (the L1
  forms with a rate table spill 16-32 bytes);  s, class weights and L1: persistent and per-step;  logistic (fp32 rows): steps,
  two workers, L1 with a rate table, class weights;
- writers of state only: s on (none -> s), s -> s', s off, class weights (1, 1) -> (2, 1/2) and back under s, L1 on under s,
  and a reload under s on a context of its own (it drops the weights);
- the weighted readers after every writer of test_gpu_resident_options.py, with no sample weights (c_i = w_y).

Readers: everything read_all and read_more read; eval_weighted over N_STREAM rows and over N_SMALL rows, its sampled and list
forms; the weighted curve over a range with points and words only, its sampled and list forms; and the sample-weighted
gradient (k_rows<..., kSampleWeighted, ...> at any size) below and above 2 048 ids.  w == NULL against the weights from
get_weights: every weighted sum and count, weighted-curve word, threshold and point weight, AUC and AP bit for bit; ||w||^2
bit for bit on dyadic rows, else within 1e-12 (the step kernels sum it in another order).  The explicit reads against the
checkers: oracle/sw.eval_weighted bit for bit (the logistic S within rtol 1e-13), oracle/wcurve.wcurve over the device's own
margins bit for bit, oracle/sw.gradient exactly on dyadic rows and else within 1e-13 of the summed magnitudes of its terms,
sum_i c_i |x_ij| + 2 lambda sum_j |w_j d_j| (c = 2 lambda (w . d) cancels, and each path sums it in its own order).  The readers
that stay unweighted under sample weights (eval_sums, eval_counts, metrics, curves, calibration, eval_class) still match
their checkers.

The next step after every writer, on both paths with the options on: the same weights and loss as the same step after
set_weights(w), and oracle/sw.sync_steps (oracle/cw or oracle/l1 without sample weights); on dyadic rows bit for bit.

Dyadic constants (test_gpu_resident_state.py: values multiples of 1/2, weights of 2^-5, lr 2 lambda d = 1): sample weights
from {0, 1/2, 1, 2} with zeros, class weights 2 and 1/2, so c in {0, 1/4, 1/2, 1, 2, 4}; lambda1 and the rate tables of
consts().  Every weight after a writer and on the checker's next step is asserted to be a multiple of 2^-10 below 2^7 (the
per-step path's 32 G + 1 rows at c up to 4 carry a few weights past 2^6): then w_j^2 is a multiple of 2^-20 below 2^14,
||w||^2 of 56 000 weights stays below 2^30 (50 bits), ||w||_1 below 2^23, and every sum is exact in any order.

Every case first shows on the checker that stale state would fail: for the step writers at least 1 % of the streaming pass's
rows change prediction and ||w||^2 moves; for the writers of state only, the next per-step loss and eval_weighted's S under the old sample
or class weights (or lambda1) differ from the right ones.

Then: the persistent kernel's hinge codes across launches of other grid sizes, step counts and batches; the weighted curve,
curve, metrics, calibration and eval_weighted passes interleaved on one context at growing and shrinking sizes against fresh
contexts; and eval_weighted on an async context after the async writers.
"""
import functools
import math
import zlib

import numpy as np
import pytest

from oracle import sw as SW
from oracle import wcurve as OW
from test_gpu_resident_options import (CLASS_W, LOGISTIC_CASES, SVM_CASES, _big_step, _bits, _ctx_of, _set_options,
                                       check_all_readers, check_next_step, consts, write)
from test_gpu_resident_options import step_ref as step_ref_unweighted
from test_gpu_resident_state import (ASYNC_WRITERS, BATCH, DIMS, KEY, KINDS, N_ROWS, N_SMALL, N_STREAM, S, _moved, _reset,  # noqa: F401
                                     _steps, async_write, envs, witness)
from test_gpu_weighted_curve import dyadic_data as curve_rows

pytestmark = pytest.mark.gpu

SW_VALUES = np.array([0.0, 0.5, 1.0, 2.0])
GRID, WMAX = 2.0 ** -10, 2.0 ** 7   # every dyadic weight is a multiple of GRID below WMAX: every sum is exact in any order


@pytest.fixture(scope="module", autouse=True)
def _device():
    """Skips the module where there is no CUDA device (before the module's contexts are made)."""
    from distributed_sgd_b200.native import DsgdError, NativeCtx
    try:
        NativeCtx(0, 16, 0.0).close()
    except DsgdError as e:
        if "no usable CUDA device" not in str(e):
            raise
        pytest.skip(f"needs a GPU: {e}")


def sample_weights(env, which):
    """The env's sample weights s (which 0) and s' (which 1), drawn from SW_VALUES."""
    if not hasattr(env, "sw"):
        env.sw = {}
    if which not in env.sw:
        rng = np.random.default_rng([env.dim, 0 if env.kind == "dyadic" else 1, 71 + which])
        env.sw[which] = rng.choice(SW_VALUES, size=N_ROWS)
    return env.sw[which]


def on_grid(w, what):
    q = w / GRID
    assert np.array_equal(q, np.round(q)) and np.abs(w).max() < WMAX, f"{what}: the weights leave the grid of 2^-10 below 2^7"


def _c_scale(env, idx, cvec):
    """sum_i c_i |x_ij| per column over the listed rows: the scale of a weighted gradient entry's rounding."""
    data = env.data
    lo, hi = data.row_ptr[idx], data.row_ptr[idx + 1]
    pos = np.concatenate([np.arange(a, b) for a, b in zip(lo, hi)])
    rows = np.repeat(np.asarray(idx), hi - lo)
    return np.bincount(data.col[pos], weights=np.abs(data.val[pos].astype(np.float64)) * cvec[rows], minlength=env.dim)


# ---- the weighted readers ---------------------------------------------------------------------------------------------------

def read_weighted(ctx, env, w):
    """Every weighted reader once, at the weights w (None: resident).  {reader: value}."""
    ids = env.ids
    return {
        "we_range": ctx.eval_weighted(0, N_STREAM, w),
        "we_rows": ctx.eval_weighted(N_STREAM, N_STREAM + N_SMALL, w),
        "we_sampled": ctx.eval_sampled_weighted(0, N_ROWS, KEY, 0, 2500, w),
        "we_list": ctx.eval_samples_weighted(ids["samples"], w),
        "wc_range": ctx.eval_weighted_curve(0, N_STREAM, w),
        "wc_words": ctx.eval_weighted_curve(0, N_STREAM, w, curve=False),
        "wc_sampled": ctx.eval_sampled_weighted_curve(0, N_ROWS, KEY, 100, 1100, w),
        "wc_list": ctx.eval_samples_weighted_curve(ids["samples"], w),
    }


WEIGHTED_IDS = {"we_range": lambda env: np.arange(N_STREAM), "we_rows": lambda env: np.arange(N_STREAM, N_STREAM + N_SMALL),
                "we_sampled": lambda env: env.sampled[:2500], "we_list": lambda env: env.ids["samples"],
                "wc_range": lambda env: np.arange(N_STREAM), "wc_words": lambda env: np.arange(N_STREAM),
                "wc_sampled": lambda env: env.sampled[100:1100], "wc_list": lambda env: env.ids["samples"]}


def check_weighted_readers(ctx, env, orc, sw, model, exact_resident, exact_oracle, what):
    """The weighted readers at w == NULL against the explicit weights, and those against oracle/sw and oracle/wcurve."""
    w = ctx.get_weights()
    wp, wn = ctx.get_class_weights()
    res, exp = read_weighted(ctx, env, None), read_weighted(ctx, env, w)
    bad = []
    for k, v in exp.items():
        r = res[k]
        if k.startswith("we_") and not exact_resident:     # ||w||^2: the step kernels sum it in another order
            if abs(r.norm_squared - v.norm_squared) > 1e-12 * v.norm_squared:
                bad.append(f"{k}.norm_squared: {r.norm_squared!r} against {v.norm_squared!r}")
            r, v = r._replace(norm_squared=0.0), v._replace(norm_squared=0.0)
        if _bits(r) != _bits(v):
            bad.append(k)
    assert not bad, f"{what}, weighted readers at w == NULL against the explicit weights: {bad}"

    lab = np.asarray(env.data.label)
    cvec = OW.weights(lab, wp, wn, sw)
    n2 = math.fsum(w * w)
    for k, v in exp.items():
        ids = WEIGHTED_IDS[k](env)
        if k.startswith("we_"):
            sums, counts = SW.eval_weighted(orc, w, ids, wp, wn, sw, logistic=model == "logistic")
            if [v.n, v.correct] != list(counts) or [v.correct_weight, v.weight_sum] != list(sums[1:]):
                bad.append(f"{k}: {v} against sums {tuple(sums)}, counts {tuple(counts)}")
            if not (abs(v.loss_sum - sums[0]) <= 1e-13 * abs(sums[0]) if model == "logistic" else v.loss_sum == sums[0]):
                bad.append(f"{k}: S {v.loss_sum!r} against {sums[0]!r}")
            if not (v.norm_squared == n2 if exact_oracle else abs(v.norm_squared - n2) <= 1e-12 * n2):
                bad.append(f"{k}: ||w||^2 {v.norm_squared!r} against {n2!r}")
            continue
        ref = OW.wcurve(ctx.margins(ids, w), lab[ids], cvec[ids])
        if not (np.array_equal(v.words, ref.words) and _bits(v.wsums) == _bits(ref.wsums) and v.n_points == len(ref.thr)
                and _bits((v.auc, v.ap)) == _bits((ref.auc, ref.ap))):
            bad.append(f"{k}: words, weighted words, point count, AUC or AP against the checker")
        if k == "wc_words":
            if len(v.thr) or len(v.tpw) or len(v.fpw):
                bad.append(f"{k}: points from a words-only pass")
        elif _bits((v.thr, v.tpw, v.fpw)) != _bits((ref.thr, ref.tpw, ref.fpw)):
            bad.append(f"{k}: points against the checker")
    assert not bad, f"{what}, weighted readers against the checkers:\n" + "\n".join(bad)


def check_sw_gradients(sw, ctx, env, orc, w, c, got_res, got_exp, model, exact, what):
    """The gradient requests at w == NULL and at w against oracle/sw.gradient under the context's class weights and sw."""
    wp, wn = ctx.get_class_weights()
    cvec = OW.weights(env.data.label, wp, wn, sw)
    for name in ("grad_stream", "grad_rows"):
        idx = env.ids[name]
        (g_res, l_res), (g, loss) = [(d[name]["grad"], d[name]["loss"]) for d in (got_res, got_exp)]
        g_ref, loss_ref, _ = SW.gradient(orc, w, idx, sw, wp, wn, logistic=model == "logistic")
        if exact:
            assert np.array_equal(g_res, g) and l_res == loss, f"{what}: {name} at w == NULL against the explicit weights"
            assert np.array_equal(g, g_ref) and loss == loss_ref, f"{what}: {name} against the checker"
            continue
        # the summed magnitudes of a column's terms: sum_i c_i |x_ij|, and c's own, 2 lambda sum_j |w_j d_j|
        tol = 1e-13 * (_c_scale(env, idx, cvec) + 2.0 * env.lam * math.fsum(np.abs(w * env.d)))
        for a, who in ((g_res, "w == NULL"), (g, "explicit weights")):
            assert np.array_equal(a != 0, g_ref != 0), f"{what}: {name} ({who}): supports differ from the checker's"
            j = np.flatnonzero(np.abs(a - g_ref) > tol)
            assert j.size == 0, f"{what}: {name} ({who}) column {j[0]}: {a[j[0]]!r} against {g_ref[j[0]]!r}"
        for v, who in ((l_res, "w == NULL"), (loss, "explicit weights")):
            assert abs(v - loss_ref) <= 1e-12 * abs(loss_ref), f"{what}: {name} loss ({who}) {v!r} against {loss_ref!r}"


# ---- the next step ------------------------------------------------------------------------------------------------------------

def step_ref(ctx, orc, w, ids, batch, lrs, model, sw=None, exact=False):
    """The next step of the checker under the context's options: oracle/sw with sample weights loaded (sw), else the
    checker test_gpu_resident_options.step_ref picks from the class weights.  exact: its weights must stay on the grid."""
    assert ctx.info()["sample_weights"] is (sw is not None), "the checker's sample weights are not the context's"
    if sw is None:
        w_ref, loss = step_ref_unweighted(ctx, orc, w, ids, batch, lrs, model)
    else:
        w_ref, losses = SW.sync_steps(orc, w, ids, [batch], lrs, sw, *ctx.get_class_weights(), logistic=model == "logistic",
                                      lambda1=ctx.info()["lambda1"])
        loss = losses[0]
    if exact:
        on_grid(w_ref, "the checker's next step")
    return w_ref, loss


# ---- writers ------------------------------------------------------------------------------------------------------------------

SW_SVM_CASES = [
    # (options at the reset, besides the sample weights s; writer)
    *[("", wr) for wr in ("set_weights", "persistent", "persistent_grid2", "per_step", "sync_step", "two_workers", "staged",
                          "avg_persistent", "avg_per_step", "table_persistent", "table_per_step")],
    *[("cw", wr) for wr in ("persistent", "per_step", "two_workers", "staged")],
    *[("l1", wr) for wr in ("persistent", "per_step", "table_persistent", "table_per_step")],
    *[("cw+l1", wr) for wr in ("persistent", "per_step")],
    ("", "sw_on"), ("", "sw_change"), ("", "sw_off"), ("", "cw_on"), ("cw", "cw_off"), ("", "l1_on"), ("", "reload"),
]
SW_LOGISTIC_CASES = [("", "steps"), ("", "two_workers"), ("l1", "table_steps"), ("cw", "steps")]
SW_STATE_ONLY = ("sw_on", "sw_change", "sw_off", "cw_on", "cw_off", "l1_on", "reload")


def write_sw(ctx, env, S, writer, rng):
    """Runs the writer on ctx (its options and s already loaded, none for sw_on); returns the sample weights it leaves."""
    s0, s1 = sample_weights(env, 0), sample_weights(env, 1)
    if writer == "sw_on":
        ctx.set_sample_weights(s0)
    elif writer == "sw_change":
        ctx.set_sample_weights(s1)
        return s1
    elif writer == "sw_off":
        ctx.set_sample_weights(None)
        return None
    elif writer == "cw_on":
        ctx.set_class_weights(*CLASS_W)
    elif writer == "cw_off":
        ctx.set_class_weights(1.0, 1.0)
    elif writer == "l1_on":
        ctx.set_weights(env.w1)                     # with the penalty off
        ctx.set_l1(consts(env)[0])
    elif writer == "reload":                        # the same rows: the readers' checkers still hold
        d = env.data
        ctx.load_csr(d.row_ptr, d.col, d.val, d.label)
        return None
    elif writer == "sync_step":
        for _ in range(2):
            ctx.sync_step(_steps(rng, BATCH, 1), env.lr)
    else:
        write(ctx, env, S, writer, rng)
    return s0


def step_witness(env, orc, w_after):
    """test_gpu_resident_state.witness without c: at least 1 % of the streaming pass's rows change prediction and ||w||^2
    moves.  c = 2 lambda (w . d) moves only when a step's rows hold the one column d weighs (8 % of them) and pass the gate at
    a non-zero weight, which two steps of 64 rows do not always do."""
    rows = np.arange(N_STREAM, dtype=np.int32)
    flips = np.mean(orc.forward(env.w0, rows) != orc.forward(w_after, rows))
    assert flips >= 0.01, f"only {flips:.2%} of the streaming pass's rows change prediction"
    assert _moved(math.fsum(env.w0 * env.w0), math.fsum(w_after * w_after)), "||w||^2 does not move"


def _differs(a, b):
    """a and b differ by far more than the 1e-12 the next step's loss is checked to: lambda ||w||^2 of 56 000 weights is
    most of a loss, and one row's weight moves it by less than test_gpu_resident_state._moved's 1e-6."""
    return abs(a - b) > 1e-9 * max(abs(a), abs(b))


def state_witness(env, orc, S, writer, w, sw, class_w, lam1, model):
    """The next per-step loss and eval_weighted's S under the state from before a writer of state only differ from the
    right ones (for l1_on only the loss: the evaluation has no penalty)."""
    s0 = sample_weights(env, 0)
    sw_old = {"sw_on": None, "sw_change": s0, "sw_off": s0, "reload": s0}.get(writer, sw)
    cw_old = {"cw_on": (1.0, 1.0), "cw_off": CLASS_W}.get(writer, class_w)
    lam1_old = 0.0 if writer == "l1_on" else lam1
    ids = _big_step(env, S)
    lrs = np.array([env.lr])
    right = SW.sync_steps(orc, w, ids, [ids.size], lrs, sw, *class_w, logistic=model == "logistic", lambda1=lam1)[1][0]
    stale = SW.sync_steps(orc, w, ids, [ids.size], lrs, sw_old, *cw_old, logistic=model == "logistic", lambda1=lam1_old)[1][0]
    assert _differs(right, stale), f"{writer}: the next loss under the stale state ({stale!r}) is the right one ({right!r})"
    if writer != "l1_on":
        rows = np.arange(N_STREAM)
        right = SW.eval_weighted(orc, w, rows, *class_w, sw, logistic=model == "logistic")[0][0]
        stale = SW.eval_weighted(orc, w, rows, *cw_old, sw_old, logistic=model == "logistic")[0][0]
        assert _differs(right, stale), f"{writer}: eval_weighted's S under the stale state ({stale!r}) is the right one"


def run_case(ctx_of, env, S, options, writer, model):
    kind = env.kind
    what = f"{'logistic' if model == 'logistic' else 'SVM'} [s {options}], {kind}, dim {env.dim}, {writer}"
    exact = kind == "dyadic"
    table = "table" in writer
    for i, path in enumerate(("per_step", "persistent")):
        rng = np.random.default_rng([zlib.crc32(f"sw/{options}/{writer}".encode()), env.dim])
        ctx, own = ctx_of(writer)
        try:
            _reset(ctx, env, env.w0)
            _set_options(ctx, env, options)
            ctx.set_sample_weights(None if writer == "sw_on" else sample_weights(env, 0))
            sw = write_sw(ctx, env, S, writer, rng)
            assert ctx.info()["sample_weights"] is (sw is not None), f"{what}: sample weights loaded"
            class_w = ctx.get_class_weights()
            w_after = ctx.get_weights()
            orc = env.oracle(env.d, model=model)
            if exact:
                on_grid(w_after, what)
            if i == 0:
                if writer in SW_STATE_ONLY:
                    state_witness(env, orc, S, writer, w_after, sw, class_w, ctx.info()["lambda1"], model)
                else:
                    step_witness(env, orc, w_after)
                    if ctx.info()["lambda1"] > 0:
                        assert _moved(math.fsum(np.abs(env.w0)), math.fsum(np.abs(w_after))), "||w||_1 does not move"
                weighted = sw is not None or class_w != (1.0, 1.0)
                w, c = check_all_readers(ctx, env, orc, model, exact, exact, what, weighted=weighted,
                                         check_gradients=functools.partial(check_sw_gradients, sw))
                check_weighted_readers(ctx, env, orc, sw, model, exact, exact, what)
            else:
                w, c = w_after, 2.0 * env.lam * math.fsum(w_after * env.d)
            cmax = max(class_w) * (1.0 if sw is None else float(sw.max()))
            check_next_step(ctx, env, orc, S, w, c, exact, path, table, model, what,
                            ref=functools.partial(step_ref, sw=sw, exact=exact), cmax=cmax)
        finally:
            if own:
                ctx.close()


def _own_ctx_of(env, which):
    def get(writer):
        if writer != "reload":
            return env.ctx(which), False
        from distributed_sgd_b200.native import NativeCtx
        c = NativeCtx(0, env.dim, env.lam, logistic=which == "logistic")
        c.load_csr(env.data.row_ptr, env.data.col, env.data.val, env.data.label)
        return c, True
    return get


def _clear(ctx, env):
    ctx.set_sample_weights(None)
    _set_options(ctx, env, "")


@pytest.mark.parametrize("options,writer", SW_SVM_CASES, ids=[f"{o or 'sw'}-{w}" for o, w in SW_SVM_CASES])
@pytest.mark.parametrize("dim", DIMS)
@pytest.mark.parametrize("kind", KINDS)
def test_svm(envs, S, kind, dim, options, writer):
    env = envs(kind, dim)
    try:
        run_case(_own_ctx_of(env, "sync"), env, S, options, writer, "svm")
    finally:
        _clear(env.ctx("sync"), env)


@pytest.mark.parametrize("options,writer", SW_LOGISTIC_CASES, ids=[f"{o or 'sw'}-{w}" for o, w in SW_LOGISTIC_CASES])
@pytest.mark.parametrize("dim", DIMS)
def test_logistic(envs, S, dim, options, writer):
    """fp32 rows only: the logistic loss of dyadic rows is not dyadic.  The logistic model always takes the per-step path."""
    env = envs("fp32", dim)
    try:
        run_case(_own_ctx_of(env, "logistic"), env, S, options, writer, "logistic")
    finally:
        _clear(env.ctx("logistic"), env)


# ---- the weighted readers after the writers without sample weights -----------------------------------------------------------

def run_unweighted_case(ctx_of, env, S, options, writer, model):
    """A writer of test_gpu_resident_options.py, then the weighted readers (c_i = w_y).  The witness: a writer that moves the
    weights moves the predictions, c and ||w||^2; a class-weight writer moves eval_weighted's S.  The L1 and dimSparsity
    writers that keep the weights change nothing the weighted readers read, which must still give the bits of the weights."""
    what = f"{'logistic' if model == 'logistic' else 'SVM'} [{options or 'no options'}], {env.kind}, dim {env.dim}, {writer}"
    rng = np.random.default_rng([zlib.crc32(f"{options}/{writer}".encode()), env.dim])
    ctx, own = ctx_of(writer)
    try:
        _reset(ctx, env, env.w0)
        _set_options(ctx, env, options)
        ctx.set_sample_weights(None)
        write(ctx, env, S, writer, rng)
        assert ctx.info()["sample_weights"] is False
        w_after = ctx.get_weights()
        orc = env.oracle(env.d, model=model)
        if writer in ("cw_on", "cw_off"):
            old = (1.0, 1.0) if writer == "cw_on" else CLASS_W
            rows = np.arange(N_STREAM)
            right = SW.eval_weighted(orc, w_after, rows, *ctx.get_class_weights(), logistic=model == "logistic")[0][0]
            stale = SW.eval_weighted(orc, w_after, rows, *old, logistic=model == "logistic")[0][0]
            assert _moved(right, stale), f"{what}: S under the old class weights is the right one"
        elif not np.array_equal(w_after, env.w0):
            witness(env, "w", env.w0, w_after, env.d, env.d, orc_before=orc, orc_after=orc)
        exact = env.kind == "dyadic"
        check_weighted_readers(ctx, env, orc, None, model, exact, exact, what)
    finally:
        if own:
            ctx.close()


@pytest.mark.parametrize("options,writer", SVM_CASES, ids=[f"{o or 'none'}-{w}" for o, w in SVM_CASES])
@pytest.mark.parametrize("dim", DIMS)
@pytest.mark.parametrize("kind", KINDS)
def test_weighted_readers_after_svm_writers(envs, S, kind, dim, options, writer):
    env = envs(kind, dim)
    try:
        run_unweighted_case(_ctx_of(env, "sync"), env, S, options, writer, "svm")
    finally:
        _clear(env.ctx("sync"), env)


@pytest.mark.parametrize("options,writer", LOGISTIC_CASES, ids=[f"{o}-{w}" for o, w in LOGISTIC_CASES])
@pytest.mark.parametrize("dim", DIMS)
def test_weighted_readers_after_logistic_writers(envs, S, dim, options, writer):
    env = envs("fp32", dim)
    try:
        run_unweighted_case(_ctx_of(env, "logistic"), env, S, options, writer, "logistic")
    finally:
        _clear(env.ctx("logistic"), env)


# ---- the persistent kernel's hinge codes across launches ---------------------------------------------------------------------

HINGE_LR = 2.0 ** -4


def hinge_code_calls(sm_count):
    """(grid limit, batch, rates) of every call: grid limits 2 -> 0 -> 7 -> 1, step counts 3 -> 40 -> 2 -> 17 and batches 1,
    G, 32 G and 32 G + 1 alternating, then one call with a rate table that includes 0."""
    calls = []
    for r, grid in enumerate((2, 0, 7, 1)):
        G = grid or sm_count
        for k, batch in enumerate(np.roll([1, G, 32 * G, 32 * G + 1], -r)):
            calls.append((grid, int(batch), np.full((3, 40, 2, 17)[(r + k) % 4], HINGE_LR)))
    calls.append((0, 32 * sm_count, np.array([HINGE_LR, 0.0, HINGE_LR / 2, 0.0, HINGE_LR])))
    return calls


def test_hinge_codes_across_launches(envs):
    """One sample-weighted context with class weights (2, 1/2), lambda = 0 and dyadic rows (every loss exact), run through
    calls whose grid size, step count and batch differ from the call before, with no set_weights in between: every call's
    losses and weights bit for bit those of oracle/sw.sync_steps.  The persistent kernel's hinge-code words t G + b of one
    launch are where the next launch, at another S or G, would find stale codes."""
    from distributed_sgd_b200.native import NativeCtx
    from oracle.oracle import Oracle
    env = envs("dyadic", 700)
    dt = env.data
    orc = Oracle(dt.row_ptr, dt.col, dt.val, dt.label, env.dim, 0.0)
    orc.set_dim_sparsity(env.d)
    sw = sample_weights(env, 0)
    rng = np.random.default_rng(19)
    with NativeCtx(0, env.dim, 0.0) as ctx:
        ctx.load_csr(dt.row_ptr, dt.col, dt.val, dt.label)
        ctx.set_dim_sparsity(env.d)
        ctx.set_class_weights(*CLASS_W)
        ctx.set_sample_weights(sw)
        w = env.w0
        ctx.set_weights(w)
        sm_count = int(ctx.info()["sm_count"])
        for grid, batch, lrs in hinge_code_calls(sm_count):
            what = f"grid limit {grid}, batch {batch}, {lrs.size} steps"
            ctx.set_grid_limit(grid)
            idx = rng.integers(0, N_ROWS, size=batch * lrs.size).astype(np.int32)
            n0 = ctx.launch_count()
            if np.all(lrs == HINGE_LR):
                losses = ctx.sync_steps(idx, batch, lrs.size, HINGE_LR)
            else:
                losses = ctx.sync_steps_lr(idx, batch, lrs)
            persistent = batch <= 32 * (grid or sm_count)
            assert (ctx.launch_count() - n0 == 2) == persistent, f"{what}: not the expected path"
            w, l_ref = SW.sync_steps(orc, w, idx, [batch], lrs, sw, *CLASS_W)
            on_grid(w, what)
            got = ctx.get_weights()
            diff = np.flatnonzero(got != w)
            assert diff.size == 0, f"{what}: {diff.size} weights differ from the checker's, first column {diff[0]}"
            bad = np.flatnonzero(losses != l_ref)
            assert bad.size == 0, f"{what}: step {bad[0]}'s loss {losses[bad[0]]!r} against {l_ref[bad[0]]!r}"


# ---- shared scratch buffers ----------------------------------------------------------------------------------------------------

SCRATCH_SIZES = [1, 33, 2048, 100_000, 2048, 33, 1]
SCRATCH_LAM = 1e-4


def _outcome(call, ctx):
    from distributed_sgd_b200.native import DsgdError
    try:
        return call(ctx)
    except DsgdError as e:
        return ("error", type(e).__name__, str(e))


def test_shared_scratch_buffers():
    """The weighted curve (range, sampled and list, with points and words only), eval_curve, eval_metrics, calibrate and
    eval_weighted share their scratch buffers (m_keys, m_alt, m_tmp, m_cnt; the weighted pass's m_val, m_valt and c_pre).
    On one context with sample and class weights they run in a fixed shuffled order at sizes that grow and then shrink;
    every result has the bits of the same call on a fresh context with the same rows and weights, and the weighted curves
    those of the weighted-curve checker over the device's margins."""
    from distributed_sgd_b200.native import NativeCtx, host_lib
    data = curve_rows(3, 110_000)
    n_rows = data.n_rows
    rng = np.random.default_rng(31)
    sw = rng.choice(SW_VALUES, size=n_rows)
    w = rng.integers(-2, 3, size=data.dim) / 4.0
    cvec = OW.weights(data.label, *CLASS_W, sw)
    h = host_lib()

    def fresh():
        c = NativeCtx(0, data.dim, SCRATCH_LAM)
        c.load_csr(data.row_ptr, data.col, data.val, data.label)
        c.set_class_weights(*CLASS_W)
        c.set_sample_weights(sw)
        return c

    order = np.random.default_rng(5)
    shared = fresh()
    try:
        for n in SCRATCH_SIZES:
            b = int(rng.integers(0, n_rows - n + 1))
            ids = rng.integers(0, n_rows, size=n).astype(np.int32)
            key = 0xC0DE + n
            drawn = np.array([h.dsgd_feistel_pos(p, n_rows, key) for p in range(n)], dtype=np.int32)
            readers = {
                "weighted_curve_range": (lambda c: c.eval_weighted_curve(b, b + n, w), np.arange(b, b + n)),
                "weighted_curve_range_words": (lambda c: c.eval_weighted_curve(b, b + n, w, curve=False), None),
                "weighted_curve_sampled": (lambda c: c.eval_sampled_weighted_curve(0, n_rows, key, 0, n, w), drawn),
                "weighted_curve_sampled_words": (lambda c: c.eval_sampled_weighted_curve(0, n_rows, key, 0, n, w, curve=False),
                                                 None),
                "weighted_curve_list": (lambda c: c.eval_samples_weighted_curve(ids, w), ids),
                "weighted_curve_list_words": (lambda c: c.eval_samples_weighted_curve(ids, w, curve=False), None),
                "curve": (lambda c: c.eval_curve(b, b + n, w), None),
                "metrics": (lambda c: c.eval_metrics(b, b + n, w), None),
                "calibrate": (lambda c: c.calibrate(b, b + n, w), None),
                "weighted": (lambda c: c.eval_weighted(b, b + n, w), None),
            }
            for name in order.permutation(sorted(readers)):
                call, rows = readers[name]
                got = _outcome(call, shared)
                other = fresh()
                try:
                    want = _outcome(call, other)
                finally:
                    other.close()
                assert _bits(got) == _bits(want), f"{name} over {n} rows: the shared context against a fresh one"
                if rows is not None:
                    ref = OW.wcurve(shared.margins(rows, w), data.label[rows], cvec[rows])
                    assert _bits((got.words, got.wsums, got.thr, got.tpw, got.fpw)) == \
                        _bits((ref.words, ref.wsums, ref.thr, ref.tpw, ref.fpw)), f"{name} over {n} rows against the checker"
    finally:
        shared.close()


# ---- async contexts ----------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("writer", ASYNC_WRITERS)
@pytest.mark.parametrize("dim", DIMS)
@pytest.mark.parametrize("kind", KINDS)
def test_async_weighted_evaluation(envs, kind, dim, writer):
    """After the async writers of test_gpu_resident_state.py, eval_weighted in its three forms at w == NULL reads a snapshot
    of the replica as it is when the call starts (c_i = 1: an async context has no class or sample weights): the bits of
    the explicit replica weights, and the checker's sums (||w||^2 exactly on dyadic weights)."""
    env = envs(kind, dim)
    what = f"async, {kind}, dim {dim}, {writer}"
    peers = []
    try:
        ctx, w_before = async_write(env, writer, peers)
        w = ctx.get_weights()
        orc = env.oracle(env.d)
        witness(env, "w", w_before, w, env.d, env.d, orc_after=orc)
        n2 = math.fsum(w * w)
        for name, call, ids in (
                ("range", lambda x: ctx.eval_weighted(0, N_STREAM, x), np.arange(N_STREAM)),
                ("rows", lambda x: ctx.eval_weighted(N_STREAM, N_STREAM + N_SMALL, x), np.arange(N_STREAM, N_STREAM + N_SMALL)),
                ("sampled", lambda x: ctx.eval_sampled_weighted(0, N_ROWS, KEY, 0, 2500, x), env.sampled[:2500]),
                ("list", lambda x: ctx.eval_samples_weighted(env.ids["samples"], x), env.ids["samples"])):
            res, exp = call(None), call(w)
            assert _bits(res) == _bits(exp), f"{what}: eval_weighted ({name}) at w == NULL {res} against {exp}"
            sums, counts = SW.eval_weighted(orc, w, ids)
            assert [exp.n, exp.correct] == list(counts) and [exp.loss_sum, exp.correct_weight, exp.weight_sum] == list(sums), \
                f"{what}: eval_weighted ({name}) {exp} against the checker's {tuple(sums)}, {tuple(counts)}"
            assert exp.norm_squared == n2 if kind == "dyadic" else abs(exp.norm_squared - n2) <= 1e-12 * n2
    finally:
        if writer == "loop_ended":
            env.ctx("async").stop_async()
        for p in peers:
            p.close()
