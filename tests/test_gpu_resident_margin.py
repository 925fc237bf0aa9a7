"""Every resident-weight read (w == NULL) after every writer of a SparseSquaredHinge or SparseModifiedHuber context.

Writers: set_weights, sync_steps, sync_step, two virtual workers, staged steps, averaging, a rate table, L1 on, class weights
on and off, sample weights on, changed and off, set_dim_sparsity and a reload.  Readers: those of
tests/test_gpu_resident_state.py in their *_sums forms (the *_counts calls refuse these models), eval_class, eval_weighted,
eval_metrics, eval_curve and, for modified Huber, probabilities.

Checks, as in the other resident modules:
  * every reader at w == NULL gives the same reader's values at the explicit resident weights: bit for bit on dyadic
    rows, within the fp32 tolerances on fp32 rows (the fp64 REDs of a gradient and ||w||^2 after a step add in another
    order there);
  * the explicit reads match the margin checker (oracle/margin.py): bit for bit on dyadic rows, within the fp32 tolerances
    of tests/test_gpu_resident_state.py on fp32 rows, gradient entries scaled by the rows' |s_i c_i| (these scales exceed 1);
  * one more step from the resident state matches the same step after set_weights re-derives the state, and the checker's;
  * first, on the checker, a reader still using the state before the writer would read other values.
The steps of the scale 2 t make the weights' bits longer with every step, so the writers that step run on fp32 rows only;
the dyadic cases are the writers that change the weights, dimSparsity, rows or weighting without a step, where every sum
of the readers is exact in any order."""
import math

import numpy as np
import pytest

from test_gpu_resident_state import (BATCH, DIMS, N_ROWS, N_SMALL, N_STREAM, _moved, _one_worker, _reset, _steps,  # noqa: F401
                                     compare, envs, oracle_all, read_all, witness)
from test_oracle_sample_weight import dyadic_weights

pytestmark = pytest.mark.gpu

MODELS = ("squared_hinge", "modified_huber")
STEPPING = ["sync_steps", "sync_step", "two_workers", "staged", "averaging", "rate_table", "l1"]
STILL = ["set_weights", "class_on", "class_off", "sample_on", "sample_changed", "sample_off", "set_dim_sparsity", "reload"]
CASES = [(w, "fp32") for w in STEPPING] + [(w, k) for w in STILL for k in ("dyadic", "fp32")]
CLASS_W = (2.0, 0.5)


def _sw(env, k):
    return dyadic_weights(np.random.default_rng(env.dim + k), N_ROWS)


def _dots(data, w, ids):
    lo, hi = data.row_ptr[ids], data.row_ptr[ids + 1]
    return np.array([float(np.dot(data.val[a:b].astype(np.float64), w[data.col[a:b]])) for a, b in zip(lo, hi)])


def read_extra(ctx, env, w, model):
    ce = ctx.eval_class(0, N_STREAM, w)
    we = ctx.eval_weighted(N_STREAM, N_STREAM + N_SMALL, w)
    out = {"class": {"loss_pos": ce.loss_pos, "loss_neg": ce.loss_neg, "correct_pos": ce.correct_pos,
                     "correct_neg": ce.correct_neg},
           "weighted": {"loss_sum": we.loss_sum, "correct_weight": we.correct_weight, "weight_sum": we.weight_sum},
           "metrics": {"words": np.asarray(ctx.eval_metrics(0, N_STREAM, w), dtype=np.float64)}}
    words, ap, thr, tp, fp = ctx.eval_curve(N_STREAM, N_STREAM + N_SMALL, w)
    out["curve"] = {"words": words.astype(np.float64), "ap": ap, "thr": thr, "tp": tp.astype(np.float64),
                    "fp": fp.astype(np.float64)}
    if model == "modified_huber":
        out["probs"] = {"p": ctx.probabilities(env.ids["fwd_rows"], w)}
    return out


def oracle_extra(orc, env, w, model, data):
    from oracle import margin as M
    sums, counts = M.eval_class(orc.base, model, w, np.arange(N_STREAM))
    ids = np.arange(N_STREAM, N_STREAM + N_SMALL)
    wsums, _ = M.eval_weighted(orc.base, model, w, ids, orc.w_pos, orc.w_neg, orc.sw)
    out = {"class": {"loss_pos": sums[0], "loss_neg": sums[1], "correct_pos": int(counts[0]), "correct_neg": int(counts[1])},
           "weighted": {"loss_sum": wsums[0], "correct_weight": wsums[1], "weight_sum": wsums[2]}}
    if model == "modified_huber":
        out["probs"] = {"p": (np.clip(-_dots(data, w, env.ids["fwd_rows"]), -1.0, 1.0) + 1.0) / 2.0}
    return out


def _grad_scale(env, orc, model, data, w, idx, c):
    """Per column: the sum over the rows idx of |x_ij s_i c_i|, + |c| (the scale of a gradient entry's rounding)"""
    from oracle import margin as M
    y = data.label[idx].astype(np.float64)
    s = np.array([M.row(model, float(v))[1] for v in y * _dots(data, w, idx)])
    cw = np.where(y > 0, orc.w_pos, orc.w_neg) * (orc.sw[idx] if orc.sw is not None else 1.0)
    lo, hi = data.row_ptr[idx], data.row_ptr[idx + 1]
    pos = np.concatenate([np.arange(a, b) for a, b in zip(lo, hi)])
    sc = np.repeat(np.abs(s * cw), hi - lo)
    return np.bincount(data.col[pos], weights=np.abs(data.val[pos].astype(np.float64)) * sc, minlength=env.dim) + abs(c)


def _scales(env, orc, model, data, w, c):
    out = {name: _grad_scale(env, orc, model, data, w, env.ids[name], c) for name in ("grad_stream", "grad_rows")}
    out["probs"] = np.ones(len(env.ids["fwd_rows"]))
    return out


def check_readers(ctx, env, orc, model, exact, what, data):
    w = ctx.get_weights()
    res = read_all(ctx, env, None, model)
    res.update(read_extra(ctx, env, None, model))
    exp = read_all(ctx, env, w, model)
    exp.update(read_extra(ctx, env, w, model))
    want, c = oracle_all(orc, env, w, model)
    want.update(oracle_extra(orc, env, w, model, data))
    scales = _scales(env, orc, model, data, w, c)
    # the scores are the row fold of the same weights on either path: the ranking words and curves keep their bits
    ranking = ("metrics", "curve")
    compare({k: res[k] for k in ranking}, {k: exp[k] for k in ranking}, True,
            f"{what}, w == NULL against the explicit weights", scales)
    compare({k: v for k, v in res.items() if k not in ranking}, {k: v for k, v in exp.items() if k not in ranking}, exact,
            f"{what}, w == NULL against the explicit weights", scales)
    compare(exp, want, exact, f"{what}, explicit weights against the checker", scales)
    return w, scales


def check_next_step(ctx, env, orc, w, exact, what, data):
    _one_worker(ctx)
    ids = env.ids["step"]
    loss = ctx.sync_steps(ids, BATCH, 1, env.lr)[0]
    w1 = ctx.get_weights()
    ctx.set_weights(w)
    loss_twin = ctx.sync_steps(ids, BATCH, 1, env.lr)[0]
    w1_twin = ctx.get_weights()
    w_ref, loss_ref = orc.sync_steps(w, ids, [BATCH], env.lr)
    if exact:
        assert loss == loss_twin == loss_ref[0], f"{what}, next step's loss: {loss!r} / {loss_twin!r} / {loss_ref[0]!r}"
        for a, name in ((w1, "resident"), (w1_twin, "re-set")):
            diff = np.flatnonzero(a != w_ref)
            assert diff.size == 0, f"{what}, next step from the {name} state, column {diff[0]}: {a[diff[0]]!r} against " \
                                   f"{w_ref[diff[0]]!r}"
        return
    assert abs(loss - loss_twin) <= 1e-12 * abs(loss_twin), f"{what}, next step's loss {loss!r} against {loss_twin!r}"
    np.testing.assert_allclose(loss_twin, loss_ref[0], rtol=1e-12, err_msg=f"{what}: next step's loss against the checker")
    tol = 1e-12 * (np.abs(w1_twin) + env.lr * _grad_scale(env, orc, orc.model, data, w, ids, 0.0) + 1e-300)
    for a, b, tag in ((w1, w1_twin, "resident against re-set"), (w1_twin, w_ref, "re-set against the checker")):
        assert np.array_equal(a != 0, b != 0), f"{what}, next step: supports differ ({tag})"
        bad = np.flatnonzero(np.abs(a - b) > tol)
        assert bad.size == 0, f"{what}, next step, {tag}, column {bad[0]}: {a[bad[0]]!r} against {b[bad[0]]!r}"


def _weighting(env, writer):
    """(weighting before the writer, after it): each (w_pos, w_neg, sw)"""
    none = (1.0, 1.0, None)
    return {"class_on": (none, (*CLASS_W, None)), "class_off": ((*CLASS_W, None), none),
            "sample_on": (none, (1.0, 1.0, _sw(env, 1))), "sample_changed": ((1.0, 1.0, _sw(env, 1)), (1.0, 1.0, _sw(env, 2))),
            "sample_off": ((1.0, 1.0, _sw(env, 1)), none)}.get(writer, (none, none))


def _install(ctx, weighting):
    w_pos, w_neg, sw = weighting
    ctx.set_class_weights(w_pos, w_neg)
    ctx.set_sample_weights(sw)


@pytest.mark.parametrize("writer,kind", CASES)
@pytest.mark.parametrize("model", MODELS)
def test_resident_reads_after_margin_writer(envs, model, writer, kind):
    from distributed_sgd_b200.native import NativeCtx
    env = envs(kind, DIMS[0])
    what = f"{model}, {kind}, dim {env.dim}, {writer}"
    rng = np.random.default_rng(len(writer) * 1000 + len(model))
    before, after = _weighting(env, writer)
    lam1 = 1e-3 if writer == "l1" else 0.0
    own = None
    if writer == "reload":
        own = NativeCtx(0, env.dim, env.lam, model=model)
        own.load_csr(env.data.row_ptr, env.data.col, env.data.val, env.data.label)
        ctx = own
    else:
        ctx = env.ctx(model)
    d_after, data = env.d, env.data
    try:
        _one_worker(ctx)
        ctx.average_end()
        ctx.set_l1(0.0)
        _install(ctx, before)
        _reset(ctx, env, env.w0, sync=False)
        if writer == "set_weights":
            ctx.set_weights(env.w1)
        elif writer in ("sync_steps", "averaging", "l1"):
            if writer == "averaging":
                ctx.average_begin()
            ctx.set_l1(lam1)
            ctx.sync_steps(_steps(rng, BATCH, 2), BATCH, 2, env.lr)
            if writer == "averaging":
                ctx.average_end()
        elif writer == "sync_step":
            for _ in range(2):
                ctx.sync_step(_steps(rng, BATCH, 1), env.lr)
        elif writer == "two_workers":
            ctx.set_workers([40, 24], 2)
            ctx.sync_steps(_steps(rng, BATCH, 2), BATCH, 2, env.lr)
        elif writer == "staged":
            ctx.stage_samples(_steps(rng, BATCH, 5))
            ctx.sync_steps_staged(BATCH, BATCH, 3, env.lr)
        elif writer == "rate_table":
            ctx.sync_steps_lr(_steps(rng, BATCH, 3), BATCH, env.lr * np.array([1.0, 0.5, 0.25]))
        elif writer == "set_dim_sparsity":
            ctx.set_dim_sparsity(env.d2)
            d_after = env.d2
        elif writer == "reload":
            ctx.load_csr(env.data2.row_ptr, env.data2.col, env.data2.val, env.data2.label)
            data = env.data2
        elif writer in ("class_on", "class_off", "sample_on", "sample_changed", "sample_off"):
            _install(ctx, after)
        w_after = ctx.get_weights()
        orc = env.oracle(d_after, model=model, data=data, w_pos=after[0], w_neg=after[1], sw=after[2], lambda1=lam1)
        # the witness: a reader or step still using the state before the writer would give other values
        if writer == "reload":
            witness(env, "rows", env.w0, w_after, env.d, d_after, orc_after=env.oracle(d_after, data=data))
        elif writer == "set_dim_sparsity":
            witness(env, "d", env.w0, w_after, env.d, d_after)
        elif writer in STEPPING or writer == "set_weights":
            witness(env, "w", env.w0, w_after, env.d, d_after)
        else:
            stale = env.oracle(d_after, model=model, data=data, w_pos=before[0], w_neg=before[1], sw=before[2])
            ids = env.ids["grad_rows"]
            assert _moved(stale.gradient_loss(w_after, ids), orc.gradient_loss(w_after, ids)), "the weighting changes no loss"
        if writer == "l1":
            stale = env.oracle(d_after, model=model, data=data)
            ids = env.ids["step"]
            assert _moved(stale.sync_steps(w_after, ids, [BATCH], env.lr)[1][0],
                          orc.sync_steps(w_after, ids, [BATCH], env.lr)[1][0]), "L1 changes no step loss"
        exact = kind == "dyadic"
        w, _ = check_readers(ctx, env, orc, model, exact, what, data)
        check_next_step(ctx, env, orc, w, exact, what, data)
    finally:
        ctx.set_l1(0.0)
        _install(ctx, (1.0, 1.0, None))
        if own is not None:
            own.close()
