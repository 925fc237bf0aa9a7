"""Every fp64 row dot on the device is the row fold (dsgd_kernels.cuh, row_fold), so a row's margin, prediction and gate do
not depend on which kernel takes it, on the request size, on the grid or on the other rows of a sync step.

The rows (tests/row_fold_model.py) are built so that other summation orders give other signs: row A and short rows whose
16-byte-unit fold differs from the row fold, and rows of 256 to 960 pairs whose whole-window lane fold differs from it;
interleaved with ordinary rows (dyadic x, non-dyadic weights) and empty rows, labels of both signs.  The reference is the
numpy model of the row fold; at lambda = 0 with dyadic x every gradient sum is exact, so every check is exact equality:
margins bit for bit, predictions, counters and metric words, gradients, sync trajectories on every path and grid, and
Hogwild replays."""
import numpy as np
import pytest

import row_fold_model as M
from helpers import data_from_csr, fused_ranks

pytestmark = pytest.mark.gpu

STREAM_MIN = 2048          # kStreamMinRows: SVM requests of this many rows take the streaming pass
LR = 2.0 ** -4


@pytest.fixture(scope="module")
def S():
    from distributed_sgd_b200.native import NativeCtx
    with NativeCtx(0, 16, 0.0) as c:
        return int(c.info()["sm_count"])


@pytest.fixture(scope="module")
def setup(S):
    d = M.build_rows(11, n_ordinary=32 * S + 200, ord_nnz=(1, 120))
    rp, col, val = M.to_csr(d["rows"])
    data = data_from_csr(rp, col, val, d["labels"], d["dim"])
    model = M.Model(rp, col, val, d["labels"], d["dim"])
    kind = d["kind"]
    adv = np.flatnonzero(np.isin(kind, ["row_a", "short", "long"])).astype(np.int32)
    return dict(data=data, model=model, w=d["w"], kind=kind, adv=adv, long=np.flatnonzero(kind == "long").astype(np.int32))


def _ctx(data, logistic=False, is_async=False):
    """A context at lambda = 0 with the rows loaded; dimSparsity only enters c = 2 lambda (w . d), so zeros do."""
    from distributed_sgd_b200.native import NativeCtx
    ctx = NativeCtx(0, data.dim, 0.0, logistic=logistic, is_async=is_async)
    ctx.load_csr(data.row_ptr, data.col, data.val, data.label)
    ctx.set_dim_sparsity(np.zeros(data.dim))
    return ctx


@pytest.fixture(scope="module")
def svm(setup):
    ctx = _ctx(setup["data"])
    yield ctx
    ctx.close()


def _ids(setup, n, seed):
    """n row ids, shuffled, with repeats: every adversarial row (as far as n allows), then random rows of every kind."""
    rng = np.random.default_rng(seed)
    adv = rng.permutation(setup["adv"])[:n]
    rest = rng.integers(0, setup["data"].n_rows, size=n - adv.size)
    return rng.permutation(np.concatenate([adv, rest])).astype(np.int32)


def _bits(a):
    return np.ascontiguousarray(a, np.float64).view(np.int64)


SIZES = [1, 31, STREAM_MIN - 1, STREAM_MIN, "all"]


def _n(setup, n):
    return setup["data"].n_rows if n == "all" else n


# ---- 1. margins and probabilities -----------------------------------------------------------------------------------

@pytest.mark.parametrize("n", SIZES)
def test_margins_are_the_row_fold_bit_for_bit(setup, svm, n):
    n = _n(setup, n)
    ids = _ids(setup, n, 1) if n > 1 else setup["long"][:1]
    got = svm.margins(ids, setup["w"])
    ref = setup["model"].margins(setup["w"], ids)
    bad = np.flatnonzero(_bits(got) != _bits(ref))
    assert bad.size == 0, f"{bad.size} of {n} margins differ; first rows {ids[bad[:5]]}: {got[bad[:5]]} vs {ref[bad[:5]]}"


def test_probabilities_follow_the_row_fold(setup):
    ctx = _ctx(setup["data"], logistic=True)
    try:
        ids = _ids(setup, setup["data"].n_rows, 2)
        got = ctx.probabilities(ids, setup["w"])
    finally:
        ctx.close()
    t = -setup["model"].margins(setup["w"], ids)
    with np.errstate(over="ignore"):
        e = np.exp(np.where(t >= 0, -t, t))
        ref = np.where(t >= 0, 1.0 / (1.0 + e), e / (1.0 + e))
    assert (np.abs(got - ref) <= 2 * np.spacing(ref)).all()


# ---- 2. predictions -----------------------------------------------------------------------------------------------

@pytest.mark.parametrize("n", [STREAM_MIN - 1, STREAM_MIN, STREAM_MIN + 1, "all"])
def test_forward_is_minus_signum_of_the_row_fold(setup, svm, n):
    n = _n(setup, n)
    ids = _ids(setup, n, 3)
    before = svm.stream_exact_rows()
    got = svm.forward(ids, setup["w"])
    recomputed = svm.stream_exact_rows() - before
    ref = M.pred(setup["model"].margins(setup["w"], ids))
    bad = np.flatnonzero(got != ref)
    assert bad.size == 0, f"{bad.size} of {n} predictions differ; rows {ids[bad[:8]]} kinds {setup['kind'][ids[bad[:8]]]}"
    n_adv = int(np.isin(ids, setup["adv"]).sum())
    if n >= STREAM_MIN:
        assert recomputed >= n_adv > 0     # the streaming pass decided the adversarial rows in fp64
    else:
        assert recomputed == 0


# ---- 3 and 4. evaluations, metric words and curves ------------------------------------------------------------------

def _host_ids(row_begin, row_end, key, lo, hi):
    from distributed_sgd_b200.native import host_lib
    h, n = host_lib(), row_end - row_begin
    pos = np.fromiter((h.dsgd_feistel_pos(p, n, key) for p in range(lo, hi)), dtype=np.int64, count=hi - lo)
    return (row_begin + pos).astype(np.int32)


def _forms(setup):
    """(name, row ids, counts call, metrics call, curve call) for ranges, device-drawn samples and id lists on both sides
    of the streaming threshold."""
    N = setup["data"].n_rows
    key = 0x5EED
    out = []
    for b, e in [(0, STREAM_MIN - 1), (0, STREAM_MIN), (7, N)]:
        out.append((f"range [{b}, {e})", np.arange(b, e, dtype=np.int32),
                    lambda c, w, b=b, e=e: c.eval_counts(b, e, w), lambda c, w, b=b, e=e: c.eval_metrics(b, e, w), None))
    for lo, hi in [(0, STREAM_MIN - 1), (5, STREAM_MIN + 5)]:
        out.append((f"sampled [{lo}, {hi})", _host_ids(0, N, key, lo, hi),
                    lambda c, w, lo=lo, hi=hi: c.eval_sampled_counts(0, N, key, lo, hi, w),
                    lambda c, w, lo=lo, hi=hi: c.eval_sampled_metrics(0, N, key, lo, hi, w), None))
    for n in [31, STREAM_MIN - 1, STREAM_MIN, N + 100]:
        ids = _ids(setup, n, 10 + n)
        out.append((f"list of {n}", ids, lambda c, w, ids=ids: c.eval_samples_counts(ids, w),
                    lambda c, w, ids=ids: c.eval_samples_metrics(ids, w), lambda c, w, ids=ids: c.eval_samples_curve(ids, w)))
    return out


def test_evaluations_count_the_row_folds_decisions(setup, svm):
    """hinge and correct of every dsgd_eval_* form; dsgd_eval_sums and dsgd_eval on the same ranges."""
    w, model = setup["w"], setup["model"]
    fails = []
    for name, ids, counts, _, _ in _forms(setup):
        h, c, _ = counts(svm, w)
        ref = model.counts(w, ids)
        if (h, c) != ref:
            fails.append(f"{name}: (hinge, correct) {(h, c)} vs {ref}")
        if name.startswith("range"):
            b, e = int(ids[0]), int(ids[-1]) + 1
            ls, cs, _ = svm.eval_sums(b, e, w)
            loss, acc = svm.eval(b, e, w)
            if (ls, cs, loss, acc) != (float(ref[0]), ref[1], ref[0] / (e - b), ref[1] / (e - b)):
                fails.append(f"{name}: eval_sums / eval {(ls, cs, loss, acc)} vs counts {ref}")
    assert not fails, "\n".join(fails)


def test_metric_words_agree_with_the_evaluations(setup, svm):
    """TP + TN is the correct count of the matching dsgd_eval_* call, words 2 + 5 count the rows whose dot is 0, all
    eight words are the checker's on the model's margins, and curve thresholds are the distinct -(x . w), highest first."""
    from oracle import metrics as metrics_oracle
    from oracle.oracle import Oracle
    data, w, model = setup["data"], setup["w"], setup["model"]
    orc = Oracle(data.row_ptr, data.col, data.val, data.label, data.dim, 0.0)
    fails = []
    for name, ids, counts, metrics, curve in _forms(setup):
        m = model.margins(w, ids)
        words = metrics(svm, w)
        _, correct, _ = counts(svm, w)
        ref = metrics_oracle.metrics(orc, w, idx=ids, margins=m)
        if not np.array_equal(words, ref):
            fails.append(f"{name}: words {words.tolist()} vs {ref.tolist()}")
        if words[0] + words[4] != correct:
            fails.append(f"{name}: TP + TN = {words[0] + words[4]}, correct = {correct}")
        if words[2] + words[5] != int(np.sum(m == 0.0)):
            fails.append(f"{name}: no-prediction words {words[2] + words[5]}, rows with dot 0: {int(np.sum(m == 0.0))}")
        if curve is not None:
            cw, _, thr, _, _ = curve(svm, w)
            want = np.unique(-m)[::-1]
            if not np.array_equal(cw, words) or not np.array_equal(thr, want):
                fails.append(f"{name}: curve words or thresholds differ ({thr.size} vs {want.size} points)")
    assert not fails, "\n".join(fails)


# ---- 5. gradients ---------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("n", [STREAM_MIN - 1, STREAM_MIN, "all"])
def test_gradient_is_the_row_fold_gated_sum(setup, svm, n):
    n = _n(setup, n)
    ids = _ids(setup, n, 20)
    got = svm.gradient(ids, setup["w"])
    ref, _ = setup["model"].raw_gradient(setup["w"], ids)
    assert np.array_equal(got != 0, ref != 0), "supports differ"
    assert np.array_equal(_bits(got), _bits(ref))


# ---- 6. sync steps --------------------------------------------------------------------------------------------------

def _chunk_layout(lengths, G):
    """Per position of a step: listed in its CTA's chunk list (the producer's prefix rule, k_sync_persistent)."""
    pairs = 2 * ((np.asarray(lengths) + 1) // 2)
    chunks = (pairs + 127) // 128
    listed = np.zeros(len(lengths), bool)
    for b in range(G):
        pos = np.arange(b, len(lengths), G)
        listed[pos] = np.cumsum(chunks[pos]) <= 128
    return listed


def _long_steps(setup, n_steps, seed):
    """32 long rows per step, longest groups first: at one CTA the last rows miss the chunk list, at two they are listed."""
    data, rng = setup["data"], np.random.default_rng(seed)
    long = setup["long"]
    lens = (data.row_ptr[long + 1] - data.row_ptr[long]).astype(np.int64)
    steps = []
    for _ in range(n_steps):
        order = np.concatenate([rng.permutation(long[lens == n]) for n in sorted(set(lens.tolist()), reverse=True)])
        steps.append(order[:32])
    steps = np.asarray(steps, np.int32)
    L = data.row_ptr[steps[0] + 1] - data.row_ptr[steps[0]]
    assert not _chunk_layout(L, 1).all() and _chunk_layout(L, 2).all()
    return steps


def _mixed_steps(setup, n_steps, batch, seed):
    rng = np.random.default_rng(seed)
    return np.stack([_ids(setup, batch, int(rng.integers(1 << 30))) for _ in range(n_steps)]).astype(np.int32)


def _one_ctx_run(setup, steps, grid_limit=None, workers=None):
    from helpers import make_pair
    ctx, _ = make_pair(setup["data"], 0.0)
    try:
        if grid_limit is not None:
            ctx.set_grid_limit(grid_limit)
        if workers is not None:
            ctx.set_workers(workers, k_total=len(workers))
        ctx.set_weights(setup["w"])
        losses = ctx.sync_steps(steps.reshape(-1), steps.shape[1], steps.shape[0], LR)
        return ctx.get_weights(), losses
    finally:
        ctx.close()


def _same(got, ref, what):
    w, l = got
    w_ref, l_ref = ref
    assert np.array_equal(_bits(l), _bits(l_ref)), f"{what}: losses {l} vs {l_ref}"
    bad = np.flatnonzero(_bits(w) != _bits(w_ref))
    assert bad.size == 0, f"{what}: {bad.size} weights differ, first columns {bad[:8]}"


@pytest.mark.parametrize("batch_kind", ["long", "mixed"])
def test_persistent_step_is_the_same_at_every_grid(setup, S, batch_kind):
    steps = _long_steps(setup, 3, 30) if batch_kind == "long" else _mixed_steps(setup, 3, 32, 31)
    ref = setup["model"].sync_steps(setup["w"], steps, [32], LR, 3)
    assert np.count_nonzero(ref[0] != setup["w"]) > 0
    for limit in (1, 2, S):
        _same(_one_ctx_run(setup, steps, grid_limit=limit), ref, f"{batch_kind} rows at grid limit {limit}")


def test_per_step_path_follows_the_row_fold(setup, S):
    b = 32 * S + 1
    steps = _mixed_steps(setup, 2, b, 40)
    steps[:, :32] = _long_steps(setup, 2, 41)
    ref = setup["model"].sync_steps(setup["w"], steps, [b], LR, 2)
    _same(_one_ctx_run(setup, steps), ref, f"per-step path, batch {b}")


def test_two_workers_and_two_fused_ranks_follow_the_row_fold(setup, S):
    steps = np.concatenate([_long_steps(setup, 2, 50), _mixed_steps(setup, 2, 32, 51)])
    ref = setup["model"].sync_steps(setup["w"], steps, [16, 16], LR, steps.shape[0])
    _same(_one_ctx_run(setup, steps, workers=[16, 16]), ref, "set_workers(2)")
    per_rank = [np.ascontiguousarray(steps[:, :16]), np.ascontiguousarray(steps[:, 16:])]
    res = fused_ranks(setup["data"], 0.0, None, [S // 2, S // 2], setup["w"], [(per_rank, None)], LR)
    _same((res["w"][0], res["losses"][0]), ref, f"two fused ranks at {S // 2} CTAs each")


# ---- 7. Hogwild replay ------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("batch", [1, 4])
def test_async_replay_of_long_rows_follows_the_row_fold(setup, batch):
    rng = np.random.default_rng(60 + batch)
    pool = np.concatenate([setup["long"], setup["adv"]])
    idx = np.concatenate([rng.permutation(pool) for _ in range(2)]).astype(np.int32)
    idx = idx[: idx.size // batch * batch]
    ctx = _ctx(setup["data"], is_async=True)
    try:
        ctx.async_replay(setup["w"], idx, batch, 0.125)
        w = ctx.get_weights()
    finally:
        ctx.close()
    ref = setup["model"].async_run(setup["w"], idx, batch, 0.125)
    assert np.count_nonzero(ref != setup["w"]) > 0
    bad = np.flatnonzero(_bits(w) != _bits(ref))
    assert bad.size == 0, f"batch {batch}: {bad.size} weights differ, first columns {bad[:8]}"
