"""Resident-weight reads (w == NULL) after every call that changes the weights.

A reader given w == NULL uses the resident weights and the state derived from them: c = 2 lambda (w . d), ||w||^2, the fp32
shadow the streaming pass (2048 rows or more) decides signs with, and on an async context the replica's control slot
S = w . d.  After each writer -- set_weights, the dimSparsity calls, every sync-step path, the async writers and a peer's
pushes -- every reader must give with w == NULL what it gives with the weights read back by dsgd_get_weights (whose c,
||w||^2 and shadow k_prepare / k_to_f32 derive afresh), and both must match the fp64 oracle at those weights:

- dyadic rows (values multiples of 1/2, weights of 2^-5, d = 4 on one column, lambda and lr powers of two with
  lr 2 lambda d = 1, so that no step makes the weights finer): bit for bit;
- fp32 RCV1-shaped rows: predictions, correct and hinge counts and gradient supports exact; losses and ||w||^2 rtol 1e-12;
  gradient entries within 1e-12 (sum_i |x_ij| + |c|) and the next step's weights within 1e-12 (|w_j| + lr (sum_i |x_ij| +
  |c|)): c lands on every key of a reply, and the row kernels add a batch's terms in whatever order their atomics land.
  The step kernels sum c and ||w||^2 in another order than k_prepare;
- async contexts: w == NULL and the explicit weights bit for bit on both kinds of data.

Every case first shows, on the oracle, that a reader still using the state from before the writer would fail: at least
1 % of the streaming pass's rows change prediction, and ||w||^2 and c move by more than 1e-6 relative (c alone for the
dimSparsity writers; for a reload, the predictions at the same weights).

Two more tests keep the staged sample stream honest: forward and gradient requests leave it alone, and a reload drops it.
"""
import math
import time

import numpy as np
import pytest

from helpers import data_from_csr, fused_ranks, make_pair

pytestmark = pytest.mark.gpu

N_ROWS = 5000
N_STREAM = 3000          # readers over 2048 rows or more take the streaming pass (k_stream_rows)
N_SMALL = 1000           # ... fewer: k_rows
DIMS = [700, 56000]      # 56 000: past the update threads' registers (2 x 192 x S columns), below the streaming limit
KINDS = ["dyadic", "fp32"]
KEY = 0x5EED5EED
BATCH = 64
DY_VALS = np.array([-2.0, -1.5, -1.0, -0.5, 0.5, 1.0, 1.5, 2.0])


@pytest.fixture(scope="module")
def S():
    from distributed_sgd_b200.native import NativeCtx
    with NativeCtx(0, 16, 0.0) as c:
        return int(c.info()["sm_count"])


# ---- data ----------------------------------------------------------------------------------------------------------------

def _dyadic_rows(dim, seed):
    """6 to 13 columns per row, values multiples of 1/2, and column dim // 3 (the one d weighs) in 8 % of the rows."""
    rng = np.random.default_rng(seed)
    j0 = dim // 3
    rp, cols, vals = [0], [], []
    for _ in range(N_ROWS):
        c = np.unique(rng.integers(0, dim, size=int(rng.integers(6, 14))))
        if rng.random() < 0.08:
            c = np.union1d(c, [j0])
        cols.append(c)
        vals.append(rng.choice(DY_VALS, size=c.size))
        rp.append(rp[-1] + c.size)
    return data_from_csr(rp, np.concatenate(cols), np.concatenate(vals), rng.choice([-1, 1], N_ROWS), dim)


def _fp32_rows(dim, seed):
    from distributed_sgd_b200.utils import synthetic_rcv1
    return synthetic_rcv1(n_rows=N_ROWS, dim=dim, seed=seed, mean_nnz=min(94.5, dim / 8.0), max_nnz=min(2000, dim // 2))


class Env:
    """One data set: rows, other rows of the same count (reloads), two weight vectors, two dimSparsity vectors, lambda, lr,
    the reader's ids, and the contexts on it (made on first use)."""

    def __init__(self, kind, dim):
        from oracle.oracle import Oracle
        self.kind, self.dim = kind, dim
        seed = dim + (0 if kind == "dyadic" else 1)
        rng = np.random.default_rng(seed)
        if kind == "dyadic":
            self.data, self.data2 = _dyadic_rows(dim, seed), _dyadic_rows(dim, seed + 7)
            self.lam, self.lr = 2.0 ** -2, 2.0 ** -1        # lr * 2 lambda d = 1: the weights keep their 2^-5 grid
            self.w0 = rng.integers(-64, 65, size=dim) / 32.0
            self.w1 = rng.integers(-64, 65, size=dim) / 32.0
            self.d = np.zeros(dim)
            self.d[dim // 3] = 4.0
            self.d2 = np.zeros(dim)
            self.d2[2 * dim // 3] = 4.0
        else:
            self.data, self.data2 = _fp32_rows(dim, seed), _fp32_rows(dim, seed + 7)
            self.lam, self.lr = 1e-3, 0.05
            self.w0 = rng.standard_normal(dim) * 0.1
            self.w1 = rng.standard_normal(dim) * 0.1
            self.d = Oracle(self.data.row_ptr, self.data.col, self.data.val, self.data.label, dim, 0.0).dim_sparsity(N_ROWS)
            self.d2 = self.d * 2.0
        self.n_train2 = 4096                                # compute_dim_sparsity's other n_train
        from distributed_sgd_b200.native import host_lib
        h = host_lib()
        self.sampled = np.fromiter((h.dsgd_feistel_pos(p, N_ROWS, KEY) for p in range(2500)), dtype=np.int32, count=2500)
        self.ids = {
            "fwd_stream": rng.choice(N_ROWS, size=N_STREAM, replace=False).astype(np.int32),
            "fwd_rows": rng.choice(N_ROWS, size=500, replace=False).astype(np.int32),
            "grad_stream": rng.choice(N_ROWS, size=2500, replace=False).astype(np.int32),
            "grad_rows": rng.choice(N_ROWS, size=300, replace=False).astype(np.int32),
            "samples": rng.integers(0, N_ROWS, size=700).astype(np.int32),       # repeats count every time
            "step": rng.choice(N_ROWS, size=BATCH, replace=False).astype(np.int32),
        }
        self._ctx = {}

    def oracle(self, d, model="svm", data=None, **weighting):
        """The checker of `model` ("svm", "logistic", "squared_hinge", "modified_huber") with dimSparsity d; a margin
        model's takes the weighting of its steps (oracle.margin.MarginOracle)."""
        from oracle.logistic import LogisticOracle
        from oracle.margin import MarginOracle
        from oracle.oracle import Oracle
        data = self.data if data is None else data
        orc = (LogisticOracle if model == "logistic" else Oracle)(data.row_ptr, data.col, data.val, data.label, self.dim,
                                                                 self.lam)
        orc.set_dim_sparsity(d)
        return orc if model in ("svm", "logistic") else MarginOracle(orc, model, **weighting)

    def ctx(self, which):
        """'sync' (the SVM), 'async' or another model's name: one context per kind, reset by the caller."""
        if which not in self._ctx:
            from distributed_sgd_b200.native import NativeCtx
            c = NativeCtx(0, self.dim, self.lam, is_async=which == "async",
                          model=None if which in ("sync", "async") else which)
            c.load_csr(self.data.row_ptr, self.data.col, self.data.val, self.data.label)
            self._ctx[which] = c
        return self._ctx[which]

    def close(self):
        for c in self._ctx.values():
            c.close()


@pytest.fixture(scope="module")
def envs():
    made = {}

    def get(kind, dim):
        if (kind, dim) not in made:
            made[kind, dim] = Env(kind, dim)
        return made[kind, dim]

    yield get
    for e in made.values():
        e.close()


def _one_worker(ctx):
    """dsgd_set_workers(ctx, 1, NULL, 0): one worker over the whole batch, as after dsgd_create."""
    ctx._ck(ctx._l.dsgd_set_workers(ctx._h, 1, None, 0))


def _reset(ctx, env, w, sync=True):
    if sync:
        ctx.set_grid_limit(0)
        _one_worker(ctx)
        ctx.average_end()
    ctx.set_dim_sparsity(env.d)
    ctx.set_weights(w)


def _steps(rng, batch, steps):
    return np.concatenate([rng.choice(N_ROWS, size=batch, replace=False) for _ in range(steps)]).astype(np.int32)


# ---- the witness: a reader still using the previous state would fail --------------------------------------------------

def _c(lam, w, d):
    return 2.0 * lam * math.fsum(w * d)


def _moved(a, b):
    return abs(a - b) > 1e-6 * max(abs(a), abs(b))


def witness(env, what, w_before, w_after, d_before, d_after, orc_before=None, orc_after=None):
    rows = np.arange(N_STREAM, dtype=np.int32)
    orc_before = orc_before or env.oracle(d_before)
    orc_after = orc_after or env.oracle(d_after)
    if what == "rows":
        flips = np.mean(orc_before.forward(w_after, rows) != orc_after.forward(w_after, rows))
        assert flips >= 0.01, f"the new rows change only {flips:.2%} of the predictions"
        return
    assert _moved(_c(env.lam, w_before, d_before), _c(env.lam, w_after, d_after)), "c does not move"
    if what == "d":
        return
    flips = np.mean(orc_before.forward(w_before, rows) != orc_after.forward(w_after, rows))
    assert flips >= 0.01, f"only {flips:.2%} of the streaming pass's rows change prediction"
    assert _moved(math.fsum(w_before * w_before), math.fsum(w_after * w_after)), "||w||^2 does not move"


# ---- readers -------------------------------------------------------------------------------------------------------------

def read_all(ctx, env, w, model):
    """Every reader once, at the weights w (None: resident).  {reader: {field: value}}.  Every model but the SVM reads the
    *_sums forms (its loss sum is not an integer)."""
    ids = env.ids
    out = {}
    out["eval_stream"] = dict(zip(("loss", "acc"), ctx.eval(0, N_STREAM, w)))
    out["eval_rows"] = dict(zip(("loss", "acc"), ctx.eval(N_STREAM, N_STREAM + N_SMALL, w)))
    if model != "svm":
        fields = ("loss_sum", "correct", "n2")
        out["sums"] = dict(zip(fields, ctx.eval_sums(0, N_STREAM, w)))
        out["sampled_stream"] = dict(zip(fields, ctx.eval_sampled_sums(0, N_ROWS, KEY, 0, 2500, w)))
        out["sampled_rows"] = dict(zip(fields, ctx.eval_sampled_sums(0, N_ROWS, KEY, 100, 1100, w)))
        out["samples"] = dict(zip(fields, ctx.eval_samples_sums(ids["samples"], w)))
    else:
        fields = ("hinge", "correct", "n2")
        out["sums"] = dict(zip(fields, ctx.eval_counts(0, N_STREAM, w)))
        out["sampled_stream"] = dict(zip(fields, ctx.eval_sampled_counts(0, N_ROWS, KEY, 0, 2500, w)))
        out["sampled_rows"] = dict(zip(fields, ctx.eval_sampled_counts(0, N_ROWS, KEY, 100, 1100, w)))
        out["samples"] = dict(zip(fields, ctx.eval_samples_counts(ids["samples"], w)))
    for name in ("fwd_stream", "fwd_rows"):
        out[name] = {"preds": ctx.forward(ids[name], w)}
    for name in ("grad_stream", "grad_rows"):
        g, loss = ctx.gradient(ids[name], w, want_loss=True)
        out[name] = {"grad": g, "loss": loss}
    return out


def oracle_all(orc, env, w, model):
    """What read_all must give at the weights w, and c.  A margin model's gradient loss is that of its weighting."""
    ids = env.ids
    n2 = math.fsum(w * w)
    out = {}

    def sums(idx=None, begin=0, n=None):
        loss, acc = orc.loss_acc(w, idx=idx, begin=begin, n=n)
        k = len(idx) if idx is not None else n
        if model != "svm":
            return {"loss_sum": math.fsum(orc.sample_losses(w, idx=idx, begin=begin, n=n)), "correct": round(acc * k),
                    "n2": n2}
        return {"hinge": round((loss - env.lam * n2) * k), "correct": round(acc * k), "n2": n2}

    for name, (b, n) in (("eval_stream", (0, N_STREAM)), ("eval_rows", (N_STREAM, N_SMALL))):
        out[name] = dict(zip(("loss", "acc"), orc.loss_acc(w, begin=b, n=n)))
    out["sums"] = sums(begin=0, n=N_STREAM)
    out["sampled_stream"] = sums(idx=env.sampled[:2500])
    out["sampled_rows"] = sums(idx=env.sampled[100:1100])
    out["samples"] = sums(idx=ids["samples"])
    for name in ("fwd_stream", "fwd_rows"):
        out[name] = {"preds": orc.forward(w, ids[name])}
    c = None
    for name in ("grad_stream", "grad_rows"):
        g, c = orc.gradient(w, ids[name])
        loss = orc.gradient_loss(w, ids[name]) if model not in ("svm", "logistic") else orc.loss_acc(w, idx=ids[name])[0]
        out[name] = {"grad": g, "loss": loss}
    return out, c


def _grad_scale(env, data, idx, c):
    """sum over the batch of |x_ij| + |c| per column: the scale of a gradient entry's rounding (|sigma|, |y| <= 1)."""
    lo, hi = data.row_ptr[idx], data.row_ptr[idx + 1]
    pos = np.concatenate([np.arange(a, b) for a, b in zip(lo, hi)])
    return np.bincount(data.col[pos], weights=np.abs(data.val[pos].astype(np.float64)), minlength=env.dim) + abs(c)


def compare(got, want, exact, what, scales):
    """got / want as read_all gives them.  exact: every value bit for bit.  Else counts, accuracies, predictions and gradient
    supports exact, losses and ||w||^2 rtol 1e-12, gradient entries within 1e-12 scales[reader]."""
    bad = []
    for reader, fields in want.items():
        for field, v in fields.items():
            g = got[reader][field]
            tag = f"{what}: {reader}.{field}"
            if isinstance(v, np.ndarray):
                if exact or field == "preds":
                    if not np.array_equal(g, v):
                        j = int(np.flatnonzero(g != v)[0])
                        bad.append(f"{tag}[{j}]: {g[j]!r} against {v[j]!r} ({np.count_nonzero(g != v)} entries differ)")
                    continue
                if not np.array_equal(g == 0, v == 0):
                    bad.append(f"{tag}: supports differ in {np.count_nonzero((g == 0) != (v == 0))} columns")
                    continue
                err = np.abs(g - v) > 1e-12 * scales[reader]
                if err.any():
                    j = int(np.flatnonzero(err)[0])
                    bad.append(f"{tag}[{j}]: {g[j]!r} against {v[j]!r}")
            elif exact or field in ("acc", "correct", "hinge"):
                if not g == v:
                    bad.append(f"{tag}: {g!r} against {v!r}")
            elif not abs(g - v) <= 1e-12 * abs(v):
                bad.append(f"{tag}: {g!r} against {v!r} (rtol {abs(g - v) / abs(v):.1e})")
    assert not bad, "\n".join(bad)


def check_readers(ctx, env, orc, model, exact_resident, exact_oracle, what, data=None):
    """Every reader at w == NULL against the explicit weights, and those against the oracle; returns the weights."""
    w = ctx.get_weights()
    resident = read_all(ctx, env, None, model)
    explicit = read_all(ctx, env, w, model)
    want, c = oracle_all(orc, env, w, model)
    data = env.data if data is None else data
    scales = {n: _grad_scale(env, data, env.ids[n], c) for n in ("grad_stream", "grad_rows")}
    compare(resident, explicit, exact_resident, f"{what}, w == NULL against the explicit weights", scales)
    compare(explicit, want, exact_oracle, f"{what}, explicit weights against the oracle", scales)
    return w, c


def check_next_step(ctx, env, orc, w, c, exact, what, data=None):
    """One more sync step from the resident state, against the same step after set_weights(w) re-derives it, and the
    oracle's."""
    _one_worker(ctx)
    ctx.set_grid_limit(0)
    ids = env.ids["step"]
    loss = ctx.sync_steps(ids, BATCH, 1, env.lr)[0]
    w1 = ctx.get_weights()
    ctx.set_weights(w)
    loss_twin = ctx.sync_steps(ids, BATCH, 1, env.lr)[0]
    w1_twin = ctx.get_weights()
    w_ref, loss_ref = orc.sync_steps(w, ids, [BATCH], env.lr, n_steps=1)
    if exact:
        assert loss == loss_twin == loss_ref[0], f"{what}, next step's loss: {loss!r} / {loss_twin!r} / {loss_ref[0]!r}"
        for a, name in ((w1, "resident"), (w1_twin, "re-set")):
            diff = np.flatnonzero(a != w_ref)
            assert diff.size == 0, f"{what}, next step from the {name} state, column {diff[0]}: {a[diff[0]]!r} against " \
                                   f"{w_ref[diff[0]]!r}"
        return
    assert abs(loss - loss_twin) <= 1e-12 * abs(loss_twin), f"{what}, next step's loss {loss!r} against {loss_twin!r}"
    np.testing.assert_allclose(loss_twin, loss_ref[0], rtol=1e-12, err_msg=f"{what}: next step's loss against the oracle")
    tol = 1e-12 * (np.abs(w1_twin) + env.lr * _grad_scale(env, env.data if data is None else data, ids, c))
    assert np.array_equal(w1 != 0, w1_twin != 0), f"{what}: next step's supports differ"
    bad = np.flatnonzero(np.abs(w1 - w1_twin) > tol)
    assert bad.size == 0, f"{what}, next step, column {bad[0]}: {w1[bad[0]]!r} against {w1_twin[bad[0]]!r}"
    assert np.array_equal(w1_twin != 0, w_ref != 0), f"{what}: next step's supports differ from the oracle's"
    np.testing.assert_allclose(w1_twin, w_ref, rtol=1e-11, atol=1e-15, err_msg=f"{what}: next step against the oracle")


# ---- sync SVM ------------------------------------------------------------------------------------------------------------

SYNC_WRITERS = ["set_weights", "persistent", "persistent_grid2", "fallback", "sync_step", "two_workers", "staged",
                "set_dim_sparsity", "compute_dim_sparsity", "avg_persistent", "avg_fallback", "load_csr"]


@pytest.mark.parametrize("writer", SYNC_WRITERS)
@pytest.mark.parametrize("dim", DIMS)
@pytest.mark.parametrize("kind", KINDS)
def test_sync_svm(envs, S, kind, dim, writer):
    env = envs(kind, dim)
    what = f"sync SVM, {kind}, dim {dim}, {writer}"
    rng = np.random.default_rng(len(writer) * 1000 + dim)
    d_after, data = env.d, env.data
    own = None
    if writer == "load_csr":           # a context of its own: the module's keeps its rows
        own, _ = make_pair(env.data, env.lam)
        ctx = own
    else:
        ctx = env.ctx("sync")
    try:
        _reset(ctx, env, env.w0)
        w_before = env.w0
        if writer == "set_weights":
            ctx.set_weights(env.w1)
        elif writer in ("persistent", "avg_persistent", "persistent_grid2"):
            if writer == "avg_persistent":
                ctx.average_begin()
            if writer == "persistent_grid2":
                ctx.set_grid_limit(2)                     # batch 64 = 32 G: still the persistent kernel
            ctx.sync_steps(_steps(rng, BATCH, 2), BATCH, 2, env.lr)
        elif writer in ("fallback", "avg_fallback"):
            if writer == "avg_fallback":
                ctx.average_begin()
            b = 32 * S + 1                                # k_rows + k_update<true>
            ctx.sync_steps(_steps(rng, b, 2), b, 2, env.lr)
        elif writer == "sync_step":
            for _ in range(2):
                ctx.sync_step(_steps(rng, BATCH, 1), env.lr)
        elif writer == "two_workers":
            ctx.set_workers([40, 24], 2)
            ctx.sync_steps(_steps(rng, BATCH, 2), BATCH, 2, env.lr)
        elif writer == "staged":
            ctx.stage_samples(_steps(rng, BATCH, 5))
            ctx.sync_steps_staged(BATCH, BATCH, 3, env.lr)
        elif writer == "set_dim_sparsity":
            ctx.set_dim_sparsity(env.d2)
            d_after = env.d2
        elif writer == "compute_dim_sparsity":
            d_after = ctx.compute_dim_sparsity(env.n_train2)
            assert np.array_equal(d_after, env.oracle(env.d).dim_sparsity(env.n_train2))
        elif writer == "load_csr":
            d2 = env.data2
            ctx.load_csr(d2.row_ptr, d2.col, d2.val, d2.label)
            data = d2
        if writer.startswith("avg_"):
            ctx.average_end()
        w_after = ctx.get_weights()
        orc = env.oracle(d_after, data=data)
        if writer == "load_csr":
            witness(env, "rows", w_before, w_after, env.d, d_after, orc_after=orc)
        else:
            witness(env, "d" if "dim_sparsity" in writer else "w", w_before, w_after, env.d, d_after, orc_after=orc)
        # dyadic rows give exact sums, except with compute_dim_sparsity's d = 1 / (df + 1)
        exact_oracle = kind == "dyadic" and writer != "compute_dim_sparsity"
        w, c = check_readers(ctx, env, orc, "svm", kind == "dyadic", exact_oracle, what, data=data)
        check_next_step(ctx, env, orc, w, c, exact_oracle, what, data=data)
    finally:
        if own is not None:
            own.close()


# ---- logistic ------------------------------------------------------------------------------------------------------------

LOGISTIC_WRITERS = ["set_weights", "sync_steps", "two_workers", "set_dim_sparsity"]


@pytest.mark.parametrize("writer", LOGISTIC_WRITERS)
@pytest.mark.parametrize("dim", DIMS)
def test_logistic(envs, dim, writer):
    """fp32 rows only: the logistic loss of dyadic rows is not dyadic."""
    env = envs("fp32", dim)
    what = f"logistic, dim {dim}, {writer}"
    rng = np.random.default_rng(len(writer) * 1000 + dim + 1)
    ctx = env.ctx("logistic")
    _reset(ctx, env, env.w0)
    d_after = env.d
    if writer == "set_weights":
        ctx.set_weights(env.w1)
    elif writer == "sync_steps":
        ctx.sync_steps(_steps(rng, BATCH, 2), BATCH, 2, env.lr)
    elif writer == "two_workers":
        ctx.set_workers([40, 24], 2)
        ctx.sync_steps(_steps(rng, BATCH, 2), BATCH, 2, env.lr)
    elif writer == "set_dim_sparsity":
        ctx.set_dim_sparsity(env.d2)
        d_after = env.d2
    orc = env.oracle(d_after, model="logistic")
    witness(env, "d" if writer == "set_dim_sparsity" else "w", env.w0, ctx.get_weights(), env.d, d_after,
            orc_before=env.oracle(env.d, model="logistic"), orc_after=orc)
    w, c = check_readers(ctx, env, orc, "logistic", False, False, what)
    check_next_step(ctx, env, orc, w, c, False, what)


# ---- async ---------------------------------------------------------------------------------------------------------------

ASYNC_WRITERS = ["update_grad", "replay_from_replica", "replay_from_w0", "loop_stopped", "loop_ended", "peer_push"]
REPLAY_BATCH, REPLAY_UPDATES, LOOP_UPDATES = 4, 100, 2000


def _wait_for_loop(ctx):
    t0 = time.time()
    while ctx.async_running() and time.time() - t0 < 60:
        time.sleep(0.002)
    assert not ctx.async_running(), "the async loop did not end by itself"


def async_write(env, writer, peers):
    """Runs an async writer on the env's async context (peer_push: on two new ranks, appended to peers); returns the
    context to read and the weights before the writer."""
    from distributed_sgd_b200.native import REPLICA_SELF
    rng = np.random.default_rng(len(writer) * 1000 + env.dim + 2)
    replay = _steps(rng, REPLAY_BATCH, REPLAY_UPDATES)
    ctx = env.ctx("async")
    _reset(ctx, env, env.w0, sync=False)
    w_before = env.w0
    if writer == "update_grad":                      # SlaveImpl.updateGrad: w -= delta, here onto w1
        delta = env.w0 - env.w1
        idx = np.flatnonzero(delta).astype(np.int32)
        ctx.update_grad(idx, delta[idx])
    elif writer == "replay_from_replica":
        ctx.async_replay(None, replay, REPLAY_BATCH, env.lr)
    elif writer == "replay_from_w0":
        ctx.set_weights(env.w1)
        w_before = env.w1
        ctx.async_replay(env.w0, replay, REPLAY_BATCH, env.lr)
    elif writer in ("loop_stopped", "loop_ended"):
        ctx.start_async(None, np.arange(N_ROWS, dtype=np.int32), batch=1, lr=env.lr, concurrency=1,
                        max_updates=LOOP_UPDATES, seed=env.dim)
        _wait_for_loop(ctx)
        if writer == "loop_stopped":
            ctx.stop_async()
    elif writer == "peer_push":                      # rank 0's replay pushes every delta into rank 1's replica
        for r in range(2):
            p, _ = make_pair(env.data, env.lam, rank=r, world=2, is_async=True)
            p.set_dim_sparsity(env.d)
            p.set_weights(env.w0)
            peers.append(p)
        peers[0].peer_attach(1, peers[1], REPLICA_SELF)
        peers[0].async_replay(None, replay, REPLAY_BATCH, env.lr)
        ctx = peers[1]
    return ctx, w_before


@pytest.mark.parametrize("writer", ASYNC_WRITERS)
@pytest.mark.parametrize("dim", DIMS)
@pytest.mark.parametrize("kind", KINDS)
def test_async(envs, kind, dim, writer):
    """Readers between writers, with no loop running; w == NULL reads the replica as it is when the call starts."""
    env = envs(kind, dim)
    what = f"async, {kind}, dim {dim}, {writer}"
    peers = []
    try:
        ctx, w_before = async_write(env, writer, peers)
        w_after = ctx.get_weights()
        orc = env.oracle(env.d)
        witness(env, "w", w_before, w_after, env.d, env.d, orc_after=orc)
        check_readers(ctx, env, orc, "svm", True, kind == "dyadic", what)
    finally:
        if writer == "loop_ended":
            env.ctx("async").stop_async()
        for p in peers:
            p.close()


# ---- fused K = 2 on one GPU --------------------------------------------------------------------------------------------

@pytest.mark.parametrize("kind", KINDS)
def test_fused_two_ranks_averaging(envs, S, kind):
    """Two ranks of the fused peer-exchange step on one GPU with averaging on; every reader on both ranks afterwards."""
    env = envs(kind, 700)
    G = S // 2
    rng = np.random.default_rng(77)
    per_rank = [np.stack([rng.choice(N_ROWS, size=BATCH, replace=False) for _ in range(2)]).astype(np.int32)
                for _ in range(2)]
    orc = env.oracle(env.d)

    def after(r, ctx):
        what = f"fused K = 2, {kind}, rank {r}"
        w = ctx.get_weights()
        witness(env, "w", env.w0, w, env.d, env.d, orc_after=orc)
        check_readers(ctx, env, orc, "svm", kind == "dyadic", kind == "dyadic", what)
        assert ctx.average_weights()[1] == 2
        return w

    res = fused_ranks(env.data, env.lam, env.d, [G, G], env.w0, [(per_rank, None)], env.lr,
                      before=lambda r, ctx: ctx.average_begin(), after=after)
    w_ref, _ = orc.sync_steps(env.w0, np.concatenate(per_rank, axis=1).reshape(-1), [BATCH, BATCH], env.lr, n_steps=2)
    if kind == "dyadic":
        np.testing.assert_array_equal(res["after"][0], w_ref)
    else:
        np.testing.assert_allclose(res["after"][0], w_ref, rtol=1e-11, atol=1e-15)


# ---- the staged sample stream --------------------------------------------------------------------------------------------

def test_requests_leave_the_staged_stream(envs):
    """Stage an epoch, serve forward and gradient requests on other ids (fewer and more than the stream holds), then run
    the staged steps: the same losses and weights, bit for bit, as with no request in between."""
    env = envs("fp32", 700)
    ctx = env.ctx("sync")
    rng = np.random.default_rng(3)
    stream = _steps(rng, BATCH, 4)
    runs = []
    for requests in (False, True):
        _reset(ctx, env, env.w0)
        ctx.stage_samples(stream)
        if requests:
            for n in (100, N_STREAM):
                other = rng.choice(N_ROWS, size=n, replace=False).astype(np.int32)
                ctx.forward(other)
                ctx.gradient(other, want_loss=True)
                ctx.forward(other, env.w1)
                ctx.gradient(other, env.w1)
        ctx.sync_steps_staged(0, BATCH, 4, env.lr, want_losses=True)
        runs.append((ctx.read_losses(4), ctx.get_weights()))
    np.testing.assert_array_equal(runs[1][0], runs[0][0])
    np.testing.assert_array_equal(runs[1][1], runs[0][1])
    w_ref, losses_ref = env.oracle(env.d).sync_steps(env.w0, stream, [BATCH], env.lr, n_steps=4)
    np.testing.assert_allclose(runs[0][0], losses_ref, rtol=1e-12)
    np.testing.assert_allclose(runs[0][1], w_ref, rtol=1e-11, atol=1e-15)


def test_reload_drops_the_staged_stream(envs):
    """A reload (here of as many rows) drops the staged stream, which was checked against the previous rows."""
    from distributed_sgd_b200.native import DsgdRange
    env = envs("fp32", 700)
    ctx, _ = make_pair(env.data, env.lam)
    try:
        ctx.set_weights(env.w0)
        ctx.stage_samples(_steps(np.random.default_rng(4), BATCH, 2))
        d2 = env.data2
        ctx.load_csr(d2.row_ptr, d2.col, d2.val, d2.label)
        with pytest.raises(DsgdRange, match="staged samples exhausted"):
            ctx.sync_steps_staged(0, BATCH, 1, env.lr)
        ctx.stage_samples(np.arange(BATCH, dtype=np.int32))         # staging again works on the new rows
        ctx.sync_steps_staged(0, BATCH, 1, env.lr)
    finally:
        ctx.close()
