"""Averaged SGD on the device (dsgd_average_*, MasterSync.fit(average_from=...)) against the fp64 oracle.

The reference average replays the oracle one step at a time, adds the weights after every step to A in numpy (step order,
plain fp64 additions) and reads A / n out through the 1e-20 filter.  Checked:

1. Against the oracle in every regime test_gpu_sync_regimes.py reaches: grids 1, 2, 7 and S (plain and cooperative launch),
   dims U - 1, 2 U + 1 and 47 237, batches 32 G (persistent kernel) and 32 G + 1 (k_rows + k_update), two virtual workers,
   the logistic single- and two-worker paths, fused K = 2 and K = 3 on one GPU.  RCV1-shaped fp32 rows: rtol 1e-11 over the
   20 steps; logistic: max |diff| <= 1e-11 max |w|; dyadic rows: bit for bit.
2. Bit for bit on dyadic rows: one call of 20 steps against four calls of 5, a run that alternates persistent and fallback
   batches and grid sizes, fused ranks holding identical averages.
3. No interference: with averaging on, every path gives weights and per-step losses bit-identical to the run with it off
   (rows of disjoint columns, so that every run of a path is deterministic).
4. Lifecycle: steps before begin are not counted, end freezes the sum, a second begin restarts, set_weights and zero-step
   calls leave it alone; the error codes on sync and async contexts.
5. End to end: MasterSync.fit(average_from=1) returns ctx.average_weights(), and its last losses are evaluations of them.
"""
import numpy as np
import pytest

from helpers import data_from_csr, make_pair, retry_once_if_not_coscheduled, run_ranks

pytestmark = pytest.mark.gpu

UPD_THREADS = 6 * 32            # update threads per CTA; U = UPD_THREADS * G register columns of the persistent kernel
EPS = 1e-20
STEPS = 20
SPLIT = (17, 3)                 # the 20 steps as two calls, without begin or set_weights in between


@pytest.fixture(scope="module")
def S():
    from distributed_sgd_b200.native import NativeCtx
    ctx = NativeCtx(0, 8, 0.0)
    s = int(ctx.info()["sm_count"])
    ctx.close()
    return s


# ---- reference ------------------------------------------------------------------------------------------------------

def readout(A, n):
    v = A / n
    return np.where(np.abs(v) > EPS, v, 0.0)


def ref_average(orc, w0, steps_ids, counts, lr, A=None):
    """steps_ids: [steps, sum(counts)] ids, workers' slices side by side.  Adds the weights after every step to A (zeros if
    None), in step order.  Returns (last weights, A, per-step losses)."""
    w = np.asarray(w0, np.float64)
    A, losses = (np.zeros_like(w) if A is None else A.copy()), []
    for ids in steps_ids:
        w, ls = orc.sync_steps(w, np.ascontiguousarray(ids, np.int32), counts, lr, n_steps=1)
        A = A + w
        losses.append(ls)
    return w, A, np.concatenate(losses)


def _run(ctx, steps_ids, lr, split=SPLIT):
    """The steps in calls of `split` steps each; returns the losses of all of them."""
    out, s = [], 0
    for n in split:
        part = steps_ids[s:s + n]
        out.append(ctx.sync_steps(part.reshape(-1), part.shape[1], n, lr))
        s += n
    return np.concatenate(out)


# ---- data -------------------------------------------------------------------------------------------------------------

def _synth(dim, n_rows, seed):
    from distributed_sgd_b200.utils import synthetic_rcv1
    return synthetic_rcv1(n_rows=n_rows, dim=dim, seed=seed, mean_nnz=min(94.5, dim / 8.0), max_nnz=min(2000, dim // 2))


def _dyadic(dim, n_rows, seed):
    """Rows of 1 to 40 distinct columns with values k / 16, weights k / 8 on 30 % of the columns: with lambda = 0 and a
    dyadic learning rate every gradient sum and every weight is exact, so the trajectories are the oracle's bit for bit."""
    rng = np.random.default_rng(seed)
    nnz = rng.integers(1, 41, size=n_rows)
    rp = np.concatenate([[0], np.cumsum(nnz)])
    col = np.concatenate([rng.choice(dim, size=k, replace=False) for k in nnz])
    val = rng.integers(1, 33, size=int(rp[-1])) / 16.0
    lab = rng.choice([-1, 1], size=n_rows)
    w0 = rng.integers(-32, 33, size=dim) / 8.0 * (rng.random(dim) < 0.3)
    return data_from_csr(rp, col, val, lab, dim), w0


def _disjoint(n_rows, per_row, seed):
    """Row i holds columns [per_row i, per_row (i + 1)), random fp32 values: no two rows share a column, so every gradient
    entry of a step is ONE addend and every run of a path gives the same bits."""
    rng = np.random.default_rng(seed)
    dim = n_rows * per_row
    rp = np.arange(n_rows + 1, dtype=np.int64) * per_row
    col = np.arange(dim, dtype=np.int32)
    val = (rng.random(dim) * 2.0 + 1e-3).astype(np.float32)
    lab = rng.choice([-1, 1], size=n_rows)
    w0 = rng.standard_normal(dim) * (rng.random(dim) < 0.3) * 0.1
    return data_from_csr(rp, col, val, lab, dim), w0


def _ids(rng, n_rows, steps, batch):
    return np.stack([rng.choice(n_rows, size=batch, replace=False) for _ in range(steps)]).astype(np.int32)


def _logistic_pair(data, lam):
    from distributed_sgd_b200.native import NativeCtx
    from oracle.logistic import LogisticOracle
    ctx = NativeCtx(0, data.dim, lam, logistic=True)
    ctx.load_csr(data.row_ptr, data.col, data.val, data.label)
    orc = LogisticOracle(data.row_ptr, data.col, data.val, data.label, data.dim, lam)
    d = orc.dim_sparsity(data.n_rows)
    orc.set_dim_sparsity(d)
    ctx.set_dim_sparsity(d)
    return ctx, orc


# ---- K ranks of the fused step on one GPU, averaging -----------------------------------------------------------------

def fused_average(data, lam, grids, w0, calls, lr, average=True):
    """K = len(grids) ranks on one GPU (rank r limited to grids[r] CTAs, attached to each other), one host thread each.
    Every rank calls average_begin (if `average`) BEFORE the threads start: its first call allocates.  calls: list of
    per-launch lists of rank ids arrays [steps, batch_r].  Returns [K (weights, losses, (average, n) or None)]."""
    K = len(grids)

    def attempt():
        ctxs = []
        try:
            for r in range(K):
                ctx, _ = make_pair(data, lam, rank=r, world=K)
                ctx.set_grid_limit(grids[r])
                ctx.reserve(max(c[r].size for c in calls), max(c[r].shape[0] for c in calls))
                if average:
                    ctx.average_begin()
                ctxs.append(ctx)
            for r in range(K):
                for q in range(K):
                    if q != r:
                        ctxs[r].xchg_attach(q, ctxs[q])
            out = [None] * K

            def rank_fn(r):
                def run():
                    ctx = ctxs[r]
                    ctx.set_weights(w0)
                    ls = [ctx.sync_steps(c[r].reshape(-1), c[r].shape[1], c[r].shape[0], lr) for c in calls]
                    out[r] = (ctx.get_weights(), np.concatenate(ls), ctx.average_weights() if average else None)
                return run

            run_ranks([rank_fn(r) for r in range(K)])
        finally:
            for c in ctxs:
                c.close()
        return out

    return retry_once_if_not_coscheduled(attempt)


def _fused_steps(calls):
    """The oracle's view of fused launches: per step the ranks' slices side by side; and the per-rank batch sizes."""
    steps = np.concatenate([np.concatenate(c, axis=1) for c in calls], axis=0)
    return steps, [a.shape[1] for a in calls[0]]


# ---- 1. against the oracle ----------------------------------------------------------------------------------------------

def _grid(S, name):
    limit = {"G1": 1, "G2": 2, "G7": 7, "S_plain": S, "S_coop": 0}[name]
    return limit, (limit or S)


GRID_CASES = ([("G1", k) for k in ("U-1", "2U+1", "rcv1")] + [("G2", "U-1"), ("G2", "2U+1")]
              + [("G7", k) for k in ("U-1", "2U+1", "rcv1")] + [("S_plain", "2U+1"), ("S_coop", "U-1"), ("S_coop", "rcv1")])


def _check_avg(avg, n, A_ref, steps, what, exact=False):
    assert n == steps, f"{what}: {n} steps averaged, expected {steps}"
    ref = readout(A_ref, steps)
    if exact:
        np.testing.assert_array_equal(avg, ref, err_msg=what)
    else:
        np.testing.assert_allclose(avg, ref, rtol=1e-11, atol=1e-15, err_msg=what)


@pytest.mark.parametrize("grid,dim_kind", GRID_CASES)
def test_grid_sweep_against_oracle(S, grid, dim_kind):
    limit, G = _grid(S, grid)
    U = UPD_THREADS * G
    dim = {"U-1": U - 1, "2U+1": 2 * U + 1, "rcv1": 47237}[dim_kind]
    n_rows = 32 * G + 64
    data = _synth(dim, n_rows, seed=1000 * G + dim)
    ctx, orc = make_pair(data, lam=1e-2)
    ctx.set_grid_limit(limit)
    rng = np.random.default_rng(dim + G)
    try:
        for b in (32 * G, 32 * G + 1):      # the persistent kernel's largest batch, and the fallback's smallest
            lr = 0.5 / b
            idx = _ids(rng, n_rows, STEPS, b)
            w0 = rng.standard_normal(dim) * (rng.random(dim) < 0.3) * 0.1
            ctx.set_weights(w0)
            ctx.average_begin()
            losses = _run(ctx, idx, lr)
            ctx.average_end()
            avg, n = ctx.average_weights()
            w_ref, A_ref, losses_ref = ref_average(orc, w0, idx, [b], lr)
            what = f"G {G} ({grid}), dim {dim}, batch {b}"
            np.testing.assert_allclose(losses, losses_ref, rtol=1e-12, atol=0, err_msg=what)
            np.testing.assert_allclose(ctx.get_weights(), w_ref, rtol=1e-11, atol=1e-15, err_msg=what)
            _check_avg(avg, n, A_ref, STEPS, what)
    finally:
        ctx.close()


def test_two_virtual_workers_against_oracle(S):
    dim, n_rows, b = 47237, 4096, 256
    data = _synth(dim, n_rows, seed=7)
    ctx, orc = make_pair(data, lam=1e-2)
    rng = np.random.default_rng(8)
    idx = _ids(rng, n_rows, STEPS, 2 * b)
    w0 = rng.standard_normal(dim) * (rng.random(dim) < 0.3) * 0.1
    try:
        ctx.set_workers([b, b], 2)
        ctx.set_weights(w0)
        ctx.average_begin()
        losses = _run(ctx, idx, 0.5 / b)
        avg, n = ctx.average_weights()
        w_ref, A_ref, losses_ref = ref_average(orc, w0, idx, [b, b], 0.5 / b)
        np.testing.assert_allclose(losses, losses_ref, rtol=1e-12, atol=0)
        np.testing.assert_allclose(ctx.get_weights(), w_ref, rtol=1e-11, atol=1e-15)
        _check_avg(avg, n, A_ref, STEPS, "two virtual workers")
    finally:
        ctx.close()


@pytest.mark.parametrize("counts", [[256], [128, 128]])
def test_logistic_against_oracle(counts):
    dim, n_rows = 47237, 4096
    data = _synth(dim, n_rows, seed=9)
    ctx, orc = _logistic_pair(data, 1e-3)
    rng = np.random.default_rng(10)
    tot = sum(counts)
    idx = _ids(rng, n_rows, STEPS, tot)
    w0 = rng.standard_normal(dim) * (rng.random(dim) < 0.3) * 0.1
    lr = 0.5 / tot
    try:
        ctx.set_workers(counts, len(counts))
        ctx.set_weights(w0)
        ctx.average_begin()
        _run(ctx, idx, lr)
        avg, n = ctx.average_weights()
        w_ref, A_ref, _ = ref_average(orc, w0, idx, counts, lr)
        w = ctx.get_weights()
        assert np.max(np.abs(w - w_ref)) <= 1e-11 * np.max(np.abs(w_ref))
        ref = readout(A_ref, STEPS)
        assert n == STEPS
        assert np.max(np.abs(avg - ref)) <= 1e-11 * np.max(np.abs(ref)), f"logistic {counts}"
    finally:
        ctx.close()


@pytest.mark.parametrize("K", [2, 3])
def test_fused_ranks_against_oracle_bit_for_bit(K):
    """Fused K-rank steps on one GPU, dyadic rows, two launches with different rank batches: every rank's average is the
    oracle's bit for bit, so the ranks hold identical averages."""
    G, dim, n_rows, lr = 5, 2047, 600, 2.0 ** -6
    data, w0 = _dyadic(dim, n_rows, seed=20 + K)
    rng = np.random.default_rng(K)
    calls = [[_ids(rng, n_rows, 12, 32 * G - r) for r in range(K)], [_ids(rng, n_rows, 8, 7 + r) for r in range(K)]]
    res = fused_average(data, 0.0, [G] * K, w0, calls, lr)
    _, orc = make_pair(data, 0.0)
    w, A = w0, None
    for c in calls:                         # the launches' steps in order, onto one sum
        steps, counts = _fused_steps([c])
        w, A, _ = ref_average(orc, w, steps, counts, lr, A)
    for r in range(K):
        np.testing.assert_array_equal(res[r][0], w, err_msg=f"rank {r}: weights")
        avg, n = res[r][2]
        _check_avg(avg, n, A, 20, f"fused K = {K}, rank {r}", exact=True)


# ---- 2. path and call independence, dyadic rows -------------------------------------------------------------------------

@pytest.mark.parametrize("path", ["persistent_G7", "fallback_G1", "two_workers"])
def test_one_call_against_four_bit_for_bit(S, path):
    dim, n_rows, lr = 2047, 32 * S + 64, 2.0 ** -6
    data, w0 = _dyadic(dim, n_rows, seed=30)
    ctx, orc = make_pair(data, 0.0)
    b = {"persistent_G7": 32 * 7, "fallback_G1": 33, "two_workers": 64}[path]
    counts = [b // 2, b // 2] if path == "two_workers" else [b]
    ctx.set_grid_limit(7 if path == "persistent_G7" else 1)
    if path == "two_workers":
        ctx.set_workers(counts, 2)
    idx = _ids(np.random.default_rng(31), n_rows, STEPS, b)
    try:
        got = []
        for split in ((STEPS,), (5, 5, 5, 5)):
            ctx.set_weights(w0)
            ctx.average_begin()
            _run(ctx, idx, lr, split)
            got.append((ctx.get_weights(), *ctx.average_weights()))
        w_ref, A_ref, _ = ref_average(orc, w0, idx, counts, lr)
        for w, avg, n in got:
            np.testing.assert_array_equal(w, w_ref)
            _check_avg(avg, n, A_ref, STEPS, path, exact=True)
    finally:
        ctx.close()


def test_mixed_sequence_bit_for_bit(S):
    """Persistent and fallback batches and grid sizes alternate from call to call under one begin."""
    half = S // 2 + 1
    calls = [(7, 20, 4), (7, 32 * 7 + 1, 3), (2, 64, 5), (0, 100, 2), (1, 33, 2), (half, 32 * half, 3), (0, 32 * S + 1, 2),
             (1, 1, 4)]
    dim, n_rows, lr = 2047, 32 * S + 64, 2.0 ** -8
    data, w0 = _dyadic(dim, n_rows, seed=40)
    ctx, orc = make_pair(data, 0.0)
    rng = np.random.default_rng(41)
    w, A = w0, None
    try:
        ctx.set_weights(w0)
        ctx.average_begin()
        for limit, b, n in calls:
            ctx.set_grid_limit(limit)
            idx = _ids(rng, n_rows, n, b)
            ctx.sync_steps(idx.reshape(-1), b, n, lr)
            w, A, _ = ref_average(orc, w, idx, [b], lr, A)
        np.testing.assert_array_equal(ctx.get_weights(), w)
        avg, n = ctx.average_weights()
        _check_avg(avg, n, A, sum(c[2] for c in calls), "mixed sequence", exact=True)
    finally:
        ctx.close()


# ---- 3. no interference -------------------------------------------------------------------------------------------------

INTERFERENCE_PATHS = ["persistent", "fallback", "two_workers", "logistic", "logistic_two_workers", "fused_K2"]


@pytest.mark.parametrize("path", INTERFERENCE_PATHS)
def test_averaging_does_not_change_the_step(S, path):
    """The same run with averaging off and on: weights and per-step losses bit for bit.  Rows of disjoint columns make every
    run of a path deterministic, fp32 values and all."""
    n_rows = 32 * S + 64
    data, w0 = _disjoint(n_rows, 4, seed=50)
    lam, rng = 1e-3, np.random.default_rng(51)
    if path == "fused_K2":
        G = S // 2
        calls = [[_ids(rng, n_rows, 12, 32 * G) for _ in range(2)]]
        off = fused_average(data, lam, [G, G], w0, calls, 0.01, average=False)
        on = fused_average(data, lam, [G, G], w0, calls, 0.01, average=True)
        for r in range(2):
            np.testing.assert_array_equal(on[r][0], off[r][0], err_msg=f"rank {r}: weights")
            np.testing.assert_array_equal(on[r][1], off[r][1], err_msg=f"rank {r}: losses")
            assert on[r][2][1] == 12
        np.testing.assert_array_equal(on[0][2][0], on[1][2][0])
        return
    b = 32 * S + 1 if path == "fallback" else 256
    counts = [b // 2, b // 2] if path.endswith("two_workers") else [b]
    ctx = _logistic_pair(data, lam)[0] if path.startswith("logistic") else make_pair(data, lam)[0]
    idx = _ids(rng, n_rows, STEPS, b)
    try:
        if len(counts) > 1:
            ctx.set_workers(counts, len(counts))
        runs = []
        for average in (False, True):
            ctx.set_weights(w0)
            if average:
                ctx.average_begin()
            losses = _run(ctx, idx, 0.5 / b)
            runs.append((ctx.get_weights(), losses))
        np.testing.assert_array_equal(runs[1][0], runs[0][0], err_msg=f"{path}: weights")
        np.testing.assert_array_equal(runs[1][1], runs[0][1], err_msg=f"{path}: losses")
        assert ctx.average_weights()[1] == STEPS
    finally:
        ctx.close()


# ---- 4. lifecycle -------------------------------------------------------------------------------------------------------

def test_lifecycle(S):
    from distributed_sgd_b200.native import DsgdEmpty
    dim, n_rows, lr, b = 2047, 600, 2.0 ** -6, 64
    data, w0 = _dyadic(dim, n_rows, seed=60)
    ctx, orc = make_pair(data, 0.0)
    idx = _ids(np.random.default_rng(61), n_rows, 30, b)
    try:
        ctx.set_weights(w0)
        ctx.sync_steps(idx[:5].reshape(-1), b, 5, lr)                  # before begin: not averaged
        ctx.average_begin()
        w5 = ctx.get_weights()
        ctx.sync_steps(idx[5:12].reshape(-1), b, 7, lr)
        ctx.sync_steps(np.zeros(0, np.int32), b, 0, lr)               # a call of zero steps adds nothing
        w12, A, _ = ref_average(orc, w5, idx[5:12], [b], lr)
        avg, n = ctx.average_weights()
        _check_avg(avg, n, A, 7, "steps 5..11", exact=True)
        ctx.set_weights(w0)                                            # leaves the sum and the count alone
        avg2, n2 = ctx.average_weights()
        assert n2 == 7 and np.array_equal(avg2, avg)
        ctx.sync_steps(idx[12:15].reshape(-1), b, 3, lr)               # ... and the steps go on from w0
        _, A, _ = ref_average(orc, w0, idx[12:15], [b], lr, A)
        avg, n = ctx.average_weights()
        _check_avg(avg, n, A, 10, "after set_weights", exact=True)
        ctx.average_end()                                              # end freezes the sum and the count
        ctx.sync_steps(idx[15:19].reshape(-1), b, 4, lr)
        avg3, n3 = ctx.average_weights()
        assert n3 == 10 and np.array_equal(avg3, avg)
        w_now = ctx.get_weights()
        ctx.average_begin()                                            # a second begin restarts from zero
        with pytest.raises(DsgdEmpty):
            ctx.average_weights()
        ctx.sync_steps(idx[19:21].reshape(-1), b, 2, lr)
        _, A, _ = ref_average(orc, w_now, idx[19:21], [b], lr)
        avg, n = ctx.average_weights()
        _check_avg(avg, n, A, 2, "second begin", exact=True)
    finally:
        ctx.close()


def test_error_codes():
    from distributed_sgd_b200.native import ERR_EMPTY, ERR_STATE, DsgdError, NativeCtx
    data, _ = _dyadic(64, 40, seed=70)
    ctx, _ = make_pair(data, 0.0)
    try:
        with pytest.raises(DsgdError) as e:
            ctx.average_weights()                                      # before any begin
        assert e.value.code == ERR_STATE
        ctx.average_begin()
        with pytest.raises(DsgdError) as e:
            ctx.average_weights()                                      # no step yet: the mean of an empty list
        assert e.value.code == ERR_EMPTY
        ctx.average_end()
        with pytest.raises(DsgdError) as e:
            ctx.average_weights()
        assert e.value.code == ERR_EMPTY
    finally:
        ctx.close()
    actx = NativeCtx(0, 64, 0.0, is_async=True)
    try:
        for call in (actx.average_begin, actx.average_end, actx.average_weights):
            with pytest.raises(DsgdError) as e:
                call()
            assert e.value.code == ERR_STATE, call.__name__
    finally:
        actx.close()


# ---- 5. end to end ------------------------------------------------------------------------------------------------------

def test_master_fit_returns_the_device_average():
    from distributed_sgd_b200 import MasterSync, Slave, SparseSVM
    from distributed_sgd_b200.ml import EarlyStopping
    from distributed_sgd_b200.utils import synthetic_rcv1
    data = synthetic_rcv1(n_rows=6000, seed=80)
    train, test = data.split_at(4800)
    train, _ = train.split_at(1200)                                    # 12 steps of 100 per epoch
    model = SparseSVM(1e-3)
    slave = Slave(0, 0, train, model, world=1, device=0, test_data=test)
    master = MasterSync(0, train, test, model, 1, slave=slave, seed=0)
    try:
        state = master.fit(np.zeros(data.dim), max_epochs=3, batch_size=100, learning_rate=0.5,
                           stopping_criterion=EarlyStopping.no_improvement(patience=5, min_delta=0.01), average_from=1)
        avg, n = master.ctx.average_weights()
        assert n == 24 and master.history["averaged_steps"] == 24
        np.testing.assert_array_equal(state.grad, avg)
        assert not np.array_equal(avg, master.ctx.get_weights())
        tl, ta = master.local_loss_accuracy(avg, test_data=False)
        vl, va = master.local_loss_accuracy(avg, test_data=True)
        assert master.history["losses"][-1] == tl and master.history["accs"][-1] == ta
        assert master.history["test_losses"][-1] == vl and master.history["test_accs"][-1] == va
        assert state.loss == tl
    finally:
        slave.stop()
