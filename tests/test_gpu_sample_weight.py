"""Per-row sample weights on the device (dsgd_set_sample_weights, dsgd_eval*_weighted), checked against oracle/sw.py:

* all ones is the library without weights: weights, losses, gradients and evaluation sums and counts, bit for bit on dyadic
  rows, on the persistent kernel's sample-weighted form, the per-step path and virtual workers;
* the persistent kernel's sample-weighted form at 1, 2, 7 and 132 CTAs, batches 1, G, 32 G and 32 G + 1 alternating, empty,
  multi-chunk and unlisted rows, a CTA of 32 rows at hinge 2, and every combination of averaging, rate table and L1;
* dyadic sample weights (multiples of 1/4 in [0, 4], some zeros) against the checker: weights bit for bit, losses bit for bit
  at lambda = 0 and at the first step, rtol 1e-13 after that (||w||^2 rounds by the order of its sum, DESIGN.md 4.12);
* an integer weight k equals the row listed k times; the weighted sums are order-free;
* per-row weights equal to the balanced class weights reproduce class_weight="balanced" training through MasterSync.fit;
* errors, the exchange-only refusal, and a reload dropping the weights.
"""
import numpy as np
import pytest

from helpers import csr, make_pair
from oracle import sw as SW
from test_gpu_class_weight import dyadic_data, dyadic_pair, dyadic_w0, long_dyadic_data, pair
from test_oracle_sample_weight import dyadic_weights

pytestmark = pytest.mark.gpu

G = 132   # CTAs of the persistent kernel on an H100 SXM: batches 32 G and 32 G + 1 fall on either side of its limit


def _run(ctx, idx, batch, lrs):
    l0 = ctx.sync_steps(idx[:batch * 2], batch, 2, lrs[0])
    l1 = ctx.sync_steps_lr(idx[batch * 2:], batch, lrs[2:])
    return np.concatenate([l0, l1]), ctx.get_weights()


@pytest.mark.parametrize("lam", [2.0 ** -6, 0.0])
@pytest.mark.parametrize("cw", [(1.0, 1.0), (2.0, 0.5)])
@pytest.mark.parametrize("batch,workers", [(1, None), (64, None), (32 * G, None), (32 * G + 1, None), (64, [40, 24])])
def test_unit_sample_weights_are_the_unweighted_library(batch, workers, cw, lam):
    data, rng = dyadic_data(11)
    w0 = dyadic_w0(rng, data.dim)
    lrs = [0.5, 0.5, 0.25, 0.125]
    idx = rng.integers(0, data.n_rows, size=batch * len(lrs)).astype(np.int32)
    runs = []
    for weighted in (False, True):
        ctx, _ = dyadic_pair(data, lam)
        try:
            if workers:
                ctx.set_workers(workers, len(workers))
            ctx.set_class_weights(*cw)
            if weighted:
                ctx.set_sample_weights(np.ones(data.n_rows))
            assert ctx.info()["sample_weights"] is weighted
            ctx.set_weights(w0)
            losses, w = _run(ctx, idx, batch, lrs)
            g, gl = ctx.gradient(idx[:100], w0, want_loss=True)
            runs.append((losses, w, g, gl, ctx.eval_weighted(0, data.n_rows, w0)))
        finally:
            ctx.close()
    (l_u, w_u, g_u, gl_u, e_u), (l_w, w_w, g_w, gl_w, e_w) = runs
    assert np.array_equal(w_w, w_u) and np.array_equal(g_w, g_u) and gl_w == gl_u and e_w == e_u
    # both contexts take the same path (the persistent kernel up to 32 G rows): ||w||^2 in the same order, losses bit for bit
    assert np.array_equal(l_w, l_u)


@pytest.mark.parametrize("logistic", [False, True])
def test_unit_sample_weights_gradient_and_evaluations(logistic):
    """Dyadic rows and weights: every SVM gradient sum is exact, so the streaming pass (2 048 ids or more without weights) and
    k_rows<…, kSampleWeighted, …> must give the same bits; the logistic scatter adds in the order of arrival."""
    data, rng = dyadic_data(21, n_rows=20000)
    w = dyadic_w0(rng, data.dim) / 8.0
    ctx, _ = dyadic_pair(data, 2.0 ** -6, logistic)
    try:
        ids = rng.integers(0, data.n_rows, size=262144).astype(np.int32)
        ref = {}
        for weighted in (False, True):
            if weighted:
                ctx.set_sample_weights(np.ones(data.n_rows))
            for n in (1, 2047, 2048, 262144):
                g, loss = ctx.gradient(ids[:n], w, want_loss=True)
                if not weighted:
                    ref[n] = (g, loss)
                elif logistic:
                    np.testing.assert_allclose(g, ref[n][0], rtol=1e-11, atol=1e-15)
                    assert loss == ref[n][1]
                else:
                    assert np.array_equal(g, ref[n][0]) and loss == ref[n][1]
            for b, e in ((0, 1), (0, 2047), (100, 2148), (0, 20000)):
                we = ctx.eval_weighted(b, e, w)
                loss_sum, correct, n2 = ctx.eval_sums(b, e, w)
                assert we.loss_sum == loss_sum and we.correct == correct and we.n == e - b and we.norm_squared == n2
                assert we.weight_sum == e - b and we.correct_weight == correct
                if not logistic:
                    assert ctx.eval_counts(b, e, w)[:2] == (int(loss_sum), correct)
    finally:
        ctx.close()


@pytest.mark.parametrize("lam", [2.0 ** -6, 0.0])
@pytest.mark.parametrize("cw", [(1.0, 1.0), (2.0, 0.5)])
@pytest.mark.parametrize("batch,workers", [(1, None), (64, None), (G, None), (32 * G + 1, None), (64, [40, 24])])
def test_dyadic_steps_against_the_checker(batch, workers, cw, lam):
    data, rng = dyadic_data(12)
    ctx, orc = dyadic_pair(data, lam)
    try:
        counts = workers or [batch]
        if workers:
            ctx.set_workers(workers, len(workers))
        sw = dyadic_weights(rng, data.n_rows)
        ctx.set_class_weights(*cw)
        ctx.set_sample_weights(sw)
        w0 = dyadic_w0(rng, data.dim)
        lrs = [0.5, 0.5, 0.25, 0.125]
        idx = rng.integers(0, data.n_rows, size=batch * len(lrs)).astype(np.int32)
        ctx.set_weights(w0)
        losses, w = _run(ctx, idx, batch, lrs)
        w_ref, l_ref = SW.sync_steps(orc, w0, idx, counts, lrs, sw, *cw)
        assert np.array_equal(w, w_ref)
        assert losses[0] == l_ref[0]
        if lam == 0.0:
            assert np.array_equal(losses, l_ref)
        np.testing.assert_allclose(losses, l_ref, rtol=1e-13)
    finally:
        ctx.close()


@pytest.mark.parametrize("lam", [2.0 ** -6, 0.0])
@pytest.mark.parametrize("grid", [1, 2, 7, 0])
@pytest.mark.parametrize("long_rows", [False, True])
def test_persistent_kernel_at_every_grid_size(grid, long_rows, lam):
    """The persistent kernel's sample-weighted form at 1, 2, 7 and one CTA per SM, batches of 1, G, 32 G rows (persistent)
    and 32 G + 1 (the per-step path), alternating, in calls that follow each other without set_weights; stages with empty
    rows, rows of several chunks and rows outside the chunk list."""
    data, rng = long_dyadic_data(15) if long_rows else dyadic_data(14)
    ctx, orc = dyadic_pair(data, lam)
    try:
        G_ = grid or ctx.info()["sm_count"]
        ctx.set_grid_limit(grid)
        sw = dyadic_weights(rng, data.n_rows)
        ctx.set_class_weights(2.0, 0.5)
        ctx.set_sample_weights(sw)
        w = dyadic_w0(rng, data.dim)
        ctx.set_weights(w)
        for batch, persistent in ((1, True), (32 * G_ + 1, False), (G_, True), (32 * G_, True), (32 * G_ + 1, False),
                                  (32 * G_, True)):
            lrs = [2.0 ** -3, 2.0 ** -4, 2.0 ** -5]
            idx = rng.integers(0, data.n_rows, size=batch * len(lrs)).astype(np.int32)
            n0 = ctx.launch_count()
            losses = ctx.sync_steps_lr(idx, batch, lrs)
            assert (ctx.launch_count() - n0 == 2) == persistent
            w, l_ref = SW.sync_steps(orc, w, idx, [batch], lrs, sw, 2.0, 0.5)
            if lam == 0.0:
                assert np.array_equal(ctx.get_weights(), w) and np.array_equal(losses, l_ref)
            else:   # over these 18 steps the weights outgrow the dyadic grid: c = 2 lambda (w . d) rounds by the sum's order
                np.testing.assert_allclose(ctx.get_weights(), w, rtol=1e-12, atol=1e-15)
                np.testing.assert_allclose(losses, l_ref, rtol=1e-12)
                w = ctx.get_weights()
    finally:
        ctx.close()


def test_one_cta_holds_32_rows_at_hinge_2():
    """One CTA takes all 32 rows of a step, every one mispredicted: every bit of the CTA's 64-bit code word is set."""
    rows = [(np.array([0]), np.array([1.0]))] * 32
    lab = np.array([1, -1] * 16, np.int8)
    data = csr([(np.array([0]), np.array([1.0 if y > 0 else -1.0])) for y in lab], lab, 4)
    del rows
    ctx, orc = make_pair(data, 0.0)
    try:
        ctx.set_grid_limit(1)
        w0 = np.array([1.0, 0.0, 0.0, 0.0])   # y * dot = 1 > 0 -> the prediction is -y: hinge 2 for every row
        ctx.set_weights(w0)
        sw = np.arange(1, 33) / 4.0
        ctx.set_sample_weights(sw)
        ids = np.tile(np.arange(32, dtype=np.int32), 2)
        n0 = ctx.launch_count()
        loss = ctx.sync_steps(ids, 32, 2, 2.0 ** -8)
        assert ctx.launch_count() - n0 == 2   # the persistent kernel and its record initialisation
        w_ref, l_ref = SW.sync_steps(orc, w0, ids, [32], [2.0 ** -8] * 2, sw)
        assert loss[0] == 2.0 * sw.sum() / 32
        assert np.array_equal(loss, l_ref) and np.array_equal(ctx.get_weights(), w_ref)
    finally:
        ctx.close()


@pytest.mark.parametrize("avg,table,l1", [(a, t, l) for a in (False, True) for t in (False, True) for l in (False, True)])
def test_persistent_kernel_every_combination(avg, table, l1):
    data, rng = dyadic_data(16)
    for unit in (False, True):   # dyadic weights against the checker; all ones against the same ctx without weights
        runs = []
        for weighted in ((True,) if not unit else (False, True)):
            ctx, orc = dyadic_pair(data, 2.0 ** -6)
            try:
                r2 = np.random.default_rng(7)
                sw = np.ones(data.n_rows) if unit else dyadic_weights(r2, data.n_rows)
                ctx.set_class_weights(0.5, 2.0)
                if weighted:
                    ctx.set_sample_weights(sw)
                lam1 = 2.0 ** -7 if l1 else 0.0
                if l1:
                    ctx.set_l1(lam1)
                w0 = dyadic_w0(r2, data.dim)
                lrs = [0.25, 0.125, 0.0, 0.0625] if table else [0.125] * 4
                idx = r2.integers(0, data.n_rows, size=256 * 4).astype(np.int32)
                ctx.set_weights(w0)
                if avg:
                    ctx.average_begin()
                n0 = ctx.launch_count()
                losses = ctx.sync_steps_lr(idx, 256, lrs) if table else ctx.sync_steps(idx, 256, 4, 0.125)
                assert ctx.launch_count() - n0 == 2
                a = ctx.average_weights()[0] if avg else None
                runs.append((losses, ctx.get_weights(), a))
                if not unit:
                    avg_ref = np.zeros(data.dim)
                    w_ref, l_ref = SW.sync_steps(orc, w0, idx, [256], lrs, sw, 0.5, 2.0, lambda1=lam1, avg_sum=avg_ref)
                    assert np.array_equal(ctx.get_weights(), w_ref) and losses[0] == l_ref[0]
                    np.testing.assert_allclose(losses, l_ref, rtol=1e-13)
                    if avg:
                        np.testing.assert_allclose(a, avg_ref / 4, rtol=1e-15, atol=0)
            finally:
                ctx.close()
        if unit:
            (l_u, w_u, a_u), (l_w, w_w, a_w) = runs
            assert np.array_equal(l_w, l_u) and np.array_equal(w_w, w_u)
            if avg:
                assert np.array_equal(a_w, a_u)


@pytest.mark.parametrize("option", ["l1", "avg"])
def test_dyadic_steps_with_l1_and_averaging(option):
    data, rng = dyadic_data(13)
    ctx, orc = dyadic_pair(data, 2.0 ** -6)
    try:
        sw = dyadic_weights(rng, data.n_rows)
        ctx.set_sample_weights(sw)
        lambda1 = 2.0 ** -5 if option == "l1" else 0.0
        if lambda1:
            ctx.set_l1(lambda1)
        w0 = dyadic_w0(rng, data.dim)
        ctx.set_weights(w0)
        if option == "avg":
            ctx.average_begin()
        lrs = [0.5, 0.25, 0.125]
        idx = rng.integers(0, data.n_rows, size=64 * 3).astype(np.int32)
        losses = ctx.sync_steps_lr(idx, 64, lrs)
        avg = np.zeros(data.dim)
        w_ref, l_ref = SW.sync_steps(orc, w0, idx, [64], lrs, sw, lambda1=lambda1, avg_sum=avg)
        assert np.array_equal(ctx.get_weights(), w_ref)
        np.testing.assert_allclose(losses, l_ref, rtol=1e-13)
        if option == "avg":
            a, n = ctx.average_weights()
            assert n == 3
            np.testing.assert_allclose(a, avg / 3, rtol=1e-15, atol=1e-20)
    finally:
        ctx.close()


def test_logistic_steps_against_the_checker():
    from distributed_sgd_b200.utils import synthetic_rcv1
    data = synthetic_rcv1(n_rows=6000, seed=3)
    ctx, orc = pair(data, 1e-5, logistic=True)
    try:
        rng = np.random.default_rng(2)
        sw = rng.random(data.n_rows) * 3.0
        ctx.set_class_weights(2.0, 0.5)
        ctx.set_sample_weights(sw)
        idx = rng.integers(0, data.n_rows, size=256 * 3).astype(np.int32)
        ctx.set_weights(np.zeros(data.dim))
        losses = ctx.sync_steps(idx, 256, 3, 0.5)
        w_ref, l_ref = SW.sync_steps(orc, np.zeros(data.dim), idx, [256], [0.5] * 3, sw, 2.0, 0.5, logistic=True)
        np.testing.assert_allclose(ctx.get_weights(), w_ref, rtol=1e-10, atol=1e-14)
        np.testing.assert_allclose(losses, l_ref, rtol=1e-12)
        sums, counts = SW.eval_weighted(orc, w_ref, np.arange(4000, 6000), 2.0, 0.5, sw, logistic=True)
        we = ctx.eval_weighted(4000, 6000, w_ref)
        np.testing.assert_allclose([we.loss_sum, we.correct_weight, we.weight_sum], sums, rtol=1e-13)
        assert we.weight_sum == sums[2] and [we.n, we.correct] == list(counts)
    finally:
        ctx.close()


@pytest.mark.parametrize("logistic", [False, True])
def test_integer_weight_equals_the_row_listed_k_times(logistic):
    data, rng = dyadic_data(14, n_rows=600)
    ctx, orc = dyadic_pair(data, 2.0 ** -6, logistic)
    try:
        w = dyadic_w0(rng, data.dim) / 8.0
        ids = np.arange(200, dtype=np.int32)
        sw = np.ones(data.n_rows)
        sw[:200] = rng.choice([0.0, 2.0, 4.0], size=200)
        rep = np.repeat(ids, sw[:200].astype(int)).astype(np.int32)
        g_rep = ctx.gradient(rep, w)
        s_rep = ctx.eval_samples_weighted(rep, w)
        ctx.set_sample_weights(sw)
        g_w = ctx.gradient(ids, w)
        s_w = ctx.eval_samples_weighted(ids, w)
        if logistic:   # k copies of a product summed against one product times k
            np.testing.assert_allclose(g_w, g_rep, rtol=1e-13, atol=1e-15)
        else:
            assert np.array_equal(g_w, g_rep)
        assert (s_w.loss_sum, s_w.correct_weight, s_w.weight_sum) == (s_rep.loss_sum, s_rep.correct_weight, s_rep.weight_sum)
        g_ref = SW.gradient(orc, w, ids, sw, logistic=logistic)[0]
        if not logistic:
            assert np.array_equal(g_w, g_ref)
    finally:
        ctx.close()


@pytest.mark.parametrize("logistic", [False, True])
def test_weighted_evaluation_is_order_free_and_matches_the_checker(logistic):
    from distributed_sgd_b200.utils import synthetic_rcv1
    data = synthetic_rcv1(n_rows=40000, seed=23)
    ctx, orc = pair(data, 1e-5, logistic)
    try:
        rng = np.random.default_rng(4)
        w = rng.standard_normal(data.dim) * 0.05
        sw = rng.random(data.n_rows) * 2.0
        sw[rng.random(data.n_rows) < 0.1] = 0.0
        ctx.set_class_weights(3.0, 0.5)
        ctx.set_sample_weights(sw)
        for n in (1, 33, 2048, 30000):
            b = int(rng.integers(0, data.n_rows - n + 1))
            ids = np.arange(b, b + n, dtype=np.int32)
            we = ctx.eval_weighted(b, b + n, w)
            for order in (ids[::-1], rng.permutation(ids)):
                assert ctx.eval_samples_weighted(order, w) == we
            if n > 1:
                assert ctx.eval_sampled_weighted(b, b + n, 99, 0, n, w) == we
            sums, counts = SW.eval_weighted(orc, w, ids, 3.0, 0.5, sw, logistic=logistic)
            assert [we.n, we.correct] == list(counts)
            assert we.correct_weight == sums[1] and we.weight_sum == sums[2]
            if logistic:
                assert we.loss_sum == pytest.approx(sums[0], rel=1e-13)
            else:
                assert we.loss_sum == sums[0]
    finally:
        ctx.close()


def test_errors_and_reload():
    from distributed_sgd_b200.native import DsgdInvalid, DsgdState, NativeCtx
    ctx = NativeCtx(0, 16, 0.1)
    try:
        with pytest.raises(DsgdState):
            ctx.set_sample_weights(np.ones(4))
        data, rng = dyadic_data(15, n_rows=50, dim=16)
        ctx.load_csr(data.row_ptr, data.col, data.val, data.label)
        ctx.set_dim_sparsity(np.full(16, 0.25))
        for bad in (np.ones(49), np.ones(51), np.r_[np.ones(49), -1.0], np.r_[np.nan, np.ones(49)], np.r_[np.inf, np.ones(49)]):
            with pytest.raises(DsgdInvalid):
                ctx.set_sample_weights(bad)
        assert ctx.info()["sample_weights"] is False
        ids = np.arange(50, dtype=np.int32)
        w = dyadic_w0(rng, 16)
        g0, e0 = ctx.gradient(ids, w), ctx.eval_weighted(0, 50, w)
        ctx.set_sample_weights(np.full(50, 2.0))
        assert ctx.info()["sample_weights"] is True
        assert ctx.eval_weighted(0, 50, w).weight_sum == 100.0
        ctx.set_sample_weights(None)
        assert ctx.info()["sample_weights"] is False and ctx.eval_weighted(0, 50, w) == e0
        ctx.set_sample_weights(np.full(50, 2.0))
        ctx.load_csr(data.row_ptr, data.col, data.val, data.label)   # the weights named the previous rows
        assert ctx.info()["sample_weights"] is False
        assert np.array_equal(ctx.gradient(ids, w), g0) and ctx.eval_weighted(0, 50, w) == e0
    finally:
        ctx.close()
    a = NativeCtx(0, 16, 0.1, is_async=True)
    try:
        a.load_csr(data.row_ptr, data.col, data.val, data.label)
        with pytest.raises(DsgdState):
            a.set_sample_weights(np.ones(50))
    finally:
        a.close()


def test_exchange_only_ranks_refuse_before_launching():
    from distributed_sgd_b200.native import DsgdState
    from distributed_sgd_b200.utils import synthetic_rcv1
    data = synthetic_rcv1(n_rows=2000, seed=5)
    ctxs = [make_pair(data, 1e-5, rank=r, world=2)[0] for r in range(2)]
    try:
        ctxs[0].xchg_attach(1, ctxs[1])
        ctxs[1].xchg_attach(0, ctxs[0])
        ctxs[0].set_sample_weights(np.ones(data.n_rows))
        n0 = ctxs[0].launch_count()
        with pytest.raises(DsgdState, match="sample weights"):
            ctxs[0].sync_steps(np.arange(32, dtype=np.int32), 32, 1, 0.5)
        assert ctxs[0].launch_count() == n0
    finally:
        for c in ctxs:
            c.close()


def test_balanced_sample_weights_reproduce_balanced_class_weights_through_fit():
    """Per-row weights equal to the resolved "balanced" class weights, with class weights (1, 1), train exactly like
    class_weight="balanced": the same persistent kernel arithmetic per row (c_i = 1 * w_y = w_y).  Dyadic rows with 4/5 of
    the train rows positive give the weights (5/8, 5/2), so every gradient sum is exact and the runs are bit for bit; a
    stopping rule that never fires fixes the epoch count."""
    from distributed_sgd_b200 import EarlyStopping, Master, Slave, SparseSVM
    from distributed_sgd_b200.core import Group
    data, rng = dyadic_data(31, n_rows=5000)
    lab = np.where(np.arange(5000) % 5 == 0, -1, 1).astype(np.int8)   # train rows 0..3999: 3 200 positive, 800 negative
    data.label = lab
    train, test = data.split_at(4000)
    wp, wn = 4000 / (2.0 * 3200), 4000 / (2.0 * 800)
    assert (wp, wn) == (0.625, 2.5)
    results = []
    for mode in ("class", "sample"):
        if mode == "class":
            model, tr = SparseSVM(2.0 ** -10, class_weight="balanced"), train
        else:
            tr, _ = train.split_at(train.n_rows)
            tr.weight = np.where(train.label > 0, wp, wn)
            model = SparseSVM(2.0 ** -10)
        slave = Slave(0, 0, tr, model, False, test_data=test)
        try:
            assert slave.sample_weighted is (mode == "sample")
            if mode == "class":
                assert slave.class_weight == (wp, wn)
            master = Master.create(0, tr, test, model, False, 1, slave=slave, group=Group(), seed=7)
            never = EarlyStopping.no_improvement(patience=10 ** 9, min_delta=0.0)
            state = master.fit(np.zeros(data.dim), 3, 64, 0.5, never)
            assert len(master.history["losses"]) == 3
            results.append(state.grad)
        finally:
            slave.stop()
    assert np.array_equal(results[1], results[0])
