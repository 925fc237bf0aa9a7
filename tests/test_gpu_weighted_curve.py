"""Weighted curves on the device (dsgd_eval_*weighted_curve, Master.local_*weighted_curve) against the weighted-curve checker
(oracle/dsgd_oracle_wcurve.c) over the device's own margins, bit for bit: the metrics words, the DSGD_WCURVE_WORDS weighted
words and every point.  Also the identities the words are chosen for -- against dsgd_eval_curve at c = 1, against the
metrics of the expanded id list for integer weights, against dsgd_eval_weighted's sums -- row-order independence, the
logistic model, the async refusal and the launches of the existing curve calls."""
import math

import numpy as np
import pytest

from helpers import data_from_csr, make_pair
from oracle import wcurve as ow

pytestmark = pytest.mark.gpu

LAM = 1e-4
SIZES = [1, 31, 32, 33, 2047, 2048, 100_000]


def dyadic_data(seed, n_rows, dim=192):
    """Rows of 0..24 entries (a tenth of them empty), values multiples of 1/8; a third of the rows positive."""
    rng = np.random.default_rng(seed)
    lens = np.where(rng.random(n_rows) < 0.1, 0, rng.integers(1, 25, size=n_rows))
    rp = np.concatenate([[0], np.cumsum(lens)]).astype(np.int64)
    col = np.concatenate([rng.choice(dim, size=k, replace=False) for k in lens]).astype(np.int32)
    val = (rng.integers(-8, 9, size=int(rp[-1])) / 8.0).astype(np.float32)
    lab = np.where(rng.random(n_rows) < 0.35, 1, -1).astype(np.int8)
    return data_from_csr(rp, col, val, lab, dim)


def bits(a):
    return np.asarray(a, dtype=np.float64).view(np.int64)


def check(ctx, data, ids, res, c_rows, w=None):
    """res over row ids `ids`, every row weighted by c_rows[row]: the checker over the device's margins, bit for bit."""
    ref = ow.wcurve(ctx.margins(ids, w), data.label[ids], c_rows[ids])
    assert np.array_equal(res.words, ref.words), (res.words, ref.words)
    assert np.array_equal(bits(res.wsums), bits(ref.wsums)), (res.wsums, ref.wsums)
    assert res.n_points == len(ref.thr)
    for a, b in ((res.thr, ref.thr), (res.tpw, ref.tpw), (res.fpw, ref.fpw)):
        assert np.array_equal(bits(a), bits(b))
    assert np.array_equal(bits([res.auc, res.ap]), bits([ref.auc, ref.ap]))
    return ref


def weight_cases(n_rows, seed):
    """(name, sample weights or None, class weights)"""
    rng = np.random.default_rng(seed)
    rand = rng.random(n_rows) * 3.0
    dyad = rng.integers(0, 9, n_rows) / 4.0
    zeros = np.where(rng.random(n_rows) < 0.3, 0.0, rand)
    return [("random", rand, (1.0, 1.0)), ("dyadic", dyad, (1.0, 1.0)), ("zeros", zeros, (1.0, 1.0)),
            ("class", None, (2.0, 0.5)), ("class+sample", rand, (2.0, 0.5))]


def set_weights(ctx, data, sw, cw):
    ctx.set_class_weights(*cw)
    ctx.set_sample_weights(sw)
    return ow.weights(data.label, cw[0], cw[1], sw)


@pytest.fixture(scope="module")
def dy():
    data = dyadic_data(1, 130_000)
    ctx, _ = make_pair(data, LAM)
    yield ctx, data
    ctx.close()


@pytest.mark.parametrize("n", SIZES + SIZES[-2::-1])
def test_three_forms_growing_then_shrinking(dy, n):
    """Sizes grow, then shrink, from test to test on one context."""
    ctx, data = dy
    rng = np.random.default_rng(500 + n)
    w = rng.integers(-2, 3, size=data.dim) / 4.0
    for name, sw, cw in weight_cases(data.n_rows, n):
        c = set_weights(ctx, data, sw, cw)
        ids = rng.integers(0, data.n_rows, size=n).astype(np.int32)   # repeats included
        check(ctx, data, ids, ctx.eval_samples_weighted_curve(ids, w), c, w)
        b = int(rng.integers(0, data.n_rows - n + 1))
        rng_ids = np.arange(b, b + n, dtype=np.int32)
        full = ctx.eval_weighted_curve(b, b + n, w)
        check(ctx, data, rng_ids, full, c, w)
        only = ctx.eval_weighted_curve(b, b + n, w, curve=False)
        assert np.array_equal(only.words, full.words) and np.array_equal(bits(only.wsums), bits(full.wsums))
        assert only.n_points == full.n_points and len(only.thr) == 0
        k = min(n, data.n_rows - 5)
        res = ctx.eval_sampled_weighted_curve(5, data.n_rows, 0xBEEF + n, 0, k, w)
        from distributed_sgd_b200.native import host_lib
        h = host_lib()
        drawn = np.array([5 + h.dsgd_feistel_pos(p, data.n_rows - 5, 0xBEEF + n) for p in range(k)], dtype=np.int32)
        check(ctx, data, drawn, res, c, w)
    set_weights(ctx, data, None, (1.0, 1.0))


def test_ties_nan_scores_and_one_class_sets(dy):
    ctx, data = dy
    rng = np.random.default_rng(7)
    c = set_weights(ctx, data, rng.integers(0, 5, data.n_rows) / 2.0, (2.0, 0.5))
    ids = rng.integers(0, data.n_rows, size=20_000).astype(np.int32)
    check(ctx, data, ids, ctx.eval_samples_weighted_curve(ids, np.zeros(data.dim)), c)   # every score 0: one tie group
    w = rng.integers(-1, 2, size=data.dim) / 8.0
    w[rng.random(data.dim) < 0.9] = 0.0                                                  # thousands of ties per score
    check(ctx, data, ids, ctx.eval_samples_weighted_curve(ids, w), c, w)
    pos, neg = ids[data.label[ids] > 0], ids[data.label[ids] < 0]
    for one in (pos, neg):
        r = check(ctx, data, one, ctx.eval_samples_weighted_curve(one, w), c, w)
        assert math.isnan(r.auc)
    wn = rng.integers(-2, 3, size=data.dim) / 4.0
    wn[:2] = np.inf                           # rows with both columns at opposite signs score NaN, others +-inf or finite
    r = check(ctx, data, ids, ctx.eval_samples_weighted_curve(ids, wn), c, wn)
    assert r.words[7] > 0 and math.isnan(r.auc) and math.isnan(r.ap)
    set_weights(ctx, data, None, (1.0, 1.0))


def test_row_order_does_not_change_a_bit(dy):
    ctx, data = dy
    rng = np.random.default_rng(8)
    set_weights(ctx, data, rng.random(data.n_rows) * 5.0, (2.0, 0.5))
    w = rng.standard_normal(data.dim) * 0.1
    b, e = 1000, 61_000
    a = ctx.eval_weighted_curve(b, e, w)
    ids = np.arange(b, e, dtype=np.int32)
    for order in (ids, ids[::-1].copy(), rng.permutation(ids)):
        r = ctx.eval_samples_weighted_curve(order, w)
        assert np.array_equal(r.words, a.words) and np.array_equal(bits(r.wsums), bits(a.wsums))
        assert np.array_equal(bits(r.thr), bits(a.thr)) and np.array_equal(bits(r.tpw), bits(a.tpw))
        assert np.array_equal(bits(r.fpw), bits(a.fpw))
    set_weights(ctx, data, None, (1.0, 1.0))


def test_identities(dy):
    ctx, data = dy
    rng = np.random.default_rng(9)
    w = rng.integers(-2, 3, size=data.dim) / 4.0
    ids = rng.integers(0, data.n_rows, size=30_000).astype(np.int32)
    # c = 1: the curve call's words, U2, AP and points
    set_weights(ctx, data, None, (1.0, 1.0))
    for sw in (None, np.ones(data.n_rows)):
        ctx.set_sample_weights(sw)
        r = ctx.eval_samples_weighted_curve(ids, w)
        words, ap, thr, tp, fp = ctx.eval_samples_curve(ids, w)
        assert np.array_equal(r.words, words) and np.array_equal(r.wsums[:8], words.astype(np.float64))
        assert r.ap == ap or (math.isnan(r.ap) and math.isnan(ap))
        assert np.array_equal(bits(r.thr), bits(thr)) and np.array_equal(r.tpw, tp) and np.array_equal(r.fpw, fp)
    # integer weights: U2w is the U2 of the expanded id list
    sw = rng.integers(0, 4, data.n_rows).astype(np.float64)
    ctx.set_sample_weights(sw)
    r = ctx.eval_samples_weighted_curve(ids, w)
    expanded = np.repeat(ids, sw[ids].astype(int)).astype(np.int32)
    assert r.wsums[6] == float(ctx.eval_samples_metrics(expanded, w)[6])
    # words 9 and 10: dsgd_eval_weighted's sums, bit for bit
    for cw, sw in (((2.0, 0.5), rng.random(data.n_rows) * 7.0), ((3.0, 0.25), None)):
        set_weights(ctx, data, sw, cw)
        r = ctx.eval_samples_weighted_curve(ids, w, curve=False)
        we = ctx.eval_samples_weighted(ids, w)
        assert np.array_equal(bits(r.wsums[9:11]), bits([we.correct_weight, we.weight_sum]))
        r = ctx.eval_weighted_curve(0, data.n_rows, w, curve=False)
        we = ctx.eval_weighted(0, data.n_rows, w)
        assert np.array_equal(bits(r.wsums[9:11]), bits([we.correct_weight, we.weight_sum]))
    set_weights(ctx, data, None, (1.0, 1.0))


def test_logistic_context_gives_the_svm_result(dy):
    from distributed_sgd_b200.native import NativeCtx
    ctx, data = dy
    rng = np.random.default_rng(10)
    sw = rng.random(data.n_rows)
    lg = NativeCtx(0, data.dim, LAM, logistic=True)
    try:
        lg.load_csr(data.row_ptr, data.col, data.val, data.label)
        w = rng.standard_normal(data.dim) * 0.1
        for c in (ctx, lg):
            c.set_class_weights(2.0, 0.5)
            c.set_sample_weights(sw)
        a, b = ctx.eval_weighted_curve(0, 50_000, w), lg.eval_weighted_curve(0, 50_000, w)
        assert np.array_equal(bits(a.wsums), bits(b.wsums)) and np.array_equal(bits(a.tpw), bits(b.tpw))
    finally:
        lg.close()
        set_weights(ctx, data, None, (1.0, 1.0))


def test_async_context_is_refused_before_any_launch():
    from distributed_sgd_b200.native import ERR_STATE, DsgdError
    data = dyadic_data(2, 3000)
    ctx, _ = make_pair(data, LAM, is_async=True)
    try:
        before = ctx.launch_count()
        for call in (lambda: ctx.eval_weighted_curve(0, 3000), lambda: ctx.eval_samples_weighted_curve([1, 2, 3]),
                     lambda: ctx.eval_sampled_weighted_curve(0, 3000, 5, 0, 100, curve=False)):
            with pytest.raises(DsgdError) as e:
                call()
            assert e.value.code == ERR_STATE and "async" in str(e.value)
        assert ctx.launch_count() == before
    finally:
        ctx.close()


def test_existing_curve_calls_launch_what_they_launched(dy):
    """score, count, fold (and emit with the points); the sampled form draws first.  Weights loaded change nothing."""
    ctx, data = dy
    set_weights(ctx, data, np.random.default_rng(11).random(data.n_rows), (2.0, 0.5))
    for call, k in ((lambda: ctx.eval_curve(0, 5000), 4), (lambda: ctx.eval_curve(0, 5000, curve=False), 3),
                    (lambda: ctx.eval_samples_curve(np.arange(100, dtype=np.int32)), 4),
                    (lambda: ctx.eval_sampled_curve(0, 5000, 3, 0, 700), 5),
                    (lambda: ctx.eval_weighted_curve(0, 5000), 4), (lambda: ctx.eval_weighted_curve(0, 5000, curve=False), 3)):
        before = ctx.launch_count()
        call()
        assert ctx.launch_count() - before == k
    set_weights(ctx, data, None, (1.0, 1.0))


def test_full_size_test_rows():
    """The full-size set's 140 000 test rows, class and sample weights."""
    from distributed_sgd_b200.utils import synthetic_rcv1
    data = synthetic_rcv1(n_rows=700_000, seed=0)
    ctx, _ = make_pair(data, LAM)
    try:
        rng = np.random.default_rng(12)
        c = set_weights(ctx, data, rng.random(data.n_rows) * 2.0, (2.0, 0.5))
        w = np.where(rng.random(data.dim) < 0.5, rng.standard_normal(data.dim) * 0.05, 0.0)
        b = data.n_rows - 140_000
        check(ctx, data, np.arange(b, data.n_rows, dtype=np.int32), ctx.eval_weighted_curve(b, data.n_rows, w), c, w)
    finally:
        ctx.close()


def test_master_weighted_curve(dy):
    """Master.local_weighted_curve / local_sampled_weighted_curve: weighted_curve_dict of the device's words."""
    from types import SimpleNamespace
    from distributed_sgd_b200.core.master import MasterSync, weighted_curve_dict
    from distributed_sgd_b200.ml import SparseSVM
    from distributed_sgd_b200.utils.dataset import Data
    ctx, data = dy
    sw = np.random.default_rng(13).random(data.n_rows)
    set_weights(ctx, data, sw, (2.0, 0.5))
    n_train = data.n_rows // 2   # the test rows are the other half
    tr = Data(data.row_ptr[:n_train + 1], data.col, data.val, data.label[:n_train], data.dim)
    slave = SimpleNamespace(ctx=ctx, world=1, is_async=False, n_train=n_train, n_test=data.n_rows - n_train, dim=data.dim,
                            class_weight=(2.0, 0.5), sample_weighted=True)
    m = MasterSync(0, tr, tr, SparseSVM(LAM), 1, slave=slave, seed=0)
    w = np.random.default_rng(14).standard_normal(data.dim) * 0.1
    d = m.local_weighted_curve(w, test_data=True)
    ref = weighted_curve_dict(ctx.eval_weighted_curve(n_train, data.n_rows, w))
    assert d["auc"] == ref["auc"] and d["weight_sum"] == ref["weight_sum"] and d["curve"] == ref["curve"]
    s = m.local_sampled_weighted_curve(w, 5000, curve=False)
    assert "curve" not in s and 0.0 <= s["auc"] <= 1.0
    set_weights(ctx, data, None, (1.0, 1.0))
