"""One-vs-rest topics on the device (dsgd_load_topics, dsgd_select_topic, dsgd_eval*_topics; DESIGN.md §4.21):

* select_topic(t) gives every path the results of a context freshly loaded with topic t's labels: the persistent kernel,
  the per-step path (batch above 32 G), the logistic model, the intercept, class and sample weights, the fp32 streaming
  evaluation and gradient, metrics; select_topic(-1) gives back the original results.  Bit for bit, except the logistic
  model's fp64 scatter, which adds in the order of arrival and so agrees to rounding from run to run.
* eval_topics: per topic the words of dsgd_eval_metrics after select_topic(t) with W_t, bit for bit; the row words equal the
  numpy restatement over T dsgd_margins calls, and both the C checker; T = 1, 103 and 1024, rows without topics, planted
  NaN and zero scores, the intercept, every model flag, range / sampled / list forms, a shuffled list.
* refusals launch no kernel; fit_one_vs_rest equals separate single-topic fits bit for bit, and a plain fit after it equals
  one on a fresh context."""
import ctypes as C

import numpy as np
import pytest

from oracle import topics as topics_oracle
from oracle.oracle import Oracle
from test_gpu_class_weight import dyadic_data, dyadic_w0
from topics_model import topic_words

pytestmark = pytest.mark.gpu

G = 132
LAM = 2.0 ** -6


def _with_topics(data, T, seed):
    import dataclasses
    from distributed_sgd_b200.utils import synthetic_topics
    return dataclasses.replace(data, topics=synthetic_topics(data, T, seed=seed))


def _ctx(data, labels, model="svm", intercept=False, topics=True, is_async=False):
    from distributed_sgd_b200.native import NativeCtx
    ctx = NativeCtx(0, data.dim, LAM, model=model, intercept=intercept, is_async=is_async)
    ctx.load_csr(data.row_ptr, data.col, data.val, labels)
    if is_async:
        return ctx
    d = np.zeros(data.dim)
    d[::3] = 0.25
    ctx.set_dim_sparsity(d)
    if topics:
        ctx.load_topics(data.topics.ptr, data.topics.ids, data.topics.n_topics)
    return ctx


# ---- select_topic ---------------------------------------------------------------------------------------------------------

CASES = {"persistent": ("svm", False, 64, None), "per_step": ("svm", False, 32 * G + 1, None),
         "logistic": ("logistic", False, 64, None), "intercept": ("svm", True, 64, None),
         "class_weighted": ("svm", False, 64, "class"), "sample_weighted": ("svm", False, 64, "sample")}


def _run(ctx, data, case, seed):
    """sync steps from a dyadic w0, then the weights, an evaluation (the fp32 streaming pass where it applies), a
    gradient over 2 500 ids (streamed likewise), the metrics and a weighted evaluation"""
    model, intercept, batch, weighting = case
    rng = np.random.default_rng(seed)
    if weighting == "class":
        ctx.set_class_weights(2.0, 0.5)
    if weighting == "sample":
        ctx.set_sample_weights(rng.integers(0, 9, size=data.n_rows) / 4.0)
    w0 = dyadic_w0(rng, ctx.wdim)
    idx = rng.integers(0, data.n_rows, size=3 * batch).astype(np.int32)
    gid = rng.integers(0, data.n_rows, size=2500).astype(np.int32)
    ctx.set_weights(w0)
    losses = ctx.sync_steps(idx, batch, 3, 0.5)
    w = ctx.get_weights()
    g, gl = ctx.gradient(gid, w0, want_loss=True)
    out = [losses, w, np.array(ctx.eval(0, data.n_rows, w0)), g, np.array([gl]), ctx.eval_metrics(0, data.n_rows, w),
           np.array(ctx.eval_weighted(0, data.n_rows, w))]
    if weighting == "class":
        ctx.set_class_weights(1.0, 1.0)
    if weighting == "sample":
        ctx.set_sample_weights(None)
    return out


def _same(a, b, logistic):
    for x, y in zip(a, b):
        if logistic:
            np.testing.assert_allclose(x, y, rtol=1e-11, atol=1e-15)
        else:
            assert np.array_equal(x, y, equal_nan=True), (x, y)


@pytest.mark.parametrize("name", list(CASES))
def test_select_topic_matches_a_context_loaded_with_the_topic_labels(name):
    model, intercept = CASES[name][:2]
    data = _with_topics(dyadic_data(31)[0], 5, seed=2)
    ctx = _ctx(data, data.label, model, intercept)
    try:
        for t in (0, 4, -1, 2):
            ctx.select_topic(t)
            labels = data.label if t < 0 else data.topics.labels(t)
            fresh = _ctx(data, labels, model, intercept, topics=False)
            try:
                _same(_run(ctx, data, CASES[name], 7 + t), _run(fresh, data, CASES[name], 7 + t), model == "logistic")
            finally:
                fresh.close()
    finally:
        ctx.close()


def test_reloading_topics_keeps_the_loaded_labels():
    data = _with_topics(dyadic_data(32)[0], 3, seed=1)
    ctx = _ctx(data, data.label)
    try:
        w = dyadic_w0(np.random.default_rng(0), data.dim)
        ref = ctx.eval_metrics(0, data.n_rows, w)
        ctx.select_topic(1)
        assert not np.array_equal(ctx.eval_metrics(0, data.n_rows, w), ref)
        ctx.load_topics(data.topics.ptr, data.topics.ids, 3)        # a selected topic's labels are not taken as loaded
        assert np.array_equal(ctx.eval_metrics(0, data.n_rows, w), ref)
        ctx.select_topic(2)
        ctx.select_topic(-1)
        assert np.array_equal(ctx.eval_metrics(0, data.n_rows, w), ref)
    finally:
        ctx.close()


# ---- eval_topics ----------------------------------------------------------------------------------------------------------

def _topic_data(T, n_rows=3000, dim=1500, seed=5):
    from distributed_sgd_b200.utils import synthetic_rcv1
    from distributed_sgd_b200.utils.dataset import Data
    d = synthetic_rcv1(n_rows=n_rows, dim=dim, seed=seed)
    lens = np.diff(d.row_ptr)
    lens[::97] = 0                                                  # empty rows: every score is 0
    keep = np.concatenate([np.arange(d.row_ptr[r], d.row_ptr[r] + lens[r]) for r in range(n_rows)])
    rp = np.concatenate([[0], np.cumsum(lens)]).astype(np.int64)
    return _with_topics(Data(rp, d.col[keep], d.val[keep], d.label, dim), T, seed)


def _weights(data, T, wdim, seed):
    """T weight vectors: random, topic 0 all zero (every score 0), topic 1 with +inf and -inf on the two most frequent
    columns (the values are positive: a NaN score wherever both occur, +-inf where one does)"""
    rng = np.random.default_rng(seed)
    W = rng.standard_normal((T, wdim)) * 0.3
    W[0] = 0.0
    if T > 1:
        c = np.argsort(np.bincount(data.col, minlength=data.dim))[::-1][:2]
        W[1, c[0]], W[1, c[1]] = np.inf, -np.inf
    return W


def _check_words(ctx, data, W, b, e, words):
    T = len(W)
    ids = np.arange(b, e, dtype=np.int32)
    margins = np.stack([ctx.margins(ids, W[t]) for t in range(T)])
    has = data.topics.indicator()[b:e]
    for t in range(T):
        ctx.select_topic(t)
        m = ctx.eval_metrics(b, e, W[t])
        assert np.array_equal(np.delete(words[8 * t:8 * t + 8], 6), np.delete(m, 6)) and words[8 * t + 6] == 0, t
    ctx.select_topic(-1)
    ref = topic_words(margins, has)
    assert np.array_equal(words, ref)
    orc = Oracle(data.row_ptr, data.col, data.val, data.label, data.dim, LAM)
    assert np.array_equal(topics_oracle.topics(orc, data.topics.ptr, data.topics.ids, T, begin=b, n=e - b,
                                               margins=margins), ref)
    return margins


@pytest.mark.parametrize("T,intercept", [(1, False), (103, False), (103, True), (1024, False)])
def test_eval_topics_equals_per_topic_metrics_numpy_and_the_checker(T, intercept):
    data = _topic_data(T, n_rows=1500 if T == 1024 else 3000)
    ctx = _ctx(data, data.label, intercept=intercept)
    try:
        W = _weights(data, T, ctx.wdim, T)
        b, e = 100, data.n_rows
        words = ctx.eval_topics(b, e, W)
        margins = _check_words(ctx, data, W, b, e, words)
        if T > 1:
            assert words[8 * 1 + 7] > 0 and words[8 * T + 4] == 0       # planted NaN scores; a score on every row
            assert words[8 * 0 + 2] + words[8 * 0 + 5] == e - b          # topic 0: no prediction anywhere
        assert words[8 * T + 3] > 0 and words[8 * T] == e - b            # rows without a topic
        assert np.isnan(margins).any() == (T > 1)
    finally:
        ctx.close()


def test_every_model_gives_the_same_words_and_forms_agree():
    from distributed_sgd_b200.native import NativeCtx
    T = 103
    data = _topic_data(T)
    W = _weights(data, T, data.dim, 9)
    ref = None
    for model in ("svm", "logistic", "squared_hinge", "modified_huber"):
        ctx = _ctx(data, data.label, model)
        try:
            words = ctx.eval_topics(0, data.n_rows, W)
            ref = words if ref is None else ref
            assert np.array_equal(words, ref), model
            n = data.n_rows
            # a draw of every position is a permutation of the range; two position halves add up to it
            assert np.array_equal(ctx.eval_sampled_topics(0, n, 77, 0, n, W), ref)
            halves = ctx.eval_sampled_topics(0, n, 78, 0, 1234, W) + ctx.eval_sampled_topics(0, n, 78, 1234, n, W)
            assert np.array_equal(halves, ref)
            perm = np.random.default_rng(4).permutation(n).astype(np.int32)
            assert np.array_equal(ctx.eval_samples_topics(perm, W), ref)
            assert np.array_equal(ctx.eval_samples_topics(perm[::-1].copy(), W), ref)
            rep = np.random.default_rng(5).integers(0, n, size=4000).astype(np.int32)   # repeats count every time
            margins = np.stack([ctx.margins(rep, W[t]) for t in range(T)])
            assert np.array_equal(ctx.eval_samples_topics(rep, W), topic_words(margins, data.topics.indicator()[rep]))
        finally:
            ctx.close()


def test_refusals_launch_nothing():
    from distributed_sgd_b200 import native
    data = _topic_data(4, n_rows=500)
    ctx = _ctx(data, data.label, topics=False)
    W = np.zeros((4, data.dim))
    try:
        n0 = ctx.launch_count()
        with pytest.raises(native.DsgdState, match="no topics loaded"):
            ctx.eval_topics(0, 100, W)
        with pytest.raises(native.DsgdState, match="no topics loaded"):
            ctx.select_topic(0)
        tp, ti = data.topics.ptr, data.topics.ids
        bad = [(4, tp.copy(), ti.copy()) for _ in range(5)]
        bad[0][1][3] = bad[0][1][2] - 1                             # not monotone
        bad[1][2][0] = 4                                            # an id outside [0, T)
        bad[2] = (0, tp, ti)                                        # T outside [1, 1024]
        bad[3] = (1025, tp, ti)
        r = int(np.flatnonzero(np.diff(tp) >= 2)[0])                # a row with two topics, swapped
        bad[4][2][tp[r]], bad[4][2][tp[r] + 1] = ti[tp[r] + 1], ti[tp[r]]
        for T, p, i in bad:
            with pytest.raises(native.DsgdInvalid):
                ctx.load_topics(p, i, T)
        with pytest.raises(native.DsgdState):
            ctx.select_topic(0)                                     # a refused load changed nothing
        assert ctx.launch_count() == n0
        ctx.load_topics(tp, ti, 4)
        n0 = ctx.launch_count()
        with pytest.raises(native.DsgdInvalid, match="3 weight vectors for 4"):
            ctx.eval_topics(0, 100, W[:3])
        with pytest.raises(native.DsgdInvalid, match="outside"):
            ctx.select_topic(4)
        with pytest.raises(native.DsgdRange):
            ctx.eval_samples_topics(np.array([0, 500], dtype=np.int32), W)
        out = np.zeros(40, dtype=np.int64)
        assert native.lib().dsgd_eval_topics(ctx._h, None, 4, 0, 100, out.ctypes.data_as(C.c_void_p)) == native.ERR_INVALID
        assert ctx.launch_count() == n0
        ctx.load_csr(data.row_ptr, data.col, data.val, data.label)  # drops the topics
        with pytest.raises(native.DsgdState, match="no topics loaded"):
            ctx.eval_topics(0, 100, W)
        assert ctx.launch_count() == n0 + 1                         # the repack of load_csr alone
    finally:
        ctx.close()
    actx = _ctx(data, data.label, is_async=True)
    try:
        n0 = actx.launch_count()
        with pytest.raises(native.DsgdState, match="async"):
            actx.load_topics(data.topics.ptr, data.topics.ids, 4)
        with pytest.raises(native.DsgdState, match="async"):
            actx.select_topic(0)
        with pytest.raises(native.DsgdState, match="async"):
            actx.eval_topics(0, 100, W)
        assert actx.launch_count() == n0
    finally:
        actx.close()


# ---- fit_one_vs_rest -------------------------------------------------------------------------------------------------------

def _master(train, test, seed=0):
    from distributed_sgd_b200 import MasterSync, Slave, SparseSVM
    model = SparseSVM(1e-5)
    slave = Slave(0, 0, train, model, False, test_data=test)
    return slave, MasterSync(0, train, test, model, 1, slave=slave, seed=seed)


def test_fit_one_vs_rest_equals_separate_fits():
    import dataclasses
    from distributed_sgd_b200.utils import synthetic_rcv1
    data = _with_topics(synthetic_rcv1(n_rows=6000, dim=3000, seed=8), 6, seed=8)
    train, test = data.split_at(4800)
    kw = dict(max_epochs=2, batch_size=64, learning_rate=0.5, stopping_criterion=lambda tl: False)
    w0 = np.zeros(data.dim)
    slave, m = _master(train, test)
    try:
        ovr = m.fit_one_vs_rest(w0, topics=["T0", "T3", "T5"], **kw)
        after = m.fit(w0, **kw).grad
        report = m.local_topic_report(m.fit_one_vs_rest(w0, **kw))
    finally:
        slave.stop()
    assert ovr.topics == ("T0", "T3", "T5") and ovr.weights.shape == (3, data.dim)
    for k, t in enumerate((0, 3, 5)):
        tr = dataclasses.replace(train, label=train.topics.labels(t), topics=None)
        te = dataclasses.replace(test, label=test.topics.labels(t), topics=None)
        s, fresh = _master(tr, te)
        try:
            assert np.array_equal(fresh.fit(w0, **kw).grad, ovr.weights[k]), t
            assert fresh.history["losses"] == ovr.histories[k]["losses"]
        finally:
            s.stop()
    plain = dataclasses.replace(train, topics=None), dataclasses.replace(test, topics=None)
    s, fresh = _master(*plain)
    try:
        assert np.array_equal(fresh.fit(w0, **kw).grad, after)
    finally:
        s.stop()
    assert report["rows"] == test.n_rows and len(report["topics"]) == 6 and 0.0 <= report["micro_f1"] <= 1.0
