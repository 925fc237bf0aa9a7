"""Per-topic decision thresholds on the device (dsgd_tune_topic_thresholds*, dsgd_eval*_thresholded_topics; DESIGN.md
§4.23), bit for bit:

* the thresholds and words equal the C checker and the numpy restatement over T dsgd_margins calls at T = 1, 103 and 1024,
  with the intercept, a topic whose margins are all 0 and one with NaN and +-inf margins; at T = 1024 over 140 000 rows the
  topics go in two groups, and the result is still the checker's;
* every model flag gives the same result; the sampled form over every position and a shuffled list give the range's; a
  list with repeats counts each; dsgd_select_topic changes nothing;
* the chosen candidate's (tp, predicted) is point j of dsgd_eval_curve after dsgd_select_topic(t), and its F1 is the
  highest of that curve's points;
* the thresholded evaluation at tau = 0 and -0 is dsgd_eval_topics, at +-inf it predicts every row below +inf or none, at
  the tuned thresholds it counts words 4 and 5 on the tuning rows, and it equals the numpy restatement in every form;
* every refusal leaves the launch count unchanged."""
import ctypes as C
from fractions import Fraction

import numpy as np
import pytest

from oracle import topic_thresh as thresh_oracle
from oracle.oracle import Oracle
from test_gpu_topics import LAM, _ctx, _topic_data, _weights
from topic_thresholds_model import counts_at, thresholded_words, tune

pytestmark = pytest.mark.gpu


def _margins(ctx, ids, W):
    return np.stack([ctx.margins(ids, W[t]) for t in range(len(W))])


def _same(a, b):
    """thresholds and words, bit for bit"""
    return np.array_equal(a[0].view(np.int64), b[0].view(np.int64)) and np.array_equal(a[1], b[1])


def _check(ctx, data, W, ids, got, fbr=0.0, model=True):
    T = len(W)
    margins = _margins(ctx, ids, W)
    has = data.topics.indicator()[ids]
    orc = Oracle(data.row_ptr, data.col, data.val, data.label, data.dim, LAM)
    ref = thresh_oracle.topic_thresh(orc, data.topics.ptr, data.topics.ids, T, fbr, idx=ids, margins=margins)
    assert _same(got, ref)
    if model:
        assert _same(got, tune(margins, has, fbr))
    for t in range(T):
        w = got[1][8 * t:8 * t + 8]
        assert counts_at(margins[t], has[:, t], got[0][t]) == (w[4], w[5])
    return margins, has


@pytest.mark.parametrize("T,intercept,fbr", [(1, False, 0.0), (103, False, 0.0), (103, True, 0.3), (1024, False, 0.0)])
def test_thresholds_equal_the_checker_and_numpy(T, intercept, fbr):
    data = _topic_data(T, n_rows=700 if T == 1024 else 3000)
    ctx = _ctx(data, data.label, intercept=intercept)
    try:
        W = _weights(data, T, ctx.wdim, T)
        b, e = 100, data.n_rows
        got = ctx.tune_topic_thresholds(b, e, W, fbr)
        _check(ctx, data, W, np.arange(b, e, dtype=np.int32), got, fbr)
        status = got[1][6::8]
        assert (status == 0).any() and got[1][0] == e - b
        if T > 1:
            assert got[1][2 + 8] > 0                                # topic 1's NaN margins
    finally:
        ctx.close()


def test_two_groups_of_topics_equal_the_checker():
    T, n = 1024, 140_000                                            # G = floor(2^27 / n) = 958: two groups
    data = _topic_data(T, n_rows=n, dim=600)
    ctx = _ctx(data, data.label)
    try:
        W = _weights(data, T, ctx.wdim, 21)
        got = ctx.tune_topic_thresholds(0, n, W)
        _check(ctx, data, W, np.arange(n, dtype=np.int32), got, model=False)
        perm = np.random.default_rng(3).permutation(n).astype(np.int32)
        assert _same(ctx.tune_topic_thresholds_samples(perm, W), got)
        tw = ctx.eval_thresholded_topics(0, n, W, got[0])
        assert np.array_equal(tw[0:8 * T:8], got[1][4::8]) and np.array_equal(tw[0:8 * T:8] + tw[3:8 * T:8], got[1][5::8])
    finally:
        ctx.close()


def test_every_model_and_row_form_agree_and_select_topic_changes_nothing():
    T = 103
    data = _topic_data(T)
    W = _weights(data, T, data.dim, 9)
    n = data.n_rows
    ref = None
    for model in ("svm", "logistic", "squared_hinge", "modified_huber"):
        ctx = _ctx(data, data.label, model)
        try:
            got = ctx.tune_topic_thresholds(0, n, W)
            ref = got if ref is None else ref
            assert _same(got, ref), model
            assert _same(ctx.tune_topic_thresholds_sampled(0, n, 77, 0, n, W), ref)
            assert _same(ctx.tune_topic_thresholds_samples(np.random.default_rng(4).permutation(n).astype(np.int32), W), ref)
            if model == "svm":
                rep = np.random.default_rng(5).integers(0, n, size=3000).astype(np.int32)   # repeats count every time
                _check(ctx, data, W, rep, ctx.tune_topic_thresholds_samples(rep, W, 0.1), 0.1)
                for t in (0, 5, T - 1):
                    ctx.select_topic(t)
                    assert _same(ctx.tune_topic_thresholds(0, n, W), ref)
                ctx.select_topic(-1)
        finally:
            ctx.close()


def test_chosen_candidate_is_the_best_point_of_the_curve():
    T = 103
    data = _topic_data(T)
    ctx = _ctx(data, data.label)
    try:
        W = np.random.default_rng(2).standard_normal((T, data.dim)) * 0.3
        n = data.n_rows
        thr, words = ctx.tune_topic_thresholds(0, n, W)
        checked = 0
        for t in range(T):
            rows, P, nan, D, tp, pp, status, j = (int(x) for x in words[8 * t:8 * t + 8])
            if status != 0:
                continue
            ctx.select_topic(t)
            _, _, thr_c, tp_c, fp_c = ctx.eval_curve(0, n, W[t])
            assert len(thr_c) == D and nan == 0
            assert tp_c[j] == tp and tp_c[j] + fp_c[j] == pp              # curve threshold -c_j: rows with m <= c_j
            best = max(Fraction(2 * int(a), P + int(a) + int(f)) for a, f in zip(tp_c, fp_c))
            assert Fraction(2 * tp, P + pp) == best
            assert all(Fraction(2 * int(a), P + int(a) + int(f)) < best for a, f in zip(tp_c[:j], fp_c[:j]))
            checked += 1
        ctx.select_topic(-1)
        assert checked > T // 2
    finally:
        ctx.close()


@pytest.mark.parametrize("intercept", [False, True])
def test_thresholded_evaluation(intercept):
    T = 103
    data = _topic_data(T)
    ctx = _ctx(data, data.label, intercept=intercept)
    try:
        W = _weights(data, T, ctx.wdim, 12)
        n = data.n_rows
        ids = np.arange(n, dtype=np.int32)
        m, has = _margins(ctx, ids, W), data.topics.indicator()
        plain = ctx.eval_topics(0, n, W)
        assert np.array_equal(ctx.eval_thresholded_topics(0, n, W, np.zeros(T)), plain)
        assert np.array_equal(ctx.eval_thresholded_topics(0, n, W, np.full(T, -0.0)), plain)
        for tau in (np.inf, -np.inf):
            got = ctx.eval_thresholded_topics(0, n, W, np.full(T, tau))
            assert np.array_equal(got, thresholded_words(m, has, np.full(T, tau)))
            present = got[0:8 * T:8] + got[3:8 * T:8]
            assert np.array_equal(present, (m < tau).sum(axis=1))
            if tau < 0:
                assert not present.any()
        thr, words = ctx.tune_topic_thresholds(0, 2000, W)
        tw = ctx.eval_thresholded_topics(0, 2000, W, thr)
        assert np.array_equal(tw[0:8 * T:8], words[4::8]) and np.array_equal(tw[0:8 * T:8] + tw[3:8 * T:8], words[5::8])
        assert np.array_equal(tw, thresholded_words(m[:, :2000], has[:2000], thr))
        assert np.array_equal(ctx.eval_thresholded_topics(2000, n, W, thr), thresholded_words(m[:, 2000:], has[2000:], thr))
        assert np.array_equal(ctx.eval_sampled_thresholded_topics(0, n, 5, 0, n, W, thr),
                              ctx.eval_thresholded_topics(0, n, W, thr))
        rep = np.random.default_rng(8).integers(0, n, size=2500).astype(np.int32)
        assert np.array_equal(ctx.eval_samples_thresholded_topics(rep, W, thr), thresholded_words(m[:, rep], has[rep], thr))
    finally:
        ctx.close()


def test_refusals_launch_nothing():
    from distributed_sgd_b200 import native
    T = 4
    data = _topic_data(T, n_rows=500)
    ctx = _ctx(data, data.label, topics=False)
    W = np.zeros((T, data.dim))
    lib = native.lib()
    p = lambda a: a.ctypes.data_as(C.c_void_p)
    try:
        n0 = ctx.launch_count()
        with pytest.raises(native.DsgdState, match="no topics loaded"):
            ctx.tune_topic_thresholds(0, 100, W)
        with pytest.raises(native.DsgdState, match="no topics loaded"):
            ctx.eval_thresholded_topics(0, 100, W, np.zeros(T))
        ctx.load_topics(data.topics.ptr, data.topics.ids, T)
        n0 = ctx.launch_count()
        with pytest.raises(native.DsgdInvalid, match="3 weight vectors for 4"):
            ctx.tune_topic_thresholds(0, 100, W[:3])
        for fbr in (np.nan, -0.1, 1.5):
            with pytest.raises(native.DsgdInvalid, match="fbr"):
                ctx.tune_topic_thresholds(0, 100, W, fbr)
            with pytest.raises(native.DsgdInvalid, match="fbr"):
                ctx.tune_topic_thresholds_sampled(0, 500, 3, 0, 100, W, fbr)
        with pytest.raises(native.DsgdRange):
            ctx.tune_topic_thresholds_samples(np.array([0, 500], dtype=np.int32), W)
        with pytest.raises(native.DsgdInvalid, match="NaN"):
            ctx.eval_thresholded_topics(0, 100, W, np.array([0.0, np.nan, 0.0, 0.0]))
        with pytest.raises(native.DsgdInvalid, match="NaN"):
            ctx.eval_sampled_thresholded_topics(0, 500, 3, 0, 100, W, np.array([0.0, 0.0, 0.0, np.nan]))
        with pytest.raises(native.DsgdInvalid, match="3 weight vectors for 4"):
            ctx.eval_thresholded_topics(0, 100, W[:3], np.zeros(3))
        thr, words, out = np.zeros(T), np.zeros(8 * T, dtype=np.int64), np.zeros(8 * T + 8, dtype=np.int64)
        assert lib.dsgd_tune_topic_thresholds(ctx._h, p(W), T, 0.0, 0, 100, None, p(words)) == native.ERR_INVALID
        assert lib.dsgd_tune_topic_thresholds(ctx._h, p(W), T, 0.0, 0, 100, p(thr), None) == native.ERR_INVALID
        assert lib.dsgd_tune_topic_thresholds(ctx._h, None, T, 0.0, 0, 100, p(thr), p(words)) == native.ERR_INVALID
        assert lib.dsgd_eval_thresholded_topics(ctx._h, p(W), T, None, 0, 100, p(out)) == native.ERR_INVALID
        assert lib.dsgd_eval_thresholded_topics(ctx._h, p(W), T, p(thr), 0, 100, None) == native.ERR_INVALID
        assert lib.dsgd_eval_thresholded_topics(ctx._h, None, T, p(thr), 0, 100, p(out)) == native.ERR_INVALID
        assert ctx.launch_count() == n0
    finally:
        ctx.close()
    actx = _ctx(data, data.label, is_async=True)
    try:
        n0 = actx.launch_count()
        with pytest.raises(native.DsgdState, match="async"):
            actx.tune_topic_thresholds(0, 100, W)
        with pytest.raises(native.DsgdState, match="async"):
            actx.eval_thresholded_topics(0, 100, W, np.zeros(T))
        assert actx.launch_count() == n0
    finally:
        actx.close()
