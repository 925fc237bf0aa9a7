"""Ranking a row's topics on the device (dsgd_eval*_topic_ranking, dsgd_topics_topk; DESIGN.md §4.22), bit for bit:

* the words and sums equal the numpy restatement over T dsgd_margins calls and the C checker, at T = 1, 103 and 1024 and
  k = 1, 5 and min(T, 32), with the intercept, with planted ties (two equal weight vectors and an all-zero one, so every
  score of that topic is 0) and planted NaN scores; every model flag gives the same words;
* the range, sampled and list forms agree, a shuffled list gives the range's result, and two halves' words add up to the
  whole, their merged limbs giving the whole's sums;
* hits@1 equals dsgd_eval_topics' top-1 word on rows without a NaN score;
* topics_topk equals a numpy ordering of the margins with the tie rule, also on a context without topics;
* every refusal leaves the launch count unchanged."""
import ctypes as C

import numpy as np
import pytest

from oracle import topic_rank as rank_oracle
from oracle.oracle import Oracle
from test_gpu_topics import LAM, _ctx, _topic_data, _weights
from topic_ranking_model import topic_ranking, topk

pytestmark = pytest.mark.gpu


def _planted_weights(data, T, wdim, seed):
    """_weights (topic 0 all zero, topic 1 with +-inf: NaN scores) and, with T > 3, topic 3 equal to topic 2"""
    W = _weights(data, T, wdim, seed)
    if T > 3:
        W[3] = W[2]
    return W


def _margins(ctx, ids, W):
    return np.stack([ctx.margins(ids, W[t]) for t in range(len(W))])


def _merge(words, k):
    """words (summed over calls) with the carries of every limb block propagated"""
    out = np.array(words, dtype=np.int64)
    for s in range(2 + k):
        q = out[8 + k + 7 * s:8 + k + 7 * s + 6]
        for i in range(5):
            q[i + 1] += q[i] >> 40
            q[i] &= (1 << 40) - 1
    return out


@pytest.mark.parametrize("T,intercept", [(1, False), (103, False), (103, True), (1024, False)])
def test_words_and_sums_equal_numpy_and_the_checker(T, intercept):
    from distributed_sgd_b200.ml.one_vs_rest import limbs_value
    data = _topic_data(T, n_rows=700 if T == 1024 else 3000)
    ctx = _ctx(data, data.label, intercept=intercept)
    try:
        W = _planted_weights(data, T, ctx.wdim, T)
        b, e = 100, data.n_rows
        ids = np.arange(b, e, dtype=np.int32)
        margins = _margins(ctx, ids, W)
        has = data.topics.indicator()[b:e]
        orc = Oracle(data.row_ptr, data.col, data.val, data.label, data.dim, LAM)
        for k in sorted({1, min(5, T), min(T, 32)}):
            words, sums = ctx.eval_topic_ranking(b, e, W, k)
            ref_w, ref_s = topic_ranking(margins, has, k)
            assert np.array_equal(words, ref_w), (k, words[:8 + k], ref_w[:8 + k])
            assert np.array_equal(sums, ref_s), (k, sums, ref_s)
            cw, cs = rank_oracle.topic_rank(orc, data.topics.ptr, data.topics.ids, T, k, begin=b, n=e - b, margins=margins)
            assert np.array_equal(cw, words) and np.array_equal(cs, sums)
            assert [limbs_value(words[8 + k + 7 * s:8 + k + 7 * s + 7]) for s in range(2 + k)] == list(sums)
            assert words[0] == e - b == words[1] + words[2] + words[3] and words[3] > 0 and words[1] > 0
            if T > 1:
                assert words[2] > 0                                     # the planted NaN scores
    finally:
        ctx.close()


def test_every_model_gives_the_same_words_and_forms_agree():
    T, k = 103, 5
    data = _topic_data(T)
    W = _planted_weights(data, T, data.dim, 9)
    n = data.n_rows
    ref = None
    for model in ("svm", "logistic", "squared_hinge", "modified_huber"):
        ctx = _ctx(data, data.label, model)
        try:
            words, sums = ctx.eval_topic_ranking(0, n, W, k)
            ref = (words, sums) if ref is None else ref
            assert np.array_equal(words, ref[0]) and np.array_equal(sums, ref[1]), model
            # a draw of every position is a permutation of the range; a shuffled list too
            for got in (ctx.eval_sampled_topic_ranking(0, n, 77, 0, n, W, k),
                        ctx.eval_samples_topic_ranking(np.random.default_rng(4).permutation(n).astype(np.int32), W, k)):
                assert np.array_equal(got[0], ref[0]) and np.array_equal(got[1], ref[1])
            # two halves: words add up, merged limbs give the whole's sums
            a = ctx.eval_topic_ranking(0, 1234, W, k)
            c = ctx.eval_topic_ranking(1234, n, W, k)
            assert np.array_equal(_merge(a[0] + c[0], k), ref[0])
            h = ctx.eval_sampled_topic_ranking(0, n, 78, 0, 999, W, k)[0] + ctx.eval_sampled_topic_ranking(0, n, 78, 999, n, W, k)[0]
            assert np.array_equal(_merge(h, k), ref[0])
            if model == "svm":
                rep = np.random.default_rng(5).integers(0, n, size=3000).astype(np.int32)   # repeats count every time
                got = ctx.eval_samples_topic_ranking(rep, W, k)
                ref_rep = topic_ranking(_margins(ctx, rep, W), data.topics.indicator()[rep], k)
                assert np.array_equal(got[0], ref_rep[0]) and np.array_equal(got[1], ref_rep[1])
        finally:
            ctx.close()


def test_hits_at_one_is_the_top1_word_without_nan_scores():
    T = 103
    data = _topic_data(T)
    ctx = _ctx(data, data.label)
    try:
        W = np.random.default_rng(2).standard_normal((T, data.dim)) * 0.3
        W[5] = W[7]                                                     # ties between two topics
        words, _ = ctx.eval_topic_ranking(0, data.n_rows, W, 1)
        tw = ctx.eval_topics(0, data.n_rows, W)
        assert words[2] == 0 and tw[8 * T + 4] == 0                     # no NaN score anywhere
        assert words[8] == tw[8 * T + 2] and words[3] == tw[8 * T + 3]
    finally:
        ctx.close()


@pytest.mark.parametrize("intercept,topics", [(False, True), (True, True), (False, False)])
def test_topics_topk_equals_numpy_order(intercept, topics):
    T = 103
    data = _topic_data(T)
    ctx = _ctx(data, data.label, intercept=intercept, topics=topics)
    try:
        W = _planted_weights(data, T, ctx.wdim, 3)
        ids = np.random.default_rng(6).integers(0, data.n_rows, size=2500).astype(np.int32)
        margins = _margins(ctx, ids, W)
        for k in (1, 5, 32):
            got_ids, got_m = ctx.topics_topk(ids, W, k)
            ref_ids, ref_m = topk(margins, k)
            assert got_ids.shape == (ids.size, k) and np.array_equal(got_ids, ref_ids)
            assert np.array_equal(got_m.view(np.int64)[~np.isnan(got_m)], ref_m.view(np.int64)[~np.isnan(ref_m)])
            assert np.array_equal(np.isnan(got_m), got_ids < 0)
        # every topic with +inf and -inf on the two planted columns: the rows holding both have no non-NaN score
        W2 = W.copy()
        W2[:, np.isinf(W[1])] = W[1, np.isinf(W[1])]
        m2 = _margins(ctx, ids, W2)
        got_ids, got_m = ctx.topics_topk(ids, W2, 5)
        all_nan = np.isnan(m2).all(axis=0)
        assert all_nan.any() and (got_ids[all_nan] == -1).all() and np.isnan(got_m[all_nan]).all()
        assert np.array_equal(got_ids, topk(m2, 5)[0])
        # a row whose scores all tie (topics 0 and 2 .. T-1 on an empty row: all 0; topic 1 too): the lowest ids first
        empty = np.flatnonzero(np.diff(data.row_ptr) == 0)[:1].astype(np.int32)
        if empty.size and not intercept:
            assert ctx.topics_topk(empty, W, 4)[0].tolist() == [[0, 1, 2, 3]]
    finally:
        ctx.close()


def test_refusals_launch_nothing():
    from distributed_sgd_b200 import native
    T = 4
    data = _topic_data(T, n_rows=500)
    ctx = _ctx(data, data.label, topics=False)
    W = np.zeros((T, data.dim))
    lib = native.lib()
    try:
        n0 = ctx.launch_count()
        with pytest.raises(native.DsgdState, match="no topics loaded"):
            ctx.eval_topic_ranking(0, 100, W, 2)
        ctx.load_topics(data.topics.ptr, data.topics.ids, T)
        n0 = ctx.launch_count()
        with pytest.raises(native.DsgdInvalid, match="3 weight vectors for 4"):
            ctx.eval_topic_ranking(0, 100, W[:3], 2)
        for k in (0, 5, 33):
            with pytest.raises(native.DsgdInvalid, match="k"):
                ctx.eval_topic_ranking(0, 100, W, k)
        with pytest.raises(native.DsgdRange):
            ctx.eval_samples_topic_ranking(np.array([0, 500], dtype=np.int32), W, 2)
        words, sums = np.zeros(8 + 2 + 28, dtype=np.int64), np.zeros(4)
        p = lambda a: a.ctypes.data_as(C.c_void_p)
        assert lib.dsgd_eval_topic_ranking(ctx._h, None, T, 2, 0, 100, p(words), p(sums)) == native.ERR_INVALID
        assert lib.dsgd_eval_topic_ranking(ctx._h, p(W), T, 2, 0, 100, None, p(sums)) == native.ERR_INVALID
        assert lib.dsgd_eval_topic_ranking(ctx._h, p(W), T, 2, 0, 100, p(words), None) == native.ERR_INVALID
        ids = np.arange(10, dtype=np.int32)
        for WW, k in ((W[:0].reshape(0, data.dim), 1), (np.zeros((1025, data.dim)), 1), (W, 0), (W, 5)):
            with pytest.raises(native.DsgdInvalid):
                ctx.topics_topk(ids, WW, k)
        oi, om = np.zeros(20, dtype=np.int32), np.zeros(20)
        assert lib.dsgd_topics_topk(ctx._h, p(W), T, 2, p(ids), 10, None, p(om)) == native.ERR_INVALID
        assert lib.dsgd_topics_topk(ctx._h, p(W), T, 2, p(ids), 10, p(oi), None) == native.ERR_INVALID
        assert lib.dsgd_topics_topk(ctx._h, None, T, 2, p(ids), 10, p(oi), p(om)) == native.ERR_INVALID
        with pytest.raises(native.DsgdRange):
            ctx.topics_topk(np.array([0, 500], dtype=np.int32), W, 2)
        assert ctx.launch_count() == n0
    finally:
        ctx.close()
    actx = _ctx(data, data.label, is_async=True)
    try:
        n0 = actx.launch_count()
        with pytest.raises(native.DsgdState, match="async"):
            actx.eval_topic_ranking(0, 100, W, 2)
        with pytest.raises(native.DsgdState, match="async"):
            actx.topics_topk(np.arange(10, dtype=np.int32), W, 2)
        assert actx.launch_count() == n0
    finally:
        actx.close()
