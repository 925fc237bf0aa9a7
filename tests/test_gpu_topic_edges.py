"""The topic kernels at their edges, on the planted layouts of tests/topic_edges_data.py, bit for bit against the numpy
models and the C checkers run over margins folded on the host (tests/row_fold_model.py); each test first requires the
device's dsgd_margins to equal those host margins.

* tuning (k_topic_keys, segmented sort, k_topic_tune): runs ending at thread edges (8q - 1, 8q) and tile edges
  (2048q - 1 .. 2048q + 1), a run longer than a tile with mixed has-topic bytes, a NaN run; every threshold branch (-inf
  chosen, adjacent doubles, 1e308 neighbours, a +inf last group, +inf alone) and every status, fbr equal to a best F1;
  the thresholded evaluation at the returned thresholds counts words 4 and 5;
* the group split: a last group of one topic (T = 1024 over 131 100 positions), one topic per group (T = 3 over
  67 109 825 positions: r times a base list, whose counting words it multiplies by r and whose thresholds it keeps), and
  a workspace reused across requests of different sizes and by the curve and metrics calls;
* ranking, top-k and the topic words at T = 2, 31, 32, 33, 63, 64, 65, 1023 and 1024 with k = 1, 5 and min(T, 32): ties
  of every topic, in one lane, across lanes and at +-inf, a NaN at topic T - 1 alone, rows with every topic; the
  thresholded words at thresholds equal to planted margins; with and without the intercept;
* the host fold on RCV1-shaped rows (multi-chunk) against eval_topics, eval_topic_ranking and tune_topic_thresholds."""
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import pytest

import topic_edges_data as E
from oracle import topic_rank as rank_oracle
from oracle import topic_thresh as thresh_oracle
from oracle import topics as topics_oracle
from oracle.oracle import Oracle
from topic_ranking_model import topic_ranking, topk
from topic_thresholds_model import thresholded_words, tune
from topics_model import topic_words

pytestmark = pytest.mark.gpu

LAM = 2.0 ** -6


def _ctx(lay):
    from distributed_sgd_b200.native import NativeCtx
    d = lay.data
    ctx = NativeCtx(0, d.dim, LAM, intercept=lay.intercept)
    ctx.load_csr(d.row_ptr, d.col, d.val, d.label)
    ctx.load_topics(d.topics.ptr, d.topics.ids, lay.T)
    return ctx


def _orc(data):
    return Oracle(data.row_ptr, data.col, data.val, data.label, data.dim, LAM)


def _host_margins_match(ctx, lay):
    """dsgd_margins of every row equals the host fold, bit for bit; then the host's margins of the request"""
    rows = np.arange(lay.data.n_rows, dtype=np.int32)
    m = lay.row_margins()
    for t in range(lay.T):
        assert E.same_bits(ctx.margins(rows, lay.W[t]), m[t]), t
    return m[:, lay.ids], lay.has()


def _same(a, b):
    """thresholds as int64 views and words"""
    return np.array_equal(a[0].view(np.int64), b[0].view(np.int64)) and np.array_equal(a[1], b[1])


def _check_tune(ctx, lay, got, m, has):
    d = lay.data
    assert _same(got, tune(m, has, lay.fbr))
    chk = thresh_oracle.topic_thresh(_orc(d), d.topics.ptr, d.topics.ids, lay.T, lay.fbr, idx=lay.ids, margins=m)
    assert _same(got, chk)
    thr, words = got
    T = lay.T
    tw = ctx.eval_samples_thresholded_topics(lay.ids, lay.W, thr)
    assert np.array_equal(tw[0:8 * T:8], words[4::8]) and np.array_equal(tw[0:8 * T:8] + tw[3:8 * T:8], words[5::8])
    assert np.array_equal(tw, thresholded_words(m, has, thr))


# ---- tuning: thread and tile edges, value edges ---------------------------------------------------------------------------

def test_tuning_runs_across_thread_and_tile_edges():
    lay = E.tune_tiles()
    ctx = _ctx(lay)
    try:
        m, has = _host_margins_match(ctx, lay)
        got = ctx.tune_topic_thresholds_samples(lay.ids, lay.W)
        _check_tune(ctx, lay, got, m, has)
        words = got[1]
        for t, e in lay.marks["end_at"].items():                   # the chosen group's end: pp - 1 of candidate j
            assert words[8 * t + 6] == 0 and words[8 * t + 5] == e + 1 and words[8 * t + 4] == words[8 * t + 1], t
        assert (words[2::8] == lay.marks["nan_positions"]).all()
    finally:
        ctx.close()


@pytest.mark.parametrize("intercept", [False, True])
def test_tuning_value_edges(intercept):
    lay = E.tune_values(intercept)
    ctx = _ctx(lay)
    try:
        m, has = _host_margins_match(ctx, lay)
        got = ctx.tune_topic_thresholds_samples(lay.ids, lay.W, lay.fbr)
        _check_tune(ctx, lay, got, m, has)
        thr, words = got
        w = {name: words[8 * t:8 * t + 8].tolist() for t, name in enumerate(E.VALUE_TOPICS)}
        tau = dict(zip(E.VALUE_TOPICS, thr.tolist()))
        n = lay.marks["n"]
        assert [w[x][6] for x in E.VALUE_TOPICS] == [0, 0, 0, 0, 0, 1, 2, 0, 3 if intercept else 0]
        assert tau["neg_inf_chosen"] == 0.5 and w["neg_inf_chosen"][7] == 0      # -inf chosen: tau falls back to c_1
        assert tau["adjacent_doubles"] == E.NEXT_UP                              # the midpoint rounds to 1.0
        assert tau["huge_neighbours"] == 1e308 / 2 + E.DBL_MAX / 2 < E.DBL_MAX
        assert tau["inf_last_group"] == np.inf and w["inf_last_group"][4:6] == [n - lay.marks["inf_rows"]] * 2
        assert tau["inf_only"] == np.inf and w["inf_only"][3] == 1 and w["inf_only"][4:6] == [0, 0]
        assert w["below_fbr"][7] == 0 and w["fbr_equal"][7] == 2
        assert 4 * w["fbr_equal"][4] == w["fbr_equal"][1] + w["fbr_equal"][5]           # F1 = 0.5 = fbr: not a fallback
    finally:
        ctx.close()


# ---- the group split ------------------------------------------------------------------------------------------------------

def _checker_in_chunks(lay, chunks=8):
    """the checker's (thresholds, words) from its own dots, its topics split over threads (ctypes drops the GIL)"""
    from distributed_sgd_b200.utils.dataset import Topics
    d = lay.data
    orc = _orc(d)
    has = d.topics.indicator()
    bounds = np.linspace(0, lay.T, chunks + 1).astype(int)

    def run(a, b):
        tp = Topics.from_indicator(has[:, a:b], [str(t) for t in range(a, b)])
        return thresh_oracle.topic_thresh(orc, tp.ptr, tp.ids, b - a, lay.fbr, W=lay.W[a:b], idx=lay.ids)

    with ThreadPoolExecutor(chunks) as ex:
        parts = list(ex.map(run, bounds[:-1], bounds[1:]))
    return np.concatenate([p[0] for p in parts]), np.concatenate([p[1] for p in parts])


def test_last_group_of_one_topic():
    T, n = 1024, 131_100
    assert E.tune_group(n, T) == T - 1                             # groups of 1023 topics and of 1
    lay = E.tune_groups(T, n)
    ctx = _ctx(lay)
    try:
        _host_margins_match(ctx, lay)
        got = ctx.tune_topic_thresholds_samples(lay.ids, lay.W)
        assert _same(got, _checker_in_chunks(lay))
        last = got[1][8 * (T - 1):]
        assert last[6] == 0 and last[7] > 0 and last[3] == lay.data.n_rows
        tw = ctx.eval_samples_thresholded_topics(lay.ids, lay.W, got[0])
        assert np.array_equal(tw[0:8 * T:8], got[1][4::8]) and np.array_equal(tw[0:8 * T:8] + tw[3:8 * T:8], got[1][5::8])
    finally:
        ctx.close()


def _curve_and_metrics(ctx, lay):
    c = ctx.eval_samples_curve(lay.ids, lay.W[1])
    return [np.asarray(x) for x in c] + [ctx.eval_samples_metrics(lay.ids, lay.W[2]), ctx.eval_metrics(0, 300, lay.W[0])]


def _bits(x):
    x = np.asarray(x)
    return x.view(np.int64) if x.dtype == np.float64 else x


def _equal_lists(a, b):
    return len(a) == len(b) and all(np.array_equal(_bits(x), _bits(y)) for x, y in zip(a, b))


def test_one_topic_per_group_and_a_reused_workspace():
    base = E.tune_groups(3, 1025)
    r = 65_473
    big_ids = np.tile(base.ids, r)
    assert big_ids.size > 1 << 26 and E.tune_group(big_ids.size, 3) == 1 and E.tune_group(base.ids.size, 3) == 3
    ctx = _ctx(base)
    try:
        m, has = _host_margins_match(ctx, base)
        small = ctx.tune_topic_thresholds_samples(base.ids, base.W)
        _check_tune(ctx, base, small, m, has)
        side = _curve_and_metrics(ctx, base)
    finally:
        ctx.close()
    ctx = _ctx(base)
    try:
        big = ctx.tune_topic_thresholds_samples(big_ids, base.W)
        # F1 does not change when every count is multiplied by r: thresholds, D, status and j stay, the counts scale
        assert np.array_equal(big[0].view(np.int64), small[0].view(np.int64))
        for k in range(8):
            scale = r if k in (0, 1, 2, 4, 5) else 1
            assert np.array_equal(big[1][k::8], scale * small[1][k::8]), k
        assert _equal_lists(_curve_and_metrics(ctx, base), side)
        assert _same(ctx.tune_topic_thresholds_samples(base.ids, base.W), small)
        assert _equal_lists(_curve_and_metrics(ctx, base), side)
        assert _same(ctx.tune_topic_thresholds_samples(big_ids, base.W), big)
        assert _equal_lists(_curve_and_metrics(ctx, base), side)
    finally:
        ctx.close()


# ---- ranking and topic words at every warp shape --------------------------------------------------------------------------

@pytest.mark.parametrize("intercept", [False, True])
@pytest.mark.parametrize("T", E.RANK_TS)
def test_ranking_and_topic_words_at_every_warp_shape(T, intercept):
    lay = E.rank_layout(T, intercept)
    d = lay.data
    ctx = _ctx(lay)
    try:
        m, has = _host_margins_match(ctx, lay)
        orc = _orc(d)
        K = min(T, 32)
        ref = topic_ranking(m, has, K)
        assert ref[0][4] > 0 and ref[0][2] > 0                      # rows with every topic; NaN rows
        for k in E.rank_ks(T):
            words, sums = ctx.eval_samples_topic_ranking(lay.ids, lay.W, k)
            rw, rs = E.slice_k(*ref, K, k)
            assert np.array_equal(words, rw), (k, words[:8 + k], rw[:8 + k])
            assert np.array_equal(sums.view(np.int64), rs.view(np.int64)), (k, sums, rs)
            cw, cs = rank_oracle.topic_rank(orc, d.topics.ptr, d.topics.ids, T, k, idx=lay.ids, margins=m)
            assert np.array_equal(cw, words) and np.array_equal(cs.view(np.int64), sums.view(np.int64))
            got_ids, got_m = ctx.topics_topk(lay.ids, lay.W, k)
            ref_ids, ref_m = topk(m, k)
            assert np.array_equal(got_ids, ref_ids), k
            assert E.same_bits(got_m, ref_m)
        tw = ctx.eval_samples_topics(lay.ids, lay.W)
        assert np.array_equal(tw, topic_words(m, has))
        assert np.array_equal(tw, topics_oracle.topics(orc, d.topics.ptr, d.topics.ids, T, idx=lay.ids, margins=m))
        for thr in E.rank_thresholds(lay):
            assert np.array_equal(ctx.eval_samples_thresholded_topics(lay.ids, lay.W, thr), thresholded_words(m, has, thr))
    finally:
        ctx.close()


# ---- the host fold on RCV1-shaped rows ------------------------------------------------------------------------------------

@pytest.mark.parametrize("intercept", [False, True])
def test_host_fold_on_rcv1_shaped_rows(intercept):
    from test_gpu_topics import _ctx as topic_ctx, _topic_data, _weights
    T = 103
    data = _topic_data(T, n_rows=1500)
    assert np.diff(data.row_ptr).max() > 128                        # multi-chunk rows
    ctx = topic_ctx(data, data.label, intercept=intercept)
    try:
        W = _weights(data, T, ctx.wdim, 17)
        n = data.n_rows
        rows = np.arange(n, dtype=np.int32)
        m = E.host_margins(data, W, rows, intercept)
        for t in range(T):
            assert E.same_bits(ctx.margins(rows, W[t]), m[t]), t
        has = data.topics.indicator()
        orc = _orc(data)
        tp, ti = data.topics.ptr, data.topics.ids
        words = ctx.eval_topics(0, n, W)
        assert np.array_equal(words, topic_words(m, has))
        assert np.array_equal(words, topics_oracle.topics(orc, tp, ti, T, begin=0, n=n, margins=m))
        rw, rs = ctx.eval_topic_ranking(0, n, W, 5)
        ref = topic_ranking(m, has, 5)
        assert np.array_equal(rw, ref[0]) and np.array_equal(rs.view(np.int64), ref[1].view(np.int64))
        cw, cs = rank_oracle.topic_rank(orc, tp, ti, T, 5, begin=0, n=n, margins=m)
        assert np.array_equal(cw, rw) and np.array_equal(cs.view(np.int64), rs.view(np.int64))
        got = ctx.tune_topic_thresholds(0, n, W)
        assert _same(got, tune(m, has))
        assert _same(got, thresh_oracle.topic_thresh(orc, tp, ti, T, 0.0, begin=0, n=n, margins=m))
    finally:
        ctx.close()
