"""The JNI shim's topic-ranking natives (evalTopicRanking and its sampled and list forms, topicsTopk) run against the library
through the stand-in JNIEnv of tests/test_gpu_jni.py: valid calls equal NativeCtx's results bit for bit on a plain and an
intercept context, and every array shorter than the header names (or a W of the wrong length) is refused before any launch
with the outputs untouched."""
import numpy as np
import pytest

from test_gpu_jni import F64, I64, KEY, SENTINEL, Shim, out

pytestmark = pytest.mark.gpu

T, N_ROWS, K = 6, 3000, 3
WORDS = 8 + K + 7 * (2 + K)
I32 = np.int32


@pytest.fixture(scope="module")
def setup(tmp_path_factory):
    import dataclasses
    from distributed_sgd_b200.native import NativeCtx
    from distributed_sgd_b200.utils import synthetic_rcv1, synthetic_topics
    shim = Shim(str(tmp_path_factory.mktemp("jni") / "libdsgd_jni_topic_ranking.so"))
    data = synthetic_rcv1(n_rows=N_ROWS, dim=800, seed=4)
    data = dataclasses.replace(data, topics=synthetic_topics(data, T, seed=4))
    ctxs = {}
    for intercept in (False, True):
        c = NativeCtx(0, data.dim, 1e-4, intercept=intercept)
        c.load_csr(data.row_ptr, data.col, data.val, data.label)
        c.load_topics(data.topics.ptr, data.topics.ids, T)
        ctxs[intercept] = c
    yield shim, ctxs, data
    for c in ctxs.values():
        c.close()


@pytest.mark.parametrize("intercept", [False, True])
def test_ranking_natives_match_native_ctx(setup, intercept):
    shim, ctxs, _ = setup
    ctx = ctxs[intercept]
    h = ctx._h.value
    W = np.random.default_rng(1).standard_normal((T, ctx.wdim)) * 0.2
    Wf = W.reshape(-1).copy()
    o, s = out(WORDS, I64), out(2 + K, F64)
    assert shim("evalTopicRanking", h, Wf, T, K, 100, 2100, o, s) == 0
    ref = ctx.eval_topic_ranking(100, 2100, W, K)
    assert np.array_equal(o, ref[0]) and np.array_equal(s, ref[1])
    o, s = out(WORDS, I64), out(2 + K, F64)
    assert shim("evalSampledTopicRanking", h, Wf, T, K, 0, N_ROWS, KEY - (1 << 64), 10, 900, o, s) == 0
    ref = ctx.eval_sampled_topic_ranking(0, N_ROWS, KEY, 10, 900, W, K)
    assert np.array_equal(o, ref[0]) and np.array_equal(s, ref[1])
    ids = np.random.default_rng(2).integers(0, N_ROWS, size=777).astype(np.int32)
    o, s = out(WORDS, I64), out(2 + K, F64)
    assert shim("evalSamplesTopicRanking", h, Wf, T, K, ids, o, s) == 0
    ref = ctx.eval_samples_topic_ranking(ids, W, K)
    assert np.array_equal(o, ref[0]) and np.array_equal(s, ref[1])
    oi, om = out(ids.size * K, I32), out(ids.size * K, F64)
    assert shim("topicsTopk", h, Wf, T, K, ids, oi, om) == 0
    ri, rm = ctx.topics_topk(ids, W, K)
    assert np.array_equal(oi, ri.reshape(-1)) and np.array_equal(om, rm.reshape(-1), equal_nan=True)


def test_wrong_lengths_are_refused(setup):
    from distributed_sgd_b200 import native
    shim, ctxs, _ = setup
    ctx = ctxs[False]
    h = ctx._h.value
    n0 = ctx.launch_count()
    W = np.zeros(T * ctx.dim)
    ids = np.arange(10, dtype=np.int32)
    for w, o, s in ((W[:-1].copy(), out(WORDS, I64), out(2 + K, F64)), (np.append(W, 0.0), out(WORDS, I64), out(2 + K, F64)),
                    (W, out(WORDS - 1, I64), out(2 + K, F64)), (W, out(WORDS, I64), out(1 + K, F64))):
        assert shim("evalTopicRanking", h, w, T, K, 0, 100, o, s) == native.ERR_INVALID
        assert shim("evalSampledTopicRanking", h, w, T, K, 0, N_ROWS, 5, 0, 100, o, s) == native.ERR_INVALID
        assert shim("evalSamplesTopicRanking", h, w, T, K, ids, o, s) == native.ERR_INVALID
        assert (o.view(np.uint8) == SENTINEL).all() and (s.view(np.uint8) == SENTINEL).all()
    for w, oi, om in ((W[:-1].copy(), out(10 * K, I32), out(10 * K, F64)), (W, out(10 * K - 1, I32), out(10 * K, F64)),
                      (W, out(10 * K, I32), out(10 * K - 1, F64))):
        assert shim("topicsTopk", h, w, T, K, ids, oi, om) == native.ERR_INVALID
        assert (oi.view(np.uint8) == SENTINEL).all() and (om.view(np.uint8) == SENTINEL).all()
    assert shim("topicsTopk", h, W, T, 0, ids, out(10, I32), out(10, F64)) == native.ERR_INVALID
    assert shim("topicsTopk", h, W, T, 33, ids, out(10 * 33, I32), out(10 * 33, F64)) == native.ERR_INVALID
    assert ctx.launch_count() == n0
