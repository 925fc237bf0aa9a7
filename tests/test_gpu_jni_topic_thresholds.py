"""The JNI shim's topic threshold natives (tuneTopicThresholds, evalThresholdedTopics and their sampled and list forms) run
against the library through the stand-in JNIEnv of tests/test_gpu_jni.py: valid calls equal NativeCtx's results bit for bit
on a plain and an intercept context, and every array shorter than the header names (or a W of the wrong length) is refused
before any launch with the outputs untouched."""
import numpy as np
import pytest

from test_gpu_jni import F64, I64, KEY, SENTINEL, Shim, out

pytestmark = pytest.mark.gpu

T, N_ROWS = 6, 3000
WORDS = 8 * T + 8


@pytest.fixture(scope="module")
def setup(tmp_path_factory):
    import dataclasses
    from distributed_sgd_b200.native import NativeCtx
    from distributed_sgd_b200.utils import synthetic_rcv1, synthetic_topics
    shim = Shim(str(tmp_path_factory.mktemp("jni") / "libdsgd_jni_topic_thresholds.so"))
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


def _bits(a, b):
    return np.array_equal(np.asarray(a).view(np.int64), np.asarray(b).view(np.int64))


@pytest.mark.parametrize("intercept", [False, True])
def test_threshold_natives_match_native_ctx(setup, intercept):
    shim, ctxs, _ = setup
    ctx = ctxs[intercept]
    h = ctx._h.value
    W = np.random.default_rng(1).standard_normal((T, ctx.wdim)) * 0.2
    Wf = W.reshape(-1).copy()
    ids = np.random.default_rng(2).integers(0, N_ROWS, size=777).astype(np.int32)
    t, w = out(T, F64), out(8 * T, I64)
    assert shim("tuneTopicThresholds", h, Wf, T, 0.1, 100, 2100, t, w) == 0
    ref = ctx.tune_topic_thresholds(100, 2100, W, 0.1)
    assert _bits(t, ref[0]) and np.array_equal(w, ref[1])
    t, w = out(T, F64), out(8 * T, I64)
    assert shim("tuneTopicThresholdsSampled", h, Wf, T, 0.0, 0, N_ROWS, KEY - (1 << 64), 10, 900, t, w) == 0
    ref = ctx.tune_topic_thresholds_sampled(0, N_ROWS, KEY, 10, 900, W)
    assert _bits(t, ref[0]) and np.array_equal(w, ref[1])
    t, w = out(T, F64), out(8 * T, I64)
    assert shim("tuneTopicThresholdsSamples", h, Wf, T, 0.0, ids, t, w) == 0
    ref = ctx.tune_topic_thresholds_samples(ids, W)
    assert _bits(t, ref[0]) and np.array_equal(w, ref[1])
    thr = ref[0].copy()
    o = out(WORDS, I64)
    assert shim("evalThresholdedTopics", h, Wf, T, thr, 100, 2100, o) == 0
    assert np.array_equal(o, ctx.eval_thresholded_topics(100, 2100, W, thr))
    o = out(WORDS, I64)
    assert shim("evalSampledThresholdedTopics", h, Wf, T, thr, 0, N_ROWS, KEY - (1 << 64), 10, 900, o) == 0
    assert np.array_equal(o, ctx.eval_sampled_thresholded_topics(0, N_ROWS, KEY, 10, 900, W, thr))
    o = out(WORDS, I64)
    assert shim("evalSamplesThresholdedTopics", h, Wf, T, thr, ids, o) == 0
    assert np.array_equal(o, ctx.eval_samples_thresholded_topics(ids, W, thr))


def test_wrong_lengths_are_refused(setup):
    from distributed_sgd_b200 import native
    shim, ctxs, _ = setup
    ctx = ctxs[False]
    h = ctx._h.value
    n0 = ctx.launch_count()
    W = np.zeros(T * ctx.dim)
    ids = np.arange(10, dtype=np.int32)
    for w, t, o in ((W[:-1].copy(), out(T, F64), out(8 * T, I64)), (np.append(W, 0.0), out(T, F64), out(8 * T, I64)),
                    (W, out(T - 1, F64), out(8 * T, I64)), (W, out(T, F64), out(8 * T - 1, I64))):
        assert shim("tuneTopicThresholds", h, w, T, 0.0, 0, 100, t, o) == native.ERR_INVALID
        assert shim("tuneTopicThresholdsSampled", h, w, T, 0.0, 0, N_ROWS, 5, 0, 100, t, o) == native.ERR_INVALID
        assert shim("tuneTopicThresholdsSamples", h, w, T, 0.0, ids, t, o) == native.ERR_INVALID
        assert (t.view(np.uint8) == SENTINEL).all() and (o.view(np.uint8) == SENTINEL).all()
    for w, thr, o in ((W[:-1].copy(), np.zeros(T), out(WORDS, I64)), (W, np.zeros(T - 1), out(WORDS, I64)),
                      (W, np.zeros(T), out(WORDS - 1, I64))):
        assert shim("evalThresholdedTopics", h, w, T, thr, 0, 100, o) == native.ERR_INVALID
        assert shim("evalSampledThresholdedTopics", h, w, T, thr, 0, N_ROWS, 5, 0, 100, o) == native.ERR_INVALID
        assert shim("evalSamplesThresholdedTopics", h, w, T, thr, ids, o) == native.ERR_INVALID
        assert (o.view(np.uint8) == SENTINEL).all()
    o = out(WORDS, I64)
    assert shim("evalThresholdedTopics", h, W, T, None, 0, 100, o) == native.ERR_INVALID   # refused by the library
    assert (o.view(np.uint8) == SENTINEL).all()
    assert ctx.launch_count() == n0
