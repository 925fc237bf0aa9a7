"""The JNI shim's topic natives (loadTopics, selectTopic, evalTopics and its sampled and list forms) run against the library
through the stand-in JNIEnv of tests/test_gpu_jni.py: the words equal NativeCtx's bit for bit on a plain and an intercept
context, selectTopic switches the labels the metrics native sees, and every array shorter or longer than the header names
is refused before any launch with the output untouched."""
import numpy as np
import pytest

from test_gpu_jni import I64, KEY, SENTINEL, Shim, out

pytestmark = pytest.mark.gpu

T, N_ROWS = 5, 3000


@pytest.fixture(scope="module")
def setup(tmp_path_factory):
    import dataclasses
    from distributed_sgd_b200.native import NativeCtx
    from distributed_sgd_b200.utils import synthetic_rcv1, synthetic_topics
    shim = Shim(str(tmp_path_factory.mktemp("jni") / "libdsgd_jni_topics.so"))
    data = synthetic_rcv1(n_rows=N_ROWS, dim=800, seed=4)
    data = dataclasses.replace(data, topics=synthetic_topics(data, T, seed=4))
    ctxs = {}
    for intercept in (False, True):
        c = NativeCtx(0, data.dim, 1e-4, intercept=intercept)
        c.load_csr(data.row_ptr, data.col, data.val, data.label)
        ctxs[intercept] = c
    yield shim, ctxs, data
    for c in ctxs.values():
        c.close()


@pytest.mark.parametrize("intercept", [False, True])
def test_topic_natives_match_native_ctx(setup, intercept):
    shim, ctxs, data = setup
    ctx = ctxs[intercept]
    h = ctx._h.value
    tp, ti = data.topics.ptr.copy(), data.topics.ids.copy()
    assert shim("loadTopics", h, T, tp, ti) == 0
    ctx.n_topics = T
    W = np.random.default_rng(1).standard_normal((T, ctx.wdim)) * 0.2
    Wf = W.reshape(-1).copy()
    n = 8 * T + 8
    o = out(n, I64)
    assert shim("evalTopics", h, Wf, T, 100, 2100, o) == 0
    assert np.array_equal(o, ctx.eval_topics(100, 2100, W))
    o = out(n, I64)
    assert shim("evalSampledTopics", h, Wf, T, 0, N_ROWS, KEY - (1 << 64), 10, 900, o) == 0
    assert np.array_equal(o, ctx.eval_sampled_topics(0, N_ROWS, KEY, 10, 900, W))
    ids = np.random.default_rng(2).integers(0, N_ROWS, size=777).astype(np.int32)
    o = out(n, I64)
    assert shim("evalSamplesTopics", h, Wf, T, ids, o) == 0
    assert np.array_equal(o, ctx.eval_samples_topics(ids, W))
    # selectTopic: the metrics native now counts "has topic 3"
    assert shim("selectTopic", h, 3) == 0
    m = out(8, I64)
    assert shim("evalMetrics", h, W[3].copy(), 100, 2100, m) == 0
    assert np.array_equal(np.delete(m, 6), np.delete(ctx.eval_topics(100, 2100, W)[24:32], 6))
    assert shim("selectTopic", h, -1) == 0


def test_wrong_lengths_are_refused(setup):
    from distributed_sgd_b200 import native
    shim, ctxs, data = setup
    ctx = ctxs[False]
    h = ctx._h.value
    tp, ti = data.topics.ptr.copy(), data.topics.ids.copy()
    n0 = ctx.launch_count()
    assert shim("loadTopics", h, T, tp[:-1].copy(), ti) == native.ERR_INVALID
    assert shim("loadTopics", h, T, tp, ti[:-1].copy()) == native.ERR_INVALID
    assert shim("loadTopics", h, T, tp, np.append(ti, 0).astype(np.int32)) == native.ERR_INVALID
    assert ctx.launch_count() == n0
    assert shim("loadTopics", h, T, tp, ti) == 0
    n0 = ctx.launch_count()
    W = np.zeros(T * ctx.dim)
    for w, o in ((W[:-1].copy(), out(8 * T + 8, I64)), (np.append(W, 0.0), out(8 * T + 8, I64)),
                 (W, out(8 * T + 7, I64))):
        assert shim("evalTopics", h, w, T, 0, 100, o) == native.ERR_INVALID
        assert (o.view(np.uint8) == SENTINEL).all()
        assert shim("evalSamplesTopics", h, w, T, np.arange(10, dtype=np.int32), o) == native.ERR_INVALID
    assert shim("evalTopics", h, W[:ctx.dim * (T - 1)].copy(), T - 1, 0, 100, out(8 * T, I64)) == native.ERR_INVALID
    assert ctx.launch_count() == n0
