"""The weighted Poisson bootstrap on the device (dsgd_eval_*weighted_bootstrap, Master.local_bootstrap(weighted=True)).

Replicate b is defined as the weighted calls over the expanded list -- the request's ids with position i repeated m_i(b)
times, every copy weighing c_i = fl(w_y * s_i) -- so every replicate's 13 weighted words and its weighted loss sum must be
the bits dsgd_eval_samples_weighted_curve and dsgd_eval_samples_weighted return over that list."""
import math

import numpy as np
import pytest

from oracle import bootstrap as ob
from test_gpu_bootstrap import LAM, MODELS, _ctx, _trained_master, _weights, dyadic_rows, host_ids

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def datasets():
    from distributed_sgd_b200.utils import synthetic_rcv1
    return {"dyadic": dyadic_rows(3), "rcv1": synthetic_rcv1(n_rows=6000, seed=21)}


def _bits(x):
    return np.asarray(x, np.float64).view(np.int64)


def _same_bits(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return np.array_equal(_bits(a), _bits(b)) or np.array_equal(np.isnan(a), np.isnan(b)) and np.array_equal(
        _bits(np.where(np.isnan(a), 0.0, a)), _bits(np.where(np.isnan(b), 0.0, b)))


def check_expanded(ctx, w, ids, bkey, b0, res):
    """Every replicate of res = (words, wsums, loss) from replicates b0.. over the request `ids`, against the weighted curve
    and the weighted evaluation over its expanded list."""
    words, wsums, loss = res
    for j in range(len(loss)):
        m = ob.multiplicities(bkey, b0 + j, len(ids))
        ex = np.repeat(np.asarray(ids, np.int32), m)
        assert words[j, 0] == m.sum()
        if ex.size == 0:
            assert words[j, 1] == 0 and not _bits(wsums[j]).any() and _bits(loss[j]) == 0
            continue
        wc = ctx.eval_samples_weighted_curve(ex, w, curve=False)
        assert words[j, 1] == wc.words[7], j
        assert _same_bits(wsums[j], wc.wsums), (j, wsums[j], wc.wsums)
        ls = ctx.eval_samples_weighted(ex, w).loss_sum
        assert _same_bits(loss[j], ls), (j, loss[j], ls)


def _weightings(data):
    """(name, class weights, sample weights) of the weightings every model is checked under"""
    rng = np.random.default_rng(8)
    n = data.n_rows
    dyadic = rng.integers(0, 5, size=n) / 2.0          # multiples of 1/2, a fifth of them 0
    return [("class", (2.0, 0.5), None), ("dyadic", (1.0, 1.0), dyadic),
            ("fp64", (1.0, 1.0), rng.random(n) * 3.0), ("ones", (1.0, 1.0), None)]


def _set(ctx, cw, sw):
    ctx.set_class_weights(*cw)
    ctx.set_sample_weights(sw)


@pytest.mark.parametrize("intercept", [False, True], ids=["plain", "intercept"])
@pytest.mark.parametrize("model", MODELS)
def test_replicates_equal_the_expanded_list(model, intercept, datasets):
    for name, data in datasets.items():
        ctx = _ctx(model, data, intercept)
        try:
            n = data.n_rows
            for wname, cw, sw in _weightings(data):
                _set(ctx, cw, sw)
                for nan in ((False, True) if name == "dyadic" else (False,)):
                    w = _weights(name, data, intercept, nan)
                    bkey = 0x5EED + 17 * nan
                    check_expanded(ctx, w, np.arange(100, 1700), bkey, 3, ctx.eval_weighted_bootstrap(100, 1700, bkey, 3, 5, w))
                    ids = host_ids(0, n, 77, 0, 900)
                    check_expanded(ctx, w, ids, bkey, 0, ctx.eval_sampled_weighted_bootstrap(0, n, 77, 0, 900, bkey, 0, 2, w))
                    lst = np.random.default_rng(5).integers(0, n, size=1200).astype(np.int32)
                    check_expanded(ctx, w, lst, bkey, 10, ctx.eval_samples_weighted_bootstrap(lst, bkey, 10, 12, w))
                if wname == "dyadic":   # one class, and n = 1
                    w = _weights(name, data, intercept)
                    pos = np.flatnonzero(data.label > 0)[:300].astype(np.int32)
                    check_expanded(ctx, w, pos, 1, 0, ctx.eval_samples_weighted_bootstrap(pos, 1, 0, 2, w))
                    check_expanded(ctx, w, [7], 1, 0, ctx.eval_weighted_bootstrap(7, 8, 1, 0, 8, w))
        finally:
            ctx.close()


@pytest.mark.parametrize("model", ["svm", "logistic"])
def test_one_group_over_every_tile_and_the_range_edges(model, datasets):
    data = datasets["dyadic"]
    ctx = _ctx(model, data, False)
    try:
        sw = np.random.default_rng(2).integers(0, 4, size=data.n_rows) / 4.0
        _set(ctx, (1.0, 1.0), sw)
        w0 = np.zeros(data.dim)   # every score +0: one tie group of all rows, over many tiles
        check_expanded(ctx, w0, np.arange(0, 3000), 9, 0, ctx.eval_weighted_bootstrap(0, 3000, 9, 0, 4, w0))
        w = _weights("dyadic", data, False)
        for big in (2.0 ** 52, 2.0 ** 1000):   # a c of 2^52, and c = inf (2^1000 * 2^1000)
            s = sw.copy()
            s[np.flatnonzero(data.label > 0)[3]] = big
            s[np.flatnonzero(data.label < 0)[5]] = big
            _set(ctx, (1.0, 2.0 ** 1000) if big > 2.0 ** 52 else (1.0, 1.0), s)
            res = ctx.eval_weighted_bootstrap(0, 3000, 4, 0, 6, w)
            check_expanded(ctx, w, np.arange(0, 3000), 4, 0, res)
            assert np.isnan(res[1]).any()
    finally:
        ctx.close()


@pytest.mark.parametrize("model", MODELS)
def test_identities_with_the_unweighted_bootstrap(model, datasets):
    data = datasets["rcv1"]
    ctx = _ctx(model, data, False)
    try:
        w = _weights("rcv1", data, False)
        words, ap, loss = ctx.eval_bootstrap(0, 5000, 21, 0, 40, w)
        _set(ctx, (1.0, 1.0), None)   # c = 1
        ww, ws, wl = ctx.eval_weighted_bootstrap(0, 5000, 21, 0, 40, w)
        assert np.array_equal(ww[:, 0], words[:, 8]) and np.array_equal(ww[:, 1], words[:, 7])
        assert _same_bits(ws[:, :8], words[:, :8].astype(np.float64))
        assert _same_bits(ws[:, 8] / ws[:, 11], ap)
        assert _same_bits(wl, loss)
        _set(ctx, (1.0, 1.0), np.full(data.n_rows, 2.0))   # c = 2: every ratio as at c = 1
        from distributed_sgd_b200.core.master import bootstrap_values, weighted_bootstrap_values
        a = bootstrap_values(words, ap, loss, 0.0)
        b = weighted_bootstrap_values(*ctx.eval_weighted_bootstrap(0, 5000, 21, 0, 40, w), 0.0)
        for k in ("auc", "ap", "accuracy", "precision", "recall", "f1"):
            assert _same_bits(a[k], b[k]), k
    finally:
        ctx.close()


def test_splits_keys_chunks_and_row_forms(datasets):
    data = datasets["rcv1"]
    ctx = _ctx("logistic", data, False)
    try:
        _set(ctx, (3.0, 0.75), np.random.default_rng(1).random(data.n_rows))
        w = _weights("rcv1", data, False)
        whole = ctx.eval_weighted_bootstrap(0, 5000, 11, 0, 300, w)
        a, b = ctx.eval_weighted_bootstrap(0, 5000, 11, 0, 137, w), ctx.eval_weighted_bootstrap(0, 5000, 11, 137, 300, w)
        for x, y, z in zip(whole, a, b):
            assert _same_bits(x, np.concatenate([y, z]))
        for x, y in zip(whole, ctx.eval_weighted_bootstrap(0, 5000, 11, 0, 300, w)):   # the same key: the same bits
            assert _same_bits(x, y)
        assert np.array_equal(whole[0][:, 0], ctx.eval_bootstrap(0, 5000, 11, 0, 300, w)[0][:, 8])
        for x, y in zip(whole, ctx.eval_samples_weighted_bootstrap(np.arange(5000, dtype=np.int32), 11, 0, 300, w)):
            assert _same_bits(x, y)
        big = ctx.eval_weighted_bootstrap(0, 500, 3, 0, 4200, w)   # across the 4 096-replicate chunk edge
        for x, y in zip(big, ctx.eval_weighted_bootstrap(0, 500, 3, 4090, 4100, w)):
            assert _same_bits(x[4090:4100], y)
    finally:
        ctx.close()


def test_refusals(datasets):
    import ctypes as C
    from distributed_sgd_b200 import native
    data = datasets["rcv1"]
    ctx = _ctx("svm", data, False)
    lib = native.lib()
    words, wsums, loss = np.zeros((4, 2), np.int64), np.zeros((4, 13)), np.zeros(4)
    P = native._ptr
    try:
        for name in ("dsgd_eval_weighted_bootstrap", "dsgd_eval_sampled_weighted_bootstrap",
                     "dsgd_eval_samples_weighted_bootstrap"):
            fn = getattr(lib, name)
            args = [0.0 if t is C.c_double else 0 if t in (C.c_int32, C.c_int64, C.c_uint64) else None for t in fn.argtypes[1:]]
            assert fn(None, *args) == native.ERR_INVALID
        n0 = ctx.launch_count()
        for k in range(3):
            outs = [P(words), P(wsums), P(loss)]
            outs[k] = None
            assert lib.dsgd_eval_weighted_bootstrap(ctx._h, None, 0, 100, 1, 0, 4, *outs) == native.ERR_INVALID
        with pytest.raises(native.DsgdInvalid):
            ctx.eval_weighted_bootstrap(0, 100, 1, -1, 4)
        with pytest.raises(native.DsgdEmpty):
            ctx.eval_weighted_bootstrap(0, 100, 1, 4, 4)
        with pytest.raises(native.DsgdInvalid, match="2\\^26"):
            ctx.eval_samples_weighted_bootstrap(np.zeros((1 << 26) + 1, np.int32), 1, 0, 4)
        with pytest.raises(native.DsgdInvalid, match="2\\^26"):
            ctx.eval_sampled_weighted_bootstrap(0, 6000, 1, 0, (1 << 26) + 1, 1, 0, 4)
        with pytest.raises(native.DsgdRange):
            ctx.eval_weighted_bootstrap(0, 6001, 1, 0, 4)
        assert ctx.launch_count() == n0
    finally:
        ctx.close()
    actx = native.NativeCtx(0, data.dim, LAM, is_async=True)
    try:
        actx.load_csr(data.row_ptr, data.col, data.val, data.label)
        n0 = actx.launch_count()
        with pytest.raises(native.DsgdState, match="dsgd_eval_weighted_bootstrap: "):
            actx.eval_weighted_bootstrap(0, 3000, 1, 0, 4)
        assert actx.launch_count() == n0
    finally:
        actx.close()


def test_master_weighted_bootstrap():
    master, slave, w, w0 = _trained_master()
    try:
        master.ctx.set_class_weights(*_balanced(master))
        r = master.local_bootstrap(w, n_boot=500, weighted=True)
        curve, rep = master.local_weighted_curve(w, test_data=True, curve=False), master.local_weighted_report(w, test_data=True)
        est = {"accuracy": curve["accuracy"], "loss": rep["weighted_loss"], "auc": curve["auc"],
               "ap": curve["average_precision"], "precision": curve["precision"], "recall": curve["recall"],
               "f1": curve["f1"]}
        for k, v in est.items():
            assert r[k]["estimate"] == v, k
            assert r[k]["n_defined"] == 500 and r[k]["lo"] <= v <= r[k]["hi"], (k, r[k])
        unweighted = master.local_bootstrap(w, n_boot=500)
        assert unweighted["auc"]["estimate"] != r["auc"]["estimate"]
        s = master.local_sampled_bootstrap(w, 5000, n_boot=50, weighted=True)
        assert s["auc"]["n_defined"] == 50
        same = master.compare_bootstrap(w, w, n_boot=50, weighted=True)
        for k, d in same.items():
            ok = d["replicates"][~np.isnan(d["replicates"])]
            assert d["estimate"] == 0.0 and not ok.any() and d["p_better"] == 0.0, k
    finally:
        slave.stop()


def _balanced(master):
    """scikit-learn's balanced class weights n / (2 n_y) of the train rows"""
    words = master.ctx.eval_metrics(0, master.n_train)
    P, N = int(words[0] + words[1] + words[2]), int(words[3] + words[4] + words[5])
    n = P + N
    return n / (2.0 * P), n / (2.0 * N)
