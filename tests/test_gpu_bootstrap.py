"""The Poisson bootstrap on the device (dsgd_eval_*bootstrap, Master.local_bootstrap / compare_bootstrap).

Replicate b is defined as the unweighted evaluation of the expanded list -- the request's ids with position i repeated m_i(b)
times, m_i(b) the draw of dsgd_bootstrap.h (restated in oracle/bootstrap.py) -- so every replicate's words, AP and loss sum
must be the bits dsgd_eval_samples_metrics, dsgd_eval_samples_curve and dsgd_eval_samples_sums return over that list."""
import math
import time

import numpy as np
import pytest

from helpers import data_from_csr
from oracle import bootstrap as ob

pytestmark = pytest.mark.gpu

LAM = 1e-4
MODELS = ["svm", "logistic", "squared_hinge", "modified_huber"]


def dyadic_rows(seed, n_rows=3000, dim=64):
    """Tie-heavy rows: 0..12 entries (a tenth empty: score 0), values multiples of 1/4; rows 0..19 hold both of the last two
    columns, which the NaN weights set to +inf and -inf."""
    rng = np.random.default_rng(seed)
    lens = np.where(rng.random(n_rows) < 0.1, 0, rng.integers(1, 13, size=n_rows))
    lens[:20] = 2
    cols = [rng.choice(dim - 2, size=k, replace=False) for k in lens]
    cols[:20] = [np.array([dim - 2, dim - 1])] * 20
    rp = np.concatenate([[0], np.cumsum(lens)]).astype(np.int64)
    col = np.concatenate(cols).astype(np.int32)
    val = (rng.integers(-4, 5, size=int(rp[-1])) / 4.0).astype(np.float32)
    val[:40] = 1.0
    lab = np.where(rng.random(n_rows) < 0.35, 1, -1).astype(np.int8)
    return data_from_csr(rp, col, val, lab, dim)


@pytest.fixture(scope="module")
def datasets():
    from distributed_sgd_b200.utils import synthetic_rcv1
    return {"dyadic": dyadic_rows(3), "rcv1": synthetic_rcv1(n_rows=6000, seed=21)}


def _ctx(model, data, intercept):
    from distributed_sgd_b200.native import NativeCtx
    ctx = NativeCtx(0, data.dim, LAM, model=model, intercept=intercept)
    ctx.load_csr(data.row_ptr, data.col, data.val, data.label)
    return ctx


def _weights(name, data, intercept, nan=False, seed=4):
    rng = np.random.default_rng(seed)
    if name == "dyadic":
        w = rng.integers(-2, 3, size=data.dim) / 4.0
        w[-2:] = (np.inf, -np.inf) if nan else 0.0
    else:
        w = np.where(rng.random(data.dim) < 0.5, rng.standard_normal(data.dim) * 0.2, 0.0)
    return np.append(w, 0.25) if intercept else w


def host_ids(row_begin, row_end, key, lo, hi):
    from distributed_sgd_b200.native import host_lib
    h, n = host_lib(), row_end - row_begin
    return (row_begin + np.array([h.dsgd_feistel_pos(p, n, key) for p in range(lo, hi)], np.int64)).astype(np.int32)


def _bits(x):
    return np.asarray(x, np.float64).view(np.int64)


def check_expanded(ctx, w, ids, bkey, b0, res):
    """Every replicate of res = (words, ap, loss) from replicates b0.. over the request `ids`, against the existing calls
    over its expanded list."""
    words, ap, loss = res
    for j in range(len(ap)):
        m = ob.multiplicities(bkey, b0 + j, len(ids))
        ex = np.repeat(np.asarray(ids, np.int32), m)
        assert words[j, 8] == m.sum()
        if ex.size == 0:
            assert not words[j].any() and math.isnan(ap[j]) and loss[j] == 0.0
            continue
        assert np.array_equal(words[j, :8], ctx.eval_samples_metrics(ex, w)), j
        _, cap, _ = ctx.eval_samples_curve(ex, w, curve=False)
        assert _bits(ap[j]) == _bits(cap) or (math.isnan(ap[j]) and math.isnan(cap)), (j, ap[j], cap)
        ls = ctx.eval_samples_sums(ex, w)[0]
        assert _bits(loss[j]) == _bits(ls) or (math.isnan(loss[j]) and math.isnan(ls)), (j, loss[j], ls)


@pytest.mark.parametrize("intercept", [False, True], ids=["plain", "intercept"])
@pytest.mark.parametrize("model", MODELS)
def test_replicates_equal_the_expanded_list(model, intercept, datasets):
    for name, data in datasets.items():
        ctx = _ctx(model, data, intercept)
        try:
            for nan in ((False, True) if name == "dyadic" else (False,)):
                w = _weights(name, data, intercept, nan)
                bkey = 0x5EED + 17 * nan
                n = data.n_rows
                # range form, rows [100, 1700)
                check_expanded(ctx, w, np.arange(100, 1700), bkey, 3, ctx.eval_bootstrap(100, 1700, bkey, 3, 6, w))
                # sampled form: positions [0, 900) of a draw from rows [0, n)
                ids = host_ids(0, n, 77, 0, 900)
                check_expanded(ctx, w, ids, bkey, 0, ctx.eval_sampled_bootstrap(0, n, 77, 0, 900, bkey, 0, 3, w))
                # list form with repeats; a one-class list; n = 1
                lst = np.random.default_rng(5).integers(0, n, size=1200).astype(np.int32)
                check_expanded(ctx, w, lst, bkey, 10, ctx.eval_samples_bootstrap(lst, bkey, 10, 13, w))
                pos = np.flatnonzero(data.label > 0)[:300].astype(np.int32)
                check_expanded(ctx, w, pos, bkey, 0, ctx.eval_samples_bootstrap(pos, bkey, 0, 3, w))
                for one in (np.array([25], np.int32), np.array([5], np.int32)):
                    check_expanded(ctx, w, one, bkey, 0, ctx.eval_samples_bootstrap(one, bkey, 0, 8, w))
                check_expanded(ctx, w, [7], bkey, 0, ctx.eval_bootstrap(7, 8, bkey, 0, 8, w))
        finally:
            ctx.close()


def _same(a, b):
    return all(np.array_equal(np.asarray(x).view(np.int64) if np.asarray(x).dtype == np.float64 else x,
                              np.asarray(y).view(np.int64) if np.asarray(y).dtype == np.float64 else y) for x, y in zip(a, b))


@pytest.mark.parametrize("model", ["svm", "logistic"])
def test_splits_keys_and_row_forms(model, datasets):
    data = datasets["rcv1"]
    ctx = _ctx(model, data, False)
    try:
        w = _weights("rcv1", data, False)
        whole = ctx.eval_bootstrap(0, 5000, 11, 0, 300, w)
        a, b = ctx.eval_bootstrap(0, 5000, 11, 0, 137, w), ctx.eval_bootstrap(0, 5000, 11, 137, 300, w)
        assert _same(whole, [np.concatenate([x, y]) for x, y in zip(a, b)])
        assert _same(whole, ctx.eval_bootstrap(0, 5000, 11, 0, 300, w))                  # the same key: the same bits
        other = ctx.eval_bootstrap(0, 5000, 12, 0, 300, w)
        assert not np.array_equal(whole[0][:, 8], other[0][:, 8])                        # another key: other replicates
        assert _same(whole, ctx.eval_samples_bootstrap(np.arange(5000, dtype=np.int32), 11, 0, 300, w))
        ids = host_ids(1000, 6000, 99, 200, 3200)
        assert _same(ctx.eval_sampled_bootstrap(1000, 6000, 99, 200, 3200, 11, 5, 40, w),
                     ctx.eval_samples_bootstrap(ids, 11, 5, 40, w))
        # more replicates than one chunk of the pass: the split holds across the chunk edge
        big = ctx.eval_bootstrap(0, 500, 3, 0, 5000, w)
        assert _same([x[4090:4100] for x in big], ctx.eval_bootstrap(0, 500, 3, 4090, 4100, w))
    finally:
        ctx.close()


def test_refusals(datasets):
    import ctypes as C
    from distributed_sgd_b200 import native
    data = datasets["rcv1"]
    ctx = _ctx("svm", data, False)
    lib = native.lib()
    words, ap, loss = np.zeros((4, 9), np.int64), np.zeros(4), np.zeros(4)
    P = native._ptr
    try:
        for name in ("dsgd_eval_bootstrap", "dsgd_eval_sampled_bootstrap", "dsgd_eval_samples_bootstrap"):
            fn = getattr(lib, name)
            args = [0.0 if t is C.c_double else 0 if t in (C.c_int32, C.c_int64, C.c_uint64) else None for t in fn.argtypes[1:]]
            assert fn(None, *args) == native.ERR_INVALID
        n0 = ctx.launch_count()
        for k in range(3):   # each output NULL in turn
            outs = [P(words), P(ap), P(loss)]
            outs[k] = None
            assert lib.dsgd_eval_bootstrap(ctx._h, None, 0, 100, 1, 0, 4, *outs) == native.ERR_INVALID
        with pytest.raises(native.DsgdEmpty):
            ctx.eval_bootstrap(0, 100, 1, 4, 4)
        with pytest.raises(native.DsgdInvalid, match="2\\^26"):
            ctx.eval_samples_bootstrap(np.zeros((1 << 26) + 1, np.int32), 1, 0, 4)
        with pytest.raises(native.DsgdInvalid, match="2\\^26"):
            ctx.eval_sampled_bootstrap(0, 6000, 1, 0, (1 << 26) + 1, 1, 0, 4)
        with pytest.raises(native.DsgdRange):
            ctx.eval_samples_bootstrap(np.array([0, 6000], np.int32), 1, 0, 4)
        with pytest.raises(native.DsgdRange):
            ctx.eval_bootstrap(0, 6001, 1, 0, 4)
        assert ctx.launch_count() == n0                                                   # nothing was launched
    finally:
        ctx.close()
    actx = native.NativeCtx(0, data.dim, LAM, is_async=True)
    try:
        actx.load_csr(data.row_ptr, data.col, data.val, data.label)
        actx.compute_dim_sparsity(6000)
        before = actx.eval_bootstrap(0, 3000, 1, 0, 4)                                    # an idle async ctx is served
        actx.start_async(np.zeros(data.dim), np.arange(3000, dtype=np.int32), 8, 0.1, concurrency=1, max_updates=64, seed=1)
        try:
            t0 = time.time()
            while actx.async_running() and time.time() - t0 < 60:
                time.sleep(0.01)
            with pytest.raises(native.DsgdState, match="dsgd_eval_bootstrap: "):
                actx.eval_bootstrap(0, 3000, 1, 0, 4)
        finally:
            actx.stop_async()
        assert before[0].shape == (4, 9)
    finally:
        actx.close()


def test_resident_weights_after_a_sync_step(datasets):
    data = datasets["rcv1"]
    ctx = _ctx("logistic", data, True)
    try:
        ctx.compute_dim_sparsity(5000)
        ctx.set_weights(_weights("rcv1", data, True))
        ctx.sync_step(np.arange(0, 512, dtype=np.int32), 0.5)
        w = ctx.get_weights()
        assert _same(ctx.eval_bootstrap(5000, 6000, 2, 0, 20), ctx.eval_bootstrap(5000, 6000, 2, 0, 20, w))
    finally:
        ctx.close()


def _trained_master(n_rows=100_000):
    """A MasterSync trained for two epochs on RCV1-shaped rows, its last 20 000 rows the test rows"""
    from distributed_sgd_b200 import Master, Slave, SparseSVM
    from distributed_sgd_b200.utils import synthetic_rcv1
    data = synthetic_rcv1(n_rows=n_rows, seed=5)
    train, test = data.split_at(n_rows - 20_000)
    model = SparseSVM(LAM)
    slave = Slave(0, 0, train, model, False, world=1, device=0, test_data=test)
    master = Master.create(0, train, test, model, False, 1, slave=slave, seed=1)
    w0 = np.zeros(data.dim)
    state = master.fit(w0, max_epochs=2, batch_size=100, learning_rate=0.5, stopping_criterion=lambda losses: False)
    return master, slave, state.grad, w0


def test_statistics_on_trained_weights_and_paired_self_comparison():
    master, slave, w, w0 = _trained_master()
    try:
        n = master.n_test
        r = master.local_bootstrap(w, n_boot=2000)
        b, e = master.n_train, master.n_train + n
        words = master.ctx.eval_metrics(b, e, w)
        P, N = int(words[0] + words[1] + words[2]), int(words[3] + words[4] + words[5])
        A = r["auc"]["estimate"]   # Hanley and McNeil's standard error of the AUC, from P, N and A alone
        q1, q2 = A / (2 - A), 2 * A * A / (1 + A)
        se_hm = math.sqrt((A * (1 - A) + (P - 1) * (q1 - A * A) + (N - 1) * (q2 - A * A)) / (P * N))
        assert abs(r["auc"]["se"] / se_hm - 1) <= 0.15, (r["auc"]["se"], se_hm)
        assert r["auc"]["lo"] < A < r["auc"]["hi"] and r["auc"]["n_defined"] == 2000
        sizes = master.ctx.eval_bootstrap(b, e, 0xABC, 0, 2000, w)[0][:, 8]
        assert abs(sizes.mean() - n) <= 3 * math.sqrt(n / 2000)
        same = master.compare_bootstrap(w, w, n_boot=50)
        for k, s in same.items():
            ok = s["replicates"][~np.isnan(s["replicates"])]
            assert s["estimate"] == 0.0 and not ok.any() and s["p_better"] == 0.0, k
        d = master.compare_bootstrap(w0, w, n_boot=200)
        assert d["auc"]["estimate"] > 0 and d["auc"]["p_better"] > 0.9
    finally:
        slave.stop()
