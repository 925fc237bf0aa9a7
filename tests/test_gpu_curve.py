"""ROC / precision-recall curves and average precision on the device (dsgd_eval_*curve, Master.local_*curve) against the
fp64 curve checker (oracle/dsgd_oracle_curve.c).

The curve pass ranks exactly the values dsgd_margins returns, so its points must be exactly the checker's when the checker
ranks the device's own margins; on dyadic rows every dot is exact and the checker's own dots give the same points.  AP is a
fixed-point sum of one IEEE division per positive row: the same bits in any row order, within 2 ulp of fsum(v) / P."""
import ctypes as C
import json
import math
import os
import socket
import subprocess
import sys

import numpy as np
import pytest

from helpers import data_from_csr, make_pair
from oracle import curve as oc
from oracle import metrics as om

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LAM = 1e-4
SIZES = [1, 31, 32, 33, 2047, 2048, 100_000]


def dyadic_data(seed, n_rows, dim=192):
    """Rows of 0..24 entries (a tenth of them empty), values multiples of 1/8 in [-1, 1]; a third of the rows positive."""
    rng = np.random.default_rng(seed)
    lens = np.where(rng.random(n_rows) < 0.1, 0, rng.integers(1, 25, size=n_rows))
    rp = np.concatenate([[0], np.cumsum(lens)]).astype(np.int64)
    col = np.concatenate([rng.choice(dim, size=k, replace=False) for k in lens]).astype(np.int32)
    val = (rng.integers(-8, 9, size=int(rp[-1])) / 8.0).astype(np.float32)
    lab = np.where(rng.random(n_rows) < 0.35, 1, -1).astype(np.int8)
    return data_from_csr(rp, col, val, lab, dim)


def dyadic_w(rng, dim):
    return rng.integers(-2, 3, size=dim) / 4.0


def rand_w(rng, dim):
    return np.where(rng.random(dim) < 0.6, rng.standard_normal(dim) * 0.1, 0.0)


def host_ids(row_begin, row_end, key, lo, hi):
    from distributed_sgd_b200.native import host_lib
    h, n = host_lib(), row_end - row_begin
    pos = np.fromiter((h.dsgd_feistel_pos(p, n, key) for p in range(lo, hi)), dtype=np.int64, count=hi - lo)
    return (row_begin + pos).astype(np.int32)


def same_ap(a, b, ulps=0):
    return (math.isnan(a) and math.isnan(b)) or a == b or abs(a - b) <= ulps * math.ulp(b)


@pytest.fixture(scope="module")
def dy():
    data = dyadic_data(1, 130_000)
    ctx, orc = make_pair(data, LAM)
    yield ctx, orc, data
    ctx.close()


@pytest.fixture(scope="module")
def rcv():
    from distributed_sgd_b200.utils import synthetic_rcv1
    data = synthetic_rcv1(n_rows=40_000, seed=21)
    ctx, orc = make_pair(data, LAM)
    yield ctx, orc, data
    ctx.close()


def check_curve(ctx, orc, w, ids, res, exact_dots, metrics_words=None):
    """res = (words, ap, thr, tp, fp) of a curve pass over `ids`: the checker's curve over the device's margins (and over its
    own dots when exact), the metrics words, the U2 identity and AP within 2 ulp."""
    words, ap, thr, tp, fp = res
    m = ctx.margins(ids, w)
    ref = oc.curve(orc, w, idx=ids, margins=m)
    assert np.array_equal(thr, ref.thr) and np.array_equal(tp, ref.tp) and np.array_equal(fp, ref.fp)
    assert not np.signbit(thr[thr == 0]).any()
    if exact_dots:
        own = oc.curve(orc, w, idx=ids)
        assert np.array_equal(thr, own.thr) and np.array_equal(tp, own.tp) and np.array_equal(fp, own.fp)
    assert np.array_equal(words, om.metrics(orc, w, idx=ids, margins=m))
    if metrics_words is not None:
        assert np.array_equal(words, metrics_words)
    tp0, fp0 = np.concatenate([[0], tp]), np.concatenate([[0], fp])
    assert int(np.sum(np.diff(fp0) * (tp0[1:] + tp0[:-1]))) == words[6]
    assert len(thr) <= len(ids) and (np.diff(thr) < 0).all()
    assert same_ap(ap, ref.ap, ulps=2), (ap, ref.ap)
    return ref


def ap_only_agrees(res, ap_only):
    words, ap, thr = res[:3]
    assert np.array_equal(ap_only[0], words)
    assert (math.isnan(ap) and math.isnan(ap_only[1])) or ap_only[1] == ap
    assert ap_only[2] == len(thr)


# ---- the three forms ---------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("n", SIZES)
def test_three_forms_on_dyadic_rows(dy, n):
    """Sizes grow from test to test on one context: every pass grows the buffers the previous one left."""
    ctx, orc, data = dy
    rng = np.random.default_rng(200 + n)
    w = dyadic_w(rng, data.dim)
    ids = rng.integers(0, data.n_rows, size=n).astype(np.int32)   # repeats included
    res = ctx.eval_samples_curve(ids, w)
    check_curve(ctx, orc, w, ids, res, True, ctx.eval_samples_metrics(ids, w))
    ap_only_agrees(res, ctx.eval_samples_curve(ids, w, curve=False))
    b = int(rng.integers(0, data.n_rows - n + 1))
    res = ctx.eval_curve(b, b + n, w)
    check_curve(ctx, orc, w, np.arange(b, b + n, dtype=np.int32), res, True, ctx.eval_metrics(b, b + n, w))
    ap_only_agrees(res, ctx.eval_curve(b, b + n, w, curve=False))
    rb, re, key = 5, data.n_rows, 0xBEEF + n
    lo = int(rng.integers(0, re - rb - n + 1))
    res = ctx.eval_sampled_curve(rb, re, key, lo, lo + n, w)
    hid = host_ids(rb, re, key, lo, lo + n)
    check_curve(ctx, orc, w, hid, res, True, ctx.eval_sampled_metrics(rb, re, key, lo, lo + n, w))
    ap_only_agrees(res, ctx.eval_sampled_curve(rb, re, key, lo, lo + n, w, curve=False))


def test_shrinking_sizes_on_a_fresh_context(dy):
    _, orc, data = dy
    from distributed_sgd_b200.native import NativeCtx
    rng = np.random.default_rng(19)
    w = dyadic_w(rng, data.dim)
    with NativeCtx(0, data.dim, LAM) as ctx:
        ctx.load_csr(data.row_ptr, data.col, data.val, data.label)
        for n in SIZES[::-1]:
            ids = rng.integers(0, data.n_rows, size=n).astype(np.int32)
            words, ap, thr, tp, fp = ctx.eval_samples_curve(ids, w)
            ref = oc.curve(orc, w, idx=ids)
            assert np.array_equal(thr, ref.thr) and np.array_equal(tp, ref.tp) and np.array_equal(fp, ref.fp)
            assert np.array_equal(words, om.metrics(orc, w, idx=ids)) and same_ap(ap, ref.ap, ulps=2)
            words, ap, thr, tp, fp = ctx.eval_curve(7, 7 + n, w)
            ref = oc.curve(orc, w, begin=7, n=n)
            assert np.array_equal(thr, ref.thr) and np.array_equal(tp, ref.tp) and np.array_equal(fp, ref.fp)


def test_rcv1_shaped_rows_rank_the_device_margins(rcv):
    ctx, orc, data = rcv
    rng = np.random.default_rng(4)
    w = rand_w(rng, data.dim)
    ids = rng.integers(0, data.n_rows, size=25_000).astype(np.int32)
    check_curve(ctx, orc, w, ids, ctx.eval_samples_curve(ids, w), False, ctx.eval_samples_metrics(ids, w))
    check_curve(ctx, orc, w, np.arange(1000, 31_000, dtype=np.int32), ctx.eval_curve(1000, 31_000, w), False,
                ctx.eval_metrics(1000, 31_000, w))


def test_full_size_test_rows():
    """The 140 000 test rows of the full-size synthetic set, after a few sync steps."""
    from distributed_sgd_b200.utils import synthetic_rcv1
    data = synthetic_rcv1(n_rows=700_000, seed=0)
    n_train = 560_000
    ctx, orc = make_pair(data, LAM, n_train=n_train)
    try:
        rng = np.random.default_rng(0)
        ctx.set_weights(np.zeros(data.dim))
        ctx.sync_steps(rng.integers(0, n_train, size=64 * 200).astype(np.int32), 64, 200, 0.5, want_losses=False)
        w = ctx.get_weights()
        res = ctx.eval_curve(n_train, data.n_rows)
        ids = np.arange(n_train, data.n_rows, dtype=np.int32)
        check_curve(ctx, orc, w, ids, res, False, ctx.eval_metrics(n_train, data.n_rows))
        assert 0.5 < res[1] <= 1.0
        ap_only_agrees(res, ctx.eval_curve(n_train, data.n_rows, curve=False))
    finally:
        ctx.close()


# ---- average precision -------------------------------------------------------------------------------------------------

def test_ap_does_not_depend_on_the_row_order(rcv):
    ctx, orc, data = rcv
    rng = np.random.default_rng(7)
    w = rand_w(rng, data.dim)
    ids = np.arange(3000, 23_000, dtype=np.int32)
    ref = ctx.eval_curve(3000, 23_000, w)
    for perm in (ids[::-1], rng.permutation(ids)):
        got = ctx.eval_samples_curve(perm, w)
        assert np.array_equal(got[0], ref[0]) and got[1] == ref[1]
        for a, b in zip(got[2:], ref[2:]):
            assert np.array_equal(a, b)
        assert ctx.eval_samples_curve(perm, w, curve=False)[1] == ref[1]
    assert ctx.eval_curve(3000, 23_000, w, curve=False)[1] == ref[1]


def test_ap_edge_cases(dy):
    ctx, orc, data = dy
    lab = data.label
    w = dyadic_w(np.random.default_rng(11), data.dim)
    pos = np.flatnonzero(lab > 0)[:5000].astype(np.int32)
    neg = np.flatnonzero(lab < 0)[:700].astype(np.int32)
    words, ap, thr, tp, fp = ctx.eval_samples_curve(pos, w)          # N = 0: every v_i is 1, S = P exactly
    assert ap == 1.0 and (fp == 0).all() and tp[-1] == len(pos)
    words, ap, thr, tp, fp = ctx.eval_samples_curve(neg, w)          # P = 0: AP undefined
    assert math.isnan(ap) and (tp == 0).all() and fp[-1] == len(neg)
    for ids in (pos[:1], neg[:1], np.repeat(np.concatenate([pos[:2], neg[:3]]), 300)):
        check_curve(ctx, orc, w, ids, ctx.eval_samples_curve(ids, w), True)
    # every score -0: one point with every row, each v_i = P / n
    words, ap, thr, tp, fp = ctx.eval_curve(0, 5000, np.zeros(data.dim))
    P = int((lab[:5000] > 0).sum())
    assert list(thr) == [0.0] and not np.signbit(thr[0]) and list(tp) == [P] and list(fp) == [5000 - P]
    assert same_ap(ap, P / 5000, ulps=1)
    # two infinite weights: rows with both columns of opposite signs score NaN (word 7, AP NaN), the others +-inf or finite
    wi = w.copy()
    wi[:2] = np.inf
    ids = np.arange(0, 20_000, dtype=np.int32)
    res = ctx.eval_samples_curve(ids, wi)
    assert res[0][7] > 0 and math.isnan(res[1])
    check_curve(ctx, orc, wi, ids, res, True, ctx.eval_samples_metrics(ids, wi))
    assert np.isinf(res[2]).any()


def test_a_logistic_context_gives_the_same_curve(rcv):
    from distributed_sgd_b200.native import NativeCtx
    ctx_svm, orc, data = rcv
    rng = np.random.default_rng(3)
    w = rand_w(rng, data.dim) * 20
    ids = rng.integers(0, data.n_rows, size=5000).astype(np.int32)
    with NativeCtx(0, data.dim, LAM, logistic=True) as lg:
        lg.load_csr(data.row_ptr, data.col, data.val, data.label)
        for a, b in ((lg.eval_samples_curve(ids, w), ctx_svm.eval_samples_curve(ids, w)),
                     (lg.eval_curve(100, 9000, w), ctx_svm.eval_curve(100, 9000, w))):
            assert np.array_equal(a[0], b[0]) and a[1] == b[1]
            for x, y in zip(a[2:], b[2:]):
                assert np.array_equal(x, y)


# ---- errors and launches -----------------------------------------------------------------------------------------------

def test_errors(dy):
    from distributed_sgd_b200.native import DsgdEmpty, DsgdInvalid, DsgdRange, DsgdState, NativeCtx
    ctx, orc, data = dy
    N = data.n_rows
    L, h = ctx._l, ctx._h
    words, thr = np.zeros(8, np.int64), np.zeros(16)
    tp, fp = np.zeros(16, np.int64), np.zeros(16, np.int64)
    ap, m = C.c_double(), C.c_int64()
    ids = np.arange(4, dtype=np.int32)
    W, A, M, T, TP, FP = words.ctypes.data, C.byref(ap), C.byref(m), thr.ctypes.data, tp.ctypes.data, fp.ctypes.data
    for outs in ((W, A, M, T, None, None), (W, A, M, None, TP, None), (W, A, M, None, None, FP), (W, A, M, T, TP, None),
                 (None, A, M, T, TP, FP), (W, None, M, None, None, None), (W, A, None, T, TP, FP)):
        assert L.dsgd_eval_curve(h, None, 0, 10, *outs) == -1
        assert L.dsgd_eval_sampled_curve(h, None, 0, 10, 1, 0, 5, *outs) == -1
        assert L.dsgd_eval_samples_curve(h, None, ids.ctypes.data, 4, *outs) == -1
    assert L.dsgd_eval_samples_curve(h, None, None, 4, W, A, M, T, TP, FP) == -1         # NULL ids
    for call in (lambda: ctx.eval_samples_curve([3, N]), lambda: ctx.eval_samples_curve([-1]),
                 lambda: ctx.eval_curve(0, N + 1), lambda: ctx.eval_curve(-1, 5), lambda: ctx.eval_curve(9, 8),
                 lambda: ctx.eval_sampled_curve(0, N + 1, 1, 0, 5)):
        with pytest.raises(DsgdRange):
            call()
    for call in (lambda: ctx.eval_samples_curve(np.zeros(0, np.int32)), lambda: ctx.eval_curve(4, 4),
                 lambda: ctx.eval_sampled_curve(5, 5, 1, 0, 0), lambda: ctx.eval_sampled_curve(10, 20, 1, 3, 3),
                 lambda: ctx.eval_curve(4, 4, curve=False)):
        with pytest.raises(DsgdEmpty):
            call()
    with pytest.raises(DsgdInvalid):
        ctx.eval_sampled_curve(10, 20, 1, 0, 11)
    with NativeCtx(0, data.dim, LAM) as empty:
        for call in (lambda: empty.eval_curve(0, 1), lambda: empty.eval_samples_curve([0]),
                     lambda: empty.eval_sampled_curve(0, 1, 1, 0, 1)):
            with pytest.raises(DsgdState):
                call()
    w = dyadic_w(np.random.default_rng(1), data.dim)                 # the ctx still answers correctly after the refusals
    got = ctx.eval_curve(10, 30, w)
    ref = oc.curve(orc, w, begin=10, n=20)
    assert np.array_equal(got[2], ref.thr) and np.array_equal(got[3], ref.tp) and np.array_equal(got[4], ref.fp)


def test_launch_counts(dy):
    """The kernels of one call (dsgd_launch_count; CUB's sort, merge and scan kernels are not counted): score, count, sum,
    and emit for a full curve; the drawn form adds its draw, explicit weights their copy and prepare."""
    ctx, _, data = dy
    w = dyadic_w(np.random.default_rng(2), data.dim)
    ids = np.arange(100, 3100, dtype=np.int32)

    def launches(fn):
        a = ctx.launch_count()
        fn()
        return ctx.launch_count() - a

    got = {}
    for curve in (False, True):
        for wt in (None, w):
            got[("range", curve, wt is None)] = launches(lambda: ctx.eval_curve(100, 3100, wt, curve=curve))
            got[("drawn", curve, wt is None)] = launches(lambda: ctx.eval_sampled_curve(0, 9000, 3, 0, 3000, wt, curve=curve))
            got[("list", curve, wt is None)] = launches(lambda: ctx.eval_samples_curve(ids, wt, curve=curve))
    want = {}
    for form, extra in (("range", 0), ("drawn", 1), ("list", 0)):
        for curve in (False, True):
            for resident in (True, False):
                want[(form, curve, resident)] = 3 + int(curve) + extra + (0 if resident else 2)
    assert got == want


# ---- async contexts ----------------------------------------------------------------------------------------------------

def test_async_context_reads_its_snapshot():
    from distributed_sgd_b200.utils import synthetic_rcv1
    data = synthetic_rcv1(n_rows=5000, seed=6)
    ctx, orc = make_pair(data, LAM, is_async=True)
    try:
        rng = np.random.default_rng(6)
        w = rand_w(rng, data.dim)
        ctx.set_weights(w)
        ids = rng.integers(0, 5000, size=3000)

        def same(a, b):
            return np.array_equal(a[0], b[0]) and a[1] == b[1] and all(np.array_equal(x, y) for x, y in zip(a[2:], b[2:]))

        assert same(ctx.eval_curve(0, 5000), ctx.eval_curve(0, 5000, w))
        idx = rng.choice(data.dim, size=500, replace=False).astype(np.int32)
        ctx.update_grad(idx, rng.standard_normal(500) * 0.05)          # changes the replica, not its scalars
        w2 = ctx.get_weights()
        assert not np.array_equal(w, w2)
        assert same(ctx.eval_curve(0, 5000), ctx.eval_curve(0, 5000, w2))
        assert same(ctx.eval_samples_curve(ids), ctx.eval_samples_curve(ids, w2))
        assert same(ctx.eval_sampled_curve(0, 5000, 9, 0, 2000), ctx.eval_sampled_curve(0, 5000, 9, 0, 2000, w2))
        assert ctx.eval_curve(0, 5000, curve=False)[1] == ctx.eval_curve(0, 5000, w2)[1]
    finally:
        ctx.close()


_FRESH = r"""
import sys
sys.path.insert(0, {root!r})
import numpy as np
from distributed_sgd_b200.native import DsgdState, NativeCtx
from distributed_sgd_b200.utils import synthetic_rcv1
data = synthetic_rcv1(n_rows=6000, seed=8)
ctx = NativeCtx(0, data.dim, 1e-4, is_async=True)
ctx.load_csr(data.row_ptr, data.col, data.val, data.label)
ctx.compute_dim_sparsity(4800)
w = np.zeros(data.dim)
ctx.start_async(w, np.arange(4800, dtype=np.int32), 8, 0.1, concurrency=1, max_updates=0, seed=1)
try:
    running = ctx.async_running()
    a = ctx.eval_curve(0, 6000)                             # the first curve pass of this process: sort, merge and scan
    b = ctx.eval_sampled_curve(0, 6000, 5, 0, 3000, curve=False)
    c = ctx.eval_samples_curve(np.arange(6000, dtype=np.int32)[::-1])
    try:
        ctx.eval_samples_curve(np.zeros(6001, np.int32))     # more ids than rows: the buffers would have to grow
        refused = False
    except DsgdState:
        refused = True
    print("OK", running, int(a[0][:6].sum()), int(b[0][:6].sum()), int(c[3][-1] + c[4][-1]), refused)
finally:
    ctx.stop_async()
ctx.close()
"""


def test_first_curve_call_while_the_loop_runs_returns():
    """A fresh process whose async loop runs makes its first curve calls: every kernel they launch (CUB's included) was
    loaded, and every buffer they use sized, before the loop started; a list longer than that is refused.  The loop is
    stopped in a `finally`; the subprocess has a timeout."""
    r = subprocess.run([sys.executable, "-s", "-c", _FRESH.format(root=ROOT)], cwd=ROOT, capture_output=True, text=True,
                       timeout=180)
    assert r.returncode == 0, r.stdout + r.stderr
    assert "OK True 6000 3000 6000 True" in r.stdout, r.stdout + r.stderr


# ---- Master ------------------------------------------------------------------------------------------------------------

def _setup(rank=0, world=1):
    from distributed_sgd_b200 import Slave, SparseSVM
    from distributed_sgd_b200.utils import synthetic_rcv1
    data = synthetic_rcv1(n_rows=7000, seed=13)
    train, test = data.split_at(4800)
    model = SparseSVM(LAM)
    slave = Slave(rank, 0, train, model, world=world, device=0, test_data=test)
    return data, train, test, model, slave


def _results(m, w):
    out = [m.local_curve(w, test_data=True), m.local_curve(w), m.local_sampled_curve(w, 1500, test_data=True),
           m.local_sampled_curve(w, 3000, curve=False)]
    m.ctx.set_weights(w)
    out.append(m.local_curve(test_data=True))
    return out


def test_master_curve_against_the_checker():
    from distributed_sgd_b200 import MasterSync
    from distributed_sgd_b200.core.master import metrics_dict, sampled_key
    from oracle.oracle import Oracle
    data, train, test, model, slave = _setup()
    try:
        orc = Oracle(data.row_ptr, data.col, data.val, data.label, data.dim, LAM)
        m = MasterSync(0, train, test, model, 1, slave=slave, seed=11)
        w = rand_w(np.random.default_rng(8), data.dim)
        res = _results(m, w)
        ids = [np.arange(4800, 7000), np.arange(4800), host_ids(4800, 7000, sampled_key(11, 0), 0, 1500),
               host_ids(0, 4800, sampled_key(11, 1), 0, 3000), np.arange(4800, 7000)]
        for k, (got, i) in enumerate(zip(res, ids)):
            i = i.astype(np.int32)
            mg = slave.ctx.margins(i, w)
            ref = oc.curve(orc, w, idx=i, margins=mg)
            words = om.metrics(orc, w, idx=i, margins=mg)
            assert json.dumps({x: got[x] for x in metrics_dict(words)}) == json.dumps(metrics_dict(words))
            assert same_ap(got["average_precision"], ref.ap, ulps=2) and got["n_points"] == len(ref.thr)
            if k == 3:
                assert "curve" not in got
                continue
            c = got["curve"]
            assert c["thresholds"] == list(ref.thr) and c["tp"] == list(ref.tp) and c["fp"] == list(ref.fp)
            P, N = int(ref.tp[-1]), int(ref.fp[-1])
            assert c["recall"] == c["tpr"] == [t / P for t in ref.tp]
            assert c["fpr"] == [f / N for f in ref.fp]
            assert c["precision"] == [t / (t + f) for t, f in zip(ref.tp, ref.fp)]
        assert json.dumps(res[4]) == json.dumps(res[0])
        # the sampled form consumes one draw of the sampled loss: the same key sequence
        m2 = MasterSync(0, train, test, model, 1, slave=slave, seed=11)
        m2.local_sampled_loss(w, 1500, test_data=True)
        assert json.dumps(m2.local_sampled_curve(w, 3000, curve=False)) == json.dumps(res[3])
        from distributed_sgd_b200.native import DsgdEmpty
        with pytest.raises(DsgdEmpty):
            m2.local_sampled_curve(w, 0)
        # jvm_exact: the ids of the reference's shuffle go through the list form
        from distributed_sgd_b200.core.master import curve_dict
        from distributed_sgd_b200.utils.jvm_random import JvmRandom
        mj = MasterSync(0, train, test, model, 1, slave=slave, seed=0, jvm_exact=True)
        jids = (JvmRandom(0).shuffle(np.arange(2200))[:700] + 4800).astype(np.int32)
        assert (json.dumps(mj.local_sampled_curve(w, 700, test_data=True))
                == json.dumps(curve_dict(slave.ctx.eval_samples_curve(jids, w))))
    finally:
        slave.stop()


def _free_port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def _rank(rank, world, port, q):
    sys.path.insert(0, ROOT)
    import torch.distributed as dist
    from distributed_sgd_b200 import MasterSync
    from distributed_sgd_b200.core import Group
    dist.init_process_group("gloo", init_method=f"tcp://127.0.0.1:{port}", rank=rank, world_size=world)
    try:
        data, train, test, model, slave = _setup(rank, world)
        m = MasterSync(rank, train, test, model, world, slave=slave, group=Group(), seed=11, attach=False)
        w = rand_w(np.random.default_rng(8), data.dim)
        q.put((rank, json.dumps(_results(m, w))))
        slave.stop()
    finally:
        dist.destroy_process_group()


def test_two_gloo_ranks_on_one_gpu_agree_with_one_rank():
    import torch.multiprocessing as mp
    from distributed_sgd_b200 import MasterSync
    ctxmp = mp.get_context("spawn")
    q = ctxmp.Queue()
    port = _free_port()
    procs = [ctxmp.Process(target=_rank, args=(r, 2, port, q)) for r in range(2)]
    for p in procs:
        p.start()
    try:
        res = dict(q.get(timeout=300) for _ in procs)
    finally:
        for p in procs:
            p.join(timeout=60)
            if p.is_alive():
                p.terminate()
    data, train, test, model, slave = _setup()
    try:
        one = json.dumps(_results(MasterSync(0, train, test, model, 1, slave=slave, seed=11),
                                  rand_w(np.random.default_rng(8), data.dim)))
    finally:
        slave.stop()
    assert res[0] == res[1] == one
