"""Scores and ranking metrics on the device (dsgd_margins, dsgd_probabilities, dsgd_eval_*metrics, Master.local_*metrics)
against the fp64 oracle.

The metrics pass and dsgd_margins share one dot body, so the words must be exactly the oracle's when the oracle ranks the
device's own margins.  On dyadic rows every dot is exact, so the oracle's own left-fold dots give the same words too; those
rows take few distinct scores, so hundreds of rows tie, and every zero dot is the score -0."""
import json
import math
import os
import socket
import subprocess
import sys

import numpy as np
import pytest

from helpers import data_from_csr, make_pair
from oracle import metrics as om
from oracle.oracle import Oracle

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
    return rng.integers(-2, 3, size=dim) / 4.0                     # 5 levels: few distinct dots


def rand_w(rng, dim):
    return np.where(rng.random(dim) < 0.6, rng.standard_normal(dim) * 0.1, 0.0)


def host_ids(row_begin, row_end, key, lo, hi):
    from distributed_sgd_b200.native import host_lib
    h, n = host_lib(), row_end - row_begin
    pos = np.fromiter((h.dsgd_feistel_pos(p, n, key) for p in range(lo, hi)), dtype=np.int64, count=hi - lo)
    return (row_begin + pos).astype(np.int32)


def stable_sigmoid(t):
    t = np.asarray(t, dtype=np.float64)
    out = np.empty_like(t)
    p = t >= 0
    out[p] = 1.0 / (1.0 + np.exp(-t[p]))
    e = np.exp(t[~p])
    out[~p] = e / (1.0 + e)
    return out


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


# ---- scores ------------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("n", SIZES)
def test_margins_bit_exact_on_dyadic_rows(dy, n):
    ctx, orc, data = dy
    rng = np.random.default_rng(n)
    w = dyadic_w(rng, data.dim)
    ids = rng.integers(0, data.n_rows, size=n).astype(np.int32)
    m = ctx.margins(ids, w)
    assert np.array_equal(m, om.margins(orc, w, idx=ids))
    assert np.array_equal(ctx.forward(ids, w), np.where(m > 0, -1.0, np.where(m < 0, 1.0, 0.0)))
    assert not np.signbit(m[m == 0]).any()                         # a zero dot is +0


def test_margins_on_rcv1_shaped_rows(rcv):
    ctx, orc, data = rcv
    rng = np.random.default_rng(2)
    w = rand_w(rng, data.dim)
    ids = rng.integers(0, data.n_rows, size=30_000).astype(np.int32)
    m = ctx.margins(ids, w)
    # rtol 1e-12 of sum_j |x_j w_j|: a row whose products nearly cancel has a dot far below its terms, and the device adds
    # them in another order than the oracle's left fold
    scale = om.margins(Oracle(data.row_ptr, data.col, np.abs(data.val), data.label, data.dim, LAM), np.abs(w), idx=ids)
    assert (np.abs(m - om.margins(orc, w, idx=ids)) <= 1e-12 * scale).all()
    assert np.array_equal(np.sign(m), -ctx.forward(ids, w))
    ctx.set_weights(w)
    assert np.array_equal(ctx.margins(ids), m)                     # w == NULL: the resident weights


def test_probabilities_on_a_logistic_context(rcv):
    from distributed_sgd_b200.native import DsgdState, NativeCtx
    ctx_svm, orc, data = rcv
    rng = np.random.default_rng(3)
    w = rand_w(rng, data.dim) * 20                                 # margins of several units: both sigmoid branches
    ids = rng.integers(0, data.n_rows, size=5000).astype(np.int32)
    with NativeCtx(0, data.dim, LAM, logistic=True) as lg:
        lg.load_csr(data.row_ptr, data.col, data.val, data.label)
        p = lg.probabilities(ids, w)
        m = om.margins(orc, w, idx=ids)
        assert (m > 1).any() and (m < -1).any()
        np.testing.assert_allclose(p, stable_sigmoid(-m), rtol=1e-12, atol=0)
        assert np.array_equal(lg.margins(ids, w), ctx_svm.margins(ids, w))   # the score does not depend on the model
        assert np.array_equal(lg.eval_samples_metrics(ids, w), ctx_svm.eval_samples_metrics(ids, w))
    with pytest.raises(DsgdState):
        ctx_svm.probabilities(ids, w)


# ---- metrics -----------------------------------------------------------------------------------------------------------

def check_words(ctx, orc, w, ids, got, exact_dots):
    """got = the device's words over `ids`: exactly the oracle's on the device's margins (and on its own dots when exact)."""
    m = ctx.margins(ids, w)
    assert np.array_equal(got, om.metrics(orc, w, idx=ids, margins=m))
    if exact_dots:
        assert np.array_equal(got, om.metrics(orc, w, idx=ids))
    assert got[:6].sum() == len(ids)


@pytest.mark.parametrize("n", SIZES)
def test_three_forms_on_dyadic_rows(dy, n):
    """Sizes grow from test to test on one context: every pass grows the buffers the previous one left."""
    ctx, orc, data = dy
    rng = np.random.default_rng(100 + n)
    w = dyadic_w(rng, data.dim)
    ids = rng.integers(0, data.n_rows, size=n).astype(np.int32)   # repeats included
    got = ctx.eval_samples_metrics(ids, w)
    check_words(ctx, orc, w, ids, got, exact_dots=True)
    b = int(rng.integers(0, data.n_rows - n + 1))
    got = ctx.eval_metrics(b, b + n, w)
    check_words(ctx, orc, w, np.arange(b, b + n, dtype=np.int32), got, exact_dots=True)
    assert got[0] + got[4] == ctx.eval_sums(b, b + n, w)[1]        # correct of the evaluation pass
    # the sampled form: positions [lo, lo + n) of the draw over [rb, re) equal the list form over the host's ids
    rb, re, key = 5, data.n_rows, 0xFEED + n
    lo = int(rng.integers(0, re - rb - n + 1))
    got = ctx.eval_sampled_metrics(rb, re, key, lo, lo + n, w)
    hid = host_ids(rb, re, key, lo, lo + n)
    assert np.array_equal(got, ctx.eval_samples_metrics(hid, w))
    check_words(ctx, orc, w, hid, got, exact_dots=True)
    assert got[0] + got[4] == ctx.eval_sampled_sums(rb, re, key, lo, lo + n, w)[1]


def test_heavy_ties_signed_zeros_and_one_class(dy):
    ctx, orc, data = dy
    lab = data.label
    w = np.zeros(data.dim)
    got = ctx.eval_metrics(0, 5000, w)                              # every score is -0: every pair ties
    P, N = int((lab[:5000] > 0).sum()), int((lab[:5000] < 0).sum())
    assert list(got) == [0, 0, P, 0, 0, N, P * N, 0]
    w = np.zeros(data.dim)
    w[:3] = (0.25, -0.25, 0.5)                                      # most rows score 0, the rest few values
    ids = np.arange(20_000, dtype=np.int32)
    got = ctx.eval_samples_metrics(ids, w)
    check_words(ctx, orc, w, ids, got, exact_dots=True)
    assert got[2] + got[5] > 10_000
    pos = np.flatnonzero(lab > 0)[:3000].astype(np.int32)
    neg = np.flatnonzero(lab < 0)[:300].astype(np.int32)
    w = dyadic_w(np.random.default_rng(5), data.dim)
    for ids in (pos, neg, pos[:1], neg[:1], np.repeat(pos[:2], 700)):
        got = ctx.eval_samples_metrics(ids, w)
        assert got[6] == 0
        check_words(ctx, orc, w, ids, got, exact_dots=True)


def test_shrinking_sizes_on_a_fresh_context(dy):
    _, orc, data = dy
    from distributed_sgd_b200.native import NativeCtx
    rng = np.random.default_rng(9)
    w = dyadic_w(rng, data.dim)
    with NativeCtx(0, data.dim, LAM) as ctx:
        ctx.load_csr(data.row_ptr, data.col, data.val, data.label)
        for n in SIZES[::-1]:
            ids = rng.integers(0, data.n_rows, size=n).astype(np.int32)
            got = ctx.eval_samples_metrics(ids, w)
            assert np.array_equal(got, om.metrics(orc, w, idx=ids))
            assert np.array_equal(ctx.eval_metrics(7, 7 + n, w), om.metrics(orc, w, begin=7, n=n))


def test_rcv1_shaped_rows_rank_the_device_margins(rcv):
    ctx, orc, data = rcv
    rng = np.random.default_rng(4)
    w = rand_w(rng, data.dim)
    ids = rng.integers(0, data.n_rows, size=25_000).astype(np.int32)
    got = ctx.eval_samples_metrics(ids, w)
    check_words(ctx, orc, w, ids, got, exact_dots=False)
    got = ctx.eval_metrics(1000, 31_000, w)
    check_words(ctx, orc, w, np.arange(1000, 31_000, dtype=np.int32), got, exact_dots=False)
    assert got[0] + got[4] == ctx.eval_sums(1000, 31_000, w)[1]


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
        got = ctx.eval_metrics(n_train, data.n_rows)
        ids = np.arange(n_train, data.n_rows, dtype=np.int32)
        check_words(ctx, orc, w, ids, got, exact_dots=False)
        assert got[0] + got[4] == ctx.eval_sums(n_train, data.n_rows)[1]
        auc = got[6] / (2 * got[:3].sum() * got[3:6].sum())
        assert 0.5 < auc <= 1.0
    finally:
        ctx.close()


# ---- cross-checks ------------------------------------------------------------------------------------------------------

def test_resident_weights_and_the_staged_stream():
    from distributed_sgd_b200.utils import synthetic_rcv1
    data = synthetic_rcv1(n_rows=6000, seed=9)
    rng = np.random.default_rng(4)
    batch, steps, lr = 64, 10, 0.5
    stream = np.concatenate([rng.choice(4800, size=batch, replace=False) for _ in range(steps)]).astype(np.int32)
    w0 = rand_w(rng, data.dim) * 0.1
    results = []
    for evaluate in (True, False):
        ctx, _ = make_pair(data, LAM, n_train=4800)
        ctx.set_weights(w0)
        ctx.stage_samples(stream)
        if evaluate:
            assert np.array_equal(ctx.eval_metrics(0, 6000), ctx.eval_metrics(0, 6000, w0))
            assert np.array_equal(ctx.eval_sampled_metrics(0, 6000, 3, 10, 3000), ctx.eval_sampled_metrics(0, 6000, 3, 10, 3000, w0))
            ids = rng.integers(0, 6000, size=3000)
            assert np.array_equal(ctx.eval_samples_metrics(ids), ctx.eval_samples_metrics(ids, w0))
            assert np.array_equal(ctx.margins(ids), ctx.margins(ids, w0))
        ctx.sync_steps_staged(0, batch, steps, lr, want_losses=True)
        results.append((ctx.get_weights(), ctx.read_losses(steps)))
        ctx.close()
    np.testing.assert_array_equal(results[0][0], results[1][0])
    np.testing.assert_array_equal(results[0][1], results[1][1])


def test_errors(dy):
    from distributed_sgd_b200.native import DsgdEmpty, DsgdInvalid, DsgdRange, DsgdState, NativeCtx
    ctx, orc, data = dy
    N = data.n_rows
    L = ctx._l
    out8 = np.zeros(8, np.int64)
    for call in (lambda: ctx.margins([0, N]), lambda: ctx.margins([-1]), lambda: ctx.eval_samples_metrics([3, N]),
                 lambda: ctx.eval_metrics(0, N + 1), lambda: ctx.eval_metrics(-1, 5), lambda: ctx.eval_metrics(9, 8),
                 lambda: ctx.eval_sampled_metrics(0, N + 1, 1, 0, 5)):
        with pytest.raises(DsgdRange):
            call()
    for call in (lambda: ctx.margins(np.zeros(0, np.int32)), lambda: ctx.eval_samples_metrics(np.zeros(0, np.int32)),
                 lambda: ctx.eval_metrics(4, 4), lambda: ctx.eval_sampled_metrics(5, 5, 1, 0, 0),
                 lambda: ctx.eval_sampled_metrics(10, 20, 1, 3, 3)):
        with pytest.raises(DsgdEmpty):
            call()
    with pytest.raises(DsgdInvalid):
        ctx.eval_sampled_metrics(10, 20, 1, 0, 11)
    ids = np.arange(4, dtype=np.int32)
    assert L.dsgd_margins(ctx._h, None, ids.ctypes.data, 4, None) == -1            # NULL outputs
    assert L.dsgd_eval_metrics(ctx._h, None, 0, 10, None) == -1
    assert L.dsgd_eval_sampled_metrics(ctx._h, None, 0, 10, 1, 0, 5, None) == -1
    assert L.dsgd_eval_samples_metrics(ctx._h, None, ids.ctypes.data, 4, None) == -1
    assert L.dsgd_eval_samples_metrics(ctx._h, None, None, 4, out8.ctypes.data) == -1   # NULL ids
    with pytest.raises(DsgdState):
        ctx.probabilities(ids)
    with NativeCtx(0, data.dim, LAM) as empty:
        for call in (lambda: empty.margins([0]), lambda: empty.eval_metrics(0, 1), lambda: empty.eval_samples_metrics([0]),
                     lambda: empty.eval_sampled_metrics(0, 1, 1, 0, 1)):
            with pytest.raises(DsgdState):
                call()
    w = dyadic_w(np.random.default_rng(1), data.dim)                 # the ctx still answers correctly after the refusals
    assert np.array_equal(ctx.eval_metrics(10, 20, w), om.metrics(orc, w, begin=10, n=10))


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
        assert np.array_equal(ctx.eval_metrics(0, 5000), ctx.eval_metrics(0, 5000, w))
        idx = rng.choice(data.dim, size=500, replace=False).astype(np.int32)
        ctx.update_grad(idx, rng.standard_normal(500) * 0.05)          # changes the replica, not its scalars
        w2 = ctx.get_weights()
        assert not np.array_equal(w, w2)
        assert np.array_equal(ctx.eval_metrics(0, 5000), ctx.eval_metrics(0, 5000, w2))
        assert np.array_equal(ctx.eval_samples_metrics(ids), ctx.eval_samples_metrics(ids, w2))
        assert np.array_equal(ctx.margins(ids), ctx.margins(ids, w2))
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
    a = ctx.eval_metrics(4800, 6000)                       # the first metrics pass of this process: sort kernels included
    b = ctx.eval_sampled_metrics(0, 6000, 5, 0, 3000)
    c = ctx.margins(np.arange(100))
    try:
        ctx.eval_samples_metrics(np.zeros(6001, np.int32))  # more ids than rows: the buffers would have to grow
        refused = False
    except DsgdState:
        refused = True
    print("OK", running, int(a[:6].sum()), int(b[:6].sum()), len(c), refused)
finally:
    ctx.stop_async()
ctx.close()
"""


def test_first_metrics_call_while_the_loop_runs_returns():
    """A fresh process whose async loop runs makes its first metrics calls: every kernel they launch, the sort's included,
    was loaded, and every buffer they use sized, before the loop started; a list longer than that is refused.  The loop is stopped in a `finally`; the subprocess has a timeout."""
    r = subprocess.run([sys.executable, "-s", "-c", _FRESH.format(root=ROOT)], cwd=ROOT, capture_output=True, text=True,
                       timeout=180)
    assert r.returncode == 0, r.stdout + r.stderr
    assert "OK True 1200 3000 100 True" in r.stdout, r.stdout + r.stderr


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
    out = [m.local_metrics(w, test_data=True), m.local_metrics(w), m.local_sampled_metrics(w, 1500, test_data=True),
           m.local_sampled_metrics(w, 3000)]
    m.ctx.set_weights(w)
    out.append(m.local_metrics(test_data=True))
    return out


def test_master_metrics_against_the_oracle():
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
        for got, i in zip(res, ids):
            i = i.astype(np.int32)
            want = metrics_dict(om.metrics(orc, w, idx=i, margins=slave.ctx.margins(i, w)))
            assert got == want
            tp, fn, pn, fp, tn, nn = (want[k] for k in ("tp", "fn", "pos_no_pred", "fp", "tn", "neg_no_pred"))
            assert got["precision"] == tp / (tp + fp) and got["recall"] == tp / (tp + fn + pn)
            assert math.isclose(got["f1"], 2 * got["precision"] * got["recall"] / (got["precision"] + got["recall"]),
                                rel_tol=1e-15)
            assert got["auc"] == want["u2"] / (2 * (tp + fn + pn) * (fp + tn + nn))
        assert res[0]["accuracy"] == m.local_accuracy(w, test_data=True)
        assert res[1]["accuracy"] == m.local_accuracy(w)
        assert res[4]["accuracy"] == m.local_accuracy(None, test_data=True) and res[4] == res[0]
        # the sampled form consumes one draw of the sampled loss: the same key sequence
        m2 = MasterSync(0, train, test, model, 1, slave=slave, seed=11)
        m2.local_sampled_loss(w, 1500, test_data=True)
        assert m2.local_sampled_metrics(w, 3000) == res[3]
        from distributed_sgd_b200.native import DsgdEmpty
        with pytest.raises(DsgdEmpty):
            m2.local_sampled_metrics(w, 0)
        # jvm_exact: the ids of the reference's shuffle go through the list form
        from distributed_sgd_b200.utils.jvm_random import JvmRandom
        mj = MasterSync(0, train, test, model, 1, slave=slave, seed=0, jvm_exact=True)
        jids = (JvmRandom(0).shuffle(np.arange(2200))[:700] + 4800).astype(np.int32)
        assert mj.local_sampled_metrics(w, 700, test_data=True) == metrics_dict(slave.ctx.eval_samples_metrics(jids, w))
        # Slave surface
        assert np.array_equal(slave.margins(np.arange(50), w), slave.ctx.margins(np.arange(50), w))
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
        one = json.dumps(_results(MasterSync(0, train, test, model, 1, slave=slave, seed=11), rand_w(np.random.default_rng(8), data.dim)))
    finally:
        slave.stop()
    assert res[0] == res[1] == one
