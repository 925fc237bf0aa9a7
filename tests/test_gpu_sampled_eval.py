"""Sampled evaluation (Master.localSampledLoss / localSampledAccuracy, core/Master.scala:109-118) on the device against the
fp64 oracle.

dsgd_eval_sampled_counts draws position i of its sample as row_begin + dsgd_feistel(i, ...) with k_draw_rows; the host
reproduces the same ids with dsgd_feistel_pos (libdsgd_host.so, the same source), and the oracle's loss_acc on those ids
gives the hinge and correct counts the device must return exactly.  Sample sizes cover k_rows (below 2048) and every work
split of the streaming pass over a list, derived from the SM count as stream_launch (csrc/dsgd_api.cu) picks it.
"""
import math

import numpy as np
import pytest

from helpers import make_pair

pytestmark = pytest.mark.gpu

LAM = 1e-4
ROW_BEGIN = 7                    # sampled ranges start at an odd row
MIN_STREAM_ROWS = 2048           # kStreamMinRows (csrc/dsgd_api.cu)


def split_bounds(sm_count):
    """stream_launch's rule with S SMs (W = 32 * S warps): blocks of 32 rows, lowered to 16 and then 8 while the pass has
    fewer than 6 * W blocks.  Returns (last pass with static blocks only, first pass with 16-row blocks, first pass with
    32-row blocks), in rows."""
    W = 32 * sm_count
    return 8 * W, 16 * (6 * W - 1) + 1, 32 * (6 * W - 1) + 1


def ragged(n):
    while n % 32 == 0 or n % 5 == 0:
        n += 1
    return n


# sample sizes k, resolved against the device's SM count
REGIMES = {
    "krows_1": lambda st, b16, b32: 1,
    "krows_2047": lambda st, b16, b32: MIN_STREAM_ROWS - 1,
    "static_2048": lambda st, b16, b32: MIN_STREAM_ROWS,
    "static_ragged": lambda st, b16, b32: ragged(st // 2 + 7),
    "static_last": lambda st, b16, b32: st,
    "dyn8_first": lambda st, b16, b32: st + 1,
    "dyn8_ragged": lambda st, b16, b32: ragged((st + b16) // 2),
    "blk16_first": lambda st, b16, b32: b16,
    "blk16_ragged": lambda st, b16, b32: ragged((b16 + b32) // 2),
    "blk32_first": lambda st, b16, b32: b32,
    "blk32_ragged": lambda st, b16, b32: ragged(b32 + 9000),
}


def sm_count():
    from distributed_sgd_b200.native import NativeCtx
    with NativeCtx(0, 16, 0.0) as c:
        return int(c.info()["sm_count"])


def rand_w(rng, dim):
    return np.where(rng.random(dim) < 0.6, rng.standard_normal(dim) * 0.1, 0.0)


def host_ids(row_begin, row_end, key, lo, hi):
    """Row ids of positions [lo, hi) of the draw with `key` over rows [row_begin, row_end), made on the host."""
    from distributed_sgd_b200.native import host_lib
    h, n = host_lib(), row_end - row_begin
    pos = np.fromiter((h.dsgd_feistel_pos(p, n, key) for p in range(lo, hi)), dtype=np.int64, count=hi - lo)
    return (row_begin + pos).astype(np.int32)


def check(orc, w, got, ids):
    """got = (hinge, correct, ||w||^2) from the device; the oracle's loss_acc on the same ids fixes both counts."""
    h, c, n2 = got
    k = len(ids)
    loss_ref, acc_ref = orc.loss_acc(w, idx=ids)
    n2_ref = float(np.dot(w, w))
    assert h == round((loss_ref - LAM * n2_ref) * k) and c == round(acc_ref * k), (h, c, loss_ref, acc_ref, k)
    assert c / k == acc_ref
    np.testing.assert_allclose(n2, n2_ref, rtol=1e-12)
    np.testing.assert_allclose(LAM * n2 + h / k, loss_ref, rtol=1e-12)


@pytest.fixture(scope="module")
def big():
    """Enough rows for a sample in every streaming regime; short rows keep the host side quick."""
    from distributed_sgd_b200.utils import synthetic_rcv1
    st, b16, b32 = split_bounds(sm_count())
    k_max = max(f(st, b16, b32) for f in REGIMES.values())
    data = synthetic_rcv1(n_rows=ROW_BEGIN + k_max + 4321, seed=5, mean_nnz=6.0, max_nnz=300)
    ctx, orc = make_pair(data, LAM)
    yield ctx, orc, data, (st, b16, b32)
    ctx.close()


@pytest.mark.parametrize("regime", list(REGIMES))
def test_device_draw_equals_host_draw(big, regime):
    ctx, orc, data, bounds = big
    k = REGIMES[regime](*bounds)
    rng = np.random.default_rng(len(regime) * 1000 + k)
    b, e = ROW_BEGIN, data.n_rows
    n = e - b
    assert k <= n
    w = rand_w(rng, data.dim)
    w_res = rand_w(rng, data.dim)
    ctx.set_weights(w_res)
    # explicit weights from position 0; resident weights from an offset, with a second key; again (counters cleared?)
    for key, lo, weights in ((0x1234567890ABCDEF, 0, w), (2**64 - 3, n - k, None), (99, (n - k) // 2, w)):
        ids = host_ids(b, e, key, lo, lo + k)
        got = ctx.eval_sampled_counts(b, e, key, lo, lo + k, weights)
        check(orc, w_res if weights is None else weights, got, ids)


@pytest.mark.parametrize("n", [1, 2, 3, 4, 5, 16, 17, 2047, 2048, 4096, 4097, 65536, 65537])
def test_whole_range_equals_full_pass(big, n):
    ctx, orc, data, _ = big
    w = rand_w(np.random.default_rng(n), data.dim)
    b, e = ROW_BEGIN, ROW_BEGIN + n
    for key in (0, 7, 2**63 + 11):
        assert ctx.eval_sampled_counts(b, e, key, 0, n, w) == ctx.eval_counts(b, e, w)
    ids = host_ids(b, e, 7, 0, n)
    assert sorted(ids.tolist()) == list(range(b, e))


def test_shards_add_up(big):
    ctx, orc, data, _ = big
    w = rand_w(np.random.default_rng(3), data.dim)
    b, e, key, k = ROW_BEGIN, data.n_rows, 0xC0FFEE, 60_000
    whole = ctx.eval_sampled_counts(b, e, key, 0, k, w)
    cuts = [0, 1000, 1001, 3500, 20_000, k]                # shards of 1000, 1, 2499, 16 500 and 40 000 positions
    parts = [ctx.eval_sampled_counts(b, e, key, lo, hi, w) for lo, hi in zip(cuts[:-1], cuts[1:])]
    assert (sum(p[0] for p in parts), sum(p[1] for p in parts)) == whole[:2]
    assert all(p[2] == whole[2] for p in parts)
    check(orc, w, whole, host_ids(b, e, key, 0, k))


@pytest.mark.parametrize("k", [1500, 40_000])
def test_list_with_repeats(big, k):
    ctx, orc, data, _ = big
    rng = np.random.default_rng(k)
    w = rand_w(rng, data.dim)
    first = rng.integers(ROW_BEGIN, data.n_rows, size=k - k // 3).astype(np.int32)
    ids = np.concatenate([first, first[: k // 3]])        # a third of the list repeats earlier ids
    rng.shuffle(ids)
    check(orc, w, ctx.eval_samples_counts(ids, w), ids)
    ctx.set_weights(w)
    check(orc, w, ctx.eval_samples_counts(ids), ids)


def test_errors(big):
    from distributed_sgd_b200.native import DsgdEmpty, DsgdInvalid, DsgdRange, DsgdState, NativeCtx
    ctx, orc, data, _ = big
    N = data.n_rows
    with pytest.raises(DsgdRange):
        ctx.eval_samples_counts([0, N])
    with pytest.raises(DsgdRange):
        ctx.eval_samples_counts([-1, 3])
    with pytest.raises(DsgdEmpty):
        ctx.eval_samples_counts(np.zeros(0, np.int32))
    with pytest.raises(DsgdRange):
        ctx.eval_sampled_counts(0, N + 1, 1, 0, 5)
    with pytest.raises(DsgdRange):
        ctx.eval_sampled_counts(-1, 10, 1, 0, 5)
    with pytest.raises(DsgdEmpty):
        ctx.eval_sampled_counts(5, 5, 1, 0, 0)
    for lo, hi in ((-1, 3), (0, 11), (4, 12)):
        with pytest.raises(DsgdInvalid):
            ctx.eval_sampled_counts(10, 20, 1, lo, hi)
    for lo, hi in ((3, 3), (5, 4)):
        with pytest.raises(DsgdEmpty):
            ctx.eval_sampled_counts(10, 20, 1, lo, hi)
    with NativeCtx(0, data.dim, LAM) as empty:
        with pytest.raises(DsgdState):
            empty.eval_sampled_counts(0, 1, 1, 0, 1)
        with pytest.raises(DsgdState):
            empty.eval_samples_counts([0])
    w = rand_w(np.random.default_rng(1), data.dim)         # the ctx still answers correctly after the refusals
    check(orc, w, ctx.eval_sampled_counts(10, 20, 1, 0, 10, w), host_ids(10, 20, 1, 0, 10))


def test_staged_stream_is_untouched():
    """A host that staged a sample stream for dsgd_sync_steps_staged finds it intact after sampled evaluations."""
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
            ctx.eval_sampled_counts(0, 6000, 17, 0, 5000)            # streaming pass
            ctx.eval_sampled_counts(0, 6000, 18, 100, 400)           # k_rows
            ctx.eval_samples_counts(rng.integers(0, 6000, size=3000))
            ctx.eval_samples_counts(rng.integers(0, 6000, size=50))
        ctx.sync_steps_staged(0, batch, steps, lr, want_losses=True)
        results.append((ctx.get_weights(), ctx.read_losses(steps)))
        ctx.close()
    np.testing.assert_array_equal(results[0][0], results[1][0])
    np.testing.assert_array_equal(results[0][1], results[1][1])


# ---- Master.local_sampled_* ----------------------------------------------------------------------------------------

@pytest.fixture(scope="module")
def master_setup():
    from distributed_sgd_b200 import Slave, SparseSVM
    from distributed_sgd_b200.utils import synthetic_rcv1
    from oracle.oracle import Oracle
    data = synthetic_rcv1(n_rows=7000, seed=13)
    train, test = data.split_at(4800)
    model = SparseSVM(LAM)
    slave = Slave(0, 0, train, model, world=1, device=0, test_data=test)
    orc = Oracle(data.row_ptr, data.col, data.val, data.label, data.dim, LAM)
    orc.set_dim_sparsity(model.dim_sparsity)
    yield slave, model, train, test, orc
    slave.stop()


def _master(setup, seed, **kw):
    from distributed_sgd_b200 import MasterSync
    slave, model, train, test, _ = setup
    return MasterSync(0, train, test, model, 1, slave=slave, seed=seed, **kw)


def test_master_train_and_test_samples_match_the_oracle(master_setup):
    from distributed_sgd_b200.core.master import sampled_key
    orc = master_setup[4]
    m = _master(master_setup, seed=11)
    w = rand_w(np.random.default_rng(8), m.dim)
    for t, (count, test_data, b, e) in enumerate([(3000, False, 0, 4800), (500, True, 4800, 7000),
                                                  (10_000, True, 4800, 7000), (40, False, 0, 4800)]):
        k = min(count, e - b)
        ids = host_ids(b, e, sampled_key(11, t), 0, k)
        loss, acc = m.local_sampled_loss_accuracy(w, count, test_data)
        loss_ref, acc_ref = orc.loss_acc(w, idx=ids)
        assert acc == acc_ref
        np.testing.assert_allclose(loss, loss_ref, rtol=1e-12)
    m.ctx.set_weights(w)
    k = 2500
    ids = host_ids(0, 4800, sampled_key(11, 4), 0, k)
    loss_ref, acc_ref = orc.loss_acc(w, idx=ids)
    np.testing.assert_allclose(m.local_sampled_loss(None, k), loss_ref, rtol=1e-12)
    assert m.local_sampled_accuracy(None, k) == orc.loss_acc(w, idx=host_ids(0, 4800, sampled_key(11, 5), 0, k))[1]


def test_master_draws_fresh_samples_and_repeats_with_the_seed(master_setup):
    w = rand_w(np.random.default_rng(9), master_setup[0].dim)
    runs = []
    for _ in range(2):
        m = _master(master_setup, seed=21)
        runs.append([m.local_sampled_loss_accuracy(w, 300, test_data=True) for _ in range(6)])
    assert runs[0] == runs[1]                                       # a new Master with the same seed repeats the sequence
    assert len(set(runs[0])) > 1                                    # consecutive calls draw different samples
    from distributed_sgd_b200.core.master import sampled_key
    a, b = host_ids(4800, 7000, sampled_key(21, 0), 0, 300), host_ids(4800, 7000, sampled_key(21, 1), 0, 300)
    assert set(a.tolist()) != set(b.tolist())


def test_master_whole_sample_equals_full_evaluation(master_setup):
    m = _master(master_setup, seed=2)
    w = rand_w(np.random.default_rng(10), m.dim)
    for test_data in (False, True):
        n = m.n_test if test_data else m.n_train
        for count in (n, n + 1, 10**9):
            assert m.local_sampled_loss_accuracy(w, count, test_data) == m.local_loss_accuracy(w, test_data)
    m.ctx.set_weights(w)
    assert m.local_sampled_loss_accuracy(None, 10**6) == m.local_loss_accuracy(None)


def test_master_empty_sample(master_setup):
    from distributed_sgd_b200.native import DsgdEmpty
    m = _master(master_setup, seed=2)
    with pytest.raises(DsgdEmpty):
        m.local_sampled_loss(None, 0)
    assert math.isnan(m.local_sampled_accuracy(None, 0, test_data=True))


def test_master_jvm_exact_sample(master_setup):
    from distributed_sgd_b200.ml import split_strategy
    from distributed_sgd_b200.utils.jvm_random import JvmRandom
    orc = master_setup[4]
    m = _master(master_setup, seed=0, jvm_exact=True)
    w = rand_w(np.random.default_rng(11), m.dim)
    ref = JvmRandom(0)
    ids = ref.shuffle(np.arange(2200))[:700] + 4800
    loss, acc = m.local_sampled_loss_accuracy(w, 700, test_data=True)
    loss_ref, acc_ref = orc.loss_acc(w, idx=ids)
    assert acc == acc_ref
    np.testing.assert_allclose(loss, loss_ref, rtol=1e-12)
    ids = ref.shuffle(np.arange(4800))[:2600]                        # the streaming list pass
    assert m.local_sampled_accuracy(w, 2600) == orc.loss_acc(w, idx=ids)[1]
    # the next epoch draw continues the stream where the reference's global Random would be
    groups = split_strategy.vanilla(4800, 2)
    got = m.draw_epoch(groups, 100)
    want = ref.sync_epoch(4800, 2, 100, group_size=len(groups[0]))
    assert [[g.tolist() for g in st] for st in got] == [[g.tolist() for g in st] for st in want]


def test_master_fit_is_unchanged_by_sampled_calls(master_setup):
    from distributed_sgd_b200.ml import EarlyStopping
    w = rand_w(np.random.default_rng(12), master_setup[0].dim)
    states = []
    for sample in (True, False):
        m = _master(master_setup, seed=5)
        if sample:
            m.local_sampled_loss_accuracy(w, 3000)
            m.local_sampled_accuracy(w, 100, test_data=True)
        state = m.fit(np.zeros(m.dim), max_epochs=2, batch_size=100, learning_rate=0.5,
                      stopping_criterion=EarlyStopping.no_improvement(patience=5, min_delta=0.01))
        states.append((state.grad.copy(), m.history["losses"], m.history["test_losses"]))
    np.testing.assert_array_equal(states[0][0], states[1][0])
    assert states[0][1:] == states[1][1:]
