"""Async (Hogwild) kernels at their edges, against the fp64 oracle through the C ABI.

- Replays on dyadic data, where the device's arithmetic is the oracle's operation for operation: weights equal bit for
  bit, in k_async_worker_b1 (batch 1) and k_async_worker (batch > 1), on rows on both sides of the 128 prefetched pairs,
  in any column order, with batches that share most of their columns.
- The 1e-20 filter of the reference's Sparse at every place it acts: the dot product, c, m + c, the delta and the
  result w - delta of every replica update, including dsgd_update_grad.
- The device-side batch draw, Hogwild conservation with concurrent lanes, the drift of the incremental S = w . d,
  concurrent dsgd_update_grad calls, and rows that repeat a key.
"""
import threading
import time

import numpy as np
import pytest

from helpers import FILTER_CASES, conservation_rows, csr, edge_rows, filter_case, filter_expect, make_pair

pytestmark = pytest.mark.gpu


def _batches(rng, n_rows, batch, n_updates):
    return np.stack([rng.choice(n_rows, size=batch, replace=False) for _ in range(n_updates)]).astype(np.int32).reshape(-1)


@pytest.fixture(scope="module")
def edge_data():
    return edge_rows(21)


# ---- a. replay: bit for bit at lambda = 0, and at the stated tolerance with lambda > 0 ---------------------------------

@pytest.mark.parametrize("batch,n_updates", [(1, 400), (2, 120), (31, 30), (32, 30), (33, 30), (64, 16), (256, 6)])
def test_replay_bit_exact_on_dyadic_rows(edge_data, batch, n_updates):
    """lambda = 0: c is 0, and per column the device folds the batch in row order into the lane's scratch, then forms
    sum / B, * lr and w - delta, like the oracle.  Values and w0 are dyadic and lr = 2^-3, so with a power-of-two B every
    dot product is exact too, and with B = 31 or 33 only the gates read rounded dots: weights must be equal."""
    data, w0 = edge_data
    ctx, orc = make_pair(data, lam=0.0, is_async=True)
    idx = _batches(np.random.default_rng(100 + batch), data.n_rows, batch, n_updates)
    ctx.async_replay(w0, idx, batch, 0.125)
    w = ctx.get_weights()
    w_ref = orc.async_run(w0, idx, batch, 0.125)
    assert np.count_nonzero(w != w0) > 100                     # the run moved many columns (not a vacuous pass)
    np.testing.assert_array_equal(w, w_ref)
    assert ctx.async_updates() == n_updates
    ctx.close()


@pytest.mark.parametrize("batch,n_updates", [(1, 400), (33, 30), (256, 6)])
def test_replay_with_regularizer(edge_data, batch, n_updates):
    """lambda > 0: c comes from the device's running S = w . d; weights within rtol 1e-9, supports exact, and the gate
    decisions exact (a wrong gate moves a whole row's columns by lr * x / B, far outside the tolerance)."""
    data, w0 = edge_data
    ctx, orc = make_pair(data, lam=1e-3, is_async=True)
    idx = _batches(np.random.default_rng(200 + batch), data.n_rows, batch, n_updates)
    ctx.async_replay(w0, idx, batch, 0.125)
    w = ctx.get_weights()
    w_ref = orc.async_run(w0, idx, batch, 0.125)
    assert (w == 0).tolist() == (w_ref == 0).tolist()
    np.testing.assert_allclose(w, w_ref, rtol=1e-9, atol=1e-13)
    ctx.close()


# ---- b. the 1e-20 filter, one or two hand-built updates through both kernels -------------------------------------------

def _filter_pair(name):
    from distributed_sgd_b200.native import NativeCtx
    from oracle.oracle import Oracle
    rows, labels, dim, d, lam, lr, w0 = filter_case(name)
    data = csr(rows, np.asarray(labels, np.int8), dim)
    ctx = NativeCtx(0, dim, lam, is_async=True)
    ctx.load_csr(data.row_ptr, data.col, data.val, data.label)
    ctx.set_dim_sparsity(d)
    orc = Oracle(data.row_ptr, data.col, data.val, data.label, dim, lam)
    orc.set_dim_sparsity(d)
    return ctx, orc, len(rows), lr, w0


@pytest.mark.parametrize("batch", [1, 2])
@pytest.mark.parametrize("name", FILTER_CASES)
def test_filter_edges(name, batch):
    """Batch 1 runs k_async_worker_b1; batch 2 runs k_async_worker on the same row twice (sum 2x, mean x: the same delta)."""
    ctx, orc, n_rows, lr, w0 = _filter_pair(name)
    idx = np.repeat(np.arange(n_rows, dtype=np.int32), batch)
    ctx.async_replay(w0, idx, batch, lr)
    w = ctx.get_weights()
    w_ref = orc.async_run(w0, idx, batch, lr)
    expect = filter_expect(name)
    for j, v in expect.items():
        assert w_ref[j] == v, (j, w_ref[j], v)               # the case is what it says on the oracle
        assert w[j] == v, (j, w[j], v)
    assert (w == 0).tolist() == (w_ref == 0).tolist()
    np.testing.assert_array_equal(w, w_ref)
    ctx.close()


def test_update_grad_filters_the_residual():
    """SlaveImpl.updateGrad builds a new Sparse (core/Slave.scala:180): w - v = 2^-72 must become 0."""
    ctx, _, _, _, w0 = _filter_pair("residual")
    ctx.set_weights(w0)
    ctx.update_grad([3, 5], [2.0 ** -20, 0.5])
    w = ctx.get_weights()
    assert w[3] == 0.0, w[3]
    assert w[5] == -0.5
    ctx.close()


# ---- c. the device's batch draw (free-running, one lane, lambda = 0) ---------------------------------------------------

@pytest.fixture(scope="module")
def private_columns():
    """Row i holds only column i (value 1, y = +1); from w0 = 2^10 the gate always passes, and the decrease of column i
    counts how often row i was drawn."""
    n = 2000
    return csr([([i], [1.0]) for i in range(n)], np.ones(n, np.int8), n)


def _run_free(ctx, w0, assigned, batch, lr, n_updates, lanes=1, seed=5):
    ctx.start_async(w0, np.asarray(assigned, np.int32), batch=batch, lr=lr, concurrency=lanes, max_updates=n_updates,
                    seed=seed)
    t0 = time.time()
    while ctx.async_running() and time.time() - t0 < 60:
        time.sleep(0.002)
    assert not ctx.async_running()
    ctx.stop_async()


@pytest.mark.parametrize("batch", [1, 8])
def test_device_draw_range(private_columns, batch):
    """Batch 1 draws data(assigned(i)); batch > 1 draws POSITIONS 0..n-1 and indexes `data` with them (quirk Q6,
    core/Slave.scala:87)."""
    data = private_columns
    ctx, _ = make_pair(data, lam=0.0, is_async=True)
    w0 = np.full(data.dim, 1024.0)
    lr, U = 2.0 ** -4, 3000
    _run_free(ctx, w0, np.arange(1000, 2000), batch, lr, U)
    counts = (w0 - ctx.get_weights()) / (lr / batch)
    assert np.array_equal(counts, np.round(counts))
    hit = np.flatnonzero(counts)
    lo, hi = (1000, 2000) if batch == 1 else (0, 1000)
    assert hit.min() >= lo and hit.max() < hi
    assert counts.sum() == U * batch
    assert counts.max() <= U                                   # without replacement inside a batch
    ctx.close()


@pytest.mark.parametrize("n_assigned,batch", [(33, 40), (1000, 1024)])
def test_device_draw_clips_batch_to_assigned(private_columns, n_assigned, batch):
    """`shuffle take batchSize` of a shorter list takes all of it: every position is drawn once per update, so each of
    the first n_assigned columns equals U sequential subtractions of (1 / n) * lr."""
    data = private_columns
    ctx, _ = make_pair(data, lam=0.0, is_async=True)
    w0 = np.full(data.dim, 1024.0)
    lr, U = 0.25, 150
    _run_free(ctx, w0, np.arange(500, 500 + n_assigned), batch, lr, U)
    w = ctx.get_weights()
    ref = 1024.0
    step = (1.0 / n_assigned) * lr
    for _ in range(U):
        ref = ref - step
    np.testing.assert_array_equal(w[:n_assigned], np.full(n_assigned, ref))
    np.testing.assert_array_equal(w[n_assigned:], w0[n_assigned:])
    ctx.close()


# ---- d. Hogwild conservation: concurrent lanes lose and duplicate nothing ----------------------------------------------

@pytest.fixture(scope="module")
def conservation():
    return conservation_rows()


@pytest.mark.parametrize("batch", [1, 8])
@pytest.mark.parametrize("lanes", [1, 32, 256])
def test_hogwild_conservation(conservation, lanes, batch):
    """Every entry is 2^-4, y = +1, w0 = 2^10, lr = 2^-6: the gate always passes and every partial sum is exact in any
    order.  So the update count, the total decrease, the master replica and the outbox must all be exact."""
    data, k = conservation
    ctx, _ = make_pair(data, lam=0.0, is_async=True)
    w0 = np.full(data.dim, 1024.0)
    lr, U = 2.0 ** -6, 20000
    ctx.async_host_master(w0)
    ctx.async_outbox_enable()
    _run_free(ctx, w0, np.arange(data.n_rows), batch, lr, U, lanes=lanes, seed=lanes + batch)
    w, wm, out = ctx.get_weights(), ctx.async_master_weights(), ctx.async_outbox_read()
    assert ctx.async_updates() == U
    assert (w0 - w).sum() == U * lr * k * 2.0 ** -4
    np.testing.assert_array_equal(w, wm)
    np.testing.assert_array_equal(out, w - w0)
    ctx.close()


# ---- e. drift of the incremental S = w . d ----------------------------------------------------------------------------

@pytest.fixture(scope="module")
def synth():
    from distributed_sgd_b200.utils import synthetic_rcv1
    return synthetic_rcv1(n_rows=5000, seed=9)


@pytest.mark.parametrize("batch,n_updates", [(1, 20000), (8, 5000)])
def test_incremental_s_drift(synth, batch, n_updates):
    """The device carries S = w . d by subtracting sum_j delta_j d_j per update; the oracle recomputes it every update.
    Over 20 000 (batch 1) and 5 000 (batch 8) updates with lambda = 1e-3 the weights stay within rtol 1e-9, atol 1e-13."""
    ctx, orc = make_pair(synth, lam=1e-3, n_train=4000, is_async=True)
    idx = _batches(np.random.default_rng(300 + batch), 4000, batch, n_updates)
    w0 = np.zeros(synth.dim)
    ctx.async_replay(w0, idx, batch, 0.5)
    w = ctx.get_weights()
    w_ref = orc.async_run(w0, idx, batch, 0.5)
    nz = w_ref != 0
    rel = np.abs(w - w_ref)[nz] / np.abs(w_ref[nz])
    print(f"batch {batch}: {n_updates} updates, largest relative error {rel.max():.3e}, "
          f"largest absolute error {np.abs(w - w_ref).max():.3e}")
    assert (w == 0).tolist() == (w_ref == 0).tolist()
    np.testing.assert_allclose(w, w_ref, rtol=1e-9, atol=1e-13)
    ctx.close()


# ---- f. concurrent dsgd_update_grad -----------------------------------------------------------------------------------

def test_update_grad_from_eight_threads(synth):
    """Eight host threads, 50 calls each, dyadic deltas on 64 shared keys, the loop idle: w == w0 - sum exactly.  The
    first call stages 4 096 keys, so the staging buffers never grow while the threads run."""
    ctx, _ = make_pair(synth, lam=1e-3, n_train=4000, is_async=True)
    dim = synth.dim
    w0 = np.full(dim, 1024.0)
    ctx.set_weights(w0)
    ctx.update_grad(np.arange(4096), np.zeros(4096))           # sizes the staging buffers; zeros change nothing
    keys = np.random.default_rng(5).choice(dim, size=64, replace=False)
    calls = []
    for t in range(8):
        rng = np.random.default_rng(1000 + t)
        calls.append([(rng.choice(keys, size=int(rng.integers(1, 65)), replace=False).astype(np.int32),
                       rng.integers(-512, 513, size=64) / 256.0) for _ in range(50)])
    expect = w0.copy()
    for per_thread in calls:
        for idx, val in per_thread:
            expect[idx] -= val[:len(idx)]
    start = threading.Barrier(8)
    errors = []

    def work(per_thread):
        try:
            start.wait()
            for idx, val in per_thread:
                ctx.update_grad(idx, val[:len(idx)])
        except Exception as e:  # pragma: no cover - reported below
            errors.append(e)

    threads = [threading.Thread(target=work, args=(c,)) for c in calls]
    for th in threads:
        th.start()
    for th in threads:
        th.join()
    assert not errors
    np.testing.assert_array_equal(ctx.get_weights(), expect)
    ctx.close()


# ---- g. a row is a Map: repeated keys are rejected ---------------------------------------------------------------------

@pytest.mark.parametrize("bad_row", [[3, 3, 5], [1, 4, 6, 8, 9, 1], [7, 2, 5, 2, 0]], ids=["adjacent", "distant", "unsorted"])
def test_load_csr_rejects_repeated_keys(bad_row):
    from distributed_sgd_b200.native import DsgdInvalid, NativeCtx
    ctx = NativeCtx(0, 10, 0.0, is_async=True)
    good = [([1, 2, 3], [1.0, 1.0, 1.0]), ([3, 1, 2, 9], [1.0, 1.0, 1.0, 1.0])]   # the same keys in two rows: fine
    data = csr(good, np.ones(2, np.int8), 10)
    ctx.load_csr(data.row_ptr, data.col, data.val, data.label)
    data = csr(good + [(bad_row, np.ones(len(bad_row)))], np.ones(3, np.int8), 10)
    with pytest.raises(DsgdInvalid, match="repeats column"):
        ctx.load_csr(data.row_ptr, data.col, data.val, data.label)
    ctx.close()
