"""Calibration on the device (dsgd_calibrate*, dsgd_calibrated_probabilities, dsgd_eval_calibration*; DESIGN.md §4.11)
against the checker of oracle/calib.py run over the device's own margins.

The property the design rests on: every sum over the rows is an order-free fixed-point sum and the Newton arithmetic between
the sums is one fixed sequence, so (A, B, F, iterations, status) are ONE bit pattern per (weights, row multiset) -- whatever the
row form, the row order, the grid or the model flag."""
import os
import struct
import subprocess
import sys

import numpy as np
import pytest

from helpers import csr
from oracle import calib

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LAM = 1e-4
N_ROWS, N_TRAIN = 100_000, 80_000
SIZES = [2, 31, 32, 33, 2047, 2048, 100_000]


def bits(fit):
    """A NativeCtx.calibrate* result as a comparable tuple: the bits of A, B and F, iterations, status, rows, NaN rows, points."""
    a, b, f, info = fit
    return (struct.pack("<3d", a, b, f), *[int(v) for v in info])


def trained(ctx, n_train, steps=300, batch=64, lr=0.5, seed=0):
    rng = np.random.default_rng(seed)
    ctx.set_weights(np.zeros(ctx.dim))
    ctx.sync_steps(rng.integers(0, n_train, size=steps * batch).astype(np.int32), batch, steps, lr, want_losses=False)
    return ctx.get_weights()


@pytest.fixture(scope="module")
def rcv():
    """(SVM context, SparseLogistic context, data, weights trained on the SVM context); both contexts hold the same rows."""
    from distributed_sgd_b200.native import NativeCtx
    from distributed_sgd_b200.utils import synthetic_rcv1
    data = synthetic_rcv1(n_rows=N_ROWS, seed=21)
    ctxs = []
    for logistic in (False, True):
        c = NativeCtx(0, data.dim, LAM, logistic=logistic)
        c.load_csr(data.row_ptr, data.col, data.val, data.label)
        c.compute_dim_sparsity(N_TRAIN)
        ctxs.append(c)
    w = trained(ctxs[0], N_TRAIN)
    yield ctxs[0], ctxs[1], data, w
    for c in ctxs:
        c.close()


def mixed_begin(label):
    """The first row whose successor has the other label: every range starting there holds both classes."""
    return int(np.flatnonzero(label[:-1] != label[1:])[0])


# ---- order-free bits ---------------------------------------------------------------------------------------------------

def test_one_bit_pattern_per_row_multiset(rcv):
    svm, logi, data, w = rcv
    b0 = mixed_begin(data.label)
    rng = np.random.default_rng(5)
    for n in SIZES + SIZES[-2::-1]:                                   # growing, then shrinking, on the same contexts
        b = 0 if n == N_ROWS else b0
        ids = np.arange(b, b + n, dtype=np.int32)
        ref = bits(svm.calibrate(b, b + n, w))
        assert ref[3] == n and ref[4] == 0
        assert bits(svm.calibrate_samples(ids[::-1].copy(), w)) == ref, n
        assert bits(svm.calibrate_samples(rng.permutation(ids).astype(np.int32), w)) == ref, n
        assert bits(svm.calibrate_sampled(b, b + n, 0x1234 + n, 0, n, w)) == ref, n     # the drawn sample covers the range
        assert bits(logi.calibrate(b, b + n, w)) == ref, n                              # the model flag does not matter
        print(f"n = {n}: A = {svm.calibrate(b, b + n, w)[0]!r}, iterations {ref[1]}, status {ref[2]}, points {ref[5]}")


@pytest.mark.parametrize("limit", [1, 2, 7])
def test_any_grid_limit_gives_the_same_bits(rcv, limit):
    """One CTA keeps 14 336 scores in shared memory and reads the rest of its slice from global memory: at limits 1 and 2 a
    100 000-row fit takes that path, at 7 it just fits."""
    svm, _, data, w = rcv
    b0 = mixed_begin(data.label)
    cases = [(b0, b0 + 33), (b0, b0 + 2048), (0, N_ROWS), (N_TRAIN, N_ROWS)]
    svm.set_grid_limit(0)
    want = [bits(svm.calibrate(b, e, w)) for b, e in cases]
    svm.set_grid_limit(limit)
    try:
        got = [bits(svm.calibrate(b, e, w)) for b, e in cases]
    finally:
        svm.set_grid_limit(0)
    assert got == want


# ---- against the checker -----------------------------------------------------------------------------------------------

def labels_of(data, ids):
    return np.asarray(data.label)[ids]


@pytest.mark.parametrize("rows", [(0, 2048), (0, N_TRAIN), (N_TRAIN, N_ROWS)])
def test_fit_against_the_checker_on_the_devices_margins(rcv, rows):
    svm, _, data, w = rcv
    b, e = rows
    ids = np.arange(b, e, dtype=np.int32)
    f, y = svm.margins(ids, w), labels_of(data, ids)
    a, bb, obj, info = svm.calibrate(b, e, w)
    ref = calib.fit(f, y)
    assert int(info[1]) == ref.status == calib.CONVERGED
    assert abs(a - ref.a) <= 1e-8 * max(1.0, abs(ref.a)) and abs(bb - ref.b) <= 1e-8 * max(1.0, abs(ref.b))
    assert abs(obj - ref.objective) <= 1e-10 * abs(ref.objective)
    t_pos, t_neg = calib.targets(f, y)[:2]
    s = calib.sums(f, y, t_pos, t_neg, a, bb)
    assert abs(s[0] - obj) <= 1e-12 * abs(obj)                      # F at the device's point, summed by the checker
    assert abs(s[1]) < 1.1e-5 and abs(s[2]) < 1.1e-5                # the stopping rule, with the 10 % margin
    # CUDA's exp and glibc's differ in the last bit of some terms; a line-search decision flips only if F(new) lands within
    # that of the sufficient-decrease bound, which none of these cases does: the counts are equal.
    print(f"rows {rows}: A = {a!r}, B = {bb!r}, F = {obj!r}; device {int(info[0])} iterations / {int(info[4])} points, "
          f"checker {ref.iterations} / {ref.evaluations}")
    assert (int(info[0]), int(info[4])) == (ref.iterations, ref.evaluations)
    assert a > 0                                                    # a positive row has a negative x . w


def planted(scores, labels):
    """(data, w): row i holds x = 1 in its own column i, so the weights w[i] = scores[i] give f_i = scores[i] exactly."""
    n = len(scores)
    return csr([([i], [1.0]) for i in range(n)], np.asarray(labels, np.int8), n), np.asarray(scores, np.float64)


def ctx_of(data, logistic=False, is_async=False):
    from distributed_sgd_b200.native import NativeCtx
    c = NativeCtx(0, data.dim, LAM, logistic=logistic, is_async=is_async)
    c.load_csr(data.row_ptr, data.col, data.val, data.label)
    return c


@pytest.mark.parametrize("case", ["two_rows", "separable", "all_equal", "huge", "beyond_exp"])
def test_hand_built_scores(case):
    scores, labels = {
        "two_rows": ([-1.5, 2.0], [1, -1]),
        "separable": ([-3.0, -2.0, -1.0, 1.0, 2.0, 4.0], [1, 1, 1, -1, -1, -1]),       # A grows until the targets stop it
        "all_equal": ([0.75] * 8, [1, -1, 1, -1, -1, -1, 1, -1]),                       # det H rests on the ridge
        "huge": ([-700.0, -710.0, 705.0, 720.0, -1.0, 1.0], [1, 1, -1, -1, -1, 1]),     # exp(700) overflows the naive form
        "beyond_exp": ([-1e6, 1e6, -2e6, 3e6, 0.5, -0.5], [1, -1, 1, -1, 1, -1]),
    }[case]
    data, w = planted(scores, labels)
    ctx = ctx_of(data)
    try:
        n = len(scores)
        assert np.array_equal(ctx.margins(np.arange(n), w), w)
        a, b, obj, info = ctx.calibrate(0, n, w)
        ref, lit = calib.fit(w, labels), calib.fit_literal(w, labels)
        print(case, (a, b, obj, info.tolist()), ref)
        if case == "beyond_exp":
            # dF/dA sums terms of 1e6 and is tested against 1e-5: one ulp of a p (CUDA's exp against glibc's) decides whether
            # the last point already passes.  Where it does not, the next line search cannot lower F by less than an ulp of F
            # and ends the fit at that same point: converged or line-search-failed, with the same (A, B) either way.
            assert ref.status == lit.status == calib.CONVERGED and int(info[1]) in (calib.CONVERGED, calib.LINE_SEARCH_FAILED)
        else:
            assert int(info[1]) == ref.status == lit.status
        assert np.isfinite([a, b, obj]).all()
        assert abs(obj - ref.objective) <= 1e-9 * max(1.0, abs(ref.objective))
        if ref.status == calib.CONVERGED and case != "all_equal":
            assert abs(a - ref.a) <= 1e-6 * abs(ref.a) and abs(b - ref.b) <= 1e-6 * max(1.0, abs(ref.b))
        assert bits(ctx.calibrate_samples(np.arange(n)[::-1].copy(), w)) == bits((a, b, obj, info))
    finally:
        ctx.close()


# ---- probabilities -----------------------------------------------------------------------------------------------------

def test_calibrated_probabilities(rcv):
    svm, logi, data, w = rcv
    rng = np.random.default_rng(9)
    ids = rng.integers(0, N_ROWS, size=30_000).astype(np.int32)
    assert np.array_equal(logi.calibrated_probabilities(ids, 1.0, 0.0, w), logi.probabilities(ids, w))   # bit for bit
    a, b = svm.calibrate(0, N_TRAIN, w)[:2]
    p = svm.calibrated_probabilities(ids, a, b, w)
    np.testing.assert_allclose(p, calib.probs(svm.margins(ids, w), a, b), rtol=1e-12, atol=0)
    assert np.array_equal(p, logi.calibrated_probabilities(ids, a, b, w))
    assert ((p >= 0) & (p <= 1)).all()


def test_a_fitted_link_is_no_worse_than_the_identity_on_an_under_confident_logistic_model(rcv):
    """The whole chain on a SparseLogistic context: weights shrunk tenfold, as a strong L2 penalty shrinks them, make
    sigmoid(-x . w) under-confident; the link fitted on the train rows must not lose to the identity on the test rows."""
    _, logi, data, w = rcv
    ws = 0.1 * w
    a, b, _, info = logi.calibrate(0, N_TRAIN, ws)
    fitted = logi.eval_calibration(N_TRAIN, N_ROWS, a, b, 10, ws)
    ident = logi.eval_calibration(N_TRAIN, N_ROWS, 1.0, 0.0, 10, ws)
    n = N_ROWS - N_TRAIN
    print(f"A = {a:.6g}, B = {b:.6g}, status {int(info[1])}; test log loss fitted {fitted[0][1] / n:.6f} vs identity "
          f"{ident[0][1] / n:.6f}; Brier {fitted[0][0] / n:.6f} vs {ident[0][0] / n:.6f}")
    assert int(info[1]) in (calib.CONVERGED, calib.LINE_SEARCH_FAILED) and a > 1.0
    assert fitted[0][1] <= ident[0][1] and fitted[0][0] <= ident[0][0]


# ---- the quality pass --------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("n_bins", [1, 10, 64])
def test_quality_pass_against_the_checker(rcv, n_bins):
    svm, _, data, w = rcv
    b, e = N_TRAIN, N_ROWS
    ids = np.arange(b, e, dtype=np.int32)
    a, bb = svm.calibrate(0, N_TRAIN, w)[:2]
    sums, rows, pos, psum, words = svm.eval_calibration(b, e, a, bb, n_bins, w)
    ref = calib.quality(svm.margins(ids, w), labels_of(data, ids), a, bb, n_bins)
    assert words.tolist() == [e - b, 0] == [ref.rows, ref.left_out] and rows.sum() == e - b
    np.testing.assert_allclose(sums, [ref.brier_sum, ref.log_loss_sum], rtol=1e-12)
    # a row whose p * n_bins is within 4 ulp of an integer may sit in the next bin under another exp: at most that many move
    assert np.abs(rows - ref.bin_rows).sum() <= 2 * ref.edge_rows and np.abs(pos - ref.bin_pos).sum() <= 2 * ref.edge_rows
    if ref.edge_rows == 0:
        np.testing.assert_allclose(psum, ref.bin_psum, rtol=1e-12)
    rng = np.random.default_rng(n_bins)
    for other in (svm.eval_samples_calibration(ids[::-1].copy(), a, bb, n_bins, w),
                  svm.eval_samples_calibration(rng.permutation(ids).astype(np.int32), a, bb, n_bins, w),
                  svm.eval_sampled_calibration(b, e, 77, 0, e - b, a, bb, n_bins, w)):
        for x, y in zip(other, (sums, rows, pos, psum, words)):
            assert x.tobytes() == y.tobytes()                       # the same bits in any row order


def test_quality_on_planted_rows():
    """p away from every bin edge, and p = 1.0 exactly (sigmoid(1000)) in the last bin."""
    scores = [-1000.0, -2.0, -0.1, 0.1, 2.0, 1000.0, -1000.0]
    labels = [1, 1, -1, 1, -1, -1, -1]
    data, w = planted(scores, labels)
    ctx = ctx_of(data)
    try:
        sums, rows, pos, psum, words = ctx.eval_calibration(0, len(scores), 1.0, 0.0, 4, w)
        p = calib.probs(w, 1.0, 0.0)
        assert p[0] == 1.0 and p[5] == 0.0
        assert rows.tolist() == [2, 1, 1, 3] and pos.tolist() == [0, 1, 0, 2] and words.tolist() == [7, 0]
        ref = calib.quality(w, labels, 1.0, 0.0, 4)
        assert rows.tolist() == ref.bin_rows.tolist() and pos.tolist() == ref.bin_pos.tolist()
        np.testing.assert_allclose(psum, ref.bin_psum, rtol=1e-14)
        np.testing.assert_allclose(sums, [ref.brier_sum, ref.log_loss_sum], rtol=1e-14)
    finally:
        ctx.close()


def nan_rows_data(scores, labels, n_nan):
    """planted(scores, labels) followed by n_nan positive rows holding x = 1 in two further columns whose weights are +inf and
    -inf: their score is inf - inf = NaN."""
    n = len(scores)
    rows = [([i], [1.0]) for i in range(n)] + [([n, n + 1], [1.0, 1.0])] * n_nan
    data = csr(rows, np.asarray(list(labels) + [1] * n_nan, np.int8), n + 2)
    return data, np.asarray(list(scores) + [np.inf, -np.inf], np.float64)


def test_nan_scores_are_left_out_and_counted():
    from distributed_sgd_b200.native import DsgdEmpty
    scores, labels = [-2.0, -0.5, 0.25, 1.0, 3.0, -1.0], [1, 1, 1, -1, -1, -1]
    data, w = nan_rows_data(scores, labels, 3)
    ctx = ctx_of(data)
    try:
        assert np.isnan(ctx.margins(np.arange(6, 9), w)).all()
        fit = ctx.calibrate(0, 9, w)
        assert fit[3][2:4].tolist() == [6, 3]
        assert bits(fit)[:3] == bits(ctx.calibrate(0, 6, w))[:3]        # the same fit as without those rows
        ref = calib.fit(ctx.margins(np.arange(9), w), data.label)
        assert (ref.rows, ref.nan_rows, ref.iterations, ref.status) == (6, 3, int(fit[3][0]), int(fit[3][1]))
        assert abs(fit[0] - ref.a) <= 1e-8 and abs(fit[1] - ref.b) <= 1e-8
        q = ctx.eval_calibration(0, 9, fit[0], fit[1], 5, w)
        assert q[4].tolist() == [6, 3] and q[1].sum() == 6
        with pytest.raises(DsgdEmpty):
            ctx.calibrate(6, 9, w)                                      # every score NaN
        assert ctx.eval_calibration(6, 9, 1.0, 0.0, 10, w)[4].tolist() == [0, 3]
    finally:
        ctx.close()


# ---- resident weights --------------------------------------------------------------------------------------------------

def same_as_explicit(ctx, b, e):
    w = ctx.get_weights()
    ids = np.arange(b, e, dtype=np.int32)
    assert bits(ctx.calibrate(b, e)) == bits(ctx.calibrate(b, e, w))
    a, bb = ctx.calibrate(b, e)[:2]
    assert np.array_equal(ctx.calibrated_probabilities(ids, a, bb), ctx.calibrated_probabilities(ids, a, bb, w))
    for x, y in zip(ctx.eval_calibration(b, e, a, bb, 10), ctx.eval_calibration(b, e, a, bb, 10, w)):
        assert x.tobytes() == y.tobytes()


def test_null_weights_read_the_resident_state(rcv):
    svm, logi, data, w = rcv
    rng = np.random.default_rng(3)
    for ctx in (svm, logi):
        ctx.set_weights(w)
        same_as_explicit(ctx, 0, 5000)
        ctx.sync_steps(rng.integers(0, N_TRAIN, size=20 * 64).astype(np.int32), 64, 20, 0.1, want_losses=False)   # the persistent kernel
        same_as_explicit(ctx, 0, 5000)
        ctx.sync_steps(rng.integers(0, N_TRAIN, size=2 * 6000).astype(np.int32), 6000, 2, 0.1, want_losses=False)  # one launch per step
        same_as_explicit(ctx, 0, 5000)
    svm.set_weights(w)


# ---- errors ------------------------------------------------------------------------------------------------------------

def test_errors(rcv):
    from distributed_sgd_b200 import native
    from distributed_sgd_b200.native import DsgdEmpty, DsgdInvalid, DsgdRange, DsgdState, NativeCtx
    svm, _, data, w = rcv
    L = native.lib()
    ab, f, info = np.zeros(2), np.zeros(1), np.zeros(5, np.int64)
    s2, r64, p64, ps64, w2 = np.zeros(2), np.zeros(64, np.int64), np.zeros(64, np.int64), np.zeros(64), np.zeros(2, np.int64)
    ids = np.arange(4, dtype=np.int32)
    P = lambda x: x.ctypes.data                                      # noqa: E731
    assert L.dsgd_calibrate(svm._h, None, 0, 10, None, P(f), P(info)) == -1            # NULL outputs
    assert L.dsgd_calibrate(svm._h, None, 0, 10, P(ab), None, P(info)) == -1
    assert L.dsgd_calibrate_sampled(svm._h, None, 0, 10, 1, 0, 5, P(ab), P(f), None) == -1
    assert L.dsgd_calibrate_samples(svm._h, None, None, 4, P(ab), P(f), P(info)) == -1  # NULL ids
    assert L.dsgd_calibrated_probabilities(svm._h, None, P(ids), 4, 1.0, 0.0, None) == -1
    assert L.dsgd_eval_calibration(svm._h, None, 0, 10, 1.0, 0.0, 10, None, P(r64), P(p64), P(ps64), P(w2)) == -1
    assert L.dsgd_eval_samples_calibration(svm._h, None, P(ids), 4, 1.0, 0.0, 10, P(s2), P(r64), P(p64), None, P(w2)) == -1
    for a, b in ((np.nan, 0.0), (1.0, np.inf)):
        with pytest.raises(DsgdInvalid):
            svm.calibrated_probabilities(ids, a, b, w)
        with pytest.raises(DsgdInvalid):
            svm.eval_calibration(0, 10, a, b, 10, w)
    for n_bins in (0, -1, 65):
        with pytest.raises(DsgdInvalid):
            svm.eval_calibration(0, 10, 1.0, 0.0, n_bins, w)
    for call in (lambda: svm.calibrate(0, N_ROWS + 1, w), lambda: svm.calibrate(-1, 5, w),
                 lambda: svm.calibrate_samples([0, N_ROWS], w), lambda: svm.eval_calibration(5, N_ROWS + 1, 1.0, 0.0, 10, w),
                 lambda: svm.calibrated_probabilities([-1], 1.0, 0.0, w)):
        with pytest.raises(DsgdRange):
            call()
    for call in (lambda: svm.calibrate(7, 7, w), lambda: svm.calibrate_samples([], w),
                 lambda: svm.calibrate_sampled(0, 10, 1, 3, 3, w), lambda: svm.eval_calibration(7, 7, 1.0, 0.0, 10, w)):
        with pytest.raises(DsgdEmpty):
            call()
    one = int(np.flatnonzero(np.asarray(data.label) > 0)[0])
    with pytest.raises(DsgdEmpty):
        svm.calibrate_samples([one, one, one], w)                   # one class
    empty = NativeCtx(0, 16, LAM)
    try:
        with pytest.raises(DsgdState):
            empty.calibrate(0, 1)                                    # no rows loaded
        with pytest.raises(DsgdState):
            empty.eval_calibration(0, 1, 1.0, 0.0, 10)
        with pytest.raises(DsgdState):
            empty.calibrated_probabilities([0], 1.0, 0.0)
    finally:
        empty.close()
    with pytest.raises(DsgdState):
        svm.probabilities(ids, w)                                   # the uncalibrated call still refuses an SVM context


_LOOP = r"""
import sys
sys.path.insert(0, {root!r})
import numpy as np
from distributed_sgd_b200.native import DsgdState, NativeCtx
from distributed_sgd_b200.utils import synthetic_rcv1
data = synthetic_rcv1(n_rows=6000, seed=8)
ctx = NativeCtx(0, data.dim, 1e-4, is_async=True)
ctx.load_csr(data.row_ptr, data.col, data.val, data.label)
ctx.compute_dim_sparsity(4800)
ctx.start_async(np.zeros(data.dim), np.arange(4800, dtype=np.int32), 8, 0.1, concurrency=1, max_updates=0, seed=1)
try:
    running = ctx.async_running()
    refused = 0
    for call in (lambda: ctx.calibrate(0, 4800), lambda: ctx.calibrate_sampled(0, 4800, 3, 0, 100),
                 lambda: ctx.calibrate_samples(np.arange(100))):
        try:
            call()
        except DsgdState:
            refused += 1
    q = ctx.eval_calibration(4800, 6000, 1.0, 0.0, 10)               # the first quality pass of this process
    p = ctx.calibrated_probabilities(np.arange(100), 1.0, 0.0)
    try:
        ctx.eval_samples_calibration(np.zeros(6001, np.int32), 1.0, 0.0, 10)   # more ids than rows: a buffer would have to grow
        long_refused = False
    except DsgdState:
        long_refused = True
    print("OK", running, refused, int(q[1].sum()), len(p), long_refused)
finally:
    ctx.stop_async()
w = ctx.get_weights()
a = ctx.calibrate(0, 4800)
b = ctx.calibrate(0, 4800, w)
print("AFTER", a[:3] == b[:3], a[3].tolist() == b[3].tolist(), "status", int(a[3][1]))
ctx.close()
"""


def test_beside_a_running_hogwild_loop():
    """While the loop runs the fit is refused before anything is launched (a cooperative grid cannot be assumed resident
    beside a kernel that never ends) and the two barrier-free calls work; once it is stopped the fit works, and w == NULL
    reads the replica the loop left.  The loop is stopped in a `finally`; the subprocess has a timeout."""
    r = subprocess.run([sys.executable, "-s", "-c", _LOOP.format(root=ROOT)], cwd=ROOT, capture_output=True, text=True,
                       timeout=180)
    assert r.returncode == 0, r.stdout + r.stderr
    assert "OK True 3 1200 100 True" in r.stdout, r.stdout + r.stderr
    assert "AFTER True True" in r.stdout, r.stdout + r.stderr
