"""Weighted calibration on the device (dsgd_calibrate_weighted*, dsgd_eval_*weighted_calibration) against the weighted
calibration checker (oracle/dsgd_oracle_wcalib.c) over the device's own margins, and the identities the calls are built
for: unweighted results at c = 1, repeated rows for integer weights, one bit pattern whatever the row order, the grid or
the model; the errors; and the existing calibration calls' launches and results with weights loaded."""
import struct

import numpy as np
import pytest

from oracle import calib as oc
from oracle import wcalib as ow
from test_gpu_weighted_curve import set_weights, weight_cases

pytestmark = pytest.mark.gpu

LAM = 1e-4
N_ROWS, N_TRAIN = 100_000, 80_000
SIZES = [1, 31, 2047, 100_000]


def fbits(*xs):
    return struct.pack(f"<{len(xs)}d", *xs)


def fit_bits(res):
    a, b, f, info, ws = res
    return fbits(a, b, f) + np.asarray(info).tobytes() + np.asarray(ws).tobytes()


def trained(ctx, n_train, steps=300, batch=64, lr=0.5, seed=0):
    rng = np.random.default_rng(seed)
    ctx.set_weights(np.zeros(ctx.dim))
    ctx.sync_steps(rng.integers(0, n_train, size=steps * batch).astype(np.int32), batch, steps, lr, want_losses=False)
    return ctx.get_weights()


@pytest.fixture(scope="module")
def rcv():
    """{model: context} over the same rows, the data and weights trained on the SVM context"""
    from distributed_sgd_b200.native import NativeCtx
    from distributed_sgd_b200.utils import synthetic_rcv1
    data = synthetic_rcv1(n_rows=N_ROWS, seed=21)
    ctxs = {}
    for model in ("svm", "logistic", "modified_huber"):
        c = NativeCtx(0, data.dim, LAM, model=model)
        c.load_csr(data.row_ptr, data.col, data.val, data.label)
        c.compute_dim_sparsity(N_TRAIN)
        ctxs[model] = c
    w = trained(ctxs["svm"], N_TRAIN)
    yield ctxs, data, w
    for c in ctxs.values():
        c.close()


def check_fit(res, ref):
    a, b, f, info, ws = res
    assert np.asarray(ws).tobytes() == fbits(ref.w_pos, ref.w_neg, ref.nan_weight)   # read() of exact sums: bit for bit
    assert [int(v) for v in info[[1, 2, 3]]] == [ref.status, ref.rows, ref.nan_rows]
    if ref.status == oc.NON_FINITE:
        return
    assert abs(a - ref.a) <= 1e-8 * max(1.0, abs(ref.a)) and abs(b - ref.b) <= 1e-8 * max(1.0, abs(ref.b))
    assert abs(f - ref.objective) <= 1e-10 * abs(ref.objective)


def check_quality(res, ref):
    sums, bw, bp, bs, words = res
    assert words.tolist() == [ref.rows, ref.left_out]
    assert sums[2] == ref.sums[2] and sums[3] == 0.0                  # the weight used: no exp in it, bit for bit
    # CUDA's exp and glibc's can differ in the last bit of p: the sums over p agree to rounding, and the bins exactly
    # unless a row sits within 4 ulp of a bin edge
    np.testing.assert_allclose(sums[:2], ref.sums[:2], rtol=1e-12)
    if ref.edge_rows == 0:
        assert bw.tobytes() == ref.bin_weight.tobytes() and bp.tobytes() == ref.bin_pos_weight.tobytes()
        np.testing.assert_allclose(bs, ref.bin_psum, rtol=1e-12)


@pytest.mark.parametrize("n", SIZES + SIZES[-2::-1])
def test_against_the_checker_growing_then_shrinking(rcv, n):
    from distributed_sgd_b200.native import DsgdEmpty
    ctxs, data, w = rcv
    ctx = ctxs["svm"]
    ids = np.arange(0, n, dtype=np.int32)
    f, y = ctx.margins(ids, w), np.asarray(data.label)[ids]
    try:
        for name, sw, cw in weight_cases(data.n_rows, n):
            c = set_weights(ctx, data, sw, cw)[ids]
            try:
                ref = ow.fit(f, y, c)
            except ValueError:
                with pytest.raises(DsgdEmpty):
                    ctx.calibrate_weighted(0, n, w)
                a, b = 1.3, -0.2
            else:
                res = ctx.calibrate_weighted(0, n, w)
                check_fit(res, ref)
                a, b = res[0], res[1]
            check_quality(ctx.eval_weighted_calibration(0, n, a, b, 10, w), ow.quality(f, y, c, a, b, 10))
    finally:
        set_weights(ctx, data, None, (1.0, 1.0))


def test_full_size_test_rows():
    """The full-size synthetic set's 140 000 test rows, class and sample weights; RCV1-shaped rows: the iteration counts
    agree as well."""
    from distributed_sgd_b200.native import NativeCtx
    from distributed_sgd_b200.utils import synthetic_rcv1
    data = synthetic_rcv1(n_rows=700_000, seed=0)
    n_train = int(data.n_rows * 0.8)
    ctx = NativeCtx(0, data.dim, LAM)
    try:
        ctx.load_csr(data.row_ptr, data.col, data.val, data.label)
        ctx.compute_dim_sparsity(n_train)
        w = trained(ctx, n_train)
        sw = np.random.default_rng(3).random(data.n_rows) * 2.0
        c_rows = set_weights(ctx, data, sw, (2.0, 0.5))
        ids = np.arange(n_train, data.n_rows, dtype=np.int32)
        f, y, c = ctx.margins(ids, w), np.asarray(data.label)[ids], c_rows[ids]
        res, ref = ctx.calibrate_weighted(n_train, data.n_rows, w), ow.fit(f, y, c)
        check_fit(res, ref)
        assert (int(res[3][0]), int(res[3][4])) == (ref.iterations, ref.evaluations)
        check_quality(ctx.eval_weighted_calibration(n_train, data.n_rows, res[0], res[1], 10, w),
                      ow.quality(f, y, c, res[0], res[1], 10))
    finally:
        ctx.close()


def test_one_bit_pattern_per_weighted_row_multiset(rcv):
    """A range, its ids reversed and shuffled, the drawn sample covering it, every grid limit and every model."""
    ctxs, data, w = rcv
    b, e = N_TRAIN, N_ROWS
    ids = np.arange(b, e, dtype=np.int32)
    rng = np.random.default_rng(4)
    sw = rng.random(data.n_rows) * 3.0
    try:
        for ctx in ctxs.values():
            set_weights(ctx, data, sw, (2.0, 0.5))
        ctx = ctxs["svm"]
        fit = fit_bits(ctx.calibrate_weighted(b, e, w))
        a, bb = ctx.calibrate_weighted(b, e, w)[:2]
        q = [x.tobytes() for x in ctx.eval_weighted_calibration(b, e, a, bb, 10, w)]
        for c in ctxs.values():
            for fn in (lambda: c.calibrate_weighted_samples(ids[::-1].copy(), w),
                       lambda: c.calibrate_weighted_samples(rng.permutation(ids).astype(np.int32), w),
                       lambda: c.calibrate_weighted_sampled(b, e, 77, 0, e - b, w)):
                assert fit_bits(fn()) == fit
            for res in (c.eval_samples_weighted_calibration(ids[::-1].copy(), a, bb, 10, w),
                        c.eval_sampled_weighted_calibration(b, e, 77, 0, e - b, a, bb, 10, w)):
                assert [x.tobytes() for x in res] == q
        for limit in (1, 2, 0):
            ctx.set_grid_limit(limit)
            assert fit_bits(ctx.calibrate_weighted(b, e, w)) == fit
            assert [x.tobytes() for x in ctx.eval_weighted_calibration(b, e, a, bb, 10, w)] == q
    finally:
        ctxs["svm"].set_grid_limit(0)
        for ctx in ctxs.values():
            set_weights(ctx, data, None, (1.0, 1.0))


@pytest.mark.parametrize("form", ["class 1,1", "sample ones"])
def test_unit_weights_equal_the_unweighted_calls(rcv, form):
    ctxs, data, w = rcv
    ctx = ctxs["svm"]
    sw = np.ones(data.n_rows) if form == "sample ones" else None
    try:
        set_weights(ctx, data, sw, (1.0, 1.0))
        for b, e in ((0, 2048), (0, N_TRAIN), (N_TRAIN, N_ROWS)):
            a, bb, f, info, ws = ctx.calibrate_weighted(b, e, w)
            ua, ub, uf, uinfo = ctx.calibrate(b, e, w)
            assert fbits(a, bb, f) == fbits(ua, ub, uf) and info.tobytes() == uinfo.tobytes()
            assert ws[0] + ws[1] == info[2] and ws[2] == info[3]
            sums, bw, bp, bs, words = ctx.eval_weighted_calibration(b, e, a, bb, 10, w)
            us, ur, up, ups, uw = ctx.eval_calibration(b, e, a, bb, 10, w)
            assert sums[:2].tobytes() == us.tobytes() and bs.tobytes() == ups.tobytes()
            assert np.array_equal(bw, ur) and np.array_equal(bp, up) and words.tobytes() == uw.tobytes()
            assert sums[2] == words[0]
    finally:
        set_weights(ctx, data, None, (1.0, 1.0))


def test_integer_weights_equal_the_repeated_rows(rcv):
    ctxs, data, w = rcv
    ctx = ctxs["svm"]
    b, e = N_TRAIN, N_ROWS
    sw = np.random.default_rng(5).integers(0, 4, data.n_rows).astype(np.float64)
    rep = np.repeat(np.arange(b, e, dtype=np.int32), sw[b:e].astype(int))
    try:
        unrep = ctx.calibrate_samples(rep, w)
        set_weights(ctx, data, sw, (1.0, 1.0))
        a, bb, f, info, ws = ctx.calibrate_weighted(b, e, w)
        assert ws[0] + ws[1] == unrep[3][2]
        assert abs(a - unrep[0]) <= 1e-8 * max(1.0, abs(unrep[0])) and abs(bb - unrep[1]) <= 1e-8 * max(1.0, abs(unrep[1]))
        assert abs(f - unrep[2]) <= 1e-10 * abs(unrep[2])
        sums, bw, bp, bs, words = ctx.eval_weighted_calibration(b, e, a, bb, 10, w)
        set_weights(ctx, data, None, (1.0, 1.0))
        us, ur, up, ups, uw = ctx.eval_samples_calibration(rep, a, bb, 10, w)
        assert np.array_equal(bw, ur) and np.array_equal(bp, up) and sums[:2].tobytes() == us.tobytes()
    finally:
        set_weights(ctx, data, None, (1.0, 1.0))


def test_errors(rcv):
    from distributed_sgd_b200.native import ERR_EMPTY, ERR_INVALID, ERR_STATE, DsgdError, NativeCtx
    ctxs, data, w = rcv
    ctx = ctxs["svm"]
    pos = np.asarray(data.label) > 0
    try:
        set_weights(ctx, data, np.where(pos, 0.0, 1.0), (1.0, 1.0))     # no positive weight
        for call in (lambda: ctx.calibrate_weighted(0, N_TRAIN, w), lambda: ctx.calibrate_weighted_samples(np.arange(50), w)):
            with pytest.raises(DsgdError) as ex:
                call()
            assert ex.value.code == ERR_EMPTY
        set_weights(ctx, data, None, (1.0, 1.0))
        lib, h = ctx._l, ctx._h
        out = np.zeros(8)
        assert lib.dsgd_calibrate_weighted(h, None, 0, 100, out.ctypes.data, out[2:].ctypes.data, None,
                                           out[5:].ctypes.data) == ERR_INVALID
        assert lib.dsgd_eval_weighted_calibration(h, None, 0, 100, 1.0, 0.0, 10, out.ctypes.data, None, out.ctypes.data,
                                                  out.ctypes.data, out.ctypes.data) == ERR_INVALID
    finally:
        set_weights(ctx, data, None, (1.0, 1.0))
    actx = NativeCtx(0, data.dim, LAM, is_async=True)
    try:
        actx.load_csr(data.row_ptr[:3001], data.col[:data.row_ptr[3000]], data.val[:data.row_ptr[3000]], data.label[:3000])
        before = actx.launch_count()
        for call in (lambda: actx.calibrate_weighted(0, 3000), lambda: actx.calibrate_weighted_samples([1, 2, 3]),
                     lambda: actx.calibrate_weighted_sampled(0, 3000, 5, 0, 100),
                     lambda: actx.eval_weighted_calibration(0, 3000, 1.0, 0.0),
                     lambda: actx.eval_samples_weighted_calibration([1, 2, 3], 1.0, 0.0),
                     lambda: actx.eval_sampled_weighted_calibration(0, 3000, 5, 0, 100, 1.0, 0.0)):
            with pytest.raises(DsgdError) as ex:
                call()
            assert ex.value.code == ERR_STATE and "async" in str(ex.value)
        assert actx.launch_count() == before
    finally:
        actx.close()


def test_zero_weight_rows_change_nothing(rcv):
    """Rows of zero weight (and of weight 2^-165, whose R is 0) add exactly nothing: the fit and the quality equal those of
    the list without them."""
    ctxs, data, w = rcv
    ctx = ctxs["svm"]
    b, e = N_TRAIN, N_ROWS
    rng = np.random.default_rng(6)
    sw = rng.random(data.n_rows) + 0.5
    drop = rng.random(data.n_rows) < 0.3
    sw[drop] = np.where(rng.random(int(drop.sum())) < 0.5, 0.0, 2.0 ** -165)
    keep = np.flatnonzero(~drop[b:e]).astype(np.int32) + b
    try:
        set_weights(ctx, data, sw, (1.0, 1.0))
        full, sub = ctx.calibrate_weighted(b, e, w), ctx.calibrate_weighted_samples(keep, w)
        assert fbits(*full[:3]) == fbits(*sub[:3]) and full[4].tobytes() == sub[4].tobytes()
        a, bb = full[:2]
        q_full = ctx.eval_weighted_calibration(b, e, a, bb, 10, w)
        q_sub = ctx.eval_samples_weighted_calibration(keep, a, bb, 10, w)
        for x, y in zip(q_full[:4], q_sub[:4]):
            assert x.tobytes() == y.tobytes()
    finally:
        set_weights(ctx, data, None, (1.0, 1.0))


def test_existing_calls_launch_and_return_what_they_did(rcv):
    """With class and sample weights loaded the unweighted calls launch what they launched and return the same bits; the
    weighted fit launches what the unweighted one does, and the weighted quality pass one kernel fewer (no finish kernel)."""
    ctxs, data, w = rcv
    ctx = ctxs["svm"]
    b, e = N_TRAIN, N_ROWS
    calls = {"fit": lambda: ctx.calibrate(b, e, w), "quality": lambda: ctx.eval_calibration(b, e, 1.3, -0.2, 10, w)}

    def run(call):
        before = ctx.launch_count()
        res = call()
        return ctx.launch_count() - before, [np.asarray(x).tobytes() for x in res]

    plain = {name: run(call) for name, call in calls.items()}
    try:
        set_weights(ctx, data, np.random.default_rng(7).random(data.n_rows), (2.0, 0.5))
        k_fit = run(lambda: ctx.calibrate_weighted(b, e, w))[0]
        k_quality = run(lambda: ctx.eval_weighted_calibration(b, e, 1.3, -0.2, 10, w))[0]
        for name, call in calls.items():
            assert run(call) == plain[name]
        assert k_fit == plain["fit"][0] and k_quality == plain["quality"][0] - 1
    finally:
        set_weights(ctx, data, None, (1.0, 1.0))


# ---- the weighted isotonic fit and its quality pass ---------------------------------------------------------------------

def check_iso(res, ref):
    x, y, bw, bp, info, ws = res
    assert x.tobytes() == ref.x.tobytes() and y.tobytes() == ref.y.tobytes()
    assert bw.tobytes() == ref.block_weight.tobytes() and bp.tobytes() == ref.block_pos_weight.tobytes()
    assert [int(v) for v in info] == list(ref.info) and ws.tobytes() == fbits(*ref.wsums)


@pytest.mark.parametrize("n", SIZES + SIZES[-2::-1])
def test_isotonic_against_the_checker_growing_then_shrinking(rcv, n):
    from distributed_sgd_b200.native import DsgdEmpty
    ctxs, data, w = rcv
    ctx = ctxs["svm"]
    ids = np.arange(0, n, dtype=np.int32)
    f, y = ctx.margins(ids, w), np.asarray(data.label)[ids]
    try:
        for name, sw, cw in weight_cases(data.n_rows, n):
            c = set_weights(ctx, data, sw, cw)[ids]
            try:
                ref = ow.fit_isotonic(f, y, c)
            except ValueError:
                with pytest.raises(DsgdEmpty):
                    ctx.calibrate_isotonic_weighted(0, n, w)
                continue
            res = ctx.calibrate_isotonic_weighted(0, n, w)
            check_iso(res, ref)
            q = ctx.eval_weighted_isotonic_calibration(0, n, res[0], res[1], 10, w)
            s, bw, bp, bs, words = ow.quality_isotonic(f, y, c, res[0], res[1], 10)
            assert q[4].tolist() == list(words) and q[0][2] == s[2] and q[0][3] == s[3]
            np.testing.assert_allclose(q[0][:2], s[:2], rtol=1e-12)
    finally:
        set_weights(ctx, data, None, (1.0, 1.0))


def test_isotonic_one_bit_pattern_tiles_grids_models_orders(rcv, monkeypatch):
    ctxs, data, w = rcv
    b, e = N_TRAIN, N_ROWS
    ids = np.arange(b, e, dtype=np.int32)
    rng = np.random.default_rng(8)
    sw = np.where(rng.random(data.n_rows) < 0.3, 0.0, rng.random(data.n_rows) * 3.0)
    def flat(res):
        return b"".join(np.asarray(v).tobytes() for v in res)
    try:
        for c in ctxs.values():
            set_weights(c, data, sw, (2.0, 0.5))
        ctx = ctxs["svm"]
        ref = flat(ctx.calibrate_isotonic_weighted(b, e, w))
        for c in ctxs.values():
            assert flat(c.calibrate_isotonic_weighted_samples(ids[::-1].copy(), w)) == ref
            assert flat(c.calibrate_isotonic_weighted_samples(rng.permutation(ids).astype(np.int32), w)) == ref
            assert flat(c.calibrate_isotonic_weighted_sampled(b, e, 77, 0, e - b, w)) == ref
        for tile in ("1", "7", "2048"):
            monkeypatch.setenv("DSGD_ISOTONIC_TILE", tile)
            assert flat(ctx.calibrate_isotonic_weighted(b, e, w)) == ref
        monkeypatch.delenv("DSGD_ISOTONIC_TILE")
        for limit in (1, 2, 0):
            ctx.set_grid_limit(limit)
            assert flat(ctx.calibrate_isotonic_weighted(b, e, w)) == ref
    finally:
        ctxs["svm"].set_grid_limit(0)
        for c in ctxs.values():
            set_weights(c, data, None, (1.0, 1.0))


@pytest.mark.parametrize("form", ["class 1,1", "sample ones"])
def test_isotonic_unit_weights_equal_the_unweighted_calls(rcv, form):
    ctxs, data, w = rcv
    ctx = ctxs["svm"]
    try:
        set_weights(ctx, data, np.ones(data.n_rows) if form == "sample ones" else None, (1.0, 1.0))
        for b, e in ((0, 2048), (N_TRAIN, N_ROWS)):
            x, y, bw, bp, info, ws = ctx.calibrate_isotonic_weighted(b, e, w)
            ux, uy, ur, up, uinfo = ctx.calibrate_isotonic(b, e, w)
            assert x.tobytes() == ux.tobytes() and y.tobytes() == uy.tobytes() and info.tobytes() == uinfo.tobytes()
            assert np.array_equal(bw, ur) and np.array_equal(bp, up)
            q = ctx.eval_weighted_isotonic_calibration(b, e, x, y, 10, w)
            u = ctx.eval_isotonic_calibration(b, e, x, y, 10, w)
            assert q[0][:2].tobytes() == u[0].tobytes() and q[3].tobytes() == u[3].tobytes()
            assert np.array_equal(q[1], u[1]) and np.array_equal(q[2], u[2]) and q[4].tobytes() == u[4].tobytes()
    finally:
        set_weights(ctx, data, None, (1.0, 1.0))


def test_isotonic_integer_weights_equal_the_repeated_rows(rcv):
    ctxs, data, w = rcv
    ctx = ctxs["svm"]
    b, e = N_TRAIN, N_ROWS
    sw = np.random.default_rng(9).integers(0, 4, data.n_rows).astype(np.float64)
    rep = np.repeat(np.arange(b, e, dtype=np.int32), sw[b:e].astype(int))
    try:
        ux, uy, ur, up, _ = ctx.calibrate_isotonic_samples(rep, w)
        set_weights(ctx, data, sw, (1.0, 1.0))
        x, y, bw, bp, _, _ = ctx.calibrate_isotonic_weighted(b, e, w)
        assert x.tobytes() == ux.tobytes() and y.tobytes() == uy.tobytes() and np.array_equal(bw, ur)
    finally:
        set_weights(ctx, data, None, (1.0, 1.0))


def test_isotonic_errors_and_zero_weight_extremes(rcv):
    from distributed_sgd_b200.native import ERR_EMPTY, ERR_RANGE, DsgdError
    ctxs, data, w = rcv
    ctx = ctxs["svm"]
    b, e = N_TRAIN, N_ROWS
    ids = np.arange(b, e, dtype=np.int32)
    f = ctx.margins(ids, w)
    sw = np.ones(data.n_rows)
    sw[b + int(np.argmax(-f))] = 0.0
    sw[b + int(np.argmin(-f))] = 0.0
    try:
        set_weights(ctx, data, sw, (1.0, 1.0))
        x = ctx.calibrate_isotonic_weighted(b, e, w)[0]
        assert -f.max() not in x and -f.min() not in x
        set_weights(ctx, data, np.zeros(data.n_rows), (1.0, 1.0))
        with pytest.raises(DsgdError) as ex:
            ctx.calibrate_isotonic_weighted(b, e, w)
        assert ex.value.code == ERR_EMPTY
        set_weights(ctx, data, np.full(data.n_rows, 2.0 ** 51), (1.0, 1.0))    # 20 000 * 2^51 > 2^64: accepted
        ctx.calibrate_isotonic_weighted(b, e, w)
        set_weights(ctx, data, np.full(data.n_rows, 2.0 ** 51), (2.0 ** 40, 2.0 ** 40))   # c = 2^91: total above 2^96
        with pytest.raises(DsgdError) as ex:
            ctx.calibrate_isotonic_weighted(b, e, w)
        assert ex.value.code == ERR_RANGE
    finally:
        set_weights(ctx, data, None, (1.0, 1.0))
