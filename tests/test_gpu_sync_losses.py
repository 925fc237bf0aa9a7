"""Per-step losses of the one-GPU persistent sync step (k_sync_persistent), against the fp64 oracle.

Every CTA stores its hinge count of a step in its own slot ([n_steps][CTAs]), CTA 0 stores the step's norms, and the kernel's
epilogue forms loss_t = lambda ||W_t||^2 (+ lambda1 ||W_t||_1) + hinge_t / batch after the last step.  Checked here:
* the losses to the suite's tolerance (rtol 1e-12), and the hinge part of each, (loss - lambda ||W_t||^2) * batch, an integer
  equal to the oracle's count -- at 1, 7 and S CTAs (S = SM count), with and without the L1 penalty;
* two calls without set_weights in between, the first one with and without losses;
* runs of more steps than the slots of earlier, smaller calls hold (the buffer grows), and more than 4096 steps at S CTAs.
"""
import numpy as np
import pytest

from helpers import make_pair

pytestmark = pytest.mark.gpu

LAM, LR, LAM1 = 1e-5, 0.5, 1e-4


@pytest.fixture(scope="module")
def pair():
    from distributed_sgd_b200.utils import synthetic_rcv1
    data = synthetic_rcv1(n_rows=6000, seed=23)
    ctx, orc = make_pair(data, LAM)
    S = int(ctx.info()["sm_count"])
    yield data, ctx, orc, S
    ctx.close()


def _batch(G):
    return min(255, 32 * G - 1)       # odd: hinge / batch is not a short binary fraction


def _ids(seed, n_rows, steps, batch):
    rng = np.random.default_rng(seed)
    return np.stack([rng.choice(n_rows, size=batch, replace=False) for _ in range(steps)]).astype(np.int32)


def _oracle(data, orc, w0, ids, lam1):
    """Step by step: (weights after the last step, losses, hinge counts of every step)."""
    from oracle import l1 as L1
    w, losses, hinge = w0, [], []
    y = data.label.astype(np.float64)
    for row in ids:
        hinge.append(int(np.sum(1.0 - y[row] * orc.forward(w, row))))
        if lam1 > 0.0:
            w, l = L1.sync_steps(orc, w, row, [len(row)], np.array([LR]), lam1)
        else:
            w, l = orc.sync_steps(w, row, [len(row)], LR, n_steps=1)
        losses.append(l[0])
    return w, np.array(losses), np.array(hinge)


def _check(losses, w, ref, B, what):
    w_ref, l_ref, h_ref = ref
    np.testing.assert_allclose(losses, l_ref, rtol=1e-12, atol=0, err_msg=what)
    np.testing.assert_allclose(w, w_ref, rtol=1e-11, atol=1e-15, err_msg=what)
    # the hinge part: the loss minus the oracle's penalty terms, times the batch, is the oracle's integer count
    h = (losses - (l_ref - h_ref / B)) * B
    assert np.all(np.abs(h - np.rint(h)) < 1e-6), f"{what}: hinge parts not integers"
    np.testing.assert_array_equal(np.rint(h).astype(np.int64), h_ref, err_msg=f"{what}: hinge counts")


@pytest.mark.parametrize("l1", [False, True], ids=["svm", "l1"])
@pytest.mark.parametrize("grid", ["1", "7", "S"])
def test_two_calls(pair, grid, l1):
    data, ctx, orc, S = pair
    G = {"1": 1, "7": 7, "S": S}[grid]
    B = _batch(G)
    n1, n2 = 13, 9
    ids = _ids(G * 10 + l1, data.n_rows, n1 + n2, B)
    w0 = np.zeros(data.dim)
    ref = _oracle(data, orc, w0, ids, LAM1 if l1 else 0.0)
    ctx.set_grid_limit(G)
    ctx.set_l1(LAM1 if l1 else 0.0)
    try:
        ctx.set_weights(w0)
        l_a = ctx.sync_steps(ids[:n1].reshape(-1), B, n1, LR)
        l_b = ctx.sync_steps(ids[n1:].reshape(-1), B, n2, LR)         # no set_weights: carries on from the first call
        _check(np.concatenate([l_a, l_b]), ctx.get_weights(), ref, B, f"G={G}")
        # the same steps with the first call's losses off: the second call's losses are those of the oracle's steps n1..
        ctx.set_weights(w0)
        assert ctx.sync_steps(ids[:n1].reshape(-1), B, n1, LR, want_losses=False) is None
        l_c = ctx.sync_steps(ids[n1:].reshape(-1), B, n2, LR)
        _check(l_c, ctx.get_weights(), (ref[0], ref[1][n1:], ref[2][n1:]), B, f"G={G}, first call without losses")
    finally:
        ctx.set_grid_limit(0)
        ctx.set_l1(0.0)


def test_slots_beyond_earlier_calls(pair):
    """A short call, then at S CTAs a call of more steps than any earlier one, then one of more than 4096 steps: every step's
    slots are stored by that call, none are left from an earlier one."""
    data, ctx, orc, S = pair
    B = _batch(S)
    w0 = np.zeros(data.dim)
    ctx.set_weights(w0)
    short = _ids(1, data.n_rows, 3, B)
    ctx.sync_steps(short.reshape(-1), B, 3, LR)
    for steps in (4096 // S + 7, 4100):
        ids = _ids(steps, data.n_rows, steps, B)
        ref = _oracle(data, orc, w0, ids, 0.0)
        ctx.set_weights(w0)
        losses = ctx.sync_steps(ids.reshape(-1), B, steps, LR)
        _check(losses, ctx.get_weights(), ref, B, f"{steps} steps")
