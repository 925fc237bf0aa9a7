"""SparseSquaredHinge and SparseModifiedHuber golden fixtures (tests/golden/margin/*.json, produced by the literal
restatement with tests/golden/make_golden_margin.py): the C checker reproduces them on the CPU, the CUDA path through the C
ABI on the GPU.  The fixtures' losses are left folds of the per-sample losses (the reference's reduce), not the device's
fixed-point sums: losses are compared at rtol 1e-12, weights within 1e-11 * max |w|, gradient entries within
1e-12 * (sum_i |s_i x_ij| + |c|)."""
import glob
import os

import numpy as np
import pytest

from oracle import margin as M
from oracle.oracle import Oracle
from test_golden import flat_draws, load

HERE = os.path.dirname(os.path.abspath(__file__))
FIXTURES = sorted(glob.glob(os.path.join(HERE, "golden", "margin", "*.json")))
IDS = [os.path.basename(p) for p in FIXTURES]


def _bound(f, w, probe, c):
    b = np.zeros(f["dim"])
    for r in probe:
        lo, hi = f["row_ptr"][r], f["row_ptr"][r + 1]
        cols, vals = f["col"][lo:hi], f["val"][lo:hi].astype(np.float64)
        z = float(f["label"][r]) * float(np.dot(vals, np.asarray(w)[cols]))
        b[cols] += np.abs(vals) * M.row(f["model"], z)[1]
    return b + abs(c)


def _check(f, w, losses, g, preds, loss, acc, c):
    np.testing.assert_allclose(losses, f["step_losses"], rtol=1e-12)
    ref = np.array(f["final_weights"])
    assert np.abs(w - ref).max() <= 1e-11 * np.abs(ref).max()
    g_ref = np.array(f["probe_gradient"])
    assert ((g == 0) == (g_ref == 0)).all()
    assert (np.abs(g - g_ref) <= 1e-12 * _bound(f, ref, f["probe"], c)).all()
    np.testing.assert_array_equal(preds, f["probe_predictions"])
    assert acc == f["test_accuracy"] and loss == pytest.approx(f["test_loss"], rel=1e-12)


def test_fixtures_exist():
    assert {load(p)["model"] for p in FIXTURES} == {"squared_hinge", "modified_huber"} and len(FIXTURES) >= 4


@pytest.mark.parametrize("path", FIXTURES, ids=IDS)
def test_c_oracle_reproduces_margin_golden(path):
    f = load(path)
    orc = Oracle(f["row_ptr"], f["col"], f["val"], f["label"], f["dim"], f["lambda"])
    d = orc.dim_sparsity(f["n_train"])
    np.testing.assert_array_equal(d, f["dim_sparsity_weight_space"])
    orc.set_dim_sparsity(d)
    steps = len(f["draws"])
    w, losses = M.sync_steps(orc, f["model"], np.zeros(f["dim"]), flat_draws(f), [f["B"]] * f["K"], [f["lr"]] * steps)
    ref = np.array(f["final_weights"])
    g, _, _ = M.gradient(orc, f["model"], ref, f["probe"])
    c = orc.lam * 2.0 * float(np.sum(np.where(np.abs(ref * d) > 1e-20, ref * d, 0.0)))
    loss, acc, _, _ = M.loss_acc(orc, f["model"], ref, begin=f["n_train"], n=len(f["label"]) - f["n_train"])
    _check(f, w, losses, g, orc.forward(ref, f["probe"]), loss, acc, c)


@pytest.mark.gpu
@pytest.mark.parametrize("path", FIXTURES, ids=IDS)
def test_gpu_reproduces_margin_golden(path):
    from distributed_sgd_b200.native import NativeCtx
    f = load(path)
    with NativeCtx(0, f["dim"], f["lambda"], model=f["model"]) as ctx:
        ctx.load_csr(f["row_ptr"], f["col"], f["val"], f["label"])
        d = ctx.compute_dim_sparsity(f["n_train"])
        np.testing.assert_array_equal(d, f["dim_sparsity_weight_space"])
        K, B = f["K"], f["B"]
        ctx.set_weights(np.zeros(f["dim"]))
        ctx.set_workers([B] * K, K)
        losses = ctx.sync_steps(flat_draws(f), K * B, len(f["draws"]), f["lr"])
        w = ctx.get_weights()
        ref = np.array(f["final_weights"])
        g = ctx.gradient(f["probe"], ref)
        c = f["lambda"] * 2.0 * float(np.sum(np.where(np.abs(ref * d) > 1e-20, ref * d, 0.0)))
        loss, acc = ctx.eval(f["n_train"], len(f["label"]), ref)
        _check(f, w, losses, g, ctx.forward(f["probe"], ref), loss, acc, c)
