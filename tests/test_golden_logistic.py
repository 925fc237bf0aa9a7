"""SparseLogistic golden fixtures (tests/golden/logistic/*.json, produced by the literal restatement with
tests/golden/make_golden.py): the C oracle reproduces them on the CPU, the CUDA path on the GPU."""
import glob
import os

import numpy as np
import pytest

from oracle.logistic import LogisticOracle
from test_golden import flat_draws, load

HERE = os.path.dirname(os.path.abspath(__file__))
FIXTURES = sorted(glob.glob(os.path.join(HERE, "golden", "logistic", "*.json")))
IDS = [os.path.basename(p) for p in FIXTURES]


def _bound(f, w, probe, c):
    """sum_i |sigma_i x_ij| + |c| per column"""
    b = np.zeros(f["dim"])
    for r in probe:
        lo, hi = f["row_ptr"][r], f["row_ptr"][r + 1]
        cols, vals = f["col"][lo:hi], f["val"][lo:hi].astype(np.float64)
        z = float(f["label"][r]) * float(np.dot(vals, np.asarray(w)[cols]))
        b[cols] += np.abs(vals) * (1.0 / (1.0 + np.exp(-z)))
    return b + abs(c)


def test_fixtures_exist():
    assert len(FIXTURES) >= 2


@pytest.mark.parametrize("path", FIXTURES, ids=IDS)
def test_c_oracle_reproduces_logistic_golden(path):
    f = load(path)
    assert f["model"] == "logistic"
    orc = LogisticOracle(f["row_ptr"], f["col"], f["val"], f["label"], f["dim"], f["lambda"])
    d = orc.dim_sparsity(f["n_train"])
    np.testing.assert_allclose(d, f["dim_sparsity_weight_space"], rtol=0, atol=0)
    orc.set_dim_sparsity(d)
    w, losses = orc.sync_steps(np.zeros(f["dim"]), flat_draws(f), [f["B"]] * f["K"], f["lr"], n_steps=len(f["draws"]))
    np.testing.assert_allclose(losses, f["step_losses"], rtol=1e-12)
    ref = np.array(f["final_weights"])
    assert np.abs(w - ref).max() <= 1e-11 * np.abs(ref).max()
    g, c = orc.gradient(ref, f["probe"])
    g_ref = np.array(f["probe_gradient"])
    assert ((g == 0) == (g_ref == 0)).all()
    assert (np.abs(g - g_ref) <= 1e-12 * _bound(f, ref, f["probe"], c)).all()
    np.testing.assert_array_equal(orc.forward(ref, f["probe"]), f["probe_predictions"])
    n = len(f["label"])
    loss, acc = orc.loss_acc(ref, begin=f["n_train"], n=n - f["n_train"])
    assert acc == f["test_accuracy"] and loss == pytest.approx(f["test_loss"], rel=1e-12)


@pytest.mark.gpu
@pytest.mark.parametrize("path", FIXTURES, ids=IDS)
def test_gpu_reproduces_logistic_golden(path):
    from distributed_sgd_b200.native import NativeCtx
    f = load(path)
    orc = LogisticOracle(f["row_ptr"], f["col"], f["val"], f["label"], f["dim"], f["lambda"])
    with NativeCtx(0, f["dim"], f["lambda"], logistic=True) as ctx:
        ctx.load_csr(f["row_ptr"], f["col"], f["val"], f["label"])
        d = ctx.compute_dim_sparsity(f["n_train"])
        np.testing.assert_array_equal(d, f["dim_sparsity_weight_space"])
        K, B = f["K"], f["B"]
        ctx.set_weights(np.zeros(f["dim"]))
        ctx.set_workers([B] * K, K)
        losses = ctx.sync_steps(flat_draws(f), K * B, len(f["draws"]), f["lr"])
        np.testing.assert_allclose(losses, f["step_losses"], rtol=1e-12)
        ref = np.array(f["final_weights"])
        w = ctx.get_weights()
        assert np.abs(w - ref).max() <= 1e-11 * np.abs(ref).max()
        g = ctx.gradient(f["probe"], ref)
        orc.set_dim_sparsity(d)
        _, c = orc.gradient(ref, f["probe"])
        g_ref = np.array(f["probe_gradient"])
        assert ((g == 0) == (g_ref == 0)).all()
        assert (np.abs(g - g_ref) <= 1e-12 * _bound(f, ref, f["probe"], c)).all()
        np.testing.assert_array_equal(ctx.forward(f["probe"], ref), f["probe_predictions"])
        n = len(f["label"])
        loss, acc = ctx.eval(f["n_train"], n, ref)
        assert acc == f["test_accuracy"] and loss == pytest.approx(f["test_loss"], rel=1e-12)
