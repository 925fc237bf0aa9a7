"""SparseLogistic in the oracle: the literal map-based restatement (oracle/scala_semantics_logistic.py) against the C
restatement (model 1 of oracle/dsgd_oracle_margin.c, as LogisticOracle) on random problems, the known answers, margins far out in both directions, and the 1e-20 product filter where sigma(z) * x crosses it."""
import math

import numpy as np
import pytest

from oracle import scala_semantics as S
from oracle import scala_semantics_logistic as L
from oracle.logistic import LogisticOracle
from conftest import random_csr
from test_oracle_c_vs_literal import literal_to_w, to_literal, w_to_literal


def _problem(seed, n=50, dim=30, lam=0.05, n_train=40):
    rng = np.random.default_rng(seed)
    rp, col, val, lab = random_csr(rng, n, dim, max_nnz=8)
    orc = LogisticOracle(rp, col, val, lab, dim, lam)
    data = to_literal(rp, col, val, lab, dim)
    d_lit = S.dim_sparsity(data[:n_train])
    orc.set_dim_sparsity(orc.dim_sparsity(n_train))
    return rng, orc, data, L.SparseLogistic(lam, d_lit)


def _close_per_entry(g, g_ref, bound):
    assert ((g == 0) == (g_ref == 0)).all()
    assert (np.abs(g - g_ref) <= 1e-12 * bound).all()


@pytest.mark.parametrize("seed", [0, 1, 2])
def test_gradient_and_loss_match_the_literal_restatement(seed):
    rng, orc, data, model = _problem(seed)
    dim, n = orc.dim, orc.n_rows
    for trial in range(5):
        w = np.where(rng.random(dim) < 0.6, rng.standard_normal(dim), 0.0) if trial else np.zeros(dim)
        wl = w_to_literal(w, dim)
        idx = rng.choice(n, size=int(rng.integers(1, 20)), replace=False).astype(np.int32)
        g_ref = literal_to_w(S.slave_gradient(model, data, wl, idx.tolist()), dim)
        g, c = orc.gradient(w, idx)
        bound = np.zeros(dim)
        for i in idx:
            x, y = data[i]
            s = L.sigmoid(y * x.dot(wl))
            for k, v in x.map.items():
                bound[k - 1] += abs(v) * s
        _close_per_entry(g, g_ref, bound + abs(c))
        loss, acc = orc.loss_acc(w, idx=idx)
        batch = [data[i] for i in idx]
        assert math.isclose(loss, S.local_loss(model, wl, batch), rel_tol=1e-12)
        assert acc == S.local_accuracy(model, wl, batch)


@pytest.mark.parametrize("K", [1, 2, 3])
def test_sync_steps_match_the_literal_restatement(K):
    rng, orc, data, model = _problem(10 + K)
    dim = orc.dim
    counts = [int(x) for x in rng.integers(1, 8, size=K)]
    w = np.zeros(dim)
    wl = w_to_literal(w, dim)
    steps = 4
    idx = np.concatenate([rng.choice(40, size=sum(counts), replace=False) for _ in range(steps)]).astype(np.int32)
    w_c, losses = orc.sync_steps(w, idx, counts, lr=0.5, n_steps=steps)
    off = 0
    for s in range(steps):
        batches, o = [], off
        for k in counts:
            batches.append(idx[o:o + k].tolist())
            o += k
        all_rows = [data[i] for b in batches for i in b]
        assert math.isclose(losses[s], S.local_loss(model, wl, all_rows), rel_tol=1e-12)
        wl = S.master_sync_step(model, data, wl, batches, 0.5)
        off = o
    w_lit = literal_to_w(wl, dim)
    assert np.abs(w_c - w_lit).max() <= 1e-11 * np.abs(w_lit).max()
    assert ((w_c == 0) == (w_lit == 0)).all()


def test_known_answers_at_zero_weights():
    rng, orc, data, model = _problem(5)
    w = np.zeros(orc.dim)
    idx = np.arange(20, dtype=np.int32)
    g, c = orc.gradient(w, idx)
    assert c == 0.0
    half = np.zeros(orc.dim)
    for i in idx:
        x, y = data[i]
        for k, v in x.map.items():
            half[k - 1] += 0.5 * y * v
    np.testing.assert_allclose(g, half, rtol=1e-15, atol=0)
    loss, acc = orc.loss_acc(w, idx=idx)
    assert math.isclose(loss, math.log(2.0), rel_tol=1e-15) and acc == 0.0
    assert (orc.sample_losses(w, idx) == math.log1p(1.0)).all()


@pytest.mark.parametrize("t", [0.0, 1e-300, 1e-8, 0.5, 1.0, 3.7, 20.0, 36.0, 40.0, 100.0, 700.0])
def test_symmetries(t):
    sp, sg = L.softplus, L.sigmoid
    assert abs((sp(t) - sp(-t)) - t) <= 4 * math.ulp(max(sp(t), 1.0))
    assert abs(sg(t) + sg(-t) - 1.0) <= 2 * math.ulp(1.0)


@pytest.mark.parametrize("z", [700.0, -700.0, 800.0, -800.0, 1e4, -1e4])
def test_no_overflow_far_out(z):
    # two one-entry rows of opposite labels, both at margin z
    rp = np.array([0, 1, 2], dtype=np.int64)
    orc = LogisticOracle(rp, np.array([0, 1], np.int32), np.array([1.0, 1.0], np.float32), np.array([1, -1], np.int8), 2,
                         1e-5)
    w = np.array([z, -z])
    g, _ = orc.gradient(w, [0, 1])
    loss, _ = orc.loss_acc(w, idx=[0, 1])
    assert np.isfinite(g).all() and math.isfinite(loss)
    expect = np.array([1.0, -1.0]) if z > 0 else np.zeros(2)
    np.testing.assert_allclose(g, expect, rtol=0, atol=1e-300 if z < 0 else 1e-15)
    sp = L.softplus(z)
    assert math.isclose(loss, 1e-5 * 2 * z * z + sp, rel_tol=1e-15)


def test_product_filter_near_z_minus_46():
    zs = [-45.9, -46.0, -46.05, -46.2, -47.0]
    n = len(zs)
    rp = np.arange(n + 1, dtype=np.int64)
    orc = LogisticOracle(rp, np.arange(n, dtype=np.int32), np.ones(n, np.float32), np.ones(n, np.int8), n, 1e-5)
    kept = []
    for z in zs:
        prod = L.sigmoid(z)
        assert abs(prod - 1e-20) >= 1e-9 * 1e-20          # far enough from the threshold for a last-ulp exp difference
        kept.append(prod > 1e-20)
    g, _ = orc.gradient(np.array(zs), np.arange(n, dtype=np.int32))
    assert ((g != 0) == np.array(kept)).all() and any(kept) and not all(kept)
