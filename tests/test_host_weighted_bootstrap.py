"""Host side of the weighted bootstrap (Master.local_bootstrap / local_sampled_bootstrap / compare_bootstrap with
weighted=True, the `bootstrap-weighted` configuration key) with a stand-in for NativeCtx: the 16-word replicate layout as it
is packed and gathered, the metric formulas against weighted_curve_dict's, and the estimates from the weighted calls."""
import math

import numpy as np
import pytest

LAM = 1e-5


def _wreps(key, lo, hi, scale):
    """Weighted replicate words that depend on (key, b) alone: replicate b = 7 has no positive weight, b = 9 a NaN score."""
    words, wsums, loss = [], [], []
    for b in range(lo, hi):
        r = np.random.default_rng([key & 0xFFFFFFFF, b])
        tp, fn, pz, fp, tn, nz = (float(x) for x in r.random(6) * 40.0)
        if b == 7:
            tp = fn = pz = 0.0
        nan_w = 0.0 if b != 9 else 0.5
        wp, wn = tp + fn + pz, fp + tn + nz
        u2w = float(r.random() * 2.0 * wp * wn)
        sap = float(r.random() * wp) * scale
        words.append([int(r.integers(10, 99)), int(b == 9)])
        wsums.append([tp, fn, pz, fp, tn, nz, u2w, nan_w, sap, tp + tn, wp + wn, wp, wn])
        loss.append(float(r.integers(0, 100)) * scale)
    return np.array(words, np.int64).reshape(-1, 2), np.array(wsums).reshape(-1, 13), np.array(loss)


class _WC:
    """A NativeCtx.eval_*weighted_curve result's fields that weighted_curve_dict reads"""

    def __init__(self, words, wsums):
        from distributed_sgd_b200.native import weighted_auc_ap
        self.words, self.wsums, self.n_points = words, wsums, 7
        self.auc, self.ap = weighted_auc_ap(words, wsums)


class WBootCtx:
    def __init__(self, dim):
        self.dim, self.calls = dim, []

    def _scale(self, w):
        return 1.0 if w is None else float(np.asarray(w)[0])

    def eval_weighted_bootstrap(self, b, e, key, lo, hi, w=None):
        self.calls.append(("eval_weighted_bootstrap", b, e, key, lo, hi))
        return _wreps(key, lo, hi, self._scale(w))

    def eval_sampled_weighted_bootstrap(self, b, e, skey, plo, phi, key, lo, hi, w=None):
        self.calls.append(("eval_sampled_weighted_bootstrap", b, e, skey, plo, phi, key, lo, hi))
        return _wreps(key, lo, hi, self._scale(w))

    def eval_weighted_curve(self, b, e, w=None, curve=True):
        self.calls.append(("eval_weighted_curve", b, e))
        return _WC(np.array([30, 10, 0, 5, 55, 0, 3000, 0]),
                   np.array([15.0, 5.0, 0.0, 10.0, 27.5, 0.0, 900.0, 0.0, 14.0 * self._scale(w), 42.5, 57.5, 20.0, 37.5]))

    def eval_sampled_weighted_curve(self, b, e, key, lo, hi, w=None, curve=True):
        self.calls.append(("eval_sampled_weighted_curve", b, e, key, lo, hi))
        return _WC(np.array([3, 1, 0, 1, 5, 0, 30, 0]),
                   np.array([1.5, 0.5, 0.0, 1.0, 2.5, 0.0, 9.0, 0.0, 1.5, 4.0, 5.5, 2.0, 3.5]))

    def eval_weighted(self, b, e, w=None):
        from distributed_sgd_b200.native import WeightedEval
        self.calls.append(("eval_weighted", b, e))
        return WeightedEval(4.0, 60.0 * self._scale(w), 42.5, 57.5, 100, 85)

    def eval_sampled_weighted(self, b, e, key, lo, hi, w=None):
        from distributed_sgd_b200.native import WeightedEval
        return WeightedEval(4.0, 6.0, 4.0, 5.5, 10, 8)

    def comm_init(self, uid):
        pass


class WBootSlave:
    def __init__(self, world, n_train, n_test, dim):
        self.ctx, self.world, self.is_async = WBootCtx(dim), world, False
        self.n_train, self.n_test, self.dim = n_train, n_test, dim


def _stub(n, dim):
    from distributed_sgd_b200.utils.dataset import Data
    return Data(np.arange(n + 1, dtype=np.int64), np.zeros(n, np.int32), np.ones(n, np.float32), np.ones(n, np.int8), dim)


def _master(seed=3, n_train=101, n_test=100):
    from distributed_sgd_b200.core.master import MasterSync
    from distributed_sgd_b200.ml import SparseSVM
    slave = WBootSlave(1, n_train, n_test, 16)
    m = MasterSync(0, _stub(n_train, 16), _stub(n_test, 16), SparseSVM(LAM), 1, slave=slave, seed=seed, attach=False)
    return m, slave.ctx


def test_pack_and_unpack_the_replicate_layouts():
    from distributed_sgd_b200.core.master import BOOTSTRAP_LAYOUT, bootstrap_pack, bootstrap_unpack
    assert BOOTSTRAP_LAYOUT[True] == (2, 13) and sum(BOOTSTRAP_LAYOUT[True]) + 1 == 16
    a, b = _wreps(5, 0, 3, 1.0), _wreps(5, 3, 8, 1.0)
    parts = [bootstrap_pack(*a), np.zeros(0), bootstrap_pack(*b)]   # a rank with no replicates sends nothing
    assert parts[0].size == 16 * 3
    words, wsums, loss = bootstrap_unpack(parts, weighted=True)
    whole = _wreps(5, 0, 8, 1.0)
    assert words.shape == (8, 2) and wsums.shape == (8, 13) and loss.shape == (8,)
    assert np.array_equal(words, whole[0]) and np.array_equal(wsums.view(np.int64), whole[1].view(np.int64))
    assert np.array_equal(loss, whole[2])
    # the unweighted layout is unchanged: 9 words, the AP, the loss sum
    uw = (np.arange(18, dtype=np.int64).reshape(2, 9), np.array([0.5, np.nan]), np.array([1.0, 2.0]))
    w2, ap2, l2 = bootstrap_unpack([bootstrap_pack(*uw)])
    assert np.array_equal(w2, uw[0]) and ap2.shape == (2,) and np.isnan(ap2[1]) and np.array_equal(l2, uw[2])


def test_weighted_values_follow_weighted_curve_dict():
    from distributed_sgd_b200.core.master import weighted_bootstrap_values, weighted_curve_dict
    words, wsums, loss = _wreps(11, 0, 12, 1.0)
    v = weighted_bootstrap_values(words, wsums, loss, 0.25)
    for j in range(12):
        d = weighted_curve_dict(_WC(np.array([0] * 7 + [int(words[j, 1])]), wsums[j]), curve=False)
        for k, dk in (("accuracy", "accuracy"), ("auc", "auc"), ("ap", "average_precision"), ("precision", "precision"),
                      ("recall", "recall"), ("f1", "f1")):
            a, b = float(v[k][j]), float(d[dk])
            assert (math.isnan(a) and math.isnan(b)) or a == b, (j, k, a, b)
        assert v["loss"][j] == 0.25 + loss[j] / words[j, 0]
    assert np.isnan(v["auc"][7]) and np.isnan(v["ap"][7]) and np.isnan(v["recall"][7])
    assert np.isnan(v["auc"][9]) and np.isnan(v["ap"][9]) and not np.isnan(v["accuracy"][9])
    # no negative weight: AP is 1 and AUC undefined
    ws = wsums[:1].copy()
    ws[0, [3, 4, 5, 12]] = 0.0
    one = weighted_bootstrap_values(words[:1] * [1, 0], ws, loss[:1], 0.0)
    assert one["ap"][0] == 1.0 and np.isnan(one["auc"][0])


def test_local_bootstrap_weighted_estimates_and_calls():
    from distributed_sgd_b200.core.master import BOOTSTRAP_METRICS, bootstrap_key
    m, ctx = _master()
    r = m.local_bootstrap(None, n_boot=30, weighted=True)
    assert ctx.calls[-1] == ("eval_weighted_bootstrap", 101, 201, bootstrap_key(3), 0, 30)
    assert not any(c[0] in ("eval_bootstrap", "eval_curve") for c in ctx.calls)
    assert set(r) == set(BOOTSTRAP_METRICS)
    curve = m.local_weighted_curve(None, test_data=True, curve=False)
    rep = m.local_weighted_report(None, test_data=True)
    assert r["auc"]["estimate"] == curve["auc"] and r["ap"]["estimate"] == curve["average_precision"]
    assert r["accuracy"]["estimate"] == curve["accuracy"] and r["f1"]["estimate"] == curve["f1"]
    assert r["precision"]["estimate"] == curve["precision"] and r["recall"]["estimate"] == curve["recall"]
    assert r["loss"]["estimate"] == rep["weighted_loss"] == LAM * 4.0 + 60.0 / 100
    words, wsums, loss = _wreps(bootstrap_key(3), 0, 30, 1.0)
    assert np.array_equal(r["loss"]["replicates"], LAM * 4.0 + loss / words[:, 0])
    assert r["auc"]["n_defined"] == 28 and r["accuracy"]["n_defined"] == 30
    s = m.local_sampled_bootstrap(None, 30, n_boot=5, weighted=True)
    assert ctx.calls[-1][0] == "eval_sampled_weighted_bootstrap" and s["accuracy"]["estimate"] == 4.0 / 5.5


def test_compare_bootstrap_weighted_pairs_by_key():
    m, ctx = _master()
    wa, wb = np.full(16, 1.0), np.full(16, 2.0)
    r = m.compare_bootstrap(wa, wb, n_boot=20, key=5, weighted=True)
    boots = [c for c in ctx.calls if c[0] == "eval_weighted_bootstrap"]
    assert len(boots) == 2 and boots[0] == boots[1] == ("eval_weighted_bootstrap", 101, 201, 5, 0, 20)
    assert r["ap"]["estimate"] == 14.0 / 20.0 and r["ap"]["p_better"] == 1.0
    same = m.compare_bootstrap(wa, wa, n_boot=20, key=5, weighted=True)
    for k, s in same.items():
        ok = s["replicates"][~np.isnan(s["replicates"])]
        assert s["estimate"] == 0.0 and not ok.any() and s["p_better"] == 0.0, k


def test_configuration_key_and_its_async_refusal():
    from distributed_sgd_b200.main import scenario
    from distributed_sgd_b200.utils.config import load_config
    assert load_config(env={}).bootstrap_weighted is False
    cfg = load_config(env={"DSGD_BOOTSTRAP_WEIGHTED": "true", "DSGD_BOOTSTRAP": "100"})
    assert cfg.bootstrap_weighted is True and cfg.bootstrap == 100
    with pytest.raises(ValueError):
        load_config(env={"DSGD_BOOTSTRAP_WEIGHTED": "sometimes"})
    cfg = load_config(env={"DSGD_BOOTSTRAP_WEIGHTED": "true", "DSGD_ASYNC": "true"})
    with pytest.raises(ValueError, match="bootstrap-weighted"):
        scenario(cfg, None)            # refused before the data (None here) or a device is touched
