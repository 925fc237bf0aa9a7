"""Host side of the calibration calls (Master.calibrate / sampled_calibrate / local_calibration, Slave.calibrated_probabilities,
the `calibrate` configuration key) with a recording stand-in for NativeCtx: which context calls are made with which rows, and
the numbers derived on the host (ECE, MCE, empty bins)."""
import math

import numpy as np
import pytest

LAM = 1e-5


class RecordingCtx:
    def __init__(self, dim):
        self.dim, self.calls = dim, []

    def _fit(self, *call):
        self.calls.append(call)
        return 0.5, -0.25, 12.5, np.array([4, 0, 90, 1, 5], dtype=np.int64)

    def calibrate(self, b, e, w=None):
        return self._fit("calibrate", int(b), int(e))

    def calibrate_sampled(self, b, e, key, lo, hi, w=None):
        return self._fit("calibrate_sampled", int(b), int(e), int(key), int(lo), int(hi))

    def calibrate_samples(self, ids, w=None):
        return self._fit("calibrate_samples", np.asarray(ids).tolist())

    def _quality(self, n_bins, *call):
        self.calls.append(call)
        rows = np.zeros(n_bins, dtype=np.int64)
        pos = np.zeros(n_bins, dtype=np.int64)
        psum = np.zeros(n_bins)
        rows[0], pos[0], psum[0] = 6, 1, 0.6            # mean p 0.1, observed 1/6
        rows[-1], pos[-1], psum[-1] = 4, 3, 3.8         # mean p 0.95, observed 0.75
        return np.array([2.0, 5.0]), rows, pos, psum, np.array([10, 2], dtype=np.int64)

    def eval_calibration(self, b, e, a, bb, n_bins=10, w=None):
        return self._quality(n_bins, "eval_calibration", int(b), int(e), a, bb, n_bins)

    def eval_sampled_calibration(self, b, e, key, lo, hi, a, bb, n_bins=10, w=None):
        return self._quality(n_bins, "eval_sampled_calibration", int(b), int(e), int(key), int(lo), int(hi), a, bb, n_bins)

    def eval_samples_calibration(self, ids, a, bb, n_bins=10, w=None):
        return self._quality(n_bins, "eval_samples_calibration", np.asarray(ids).tolist(), a, bb, n_bins)

    def calibrated_probabilities(self, ids, a, b, w=None):
        self.calls.append(("calibrated_probabilities", np.asarray(ids).tolist(), a, b))
        return np.full(len(ids), 0.5)

    def comm_init(self, uid):
        pass


class RecordingSlave:
    def __init__(self, world, n_train, n_test, dim):
        self.ctx, self.world, self.is_async = RecordingCtx(dim), world, False
        self.n_train, self.n_test, self.dim = n_train, n_test, dim


def _stub(n, dim):
    from distributed_sgd_b200.utils.dataset import Data
    return Data(np.arange(n + 1, dtype=np.int64), np.zeros(n, np.int32), np.ones(n, np.float32), np.ones(n, np.int8), dim)


def _master(n_train=101, n_test=40, dim=16, jvm_exact=False, seed=3):
    from distributed_sgd_b200.core.master import MasterSync
    from distributed_sgd_b200.ml import SparseSVM
    slave = RecordingSlave(1, n_train, n_test, dim)
    m = MasterSync(0, _stub(n_train, dim), _stub(n_test, dim), SparseSVM(LAM), 1, slave=slave, seed=seed, jvm_exact=jvm_exact)
    return m, slave.ctx


def test_calibration_value():
    from distributed_sgd_b200.ml import Calibration
    c = Calibration.identity()
    assert (c.a, c.b, c.status) == (1.0, 0.0, 0) and math.isnan(c.objective)
    with pytest.raises(Exception):
        c.a = 2.0                                                     # frozen


def test_master_calibrate_names_the_train_or_test_rows():
    m, ctx = _master()
    c = m.calibrate()
    assert (c.a, c.b, c.objective, c.iterations, c.status, c.rows, c.nan_rows) == (0.5, -0.25, 12.5, 4, 0, 90, 1)
    m.calibrate(test_data=True)
    assert ctx.calls == [("calibrate", 0, 101), ("calibrate", 101, 141)]


def test_sampled_forms_draw_as_the_sampled_metrics_do():
    from distributed_sgd_b200.core.master import sampled_key
    from distributed_sgd_b200.native import DsgdEmpty
    m, ctx = _master()
    m.sampled_calibrate(None, 37)
    c = m.calibrate()
    m.local_sampled_calibration(c, None, 500, test_data=True, n_bins=5)
    assert ctx.calls[0] == ("calibrate_sampled", 0, 101, sampled_key(3, 0), 0, 37)
    assert ctx.calls[2] == ("eval_sampled_calibration", 101, 141, sampled_key(3, 1), 0, 40, 0.5, -0.25, 5)
    with pytest.raises(DsgdEmpty):
        m.sampled_calibrate(None, 0)
    mj, ctxj = _master(jvm_exact=True, seed=0)
    mj.sampled_calibrate(None, 10)
    mj.local_sampled_calibration(c, None, 7)
    assert ctxj.calls[0][0] == "calibrate_samples" and len(ctxj.calls[0][1]) == 10
    assert ctxj.calls[1][0] == "eval_samples_calibration" and len(ctxj.calls[1][1]) == 7


def test_local_calibration_derives_its_numbers_on_the_host():
    from distributed_sgd_b200.ml import Calibration
    m, ctx = _master()
    q = m.local_calibration(Calibration(2.0, 0.5), test_data=True, n_bins=4)
    assert ctx.calls == [("eval_calibration", 101, 141, 2.0, 0.5, 4)]
    assert q["rows"] == 10 and q["nan_rows"] == 2
    assert q["brier"] == 0.2 and q["log_loss"] == 0.5
    gaps = [abs(0.6 / 6 - 1 / 6), abs(3.8 / 4 - 0.75)]
    assert q["ece"] == pytest.approx(0.6 * gaps[0] + 0.4 * gaps[1], rel=1e-15) and q["mce"] == pytest.approx(max(gaps), rel=1e-15)
    bins = q["bins"]
    assert bins["edges"].tolist() == [0.0, 0.25, 0.5, 0.75, 1.0]
    assert bins["rows"].tolist() == [6, 0, 0, 4] and bins["positives"].tolist() == [1, 0, 0, 3]
    assert np.isnan(bins["mean_predicted"][1:3]).all() and np.isnan(bins["observed"][1:3]).all()      # empty bins
    assert bins["mean_predicted"][0] == 0.6 / 6 and bins["observed"][3] == 0.75


def test_slave_calibrated_probabilities_passes_the_pair():
    from distributed_sgd_b200.core.slave import Slave
    from distributed_sgd_b200.ml import Calibration
    s = Slave.__new__(Slave)
    s.ctx, s._train_ids = RecordingCtx(4), lambda ids: None
    p = s.calibrated_probabilities([3, 1], Calibration(0.75, 0.125))
    assert p.tolist() == [0.5, 0.5] and s.ctx.calls == [("calibrated_probabilities", [3, 1], 0.75, 0.125)]


def test_configuration_key():
    from distributed_sgd_b200.utils.config import Config, load_config
    assert Config().calibrate is False and load_config(env={}).calibrate is False
    assert load_config(env={"DSGD_CALIBRATE": "true"}).calibrate is True
    with pytest.raises(ValueError):
        load_config(env={"DSGD_CALIBRATE": "maybe"})


class _FakeState:
    grad, updates = np.zeros(16), 0


def _scenario_calls(monkeypatch, **cfg_fields):
    """The context calls a scenario makes, with Slave and Master.create replaced so that no device is touched."""
    import distributed_sgd_b200 as pkg
    from distributed_sgd_b200.main import scenario
    from distributed_sgd_b200.utils.config import Config
    ctx = RecordingCtx(16)

    class FakeSlave:
        def __init__(self, *a, **k):
            self.ctx = ctx

        def stop(self):
            pass

    class FakeMaster:
        history = {}

        def __init__(self):
            from distributed_sgd_b200.core.master import Master
            self._m = Master

        def distributed_loss(self, w):
            return 1.0

        def distributed_accuracy(self, w):
            return 0.5

        def fit(self, *a, **k):
            return _FakeState()

        def local_loss_accuracy(self, w, test_data=False):
            return 0.5, 0.5

        def calibrate(self, w=None, test_data=False):
            from distributed_sgd_b200.core.master import _calibration
            return _calibration(ctx.calibrate(0, 8, w))

        def local_calibration(self, c, w=None, test_data=False, n_bins=10):
            from distributed_sgd_b200.core.master import calibration_dict
            return calibration_dict(ctx.eval_calibration(8, 10, c.a, c.b, n_bins, w))

    monkeypatch.setattr(pkg, "Slave", FakeSlave)
    monkeypatch.setattr(pkg.Master, "create", staticmethod(lambda *a, **k: FakeMaster()))
    lines = []
    rep = scenario(Config(node_count=1, **cfg_fields), _stub(10, 16), log=lines.append)
    return ctx.calls, rep, lines


def test_a_default_scenario_makes_no_calibration_call(monkeypatch):
    calls, rep, lines = _scenario_calls(monkeypatch)
    assert calls == [] and "calibration" not in rep and not any("calibration" in s for s in lines)


def test_scenario_with_the_key_fits_on_train_and_judges_on_test(monkeypatch):
    calls, rep, lines = _scenario_calls(monkeypatch, calibrate=True, model="logistic")
    assert [c[0] for c in calls] == ["calibrate", "eval_calibration", "eval_calibration"]
    assert calls[1][3:5] == (0.5, -0.25) and calls[2][3:5] == (1.0, 0.0)          # the fitted link, then the identity
    assert rep["calibration"]["a"] == 0.5 and "identity" in rep["calibration"]
    assert any(s.startswith("calibration: A = 0.5") and "identity link" in s for s in lines)
    calls, rep, _ = _scenario_calls(monkeypatch, calibrate=True)                   # svm: no identity link to compare with
    assert [c[0] for c in calls] == ["calibrate", "eval_calibration"] and "identity" not in rep["calibration"]
