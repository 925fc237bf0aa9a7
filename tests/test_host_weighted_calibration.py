"""Host side of the weighted calibration calls (Master.calibrate / sampled_calibrate / local_calibration /
local_sampled_calibration with weighted=True, weighted_calibration_dict, the calibration-weighted key) with a recording
stand-in for NativeCtx: which context calls are made, and the numbers derived on the host."""
import math

import numpy as np
import pytest

from test_host_calibration import RecordingCtx, RecordingSlave, _stub

LAM = 1e-5


class WeightedCtx(RecordingCtx):
    def _wfit(self, *call):
        self.calls.append(call)
        return 0.5, -0.25, 12.5, np.array([4, 0, 90, 1, 5], dtype=np.int64), np.array([30.5, 60.25, 2.0])

    def calibrate_weighted(self, b, e, w=None):
        return self._wfit("calibrate_weighted", int(b), int(e))

    def calibrate_weighted_sampled(self, b, e, key, lo, hi, w=None):
        return self._wfit("calibrate_weighted_sampled", int(b), int(e), int(key), int(lo), int(hi))

    def calibrate_weighted_samples(self, ids, w=None):
        return self._wfit("calibrate_weighted_samples", np.asarray(ids).tolist())

    def _wquality(self, n_bins, *call):
        self.calls.append(call)
        wt, pw, ps = np.zeros(n_bins), np.zeros(n_bins), np.zeros(n_bins)
        wt[0], pw[0], ps[0] = 6.0, 1.5, 0.6             # mean p 0.1, observed 0.25
        wt[-1], pw[-1], ps[-1] = 4.0, 3.0, 3.8          # mean p 0.95, observed 0.75
        return np.array([2.0, 5.0, 10.0, 0.0]), wt, pw, ps, np.array([12, 2], dtype=np.int64)

    def eval_weighted_calibration(self, b, e, a, bb, n_bins=10, w=None):
        return self._wquality(n_bins, "eval_weighted_calibration", int(b), int(e), a, bb, n_bins)

    def eval_sampled_weighted_calibration(self, b, e, key, lo, hi, a, bb, n_bins=10, w=None):
        return self._wquality(n_bins, "eval_sampled_weighted_calibration", int(b), int(e), int(key), int(lo), int(hi), a,
                              bb, n_bins)

    def calibrate_isotonic_weighted(self, b, e, w=None):
        self.calls.append(("calibrate_isotonic_weighted", int(b), int(e)))
        return (np.array([-1.0, 2.0]), np.array([0.25, 0.75]), np.array([4.0, 5.75]), np.array([1.0, 6.5]),
                np.array([2, 2, 30, 0, 9]), np.array([7.5, 2.25]))

    def _wiquality(self, n_bins, *call):
        sums, wt, pw, ps, _ = self._wquality(n_bins, *call)
        sums[3] = 0.5
        return sums, wt, pw, ps, np.array([12, 2, 1], dtype=np.int64)

    def eval_weighted_isotonic_calibration(self, b, e, x, y, n_bins=10, w=None):
        return self._wiquality(n_bins, "eval_weighted_isotonic_calibration", int(b), int(e), n_bins)

    def eval_sampled_weighted_isotonic_calibration(self, b, e, key, lo, hi, x, y, n_bins=10, w=None):
        return self._wiquality(n_bins, "eval_sampled_weighted_isotonic_calibration", int(b), int(e), n_bins)

    def eval_samples_weighted_isotonic_calibration(self, ids, x, y, n_bins=10, w=None):
        return self._wiquality(n_bins, "eval_samples_weighted_isotonic_calibration", n_bins)

    def eval_samples_weighted_calibration(self, ids, a, bb, n_bins=10, w=None):
        return self._wquality(n_bins, "eval_samples_weighted_calibration", np.asarray(ids).tolist(), a, bb, n_bins)


def _master(n_train=101, n_test=40, dim=16, jvm_exact=False):
    from distributed_sgd_b200.core.master import MasterSync
    from distributed_sgd_b200.ml import SparseSVM
    slave = RecordingSlave(1, n_train, n_test, dim)
    slave.ctx = WeightedCtx(dim)
    m = MasterSync(0, _stub(n_train, dim), _stub(n_test, dim), SparseSVM(LAM), 1, slave=slave, seed=3, jvm_exact=jvm_exact)
    return m, slave.ctx


def test_weighted_calls_and_result():
    from distributed_sgd_b200.ml import Calibration
    m, ctx = _master()
    cal = m.calibrate(weighted=True)
    assert ctx.calls == [("calibrate_weighted", 0, 101)]
    assert cal.weighted and (cal.weight_pos, cal.weight_neg, cal.nan_weight) == (30.5, 60.25, 2.0)
    assert (cal.a, cal.b, cal.iterations, cal.rows, cal.nan_rows) == (0.5, -0.25, 4, 90, 1)
    assert repr(cal) == repr(Calibration(0.5, -0.25, 12.5, 4, 0, 90, 1))     # prints as an unweighted one
    assert cal != Calibration(0.5, -0.25, 12.5, 4, 0, 90, 1)
    m.calibrate(test_data=True, weighted=True)
    assert ctx.calls[-1] == ("calibrate_weighted", 101, 141)
    q = m.local_calibration(cal, test_data=True, n_bins=5, weighted=True)
    assert ctx.calls[-1] == ("eval_weighted_calibration", 101, 141, 0.5, -0.25, 5)
    assert q["weight"] == 10.0 and q["rows"] == 12 and q["nan_rows"] == 2


def test_unweighted_calls_are_unchanged():
    m, ctx = _master()
    cal = m.calibrate()
    m.local_calibration(cal, n_bins=5)
    assert [c[0] for c in ctx.calls] == ["calibrate", "eval_calibration"] and not cal.weighted


@pytest.mark.parametrize("jvm_exact", [False, True])
def test_sampled_forms(jvm_exact):
    m, ctx = _master(jvm_exact=jvm_exact)
    cal = m.sampled_calibrate(None, 37, weighted=True)
    m.local_sampled_calibration(cal, None, 40, test_data=True, n_bins=5, weighted=True)
    names = [c[0] for c in ctx.calls]
    if jvm_exact:
        assert names == ["calibrate_weighted_samples", "eval_samples_weighted_calibration"]
    else:
        assert names == ["calibrate_weighted_sampled", "eval_sampled_weighted_calibration"]


def test_weighted_isotonic_calls():
    from distributed_sgd_b200.ml import IsotonicCalibration
    m, ctx = _master()
    iso = m.calibrate(method="isotonic", weighted=True)
    assert ctx.calls == [("calibrate_isotonic_weighted", 0, 101)]
    assert iso.weighted and (iso.weight_pos, iso.weight_neg) == (7.5, 2.25) and iso.block_rows.dtype == np.float64
    q = m.local_calibration(iso, test_data=True, n_bins=4, weighted=True)
    assert ctx.calls[-1][0] == "eval_weighted_isotonic_calibration" and q["infinite_log_loss_rows"] == 1
    assert q["log_loss"] == math.inf
    m.local_sampled_calibration(iso, None, 20, n_bins=4, weighted=True)
    assert ctx.calls[-1][0] == "eval_sampled_weighted_isotonic_calibration"
    assert not IsotonicCalibration(np.zeros(1), np.zeros(1), np.zeros(1), np.zeros(1)).weighted


def test_dict_arithmetic():
    from distributed_sgd_b200.core.master import weighted_calibration_dict
    n_bins = 4
    wt, pw, ps = np.array([6.0, 0.0, 0.0, 4.0]), np.array([1.5, 0.0, 0.0, 3.0]), np.array([0.6, 0.0, 0.0, 3.8])
    d = weighted_calibration_dict((np.array([2.0, 5.0, 10.0, 0.0]), wt, pw, ps, np.array([12, 2])))
    assert d["brier"] == 2.0 / 10.0 and d["log_loss"] == 5.0 / 10.0 and d["weight"] == 10.0
    gaps = [abs(0.6 / 6.0 - 1.5 / 6.0), abs(3.8 / 4.0 - 3.0 / 4.0)]
    assert d["ece"] == pytest.approx(0.6 * gaps[0] + 0.4 * gaps[1], rel=1e-15) and d["mce"] == max(gaps)
    assert math.isnan(d["bins"]["mean_predicted"][1]) and math.isnan(d["bins"]["observed"][2])
    assert np.array_equal(d["bins"]["weight"], wt) and len(d["bins"]["edges"]) == n_bins + 1
    inf = weighted_calibration_dict((np.array([2.0, 5.0, 10.0, 0.5]), wt, pw, ps, np.array([12, 2])))
    assert inf["log_loss"] == math.inf and inf["brier"] == 0.2
    empty = weighted_calibration_dict((np.zeros(4), np.zeros(2), np.zeros(2), np.zeros(2), np.array([3, 0])))
    assert all(math.isnan(empty[k]) for k in ("brier", "log_loss", "ece", "mce")) and empty["rows"] == 3


def test_configuration_key_and_its_refusals(tmp_path):
    from distributed_sgd_b200.main import scenario
    from distributed_sgd_b200.utils.config import load_config
    assert load_config(env={}).calibration_weighted is False
    cfg = load_config(env={"DSGD_CALIBRATION_WEIGHTED": "true", "DSGD_CALIBRATE": "true"})
    assert cfg.calibration_weighted is True
    assert load_config(env={"DSGD_CALIBRATION_WEIGHTED": "true", "DSGD_CALIBRATION_METHOD": "isotonic"}).calibration_weighted
    cfg = load_config(env={"DSGD_CALIBRATION_WEIGHTED": "true", "DSGD_ASYNC": "true"})
    with pytest.raises(ValueError, match="calibration-weighted"):
        scenario(cfg, None)            # refused before the data (None here) or a device is touched
