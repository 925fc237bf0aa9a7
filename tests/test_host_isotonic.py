"""The host side of isotonic calibration without a GPU: the configuration key, the type dispatch of Master and Slave, and
that method="sigmoid" makes exactly the calls it made before the isotonic method existed."""
import numpy as np
import pytest

from distributed_sgd_b200.ml import Calibration, IsotonicCalibration
from distributed_sgd_b200.utils.config import load_config


class RecordingCtx:
    """A NativeCtx stand-in: records every call and answers with fixed arrays."""

    def __init__(self):
        self.calls = []

    def __getattr__(self, name):
        def call(*args):
            self.calls.append((name, *args))
            if name.startswith("calibrate_isotonic"):
                return (np.array([-1.0, 2.0]), np.array([0.25, 0.75]), np.array([4, 4]), np.array([1, 3]),
                        np.array([2, 2, 8, 0, 5]))
            if name.startswith("calibrate"):
                return 0.5, -0.25, 1.0, np.array([3, 0, 8, 0, 4])
            if "calibration" in name:
                words = np.array([8, 1, 2]) if "isotonic" in name else np.array([8, 1])
                return np.array([2.0, 4.0]), np.full(10, 0) + np.eye(10, dtype=np.int64)[0] * 8, np.zeros(10, np.int64), \
                    np.eye(10)[0] * 2.0, words
            return np.zeros(len(args[0]) if args and hasattr(args[0], "__len__") else 1)
        return call


def master_with(ctx):
    from distributed_sgd_b200.core.master import Master
    m = Master.__new__(Master)
    m.ctx, m.n_train, m.n_test = ctx, 8, 2
    m._draw_sample = lambda count, test_data: (0, 8, 4, 77, None)
    return m


def test_configuration_key():
    assert load_config(env={}).calibration_method == "sigmoid"
    assert load_config(env={"DSGD_CALIBRATION_METHOD": "isotonic"}).calibration_method == "isotonic"
    with pytest.raises(ValueError):
        load_config(env={"DSGD_CALIBRATION_METHOD": "beta"})


def test_configuration_file_key(tmp_path):
    p = tmp_path / "app.conf"
    p.write_text('dsgd {\n  calibrate = true\n  calibration-method = "isotonic"\n}\n')
    cfg = load_config(str(p), env={})
    assert cfg.calibrate and cfg.calibration_method == "isotonic"


def test_sigmoid_makes_exactly_the_calls_it_always_made():
    a, b = RecordingCtx(), RecordingCtx()
    ma, mb = master_with(a), master_with(b)
    ca = ma.calibrate(None)
    cb = mb.calibrate(None, method="sigmoid")
    assert ca == cb and isinstance(cb, Calibration)
    ma.sampled_calibrate(None, 4)
    mb.sampled_calibrate(None, 4, method="sigmoid")
    ma.local_calibration(ca)
    mb.local_calibration(cb)
    assert a.calls == b.calls
    assert [c[0] for c in a.calls] == ["calibrate", "calibrate_sampled", "eval_calibration"]


def test_isotonic_dispatch():
    ctx = RecordingCtx()
    m = master_with(ctx)
    c = m.calibrate(None, method="isotonic")
    assert isinstance(c, IsotonicCalibration) and c.blocks == 2 and c.points == 2 and c.rows == 8 and c.distinct_scores == 5
    c2 = m.calibrate(None, test_data=True, method="isotonic")
    assert ctx.calls[-1][1:3] == (8, 10) and c2.blocks == 2
    m.sampled_calibrate(None, 4, method="isotonic")
    q = m.local_calibration(c, n_bins=10)
    assert q["infinite_log_loss_rows"] == 2 and q["log_loss"] == float("inf") and q["rows"] == 8
    m.local_sampled_calibration(c, None, 4)
    names = [k[0] for k in ctx.calls]
    assert names == ["calibrate_isotonic", "calibrate_isotonic", "calibrate_isotonic_sampled", "eval_isotonic_calibration",
                     "eval_sampled_isotonic_calibration"]
    x, y = ctx.calls[3][3], ctx.calls[3][4]
    assert x is c.x and y is c.y
    with pytest.raises(ValueError):
        m.calibrate(None, method="beta")


def test_slave_dispatches_on_the_calibration_type():
    from distributed_sgd_b200.core.slave import Slave
    ctx = RecordingCtx()
    s = Slave.__new__(Slave)
    s.ctx = ctx
    s._train_ids = lambda ids: None
    s.calibrated_probabilities([0, 1], Calibration(0.5, 0.1))
    iso = IsotonicCalibration(np.array([0.0, 1.0]), np.array([0.2, 0.8]), np.array([3]), np.array([1]), 1, 3, 0, 2)
    s.calibrated_probabilities([0, 1], iso)
    assert [c[0] for c in ctx.calls] == ["calibrated_probabilities", "isotonic_probabilities"]
    assert ctx.calls[1][2] is iso.x and ctx.calls[1][3] is iso.y
