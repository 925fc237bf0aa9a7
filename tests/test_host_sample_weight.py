"""Sample weights on the host side, without a GPU: Data carries them through split_at and head, the `sample-weight`
configuration key and its .npy loader, the refusals of asynchronous training before any device context is made, and what
Master asks of the device context with weights loaded -- a stand-in context defined here records the calls."""
from types import SimpleNamespace

import numpy as np
import pytest

DIM = 8


def _data(n, weight=None, labels=None):
    from distributed_sgd_b200.utils.dataset import Data
    lab = np.ones(n, np.int8) if labels is None else np.asarray(labels, np.int8)
    d = Data(np.arange(n + 1, dtype=np.int64), np.zeros(n, np.int32), np.ones(n, np.float32), lab, DIM)
    if weight is not None:
        d.weight = np.asarray(weight, np.float64)
    return d


def test_split_at_and_head_carry_the_weights():
    from distributed_sgd_b200.utils.dataset import Data, has_sample_weights, sample_weights_of
    d = _data(5, [0.5, 1.0, 0.0, 2.0, 4.0])
    a, b = d.split_at(3)
    assert list(a.weight) == [0.5, 1.0, 0.0] and list(b.weight) == [2.0, 4.0]
    assert list(d.head(2).weight) == [0.5, 1.0]
    u = _data(5)
    assert u.weight is None and all(p.weight is None for p in u.split_at(2))
    # the positional construction of before still works and is unweighted
    assert Data(u.row_ptr, u.col, u.val, u.label, DIM).weight is None
    assert not has_sample_weights(u, None) and has_sample_weights(u, b)
    assert list(sample_weights_of(a, _data(2))) == [0.5, 1.0, 0.0, 1.0, 1.0]


def test_config_key_environment_variable_and_default(tmp_path):
    from distributed_sgd_b200.utils.config import load_config
    assert load_config(env={}).sample_weight == ""
    assert load_config(env={"DSGD_SAMPLE_WEIGHT": "/data/w.npy"}).sample_weight == "/data/w.npy"
    conf = tmp_path / "application.conf"
    conf.write_text('dsgd {\n  sample-weight = "w.npy"\n  sample-weight = ${?DSGD_SAMPLE_WEIGHT}\n}\n')
    assert load_config(str(conf), env={}).sample_weight == "w.npy"
    assert load_config(str(conf), env={"DSGD_SAMPLE_WEIGHT": "v.npy"}).sample_weight == "v.npy"
    for bad in ("w.txt", "1.0", "balanced"):
        with pytest.raises(ValueError, match="sample-weight"):
            load_config(env={"DSGD_SAMPLE_WEIGHT": bad})


def test_loader_checks_shape_and_values(tmp_path):
    from distributed_sgd_b200.utils.dataset import load_sample_weights
    p = tmp_path / "w.npy"
    np.save(p, np.array([0, 1, 2], np.int32))
    w = load_sample_weights(str(p), 3)
    assert w.dtype == np.float64 and list(w) == [0.0, 1.0, 2.0]
    for bad, n in ((np.ones(4), 3), (np.ones((3, 1)), 3), (np.array([1.0, -0.5, 1.0]), 3), (np.array([1.0, np.nan, 1.0]), 3),
                   (np.array([np.inf, 1.0, 1.0]), 3), (np.array(["a", "b", "c"]), 3)):
        np.save(p, bad)
        with pytest.raises(ValueError, match="sample-weight"):
            load_sample_weights(str(p), n)


def test_async_training_refuses_sample_weights_before_any_context(monkeypatch, tmp_path):
    from distributed_sgd_b200 import native
    from distributed_sgd_b200.core.master import MasterAsync
    from distributed_sgd_b200.core.slave import Slave
    from distributed_sgd_b200.main import scenario
    from distributed_sgd_b200.ml import SparseSVM
    from distributed_sgd_b200.utils.config import Config

    def no_device(*a, **kw):
        raise AssertionError("a device context was made")
    monkeypatch.setattr(native.NativeCtx, "__init__", no_device)
    with pytest.raises(ValueError, match="sample-weight"):
        Slave(0, 0, _data(4, [1.0, 2.0, 0.0, 1.0]), SparseSVM(0.1), True)
    with pytest.raises(ValueError, match="sample-weight"):   # weights on the test rows alone count too
        Slave(0, 0, _data(4), SparseSVM(0.1), True, test_data=_data(2, [1.0, 1.0]))
    slave = SimpleNamespace(ctx=None, world=1, is_async=True, n_train=4, n_test=2, dim=DIM)
    with pytest.raises(ValueError, match="sample-weight"):
        MasterAsync(0, _data(4, np.ones(4)), _data(2), SparseSVM(0.1), 1, slave=slave)
    with pytest.raises(ValueError, match="sample-weight"):
        MasterAsync(0, _data(4), _data(2, np.ones(2)), SparseSVM(0.1), 1, slave=slave)
    p = tmp_path / "w.npy"
    np.save(p, np.ones(10))
    with pytest.raises(ValueError, match="sample-weight"):
        scenario(Config(is_async=True, sample_weight=str(p)), _data(10))


class _Ctx:
    """Stands in for NativeCtx: no arithmetic, records the name of every call."""

    def __init__(self):
        self.log = []

    def __getattr__(self, name):
        from distributed_sgd_b200.native import WeightedEval

        def call(*args, **kw):
            self.log.append(name)
            if name.endswith("_weighted"):
                return WeightedEval(0.5, 6.5, 3.25, 9.0, 20, 7)   # S 6.5, sum c [correct] 3.25, sum c 9; 7 of 20 correct
            return 14, 7, 0.5
        return call


def _master(ctx, sample_weighted, class_weight=(1.0, 1.0), n_train=20, n_test=5):
    from distributed_sgd_b200.core.master import MasterSync
    from distributed_sgd_b200.ml import SparseSVM
    slave = SimpleNamespace(ctx=ctx, world=1, is_async=False, n_train=n_train, n_test=n_test, dim=DIM,
                            class_weight=class_weight, sample_weighted=sample_weighted)
    return MasterSync(0, _data(n_train), _data(n_test), SparseSVM(0.1), 1, slave=slave, seed=0)


def test_a_sample_weighted_master_reports_penalty_plus_s_over_n():
    for cw in ((1.0, 1.0), (4.0, 0.25)):   # S already carries the class weights
        ctx = _Ctx()
        m = _master(ctx, True, cw)
        assert m.local_loss() == 0.1 * 0.5 + 6.5 / 20
        loss, acc = m.local_loss_accuracy(test_data=True)
        assert loss == 0.1 * 0.5 + 6.5 / 5 and acc == 7 / 5    # the accuracy stays the unweighted share
        assert m.local_accuracy() == 7 / 20
        assert m.local_sampled_loss(None, 10) == 0.1 * 0.5 + 6.5 / 10
        assert m.distributed_loss(None) == 0.1 * 0.5 + 6.5 / 20
        assert ctx.log == ["eval_weighted"] * 3 + ["eval_sampled_weighted", "eval_weighted"]


def test_without_the_flag_the_master_makes_the_calls_of_before():
    ctx = _Ctx()
    m = _master(ctx, False)
    m.local_loss()
    m.local_sampled_loss(None, 10)
    assert ctx.log == ["eval_counts", "eval_sampled_counts"]


def test_weighted_report():
    ctx = _Ctx()
    r = _master(ctx, True).local_weighted_report(test_data=True)
    assert ctx.log == ["eval_weighted"]
    assert r == {"n": 20, "weight_sum": 9.0, "weighted_loss": 0.1 * 0.5 + 6.5 / 20, "weighted_accuracy": 3.25 / 9.0}
    r = _master(ctx, False).local_sampled_weighted_report(None, 10)
    assert ctx.log[-1] == "eval_sampled_weighted" and r["weighted_accuracy"] == 3.25 / 9.0
