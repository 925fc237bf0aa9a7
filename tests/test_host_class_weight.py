"""Class weights on the host side, without a GPU: how "balanced" resolves, the `class-weight` configuration key, the refusals
of asynchronous training, and what Master asks of the device context with and without weights -- a stand-in context defined
here records the calls."""
from types import SimpleNamespace

import numpy as np
import pytest

DIM = 8


def test_balanced_resolves_from_the_train_labels():
    from distributed_sgd_b200.ml.class_weight import resolve_class_weight
    lab = np.array([1] * 10 + [-1] * 90, np.int8)
    assert resolve_class_weight("balanced", lab) == (100 / 20, 100 / 180)
    assert resolve_class_weight(None, lab) == (1.0, 1.0)
    assert resolve_class_weight((3, 0.5), lab) == (3.0, 0.5)
    for one_class in (np.ones(5, np.int8), -np.ones(5, np.int8)):
        with pytest.raises(ValueError, match="balanced"):
            resolve_class_weight("balanced", one_class)
    for bad in ((-1.0, 1.0), (1.0, float("inf")), (float("nan"), 1.0), (1.0,), "heavy"):
        with pytest.raises(ValueError, match="class_weight"):
            resolve_class_weight(bad, lab)


def test_config_key_environment_variable_and_default(tmp_path):
    from distributed_sgd_b200.ml.class_weight import parse_class_weight
    from distributed_sgd_b200.utils.config import load_config
    assert load_config(env={}).class_weight == "none"
    assert parse_class_weight(load_config(env={}).class_weight) is None
    assert parse_class_weight(load_config(env={"DSGD_CLASS_WEIGHT": "balanced"}).class_weight) == "balanced"
    assert parse_class_weight(load_config(env={"DSGD_CLASS_WEIGHT": "4, 0.25"}).class_weight) == (4.0, 0.25)
    conf = tmp_path / "application.conf"
    conf.write_text('dsgd {\n  class-weight = "2,1"\n  class-weight = ${?DSGD_CLASS_WEIGHT}\n}\n')
    assert parse_class_weight(load_config(str(conf), env={}).class_weight) == (2.0, 1.0)
    assert parse_class_weight(load_config(str(conf), env={"DSGD_CLASS_WEIGHT": "none"}).class_weight) is None
    for bad in ("-1,1", "1", "1,2,3", "inf,1", "heavy"):
        with pytest.raises(ValueError):
            load_config(env={"DSGD_CLASS_WEIGHT": bad})


def test_models_take_class_weight_as_a_trailing_field():
    from distributed_sgd_b200.ml import SparseLogistic, SparseSVM
    for M in (SparseSVM, SparseLogistic):
        d = np.ones(3)
        m = M(0.1, d, 0.5)                                   # positional construction as before
        assert m.lam == 0.1 and m.dim_sparsity is d and m.l1 == 0.5 and m.class_weight is None
        assert M(0.1, class_weight="balanced").class_weight == "balanced"


def _data(n, labels=None):
    from distributed_sgd_b200.utils.dataset import Data
    lab = np.ones(n, np.int8) if labels is None else np.asarray(labels, np.int8)
    return Data(np.arange(n + 1, dtype=np.int64), np.zeros(n, np.int32), np.ones(n, np.float32), lab, DIM)


def test_async_training_refuses_a_weighted_model():
    from distributed_sgd_b200.core.master import MasterAsync
    from distributed_sgd_b200.core.slave import Slave
    from distributed_sgd_b200.main import scenario
    from distributed_sgd_b200.ml import SparseSVM
    from distributed_sgd_b200.utils.config import Config
    with pytest.raises(ValueError, match="class_weight"):
        Slave(0, 0, _data(4, [1, -1, 1, -1]), SparseSVM(0.1, class_weight=(2.0, 1.0)), True)
    slave = SimpleNamespace(ctx=None, world=1, is_async=True, n_train=4, n_test=2, dim=DIM)
    with pytest.raises(ValueError, match="class_weight"):
        MasterAsync(0, _data(4, [1, 1, -1, 1]), _data(2), SparseSVM(0.1, class_weight="balanced"), 1, slave=slave)
    with pytest.raises(ValueError, match="class_weight"):
        MasterAsync(0, _data(4), _data(2), SparseSVM(0.1, class_weight=(1.0, 3.0)), 1, slave=slave)
    with pytest.raises(ValueError, match="class-weight"):
        scenario(Config(is_async=True, class_weight="balanced"), _data(10))


class _Ctx:
    """Stands in for NativeCtx: no arithmetic, records the name of every call."""

    def __init__(self):
        self.log = []

    def __getattr__(self, name):
        from distributed_sgd_b200.native import ClassEval

        def call(*args, **kw):
            self.log.append(name)
            if name.endswith("_class"):
                return ClassEval(0.5, 6.0, 8.0, 3, 4, 5, 15)     # L+ 6, L- 8; correct 3 + 4 of 5 + 15 rows
            return 14, 7, 0.5                                    # hinge sum, correct, ||w||^2
        return call


def _master(ctx, class_weight, n_train=20, n_test=5):
    from distributed_sgd_b200.core.master import MasterSync
    from distributed_sgd_b200.ml import SparseSVM
    slave = SimpleNamespace(ctx=ctx, world=1, is_async=False, n_train=n_train, n_test=n_test, dim=DIM,
                            **({} if class_weight is None else {"class_weight": class_weight}))
    return MasterSync(0, _data(n_train), _data(n_test), SparseSVM(0.1), 1, slave=slave, seed=0)


def test_an_unweighted_model_makes_no_new_context_call():
    for cw in (None, (1.0, 1.0)):
        ctx = _Ctx()
        m = _master(ctx, cw)
        assert m.local_loss() == 0.1 * 0.5 + 14 / 20
        m.local_loss_accuracy(test_data=True)
        m.local_sampled_loss(None, 10)
        m.distributed_loss(None)
        assert ctx.log == ["eval_counts", "eval_counts", "eval_sampled_counts", "eval_counts"]


def test_a_weighted_model_reports_the_weighted_loss_through_the_class_calls():
    ctx = _Ctx()
    m = _master(ctx, (4.0, 0.25))
    assert m.local_loss() == 0.1 * 0.5 + (4.0 * 6 + 0.25 * 8) / 20
    loss, acc = m.local_loss_accuracy(test_data=True)
    assert loss == 0.1 * 0.5 + 26.0 / 5 and acc == 7 / 5
    assert m.local_sampled_loss(None, 10) == 0.1 * 0.5 + 26.0 / 10
    assert m.distributed_loss(None) == 0.1 * 0.5 + 26.0 / 20
    assert ctx.log == ["eval_class", "eval_class", "eval_sampled_class", "eval_class"]


def test_class_report():
    ctx = _Ctx()
    r = _master(ctx, (4.0, 0.25)).local_class_report(test_data=True)
    assert ctx.log == ["eval_class"]
    assert (r["n_pos"], r["n_neg"], r["correct_pos"], r["correct_neg"]) == (5, 15, 3, 4)
    assert r["recall_pos"] == 3 / 5 and r["recall_neg"] == 4 / 15 and r["balanced_accuracy"] == (3 / 5 + 4 / 15) / 2
    assert r["loss"] == 0.1 * 0.5 + 14.0 / 20 and r["weighted_loss"] == 0.1 * 0.5 + 26.0 / 20
    r1 = _master(_Ctx(), None).local_sampled_class_report(None, 10)
    assert r1["class_weight"] == (1.0, 1.0) and r1["loss"] == r1["weighted_loss"]
