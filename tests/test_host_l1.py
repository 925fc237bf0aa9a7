"""The L1 penalty on the host side, without a GPU: the `l1` configuration key, the refusals of asynchronous training with
l1 > 0 (scenario, Slave, MasterAsync), and what Master asks of the device context with l1 = 0 and with l1 > 0 -- a stand-in
context defined here records the calls."""
import numpy as np
import pytest

DIM = 8
L1_NORM, NNZ = 3.0, 5


class _Ctx:
    """Stands in for NativeCtx: no arithmetic.  Records sync steps, evaluations and weights_l1 calls (with their weights)."""

    def __init__(self, dim):
        self.dim, self.log = dim, []

    def set_weights(self, w):
        self.log.append(("set_weights",))

    def get_weights(self):
        return np.full(self.dim, -1.0)

    def set_workers(self, counts, k_total):
        pass

    def sync_steps(self, samples, n_per_step, n_steps, lr, want_losses=True):
        self.log.append(("steps", n_steps))
        return np.zeros(n_steps)

    def eval_counts(self, lo, hi, w=None):
        self.log.append(("eval", None if w is None else np.array(w)))
        return hi - lo, 0, 0.5                              # hinge sum = rows, ||w||^2 = 0.5

    def eval_sampled_counts(self, b, e, key, lo, hi, w=None):
        self.log.append(("eval_sampled", None if w is None else np.array(w)))
        return hi - lo, 0, 0.5

    def weights_l1(self, w=None):
        self.log.append(("weights_l1", None if w is None else np.array(w)))
        return L1_NORM, NNZ


def _master(ctx, l1, n_train=20, n_test=5):
    from types import SimpleNamespace
    from distributed_sgd_b200.core.master import MasterSync
    from distributed_sgd_b200.ml import SparseSVM
    from distributed_sgd_b200.utils.dataset import Data
    stub = lambda n: Data(np.arange(n + 1, dtype=np.int64), np.zeros(n, np.int32), np.ones(n, np.float32),
                          np.ones(n, np.int8), DIM)
    slave = SimpleNamespace(ctx=ctx, world=1, is_async=False, n_train=n_train, n_test=n_test, dim=DIM)
    return MasterSync(0, stub(n_train), stub(n_test), SparseSVM(0.1, None, l1), 1, slave=slave, seed=0)


# ---- configuration -----------------------------------------------------------------------------------------------

def test_config_key_environment_variable_and_default(tmp_path):
    from distributed_sgd_b200.utils.config import load_config
    assert load_config(env={}).l1 == 0.0
    assert load_config(env={"DSGD_L1": "1e-4"}).l1 == 1e-4
    conf = tmp_path / "application.conf"
    conf.write_text("dsgd {\n  l1 = 0.002\n  l1 = ${?DSGD_L1}\n}\n")
    assert load_config(str(conf), env={}).l1 == 0.002
    assert load_config(str(conf), env={"DSGD_L1": "0"}).l1 == 0.0
    for bad in ("-1e-6", "inf", "nan"):
        with pytest.raises(ValueError, match="l1"):
            load_config(env={"DSGD_L1": bad})


def test_models_take_l1_as_a_trailing_field():
    from distributed_sgd_b200.ml import SparseLogistic, SparseSVM
    for M in (SparseSVM, SparseLogistic):
        assert M(0.1).l1 == 0.0
        d = np.ones(3)
        m = M(0.1, d)                                        # positional construction as before
        assert m.lam == 0.1 and m.dim_sparsity is d and m.l1 == 0.0
        assert M(0.1, None, 1e-3).l1 == 1e-3


def test_scenario_refuses_l1_with_async():
    from distributed_sgd_b200.main import scenario
    from distributed_sgd_b200.utils.config import Config
    with pytest.raises(ValueError, match="l1"):
        scenario(Config(is_async=True, l1=1e-4), data=None)     # refused before any data or device is touched


def test_slave_and_master_async_refuse_l1():
    from types import SimpleNamespace
    from distributed_sgd_b200.core.master import MasterAsync
    from distributed_sgd_b200.core.slave import Slave
    from distributed_sgd_b200.ml import SparseSVM
    data = SimpleNamespace(n_rows=4, dim=DIM)
    with pytest.raises(ValueError, match="l1"):
        Slave(0, 0, data, SparseSVM(0.1, None, 1e-3), is_async=True)
    with pytest.raises(ValueError, match="l1"):
        MasterAsync(0, data, data, SparseSVM(0.1, None, 1e-3), 1, slave=None)


# ---- the calls Master makes --------------------------------------------------------------------------------------

def _fit(m, max_epochs=2):
    return m.fit(np.zeros(DIM), max_epochs=max_epochs, batch_size=5, learning_rate=0.5, stopping_criterion=lambda tl: False)


def test_l1_zero_makes_no_new_call():
    ctx = _Ctx(DIM)
    m = _master(ctx, 0.0)
    _fit(m)
    assert not any(c[0] == "weights_l1" for c in ctx.log)
    assert "nnz" not in m.history
    assert m.local_loss(None) == 0.1 * 0.5 + 1.0
    assert m.local_sampled_loss(None, 10) == 0.1 * 0.5 + 1.0
    assert not any(c[0] == "weights_l1" for c in ctx.log)


def test_l1_adds_the_penalty_and_records_nnz():
    ctx = _Ctx(DIM)
    m = _master(ctx, 0.25)
    _fit(m, max_epochs=3)
    names = [c[0] for c in ctx.log]
    # every epoch: its steps, two evaluations each with its ||w||_1, and the nnz of the evaluated (resident) weights
    assert names.count("weights_l1") == 3 * 3
    assert m.history["nnz"] == [NNZ] * 3
    assert m.history["losses"] == [0.1 * 0.5 + 0.25 * L1_NORM + 1.0] * 3
    ctx.log.clear()
    w = np.arange(DIM, dtype=np.float64)
    assert m.local_loss(w, test_data=True) == 0.1 * 0.5 + 0.25 * L1_NORM + 1.0
    np.testing.assert_array_equal(ctx.log[-1][1], w)          # the penalty of the weights that were evaluated
    assert ctx.log[-1][0] == "weights_l1"
    assert m.local_sampled_loss(w, 10) == 0.1 * 0.5 + 0.25 * L1_NORM + 1.0
    assert ctx.log[-1][0] == "weights_l1"
    assert m.distributed_loss(w) == 0.1 * 0.5 + 0.25 * L1_NORM + 1.0


def test_accuracy_queries_make_no_l1_pass():
    ctx = _Ctx(DIM)
    m = _master(ctx, 0.25)
    w = np.arange(DIM, dtype=np.float64)
    assert m.local_accuracy(w) == 0.0
    assert m.local_sampled_accuracy(w, 10) == 0.0
    assert m.distributed_accuracy(w) == 0.0
    assert not any(c[0] == "weights_l1" for c in ctx.log)
