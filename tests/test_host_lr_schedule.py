"""The decaying learning rate on the host side, without a GPU: learning_rates, the `learning-rate-decay` and
`learning-rate-power` configuration keys, `scenario` refusing a decay in async mode, and the calls MasterSync.fit makes --
a stand-in context defined here records them."""
import math

import numpy as np
import pytest

DIM = 8


# ---- learning_rates -------------------------------------------------------------------------------------------------

def test_no_decay_is_the_constant_rate():
    from distributed_sgd_b200.ml.lr_schedule import learning_rates
    for lr0 in (0.5, 0.1, 1e-3):
        t = learning_rates(lr0, 0.0, 0.75, 17, 50)
        assert t.dtype == np.float64 and t.shape == (50,)
        assert np.all(t == lr0)


@pytest.mark.parametrize("power", [1.0, 0.75])
def test_values(power):
    from distributed_sgd_b200.ml.lr_schedule import learning_rates
    lr0, a = 0.5, 1e-2
    t = learning_rates(lr0, a, power, 0, 1000)
    assert t[0] == lr0
    for s in (1, 10, 99, 999):
        assert t[s] == pytest.approx(lr0 / (1 + a * s) ** power, rel=1e-15)
    if power == 1.0:
        assert t[100] == pytest.approx(lr0 / 2, rel=1e-15)           # 1 + a t = 2
    else:
        assert t[100] == pytest.approx(lr0 / 2 ** 0.75, rel=1e-15)
    assert np.all(np.diff(t) < 0)


def test_a_slice_equals_the_same_positions_of_a_longer_table():
    from distributed_sgd_b200.ml.lr_schedule import learning_rates
    full = learning_rates(0.5, 3e-4, 0.75, 0, 5000)
    for t0, n in ((0, 1), (1, 7), (2188, 2188), (4999, 1), (37, 0)):
        np.testing.assert_array_equal(learning_rates(0.5, 3e-4, 0.75, t0, n), full[t0:t0 + n])
        assert learning_rates(0.5, 3e-4, 0.75, t0, n).shape == (n,)
    assert learning_rates(0.5, 3e-4, 0.75, 42, 1)[0] == 0.5 / math.pow(1 + 3e-4 * 42, 0.75)


@pytest.mark.parametrize("decay,power", [(-1e-4, 1.0), (1e-4, 0.0), (1e-4, -1.0), (float("nan"), 1.0)])
def test_out_of_range_schedules_raise(decay, power):
    from distributed_sgd_b200.ml.lr_schedule import learning_rates
    with pytest.raises(ValueError):
        learning_rates(0.5, decay, power, 0, 3)


# ---- configuration -----------------------------------------------------------------------------------------------------

def test_config_keys_from_the_file_and_the_environment(tmp_path):
    from distributed_sgd_b200.utils.config import load_config
    cfg = load_config(env={})
    assert cfg.learning_rate_decay == 0.0 and cfg.learning_rate_power == 1.0           # the reference's constant rate
    cfg = load_config(env={"DSGD_LEARNING_RATE_DECAY": "1e-4", "DSGD_LEARNING_RATE_POWER": "0.75"})
    assert cfg.learning_rate_decay == 1e-4 and cfg.learning_rate_power == 0.75
    conf = tmp_path / "application.conf"
    conf.write_text("dsgd {\n  learning-rate-decay = 0.002\n  learning-rate-decay = ${?DSGD_LEARNING_RATE_DECAY}\n"
                    "  learning-rate-power = 0.5\n  learning-rate-power = ${?DSGD_LEARNING_RATE_POWER}\n}\n")
    cfg = load_config(str(conf), env={})
    assert cfg.learning_rate_decay == 0.002 and cfg.learning_rate_power == 0.5
    cfg = load_config(str(conf), env={"DSGD_LEARNING_RATE_DECAY": "0", "DSGD_LEARNING_RATE_POWER": "2"})
    assert cfg.learning_rate_decay == 0.0 and cfg.learning_rate_power == 2.0


@pytest.mark.parametrize("env,key", [({"DSGD_LEARNING_RATE_DECAY": "-1e-4"}, "learning-rate-decay"),
                                     ({"DSGD_LEARNING_RATE_POWER": "0"}, "learning-rate-power"),
                                     ({"DSGD_LEARNING_RATE_POWER": "-0.5"}, "learning-rate-power")])
def test_config_out_of_range_raises(env, key):
    from distributed_sgd_b200.utils.config import load_config
    with pytest.raises(ValueError, match=key):
        load_config(env=env)


def test_scenario_refuses_a_decay_with_async():
    from distributed_sgd_b200.main import scenario
    from distributed_sgd_b200.utils.config import Config
    with pytest.raises(ValueError, match="learning-rate-decay"):
        scenario(Config(is_async=True, learning_rate_decay=1e-4), data=None)   # refused before any data or device is touched


# ---- MasterSync.fit against a stand-in context ---------------------------------------------------------------------------

class _LrCtx:
    """Stands in for NativeCtx: no arithmetic.  Records every sync step call (scalar or table) and the averaging calls."""

    def __init__(self, dim, fail_at_call=None):
        self.dim, self.log, self.fail_at_call = dim, [], fail_at_call
        self.averaging, self.n_avg = False, 0

    def _maybe_fail(self):
        if self.fail_at_call is not None and sum(e[0] in ("steps", "steps_lr") for e in self.log) == self.fail_at_call:
            raise RuntimeError("device failure")

    def set_weights(self, w):
        self.log.append(("set_weights",))

    def get_weights(self):
        return np.full(self.dim, -1.0)

    def set_workers(self, counts, k_total):
        self.log.append(("set_workers", list(counts), k_total))

    def sync_steps(self, samples, n_per_step, n_steps, lr, want_losses=True):
        self._maybe_fail()
        self.log.append(("steps", n_steps, lr, n_per_step))
        self.n_avg += n_steps if self.averaging else 0
        return np.zeros(n_steps)

    def sync_steps_lr(self, samples, n_per_step, lrs, want_losses=True):
        self._maybe_fail()
        lrs = np.array(lrs, dtype=np.float64)
        assert np.asarray(samples).size == n_per_step * lrs.size
        self.log.append(("steps_lr", lrs, n_per_step))
        self.n_avg += lrs.size if self.averaging else 0
        return np.zeros(lrs.size)

    def eval_counts(self, lo, hi, w=None):
        return hi - lo, 0, 0.0

    def average_begin(self):
        self.log.append(("begin",))
        self.averaging, self.n_avg = True, 0

    def average_end(self):
        self.log.append(("end",))
        self.averaging = False

    def average_weights(self):
        return np.full(self.dim, float(self.n_avg)), self.n_avg


class _ScalarOnlyCtx(_LrCtx):
    """A context without sync_steps_lr, like the stand-ins of the older host tests."""

    def __getattribute__(self, name):
        if name == "sync_steps_lr":
            raise AttributeError(name)
        return object.__getattribute__(self, name)


def _master(ctx, n_train=20, n_test=5, world=1):
    from types import SimpleNamespace
    from distributed_sgd_b200.core.master import MasterSync
    from distributed_sgd_b200.ml import SparseSVM
    from distributed_sgd_b200.utils.dataset import Data
    stub = lambda n: Data(np.arange(n + 1, dtype=np.int64), np.zeros(n, np.int32), np.ones(n, np.float32),
                          np.ones(n, np.int8), DIM)
    slave = SimpleNamespace(ctx=ctx, world=world, is_async=False, n_train=n_train, n_test=n_test, dim=DIM)
    return MasterSync(0, stub(n_train), stub(n_test), SparseSVM(0.1), 1, slave=slave, seed=0)


def _fit(m, max_epochs=3, batch_size=5, decay=0.0, power=1.0, **kw):
    return m.fit(np.zeros(DIM), max_epochs=max_epochs, batch_size=batch_size, learning_rate=0.5,
                 stopping_criterion=lambda tl: False, learning_rate_decay=decay, learning_rate_power=power, **kw)


def test_no_decay_makes_only_scalar_calls():
    ctx = _ScalarOnlyCtx(DIM)
    _fit(_master(ctx), decay=0.0, power=0.75)
    steps = [e for e in ctx.log if e[0].startswith("steps")]
    assert steps and all(e[0] == "steps" and e[2] == 0.5 for e in steps)
    assert sum(e[1] for e in steps) == 12


def _tables(log):
    return [e[1] for e in log if e[0] == "steps_lr"]


@pytest.mark.parametrize("case", ["epochs", "short_last_batch", "virtual_workers", "average_from"])
def test_tables_concatenate_to_the_schedule_of_the_fit(case):
    from distributed_sgd_b200.ml.lr_schedule import learning_rates
    a, p = 0.05, 0.75
    kw, n_train, batch, per_epoch = {}, 20, 5, 4
    if case == "short_last_batch":
        n_train, batch, per_epoch = 23, 5, 5             # 4 full steps and one of 3: two calls per epoch
    elif case == "virtual_workers":
        n_train, batch, per_epoch = 23, 4, 3             # 2 groups (12, 11): steps of (4, 4) x 2, then (4, 3)
        kw["virtual_workers"] = 2
    elif case == "average_from":
        kw["average_from"] = 1
    ctx = _LrCtx(DIM)
    _fit(_master(ctx, n_train=n_train), max_epochs=3, batch_size=batch, decay=a, power=p, **kw)
    assert not any(e[0] == "steps" for e in ctx.log)
    tables = _tables(ctx.log)
    np.testing.assert_array_equal(np.concatenate(tables), learning_rates(0.5, a, p, 0, 3 * per_epoch))
    if case in ("short_last_batch", "virtual_workers"):
        assert len(tables) == 6                          # every epoch split where the counts change
    if case == "average_from":
        names = [e[0] for e in ctx.log]
        assert names.count("begin") == 1 and names[-1] == "end"
        assert sum(len(t) for t in _tables(ctx.log[names.index("begin"):])) == 2 * per_epoch


def test_a_failing_call_still_ends_averaging():
    ctx = _LrCtx(DIM, fail_at_call=2)                    # one call per epoch: epoch 2's fails
    with pytest.raises(RuntimeError, match="device failure"):
        _fit(_master(ctx), decay=1e-2, average_from=1)
    names = [e[0] for e in ctx.log]
    assert names.count("begin") == 1 and names[-1] == "end"


@pytest.mark.parametrize("decay,power", [(-1e-3, 1.0), (1e-3, 0.0), (1e-3, -2.0)])
def test_fit_refuses_out_of_range_schedules(decay, power):
    ctx = _LrCtx(DIM)
    with pytest.raises(ValueError, match="learning_rate_"):
        _fit(_master(ctx), decay=decay, power=power)
    assert ctx.log == []
