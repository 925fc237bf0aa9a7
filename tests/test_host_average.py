"""Averaged SGD on the host side, without a GPU: the `average-from` configuration key, `scenario` refusing it in async mode,
and what MasterSync.fit(average_from=e) asks of the device context -- a stand-in context defined here records the calls."""
import numpy as np
import pytest

DIM = 8


class _AvgCtx:
    """Stands in for NativeCtx: no arithmetic.  Records sync steps, evaluations (with the weights they were given) and the
    averaging calls in order; average_weights returns a vector that names the number of steps averaged."""

    def __init__(self, dim, fail_at_call=None):
        self.dim, self.log, self.fail_at_call = dim, [], fail_at_call
        self.averaging, self.n_avg, self.begun = False, 0, False
        self.last_avg = None

    def set_weights(self, w):
        self.log.append(("set_weights",))

    def get_weights(self):
        return np.full(self.dim, -1.0)                     # "the last weights"

    def set_workers(self, counts, k_total):
        pass

    def sync_steps(self, samples, n_per_step, n_steps, lr, want_losses=True):
        if self.fail_at_call is not None and sum(e[0] == "steps" for e in self.log) == self.fail_at_call:
            raise RuntimeError("device failure")
        self.log.append(("steps", n_steps))
        if self.averaging:
            self.n_avg += n_steps
        return np.zeros(n_steps)

    def eval_counts(self, lo, hi, w=None):
        self.log.append(("eval", None if w is None else np.array(w)))
        return hi - lo, 0, 0.0

    def average_begin(self):
        self.log.append(("begin",))
        self.averaging, self.n_avg, self.begun = True, 0, True

    def average_end(self):
        self.log.append(("end",))
        self.averaging = False

    def average_weights(self):
        assert self.begun
        self.log.append(("average_weights",))
        self.last_avg = np.full(self.dim, float(self.n_avg))
        return self.last_avg.copy(), self.n_avg


class _PlainCtx(_AvgCtx):
    """A context without the averaging calls (like the stand-ins of the older host tests): any use of them fails."""

    def __getattribute__(self, name):
        if name.startswith("average_"):
            raise AttributeError(name)
        return object.__getattribute__(self, name)


def _master(ctx, n_train=20, n_test=5):
    from types import SimpleNamespace
    from distributed_sgd_b200.core.master import MasterSync
    from distributed_sgd_b200.ml import SparseSVM
    from distributed_sgd_b200.utils.dataset import Data
    stub = lambda n: Data(np.arange(n + 1, dtype=np.int64), np.zeros(n, np.int32), np.ones(n, np.float32),
                          np.ones(n, np.int8), DIM)
    slave = SimpleNamespace(ctx=ctx, world=1, is_async=False, n_train=n_train, n_test=n_test, dim=DIM)
    return MasterSync(0, stub(n_train), stub(n_test), SparseSVM(0.1), 1, slave=slave, seed=0)


def _fit(m, max_epochs, average_from, stop_after=None):
    """batch 5 over 20 train rows: 4 steps per epoch.  stop_after: the stopping rule fires once that many epochs ran."""
    rule = (lambda tl: False) if stop_after is None else (lambda tl: len(tl) >= stop_after)
    return m.fit(np.zeros(DIM), max_epochs=max_epochs, batch_size=5, learning_rate=0.5, stopping_criterion=rule,
                 average_from=average_from)


def _epochs(log):
    """The log cut into epochs: [(calls before the epoch's first step, steps, evaluations)] -- an epoch ends with its two
    evaluations (train rows, test rows)."""
    out, pre, steps, evals = [], [], 0, []
    for e in log:
        if e[0] == "steps":
            steps += e[1]
        elif e[0] == "eval":
            evals.append(e[1])
            if len(evals) == 2:
                out.append((pre, steps, evals))
                pre, steps, evals = [], 0, []
        elif steps == 0 and not evals:
            pre.append(e[0])
    return out


# ---- configuration -----------------------------------------------------------------------------------------------

def test_config_key_environment_variable_and_default(tmp_path):
    from distributed_sgd_b200.utils.config import load_config
    assert load_config(env={}).average_from == -1                                   # default: off
    assert load_config(env={"DSGD_AVERAGE_FROM": "3"}).average_from == 3
    conf = tmp_path / "application.conf"
    conf.write_text("dsgd {\n  average-from = 2\n  average-from = ${?DSGD_AVERAGE_FROM}\n}\n")
    assert load_config(str(conf), env={}).average_from == 2
    assert load_config(str(conf), env={"DSGD_AVERAGE_FROM": "0"}).average_from == 0
    with pytest.raises(ValueError, match="average-from"):
        load_config(env={"DSGD_AVERAGE_FROM": "-2"})


def test_scenario_refuses_averaging_with_async():
    from distributed_sgd_b200.main import scenario
    from distributed_sgd_b200.utils.config import Config
    with pytest.raises(ValueError, match="average-from"):
        scenario(Config(is_async=True, average_from=1), data=None)       # refused before any data or device is touched


# ---- MasterSync.fit(average_from=...) against the stand-in context ---------------------------------------------------

@pytest.mark.parametrize("e", [0, 1, 2])
def test_begin_once_before_epoch_e_and_evaluations_use_the_average(e):
    ctx = _AvgCtx(DIM)
    m = _master(ctx)
    state = _fit(m, max_epochs=3, average_from=e)
    assert [c[0] for c in ctx.log].count("begin") == 1
    assert [c[0] for c in ctx.log].count("end") == 1 and ctx.log[-1] == ("end",)
    epochs = _epochs(ctx.log)
    assert len(epochs) == 3
    for k, (pre, steps, evals) in enumerate(epochs):
        assert steps == 4
        assert ("begin" in pre) == (k == e), (k, pre)                     # begin comes before the first step of epoch e
        if k < e:
            assert all(w is None for w in evals)                          # the resident (last) weights
        else:
            n = 4 * (k - e + 1)                                           # steps averaged by the end of epoch k
            for w in evals:                                               # the host vector average_weights returned
                np.testing.assert_array_equal(w, np.full(DIM, float(n)))
    assert m.history["averaged_steps"] == 4 * (3 - e)
    np.testing.assert_array_equal(state.grad, np.full(DIM, float(4 * (3 - e))))   # fit returns the average
    assert len(m.history["losses"]) == 3


def test_end_on_early_stop_after_begin():
    ctx = _AvgCtx(DIM)
    m = _master(ctx)
    state = _fit(m, max_epochs=5, average_from=1, stop_after=2)
    names = [c[0] for c in ctx.log]
    assert names.count("begin") == 1 and names.count("end") == 1 and names[-1] == "end"
    assert len(_epochs(ctx.log)) == 2
    assert m.history["averaged_steps"] == 4
    np.testing.assert_array_equal(state.grad, np.full(DIM, 4.0))


def test_early_stop_before_epoch_e_returns_the_last_weights():
    ctx = _AvgCtx(DIM)
    m = _master(ctx)
    state = _fit(m, max_epochs=5, average_from=3, stop_after=2)
    names = [c[0] for c in ctx.log]
    assert "begin" not in names and "end" not in names and "average_weights" not in names
    assert m.history["averaged_steps"] == 0
    np.testing.assert_array_equal(state.grad, np.full(DIM, -1.0))


def test_end_when_a_step_fails_while_averaging():
    ctx = _AvgCtx(DIM, fail_at_call=2)                   # one sync_steps call per epoch: epoch 2's fails
    m = _master(ctx)
    with pytest.raises(RuntimeError, match="device failure"):
        _fit(m, max_epochs=3, average_from=1)
    names = [c[0] for c in ctx.log]
    assert names.count("begin") == 1 and names[-1] == "end"


def test_no_averaging_call_without_average_from():
    ctx = _PlainCtx(DIM)
    m = _master(ctx)
    state = _fit(m, max_epochs=2, average_from=None)
    assert not any(c[0] in ("begin", "end", "average_weights") for c in ctx.log)
    assert "averaged_steps" not in m.history
    np.testing.assert_array_equal(state.grad, np.full(DIM, -1.0))
    assert all(w is None for _, _, evals in _epochs(ctx.log) for w in evals)


@pytest.mark.parametrize("e", [-1, 3, 7])
def test_average_from_outside_the_epochs_is_refused(e):
    ctx = _AvgCtx(DIM)
    m = _master(ctx)
    with pytest.raises(ValueError, match="average_from"):
        _fit(m, max_epochs=3, average_from=e)
    assert ctx.log == []
