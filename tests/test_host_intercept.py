"""The intercept (fit_intercept, DSGD_FLAG_INTERCEPT) on the host side, without a GPU: the flag constant against the header,
dsgd_create's refusal of an intercept in async mode (made before it looks for a device), the refusals of asynchronous
training and of the gRPC service, the `fit-intercept` configuration key, and the dim + 1 length checks of NativeCtx and
MasterSync.fit."""
import ctypes as C
import re
from types import SimpleNamespace

import numpy as np
import pytest

DIM = 8


def test_flag_constant_matches_the_header_and_is_a_new_bit():
    from distributed_sgd_b200 import native
    header = open(native.HEADER_PATH).read()
    flags = {name: int(v) for name, v in re.findall(r"#define DSGD_FLAG_(\w+) (\d+)u", header)}
    assert flags["INTERCEPT"] == native.FLAG_INTERCEPT == 16
    others = [native.FLAG_ASYNC, native.FLAG_LOGISTIC, native.FLAG_SQUARED_HINGE, native.FLAG_MODIFIED_HUBER]
    assert all(native.FLAG_INTERCEPT & v == 0 for v in others)
    assert 16 not in native.MODEL_FLAGS.values()


@pytest.mark.parametrize("model", ["svm", "logistic", "squared_hinge", "modified_huber"])
def test_create_refuses_an_intercept_with_async(model):
    from distributed_sgd_b200 import native
    lib = native.lib()
    h = C.c_void_p()
    flags = native.MODEL_FLAGS[model] | native.FLAG_INTERCEPT | native.FLAG_ASYNC
    rc = lib.dsgd_create(C.byref(h), 0, 16, C.c_double(0.1), 0, 1, C.c_uint32(flags))
    msg = (lib.dsgd_last_error(None) or b"").decode()
    assert rc == native.ERR_INVALID and not h.value
    if model == "svm":
        assert "async mode has no intercept" in msg
    with pytest.raises(native.DsgdInvalid):
        native.NativeCtx(0, 16, 0.1, is_async=True, model=model, intercept=True)


def test_models_take_fit_intercept_as_a_trailing_field():
    from distributed_sgd_b200.ml import SparseLogistic, SparseSVM
    from distributed_sgd_b200.ml.sparse_margin import SparseModifiedHuber, SparseSquaredHinge
    for M in (SparseSVM, SparseLogistic, SparseSquaredHinge, SparseModifiedHuber):
        m = M(0.1, None, 0.5, "balanced")                   # positional construction as before
        assert m.fit_intercept is False and m.class_weight == "balanced"
        assert M(0.1, fit_intercept=True).fit_intercept is True


def test_config_key_environment_variable_and_default(tmp_path):
    from distributed_sgd_b200.utils.config import load_config
    assert load_config(env={}).fit_intercept is False
    assert load_config(env={"DSGD_FIT_INTERCEPT": "true"}).fit_intercept is True
    conf = tmp_path / "application.conf"
    conf.write_text("dsgd {\n  fit-intercept = true\n  fit-intercept = ${?DSGD_FIT_INTERCEPT}\n}\n")
    assert load_config(str(conf), env={}).fit_intercept is True
    assert load_config(str(conf), env={"DSGD_FIT_INTERCEPT": "false"}).fit_intercept is False
    with pytest.raises(ValueError, match="boolean"):
        load_config(env={"DSGD_FIT_INTERCEPT": "maybe"})


def _data(n):
    from distributed_sgd_b200.utils.dataset import Data
    return Data(np.arange(n + 1, dtype=np.int64), np.zeros(n, np.int32), np.ones(n, np.float32),
                np.ones(n, np.int8), DIM)


def test_async_training_refuses_an_intercept():
    from distributed_sgd_b200.core.master import Master, MasterAsync
    from distributed_sgd_b200.core.slave import Slave
    from distributed_sgd_b200.main import scenario
    from distributed_sgd_b200.ml import SparseSVM
    from distributed_sgd_b200.utils.config import Config
    with pytest.raises(ValueError, match="fit_intercept"):
        Slave(0, 0, _data(4), SparseSVM(0.1, fit_intercept=True), True)
    slave = SimpleNamespace(ctx=None, world=1, is_async=True, n_train=4, n_test=2, dim=DIM)
    with pytest.raises(ValueError, match="fit_intercept"):
        MasterAsync(0, _data(4), _data(2), SparseSVM(0.1, fit_intercept=True), 1, slave=slave)
    with pytest.raises(ValueError, match="fit_intercept"):
        Master.create(0, _data(4), _data(2), SparseSVM(0.1, fit_intercept=True), True, 1, slave=slave)
    with pytest.raises(ValueError, match="fit-intercept"):
        scenario(Config(is_async=True, fit_intercept=True), _data(10))


def test_the_grpc_slave_service_refuses_an_intercept_context():
    from distributed_sgd_b200.core.wire import SlaveServicer
    with pytest.raises(ValueError, match="intercept"):
        SlaveServicer(SimpleNamespace(dim=DIM, intercept=True), 4, False)


def _bare_ctx(intercept):
    """A NativeCtx without a device context: only the host-side length checks run before the library is called."""
    from distributed_sgd_b200.native import NativeCtx
    ctx = NativeCtx.__new__(NativeCtx)
    ctx._l, ctx._h = None, None
    ctx.dim, ctx.intercept, ctx.wdim = DIM, intercept, DIM + (1 if intercept else 0)
    return ctx


def test_native_ctx_checks_every_weight_vector_against_dim_plus_one():
    from distributed_sgd_b200.native import DsgdInvalid
    ctx = _bare_ctx(True)
    for call in (lambda w: ctx.set_weights(w), lambda w: ctx.gradient([0], w), lambda w: ctx.forward([0], w),
                 lambda w: ctx.margins([0], w), lambda w: ctx.eval_sums(0, 1, w)):
        with pytest.raises(DsgdInvalid, match=f"expected {DIM + 1} elements, got {DIM}"):
            call(np.zeros(DIM))
    plain = _bare_ctx(False)
    with pytest.raises(DsgdInvalid, match=f"expected {DIM} elements, got {DIM + 1}"):
        plain.set_weights(np.zeros(DIM + 1))


def test_master_fit_refuses_initial_weights_of_the_wrong_length():
    from distributed_sgd_b200.core.master import MasterSync
    from distributed_sgd_b200.ml import SparseSVM
    from distributed_sgd_b200.ml.early_stopping import no_improvement
    for intercept, bad in ((True, DIM), (False, DIM + 1)):
        slave = SimpleNamespace(ctx=None, world=1, is_async=False, n_train=4, n_test=2, dim=DIM, intercept=intercept)
        m = MasterSync(0, _data(4), _data(2), SparseSVM(0.1, fit_intercept=intercept), 1, slave=slave, seed=0)
        assert m.wdim == DIM + intercept
        with pytest.raises(ValueError, match=f"expected {DIM + intercept} values"):
            m.fit(np.zeros(bad), 1, 2, 0.1, no_improvement(patience=1, min_delta=0.0))
