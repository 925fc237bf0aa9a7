"""SparseSquaredHinge and SparseModifiedHuber on the host side, without a GPU: the `model` configuration values, the flag
constants against the header, dsgd_create's flag checks (made before it looks for a device), the refusals of asynchronous
training (Slave, Master.create, main.scenario) and the package exports."""
import os
import re

import numpy as np
import pytest

MODELS = {"squared_hinge": "SparseSquaredHinge", "modified_huber": "SparseModifiedHuber"}


@pytest.mark.parametrize("value", list(MODELS))
def test_model_key_values(value, tmp_path):
    from distributed_sgd_b200.utils import load_config
    assert load_config(env={"DSGD_MODEL": value}).model == value
    conf = tmp_path / "application.conf"
    conf.write_text(f"dsgd {{\n  model = {value}\n}}\n")
    assert load_config(str(conf), env={}).model == value


def test_hinge_stays_refused():
    from distributed_sgd_b200.utils import load_config
    with pytest.raises(ValueError, match="model"):
        load_config(env={"DSGD_MODEL": "hinge"})


def test_flag_constants_match_the_header():
    from distributed_sgd_b200 import native
    header = open(native.HEADER_PATH).read()
    flags = {name: int(v) for name, v in re.findall(r"#define DSGD_FLAG_(\w+) (\d+)u", header)}
    assert flags["SQUARED_HINGE"] == native.FLAG_SQUARED_HINGE == 4
    assert flags["MODIFIED_HUBER"] == native.FLAG_MODIFIED_HUBER == 8
    values = [native.FLAG_ASYNC, native.FLAG_LOGISTIC, native.FLAG_SQUARED_HINGE, native.FLAG_MODIFIED_HUBER]
    assert sum(values) == 15 and all(v & (v - 1) == 0 for v in values)   # four distinct bits
    assert native.MODEL_FLAGS == {"svm": 0, "logistic": 2, "squared_hinge": 4, "modified_huber": 8}


def _create(flags):
    import ctypes as C
    from distributed_sgd_b200 import native
    lib = native.lib()
    h = C.c_void_p()
    rc = lib.dsgd_create(C.byref(h), 0, 16, C.c_double(0.1), 0, 1, C.c_uint32(flags))
    return rc, (lib.dsgd_last_error(None) or b"").decode(), h


@pytest.mark.parametrize("flags", [2 | 4, 2 | 8, 4 | 8, 2 | 4 | 8])
def test_create_refuses_two_model_flags(flags):
    from distributed_sgd_b200 import native
    rc, msg, h = _create(flags)
    assert rc == native.ERR_INVALID and not h.value and "more than one model flag" in msg


@pytest.mark.parametrize("model", list(MODELS))
def test_create_refuses_a_model_flag_with_async(model):
    from distributed_sgd_b200 import native
    rc, msg, h = _create(native.MODEL_FLAGS[model] | native.FLAG_ASYNC)
    assert rc == native.ERR_INVALID and not h.value and msg == "dsgd_create: async mode supports the SVM model only"
    with pytest.raises(native.DsgdInvalid, match="SVM model only"):
        native.NativeCtx(0, 16, 0.1, is_async=True, model=model)


def test_native_ctx_refuses_an_unknown_model_before_the_library():
    from distributed_sgd_b200 import native
    with pytest.raises(ValueError, match="model"):
        native.NativeCtx(0, 16, 0.1, model="hinge")
    with pytest.raises(ValueError, match="model"):
        native.NativeCtx(0, 16, 0.1, logistic=True, model="squared_hinge")


def _stub(n, dim=8):
    from distributed_sgd_b200.utils.dataset import Data
    return Data(np.arange(n + 1, dtype=np.int64), np.zeros(n, np.int32), np.ones(n, np.float32), np.ones(n, np.int8), dim)


@pytest.mark.parametrize("name", list(MODELS.values()))
def test_slave_refuses_async_before_any_context(name):
    import distributed_sgd_b200 as pkg
    with pytest.raises(ValueError, match=f"{name}: .*SparseSVM only"):
        pkg.Slave(0, 0, _stub(10), getattr(pkg, name)(0.1), True)


@pytest.mark.parametrize("name", list(MODELS.values()))
def test_master_create_refuses_async(name):
    import distributed_sgd_b200 as pkg
    with pytest.raises(ValueError, match=f"{name}: .*SparseSVM only"):
        pkg.Master.create(0, _stub(10), _stub(4), getattr(pkg, name)(0.1), True, 1, slave=None)


@pytest.mark.parametrize("value", list(MODELS))
def test_scenario_refuses_async(value):
    from distributed_sgd_b200.main import scenario
    from distributed_sgd_b200.utils import load_config
    cfg = load_config(env={"DSGD_MODEL": value, "DSGD_ASYNC": "true"})
    with pytest.raises(ValueError, match=f"model = {value}: asynchronous"):
        scenario(cfg, _stub(10))


def test_package_exports_the_models():
    import distributed_sgd_b200 as pkg
    from distributed_sgd_b200 import ml
    from distributed_sgd_b200.ml.sparse_margin import model_name
    for name, cls_name in MODELS.items():
        cls = getattr(ml, cls_name)
        assert getattr(pkg, cls_name) is cls and cls_name in pkg.__all__
        m = cls(0.1, l1=0.5, class_weight="balanced")
        assert (m.lam, m.dim_sparsity, m.l1, m.class_weight) == (0.1, None, 0.5, "balanced")
        assert model_name(m) == name
    assert model_name(pkg.SparseSVM(0.1)) == "svm" and model_name(pkg.SparseLogistic(0.1)) == "logistic"


def test_local_loss_takes_the_float_sums_for_every_model_but_the_svm():
    """The choice between the integer *_counts and the float *_sums evaluations, made in Master.__init__."""
    import distributed_sgd_b200 as pkg
    from distributed_sgd_b200.core.master import Master

    class Ctx:
        def __init__(self):
            self.calls = []

        def eval_sums(self, *a):
            self.calls.append("sums")
            return 1.5, 1, 0.0

        def eval_counts(self, *a):
            self.calls.append("counts")
            return 1, 1, 0.0

    class Slave:
        world, n_train, n_test, is_async = 1, 10, 4, False

        def __init__(self):
            self.ctx = Ctx()

    for cls, call in ((pkg.SparseSVM, "counts"), (pkg.SparseLogistic, "sums"), (pkg.SparseSquaredHinge, "sums"),
                      (pkg.SparseModifiedHuber, "sums")):
        s = Slave()
        m = Master(0, _stub(10), _stub(4), cls(0.1), 1, slave=s, attach=False)
        m.local_loss()
        assert s.ctx.calls == [call]


def test_jni_facade_carries_the_flags():
    from distributed_sgd_b200 import native
    src = open(os.path.join(os.path.dirname(native.__file__), "jni", "DsgdNative.scala")).read()
    assert "final val FlagSquaredHinge = 4" in src and "final val FlagModifiedHuber = 8" in src
