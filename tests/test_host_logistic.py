"""SparseLogistic on the host side, without a GPU: the `model` / DSGD_MODEL configuration key, the refusal of asynchronous
training with SparseLogistic (Slave, Master.create, main.scenario, dsgd_create), and the flag constant of the binding."""
import re

import numpy as np
import pytest


def test_model_key_defaults_to_svm():
    from distributed_sgd_b200.utils import load_config
    assert load_config(env={}).model == "svm"


def test_model_key_from_environment_and_file(tmp_path):
    from distributed_sgd_b200.utils import load_config
    assert load_config(env={"DSGD_MODEL": "logistic"}).model == "logistic"
    conf = tmp_path / "application.conf"
    conf.write_text("dsgd {\n  model = logistic\n  model = ${?DSGD_MODEL}\n}\n")
    assert load_config(str(conf), env={}).model == "logistic"
    assert load_config(str(conf), env={"DSGD_MODEL": "svm"}).model == "svm"


def test_bad_model_value_is_refused():
    from distributed_sgd_b200.utils import load_config
    with pytest.raises(ValueError, match="model"):
        load_config(env={"DSGD_MODEL": "hinge"})


def test_package_exports_the_model():
    import distributed_sgd_b200 as pkg
    from distributed_sgd_b200.ml import SparseLogistic
    assert pkg.SparseLogistic is SparseLogistic and "SparseLogistic" in pkg.__all__
    m = SparseLogistic(0.1)
    assert m.lam == 0.1 and m.dim_sparsity is None


def _stub(n, dim=8):
    from distributed_sgd_b200.utils.dataset import Data
    return Data(np.arange(n + 1, dtype=np.int64), np.zeros(n, np.int32), np.ones(n, np.float32), np.ones(n, np.int8), dim)


def test_slave_refuses_async_logistic_before_any_context():
    from distributed_sgd_b200 import Slave, SparseLogistic
    with pytest.raises(ValueError, match="SparseSVM only"):
        Slave(0, 0, _stub(10), SparseLogistic(0.1), True)


def test_master_create_refuses_async_logistic():
    from distributed_sgd_b200 import Master, SparseLogistic
    with pytest.raises(ValueError, match="SparseSVM only"):
        Master.create(0, _stub(10), _stub(4), SparseLogistic(0.1), True, 1, slave=None)


def test_scenario_refuses_logistic_with_async():
    from distributed_sgd_b200.main import scenario
    from distributed_sgd_b200.utils import load_config
    cfg = load_config(env={"DSGD_MODEL": "logistic", "DSGD_ASYNC": "true"})
    with pytest.raises(ValueError, match="logistic"):
        scenario(cfg, _stub(10))


def test_flag_constant_matches_the_header():
    import os
    from distributed_sgd_b200 import native
    header = open(os.path.join(os.path.dirname(native.HEADER_PATH), "dsgd.h")).read()
    assert int(re.search(r"#define DSGD_FLAG_LOGISTIC (\d+)u", header).group(1)) == native.FLAG_LOGISTIC == 2
    assert native.FLAG_LOGISTIC & native.FLAG_ASYNC == 0


def test_create_refuses_logistic_with_async():
    """dsgd_create checks its flags before it looks for a device: the refusal is the same with or without a GPU."""
    from distributed_sgd_b200 import native
    with pytest.raises(native.DsgdInvalid, match="SVM model only"):
        native.NativeCtx(0, 16, 0.1, is_async=True, logistic=True)
