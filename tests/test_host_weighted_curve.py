"""Weighted curves on the host side, without a GPU: weighted_curve_dict's formulas on the weighted words, the AUC and AP
rules of NativeCtx's result, and which calls Master.local_weighted_curve and local_sampled_weighted_curve make -- a
stand-in context defined here records them."""
import math
from types import SimpleNamespace

import numpy as np

DIM = 8
# TP 3, FN 1, pos none 0.5, FP 1, TN 4, neg none 0, U2w 28, NaN 0, S_ap 3.5, correct 7, total 9.5, W+ 4.5, W- 5
WSUMS = np.array([3.0, 1.0, 0.5, 1.0, 4.0, 0.0, 28.0, 0.0, 3.5, 7.0, 9.5, 4.5, 5.0])
WORDS = np.array([3, 1, 1, 1, 4, 0, 30, 0], dtype=np.int64)


def _result(curve=True, words=WORDS, wsums=WSUMS):
    from distributed_sgd_b200.native import WeightedCurve, weighted_auc_ap
    pts = (np.array([1.0, 0.0]), np.array([3.0, 4.5]), np.array([1.0, 5.0])) if curve else (np.zeros(0),) * 3
    return WeightedCurve(words, wsums, 2, *pts, *weighted_auc_ap(words, wsums))


def test_auc_and_ap_rules():
    from distributed_sgd_b200.native import weighted_auc_ap
    assert weighted_auc_ap(WORDS, WSUMS) == (28.0 / (2.0 * 4.5 * 5.0), 3.5 / 4.5)
    no_neg = WSUMS.copy()
    no_neg[12] = 0.0
    auc, ap = weighted_auc_ap(WORDS, no_neg)
    assert math.isnan(auc) and ap == 1.0
    no_pos = WSUMS.copy()
    no_pos[11] = 0.0
    assert all(math.isnan(x) for x in weighted_auc_ap(WORDS, no_pos))
    nan_row = WORDS.copy()
    nan_row[7] = 1
    assert all(math.isnan(x) for x in weighted_auc_ap(nan_row, WSUMS))


def test_weighted_curve_dict():
    from distributed_sgd_b200.core.master import weighted_curve_dict
    d = weighted_curve_dict(_result())
    assert (d["tp"], d["fn"], d["pos_no_pred"], d["fp"], d["tn"], d["neg_no_pred"]) == (3.0, 1.0, 0.5, 1.0, 4.0, 0.0)
    assert d["precision"] == 3.0 / 4.0 and d["recall"] == 3.0 / 4.5 and d["f1"] == 6.0 / (6.0 + 1.0 + 1.0 + 0.5)
    assert d["auc"] == 28.0 / 45.0 and d["average_precision"] == 3.5 / 4.5 and d["accuracy"] == 7.0 / 9.5
    assert d["weight_sum"] == 9.5 and d["n_points"] == 2 and d["nan_scores"] == 0 and d["nan_weight"] == 0.0
    c = d["curve"]
    assert c["thresholds"] == [1.0, 0.0] and c["tp_weight"] == [3.0, 4.5] and c["fp_weight"] == [1.0, 5.0]
    assert c["precision"] == [0.75, 4.5 / 9.5] and c["recall"] == [3.0 / 4.5, 1.0] and c["fpr"] == [0.2, 1.0]
    assert "curve" not in weighted_curve_dict(_result(False), curve=False)
    empty = weighted_curve_dict(_result(words=np.zeros(8, np.int64), wsums=np.zeros(13)))
    assert math.isnan(empty["precision"]) and math.isnan(empty["accuracy"]) and math.isnan(empty["auc"])


class _Ctx:
    """Stands in for NativeCtx: no arithmetic, records every call and its curve flag."""

    def __init__(self):
        self.log = []

    def __getattr__(self, name):
        def call(*args, curve=True, **kw):
            self.log.append((name, curve))
            return _result(curve)
        return call


def test_master_calls():
    from distributed_sgd_b200.core.master import MasterSync
    from distributed_sgd_b200.ml import SparseSVM
    from distributed_sgd_b200.utils.dataset import Data
    d = Data(np.arange(21, dtype=np.int64), np.zeros(20, np.int32), np.ones(20, np.float32), np.ones(20, np.int8), DIM)
    ctx = _Ctx()
    slave = SimpleNamespace(ctx=ctx, world=1, is_async=False, n_train=20, n_test=20, dim=DIM, class_weight=(2.0, 0.5),
                            sample_weighted=True)
    m = MasterSync(0, d, d, SparseSVM(0.1), 1, slave=slave, seed=0)
    assert "curve" in m.local_weighted_curve(test_data=True)
    assert "curve" not in m.local_sampled_weighted_curve(None, 10, curve=False)
    assert ctx.log == [("eval_weighted_curve", True), ("eval_sampled_weighted_curve", False)]
