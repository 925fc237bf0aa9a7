"""SparseSquaredHinge and SparseModifiedHuber -- the two standard margin losses on the same sparse rows, further choices
beside SparseSVM and SparseLogistic at the place where the reference builds its model (Main.scala:67-68).

For one sample z = y * (x . w), the activity of SparseSVM.scala:27, and t = 1 + z.  The prediction is the SVM's,
-signum(x . w), so the classifier's margin is -z and both losses vanish for z <= -1.  backward is x * (y * s):
  SparseSquaredHinge   loss t^2 above z = -1 (the L2-loss SVM, liblinear's default), s = 2 t
  SparseModifiedHuber  loss t^2 on (-1, 1] and 4 z above (scikit-learn's `modified_huber`), s = 2 t and 4;
                       P(y = +1 | x) = (clip(-x . w, -1, 1) + 1) / 2
regularize and the sync step are the SVM's.  Like SparseSVM these are parameter holders: the arithmetic exists only as CUDA
kernels in libdsgd.so.  Sync mode only: asynchronous (Hogwild) training supports SparseSVM.
"""
from __future__ import annotations

from dataclasses import dataclass
from typing import Optional

import numpy as np


@dataclass
class SparseSquaredHinge:
    lam: float                                  # `lambda`
    dim_sparsity: Optional[np.ndarray] = None   # None: computed on the device from the train rows (Main.scala:54-65)
    l1: float = 0.0                             # extension: L1 penalty l1 * ||w||_1, a proximal step in every sync step
    # extension: one weight per label on backward and loss in sync training: None, (w_pos, w_neg) or "balanced"
    class_weight: object = None
    # extension: an unregularised intercept (sync mode): weight vectors are dim + 1 long, the intercept last
    fit_intercept: bool = False


@dataclass
class SparseModifiedHuber:
    lam: float                                  # `lambda`
    dim_sparsity: Optional[np.ndarray] = None   # None: computed on the device from the train rows (Main.scala:54-65)
    l1: float = 0.0                             # extension: L1 penalty l1 * ||w||_1, a proximal step in every sync step
    # extension: one weight per label on backward and loss in sync training: None, (w_pos, w_neg) or "balanced"
    class_weight: object = None
    # extension: an unregularised intercept (sync mode): weight vectors are dim + 1 long, the intercept last
    fit_intercept: bool = False


def model_name(model) -> str:
    """The NativeCtx / configuration name of a model object: "svm", "logistic", "squared_hinge" or "modified_huber"."""
    from .sparse_logistic import SparseLogistic
    return {SparseLogistic: "logistic", SparseSquaredHinge: "squared_hinge",
            SparseModifiedHuber: "modified_huber"}.get(type(model), "svm")
