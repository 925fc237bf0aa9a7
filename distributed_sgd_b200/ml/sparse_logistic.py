"""SparseLogistic -- a logistic-loss linear model on the same sparse rows, a second choice beside SparseSVM at the place
where the reference builds its model (Main.scala:67-68).

For one sample z = y * (x . w), the activity of SparseSVM.scala:27.  forward is the SVM's, -signum(x . w); the per-sample
loss is softplus(z) = log(1 + e^z); backward is x * (y * sigmoid(z)); regularize and the sync step are the SVM's.  As z
grows the gradient tends to the SVM's active branch y * x, as z falls to its gated branch 0, so the same sign conventions and
learning rate train it.  Like SparseSVM this is a parameter holder: the arithmetic exists only as CUDA kernels in libdsgd.so.
Sync mode only: asynchronous (Hogwild) training supports SparseSVM.
"""
from __future__ import annotations

from dataclasses import dataclass
from typing import Optional

import numpy as np


@dataclass
class SparseLogistic:
    lam: float                                  # `lambda`
    dim_sparsity: Optional[np.ndarray] = None   # None: computed on the device from the train rows (Main.scala:54-65)
    l1: float = 0.0                             # extension: L1 penalty l1 * ||w||_1, a proximal step in every sync step
    # extension: one weight per label on backward and loss in sync training: None, (w_pos, w_neg) or "balanced"
    class_weight: object = None
    # extension: an unregularised intercept (sync mode): weight vectors are dim + 1 long, the intercept last
    fit_intercept: bool = False
