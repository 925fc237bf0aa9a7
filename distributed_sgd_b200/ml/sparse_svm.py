"""core/ml/SparseSVM.scala -- the model injected into Master and Slave (Main.scala:68).

Here it is a parameter holder: lambda and the dimSparsity vector (dense, weight index space).  Its
arithmetic -- forward / loss / backward / regularize (SparseSVM.scala:14-31) -- exists only as CUDA
kernels inside libdsgd.so; a Slave installs these parameters into its device context.
"""
from __future__ import annotations

from dataclasses import dataclass
from typing import Optional

import numpy as np


@dataclass
class SparseSVM:
    lam: float                                  # `lambda`
    dim_sparsity: Optional[np.ndarray] = None   # None: computed on the device from the train rows (Main.scala:54-65)
    l1: float = 0.0                             # extension: L1 penalty l1 * ||w||_1, a proximal step in every sync step
    # extension: one weight per label on backward and loss in sync training: None, (w_pos, w_neg) or "balanced"
    class_weight: object = None
    # extension: an unregularised intercept (sync mode): weight vectors are dim + 1 long, the intercept last
    fit_intercept: bool = False
