"""TEST INFRASTRUCTURE ONLY -- the SparseLogistic checker with the interface of oracle/oracle.py's Oracle.

LogisticOracle is the Oracle with the model-dependent calls (loss_acc, sample_losses, gradient, sync_steps) answered by the
checker of every model, oracle/margin.py, as model 1; forward and dimSparsity do not depend on the model and stay the SVM
oracle's.  Only tests/ and tools/ use it; the product package never does.
"""
from __future__ import annotations

from typing import Optional, Sequence

import numpy as np

from . import margin as M
from .oracle import Oracle


class LogisticOracle(Oracle):
    """CPU oracle of SparseLogistic over one CSR data set (the same constructor as Oracle)."""

    def loss_acc(self, w, idx=None, begin: int = 0, n: Optional[int] = None):
        return M.loss_acc(self, "logistic", w, idx, begin, n)[:2]

    def sample_losses(self, w, idx=None, begin: int = 0, n: Optional[int] = None) -> np.ndarray:
        """Per-sample losses softplus(z_i) (without lambda * ||w||^2) of the listed rows, or of rows [begin, begin + n)."""
        return M.sample_losses(self, "logistic", w, idx, begin, n)

    def gradient(self, w, idx):
        """(the regularized gradient sum, c = 2 lambda (w . d))"""
        g, _, _, c = M._gradient(self, "logistic", w, idx)
        return g, c

    def sync_steps(self, w, idx, counts: Sequence[int], lr: float, n_steps: int = 1, threads: int = 1):
        """Runs n_steps sync steps on a copy of w; returns (w_new, losses[n_steps]).  (Serial: `threads` is ignored.)"""
        return M.sync_steps(self, "logistic", w, idx, counts, np.full(n_steps, float(lr)))
