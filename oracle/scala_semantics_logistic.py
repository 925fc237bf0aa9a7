"""TEST INFRASTRUCTURE ONLY -- literal, map-based restatement of SparseLogistic, the logistic-loss model beside SparseSVM,
in the style of oracle/scala_semantics.py (whose Sparse vectors, folds and filters it uses unchanged).

For one sample z = y * (x . w), the activity of SparseSVM.scala:27: forward and regularize are the SVM's; the per-sample
loss is softplus(z) and backward is x * (y * sigmoid(z)), a new Sparse (products with |.| <= 1e-20 dropped).  Both in their
stable forms.  slave_gradient, master_sync_step, local_loss and local_accuracy of scala_semantics take this model as they
take SparseSVM.  Nothing under distributed_sgd_b200/ may import this module.
"""
from __future__ import annotations

import math

from .scala_semantics import Sparse, SparseSVM


def softplus(z: float) -> float:
    return (z if z > 0.0 else 0.0) + math.log1p(math.exp(-abs(z)))


def sigmoid(t: float) -> float:
    if t >= 0.0:
        return 1.0 / (1.0 + math.exp(-t))
    e = math.exp(t)
    return e / (1.0 + e)


class SparseLogistic(SparseSVM):
    def loss_sample(self, w: Sparse, x: Sparse, y: int) -> float:
        return softplus(y * x.dot(w))

    def backward(self, w: Sparse, x: Sparse, y: int) -> Sparse:
        return x * (y * sigmoid(y * x.dot(w)))
