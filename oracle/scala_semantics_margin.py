"""TEST INFRASTRUCTURE ONLY -- literal, map-based restatement of the margin models SparseSquaredHinge and
SparseModifiedHuber, in the style of oracle/scala_semantics_logistic.py (the Sparse vectors, folds and filters of
oracle/scala_semantics.py, unchanged).

For one sample z = y * (x . w), the activity of SparseSVM.scala:27, and t = 1 + z: forward and regularize are the SVM's;
  SparseSquaredHinge   loss 0 for z <= -1, else t * t;  backward x * (y * s), s = 0 for z <= -1, else 2 * t
  SparseModifiedHuber  loss 0, t * t on (-1, 1], 4 * z above;  s = 0, 2 * t, 4
(a zero scale is the SVM's gated branch: w.zeros_like()).  A weighted backward is x * ((y * s) * c).  slave_gradient,
master_sync_step and local_loss of scala_semantics take these models as they take SparseSVM; literal_sync_steps below adds
the weightings, the L1 step and the averaging sum.  Nothing under distributed_sgd_b200/ may import this module.
"""
from __future__ import annotations

from typing import Optional, Sequence

from .scala_semantics import Sparse, SparseSVM, signum, vec_sum
from .sw import literal_fixed_sum


class SparseSquaredHinge(SparseSVM):
    @staticmethod
    def loss_z(z: float) -> float:
        t = 1.0 + z
        return 0.0 if z <= -1.0 else t * t

    @staticmethod
    def scale_z(z: float) -> float:
        return 0.0 if z <= -1.0 else 2.0 * (1.0 + z)

    def loss_sample(self, w: Sparse, x: Sparse, y: int) -> float:
        return self.loss_z(y * x.dot(w))

    def backward(self, w: Sparse, x: Sparse, y: int, c: Optional[float] = None) -> Sparse:
        s = self.scale_z(y * x.dot(w))
        if s == 0.0:
            return w.zeros_like()
        return x * (y * s) if c is None else x * ((y * s) * c)


class SparseModifiedHuber(SparseSquaredHinge):
    @staticmethod
    def loss_z(z: float) -> float:
        t = 1.0 + z
        return 0.0 if z <= -1.0 else (t * t if z <= 1.0 else 4.0 * z)

    @staticmethod
    def scale_z(z: float) -> float:
        return 0.0 if z <= -1.0 else (2.0 * (1.0 + z) if z <= 1.0 else 4.0)

    def probability(self, w: Sparse, x: Sparse) -> float:
        """P(y = +1 | x) = (clip(-x . w, -1, 1) + 1) / 2."""
        m = -x.dot(w)
        m = -1.0 if m < -1.0 else (1.0 if m > 1.0 else m)
        return (m + 1.0) / 2.0


MODEL_CLASSES = {"squared_hinge": SparseSquaredHinge, "modified_huber": SparseModifiedHuber}


def _weight(y: int, r: int, w_pos: float, w_neg: float, sw, weighting: int) -> Optional[float]:
    if weighting == 0:
        return None
    wy = w_pos if y > 0 else w_neg
    return wy * (1.0 if sw is None else float(sw[r])) if weighting == 2 else wy


def literal_pass_loss(model: SparseSquaredHinge, w: Sparse, rows, label, ids, w_pos: float = 1.0, w_neg: float = 1.0,
                      sw=None, weighting: int = 0) -> float:
    """S of the listed rows in the weighting: sum R(L_i); fl(w_pos * sum_+ R(L_i)) + fl(w_neg * sum_- R(L_i));
    sum R(c_i * L_i)."""
    if weighting == 1:
        pos = [model.loss_sample(w, rows[r], int(label[r])) for r in ids if label[r] > 0]
        neg = [model.loss_sample(w, rows[r], int(label[r])) for r in ids if label[r] <= 0]
        return w_pos * literal_fixed_sum(pos) + w_neg * literal_fixed_sum(neg)
    terms = []
    for r in ids:
        y = int(label[r])
        c = _weight(y, r, w_pos, w_neg, sw, weighting)
        l = model.loss_sample(w, rows[r], y)
        terms.append(l if c is None else c * l)
    return literal_fixed_sum(terms)


def literal_correct(w: Sparse, rows, label, ids) -> int:
    return sum(1 for r in ids if -1.0 * signum(rows[r].dot(w)) == int(label[r]))


def literal_sync_steps(model: SparseSquaredHinge, rows, label, dim: int, lam: float, d, w, idx, counts: Sequence[int], lrs,
                       w_pos: float = 1.0, w_neg: float = 1.0, sw=None, weighting: int = 0, lambda1: float = 0.0,
                       avg_sum=None):
    """Sync steps with Sparse vectors: K requests per step at the same weights, regularized (SparseSVM.scala:31), their mean
    (Master.scala:194), w - lr * mean (Master.scala:197), then the L1 proximal step on every column.  Returns (w_new as a
    dense list, losses as a list); avg_sum (a list, optional) gets the weights after every step added."""
    w = Sparse({j: float(v) for j, v in enumerate(w)}, dim)
    d = Sparse({j: float(v) for j, v in enumerate(d)}, dim)
    per_step = int(sum(counts))
    losses = []
    for t, lr in enumerate(float(x) for x in lrs):
        step = [int(i) for i in idx[t * per_step:(t + 1) * per_step]]
        c = lam * 2.0 * w.dot(d)
        replies, h, off = [], None, 0
        for k in counts:
            ids = step[off:off + k]
            off += k
            grads = [model.backward(w, rows[r], int(label[r]), _weight(int(label[r]), r, w_pos, w_neg, sw, weighting))
                     for r in ids]
            g = vec_sum(grads)
            replies.append(g + g.value_like(c))
            hk = literal_pass_loss(model, w, rows, label, ids, w_pos, w_neg, sw, weighting)
            h = hk if h is None else h + hk
        n2 = 0.0
        for j in range(dim):   # ||w||^2 in column order, as the C checker (the map holds the same values)
            n2 += w.get(j) * w.get(j)
        if lambda1 > 0.0:
            l1 = literal_fixed_sum(abs(w.get(j)) for j in range(dim))
            losses.append(lam * n2 + lambda1 * l1 + h / per_step)
        else:
            losses.append(lam * n2 + h / per_step)
        w = w - lr * (vec_sum(replies) / len(counts))
        tau = lr * lambda1
        if tau > 0.0:
            w = Sparse({j: (v - tau if v > tau else (v + tau if v < -tau else 0.0)) for j, v in w.map.items()}, dim)
        if avg_sum is not None:
            for j in range(dim):
                avg_sum[j] += w.get(j)
    return [w.get(j) for j in range(dim)], losses
