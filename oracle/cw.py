"""TEST INFRASTRUCTURE ONLY -- class weights: the weighted gradient, the per-class evaluation and the weighted sync step of
both models as calls into the checker of every model (oracle/margin.py), and a literal restatement over the Sparse vectors
of oracle/scala_semantics.py that the checker is tested against.

Only tests/ and tools/ use this module; the product package never does.
"""
from __future__ import annotations

import math
from typing import Optional, Sequence

import numpy as np

from . import margin as M
from .oracle import Oracle
from .scala_semantics import Sparse, vec_sum, signum


def eval_class(orc: Oracle, w, idx, logistic: bool = False):
    """(loss sums [L_pos, L_neg], counts [correct_pos, correct_neg, n_pos, n_neg]) of the listed rows at w."""
    return M.eval_class(orc, int(logistic), w, idx)


def gradient(orc: Oracle, w, idx, w_pos: float, w_neg: float, logistic: bool = False, regularize: bool = True):
    """(gradient, loss, [L_pos, L_neg]) of one request under the class weights; regularize=False: the raw weighted sum."""
    g, loss, _ = M.gradient(orc, int(logistic), w, idx, w_pos, w_neg, regularize=regularize)
    return g, loss, eval_class(orc, w, idx, logistic)[0]


def sync_steps(orc: Oracle, w, idx, counts: Sequence[int], lrs, w_pos: float, w_neg: float, logistic: bool = False,
               lambda1: float = 0.0, avg_sum: Optional[np.ndarray] = None):
    """len(lrs) weighted sync steps of the C checker on a copy of w, with orc's rows, lambda and dimSparsity; step t at rate
    lrs[t].  Returns (w_new, losses).  avg_sum (optional, modified in place) gets the weights after every step added."""
    return M.sync_steps(orc, int(logistic), w, idx, counts, lrs, w_pos, w_neg, lambda1=lambda1, avg_sum=avg_sum)


# ---- the literal restatement over Sparse vectors: no shared code with the C checker ---------------------------------------

def _softplus(z: float) -> float:
    return max(z, 0.0) + math.log1p(math.exp(-abs(z)))


def _sigmoid(z: float) -> float:
    return 1.0 / (1.0 + math.exp(-z)) if z >= 0.0 else math.exp(z) / (1.0 + math.exp(z))


def literal_rows(row_ptr, col, val, dim: int):
    """The rows as Sparse vectors (fp32 values widened)."""
    return [Sparse({int(col[p]): float(np.float32(val[p])) for p in range(int(row_ptr[r]), int(row_ptr[r + 1]))}, dim)
            for r in range(len(row_ptr) - 1)]


def literal_backward(w: Sparse, x: Sparse, y: int, wy: float, logistic: bool) -> Sparse:
    """The model's backward with the scalar of `x * y` replaced by the weighted one."""
    z = y * x.dot(w)
    if logistic:
        return x * ((y * _sigmoid(z)) * wy)
    return w.zeros_like() if z < 0 else x * (y * wy)


def literal_loss_sums(w: Sparse, rows, label, ids, logistic: bool):
    """[L_pos, L_neg] (math.fsum: correctly rounded) and [correct_pos, correct_neg, n_pos, n_neg]."""
    terms, counts = ([], []), [0, 0, 0, 0]
    for r in ids:
        y, dot = int(label[r]), rows[r].dot(w)
        cls = 0 if y > 0 else 1
        pred = -1.0 * signum(dot)
        counts[2 + cls] += 1
        counts[cls] += int(pred == y)
        terms[cls].append(_softplus(y * dot) if logistic else max(0.0, 1.0 - y * pred))
    return [math.fsum(terms[0]), math.fsum(terms[1])], counts


def literal_sync_steps(rows, label, dim: int, lam: float, d, w, idx, counts: Sequence[int], lrs, w_pos: float,
                       w_neg: float, logistic: bool = False):
    """The weighted sync steps (no L1) with Sparse vectors.  Returns (w_new as a dense list, losses as a list)."""
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
            grads = [literal_backward(w, rows[r], int(label[r]), w_pos if label[r] > 0 else w_neg, logistic) for r in ids]
            g = vec_sum(grads)
            replies.append(g + g.value_like(c))   # regularize (SparseSVM.scala:31)
            sums, _ = literal_loss_sums(w, rows, label, ids, logistic)
            hk = w_pos * sums[0] + w_neg * sums[1]
            h = hk if h is None else h + hk
        losses.append(lam * w.norm_squared() + h / per_step)
        w = w - lr * (vec_sum(replies) / len(counts))   # Master.scala:194,197
    return [w.get(j) for j in range(dim)], losses
