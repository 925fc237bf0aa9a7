"""TEST INFRASTRUCTURE ONLY -- sample weights: the sample-weighted gradient, the weighted evaluation and the sample-weighted
sync step of both models as calls into the checker of every model (oracle/margin.py), and a literal restatement over the
Sparse vectors of oracle/scala_semantics.py that the checker is tested against.

Every call here is sample-weighted, c_i = fl(w_y * s_i); sw=None stands for every s_i = 1.  Only tests/ and tools/ use this
module; the product package never does.
"""
from __future__ import annotations

import math
from fractions import Fraction
from typing import Optional, Sequence

import numpy as np

from . import margin as M
from .cw import _sigmoid, _softplus
from .oracle import Oracle
from .scala_semantics import Sparse, signum, vec_sum


def _sw(orc: Oracle, sw):
    """The sample weights, every one 1 for sw=None: the margin checker then takes the sample-weighted pass all the same."""
    return np.ones(orc.n_rows) if sw is None else sw


def eval_weighted(orc: Oracle, w, idx, w_pos: float = 1.0, w_neg: float = 1.0, sw=None, logistic: bool = False):
    """(sums [S, sum c_i [correct], sum c_i], counts [rows, correct]) of the listed rows at w."""
    return M.eval_weighted(orc, int(logistic), w, idx, w_pos, w_neg, sw)


def gradient(orc: Oracle, w, idx, sw=None, w_pos: float = 1.0, w_neg: float = 1.0, logistic: bool = False,
             regularize: bool = True):
    """(gradient, loss, S) of one request under the sample and class weights; regularize=False: the raw weighted sum."""
    return M.gradient(orc, int(logistic), w, idx, w_pos, w_neg, _sw(orc, sw), regularize)


def sync_steps(orc: Oracle, w, idx, counts: Sequence[int], lrs, sw=None, w_pos: float = 1.0, w_neg: float = 1.0,
               logistic: bool = False, lambda1: float = 0.0, avg_sum: Optional[np.ndarray] = None):
    """len(lrs) sample-weighted sync steps of the C checker on a copy of w, with orc's rows, lambda and dimSparsity; step t at
    rate lrs[t].  Returns (w_new, losses).  avg_sum (optional, modified in place) gets the weights after every step added."""
    return M.sync_steps(orc, int(logistic), w, idx, counts, lrs, w_pos, w_neg, _sw(orc, sw), lambda1, avg_sum)


# ---- the literal restatement over Sparse vectors: no shared code with the C checker ---------------------------------------

def literal_fixed_sum(values) -> float:
    """The order-free sum of non-negative terms as the device reports it: every term rounded to a multiple of 2^-160 (ties to
    even), the exact total cut into 40-bit limbs and converted from the top limb down; NaN if a term is NaN, infinite, negative
    or 2^52 or more."""
    total = 0
    for v in values:
        v = float(v)
        if not (0.0 <= v < 2.0 ** 52):
            return math.nan
        q, r = divmod(Fraction(v) * 2 ** 160, 1)
        q = int(q)
        if r > Fraction(1, 2) or (r == Fraction(1, 2) and q & 1):
            q += 1
        total += q
    limbs = [(total >> (40 * k)) & ((1 << 40) - 1) for k in range(5)] + [total >> 200]
    s = float(limbs[5]) * 2.0 ** 40
    for k in range(4, -1, -1):
        s += float(limbs[k]) * 2.0 ** (40 * k - 160)
    return s


def combined_weight(y: int, s: float, w_pos: float, w_neg: float) -> float:
    return (w_pos if y > 0 else w_neg) * s


def literal_backward(w: Sparse, x: Sparse, y: int, c: float, logistic: bool) -> Sparse:
    """The model's backward with the scalar of `x * y` replaced by the weighted one."""
    z = y * x.dot(w)
    if logistic:
        return x * ((y * _sigmoid(z)) * c)
    return w.zeros_like() if z < 0 else x * (y * c)


def literal_eval(w: Sparse, rows, label, ids, sw, w_pos: float = 1.0, w_neg: float = 1.0, logistic: bool = False):
    """([S, sum c_i [correct], sum c_i], [rows, correct]) of the listed rows."""
    loss, ok_w, all_w, correct = [], [], [], 0
    for r in ids:
        y, dot = int(label[r]), rows[r].dot(w)
        c = combined_weight(y, 1.0 if sw is None else float(sw[r]), w_pos, w_neg)
        pred = -1.0 * signum(dot)
        ok = pred == y
        correct += int(ok)
        loss.append(c * (_softplus(y * dot) if logistic else max(0.0, 1.0 - y * pred)))
        ok_w.append(c if ok else 0.0)
        all_w.append(c)
    return [literal_fixed_sum(loss), literal_fixed_sum(ok_w), literal_fixed_sum(all_w)], [len(ids), correct]


def literal_sync_steps(rows, label, dim: int, lam: float, d, w, idx, counts: Sequence[int], lrs, sw, w_pos: float = 1.0,
                       w_neg: float = 1.0, logistic: bool = False):
    """The sample-weighted sync steps (no L1) with Sparse vectors.  Returns (w_new as a dense list, losses as a list)."""
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
            grads = [literal_backward(w, rows[r], int(label[r]),
                                      combined_weight(int(label[r]), 1.0 if sw is None else float(sw[r]), w_pos, w_neg),
                                      logistic) for r in ids]
            g = vec_sum(grads)
            replies.append(g + g.value_like(c))   # regularize (SparseSVM.scala:31)
            hk = literal_eval(w, rows, label, ids, sw, w_pos, w_neg, logistic)[0][0]
            h = hk if h is None else h + hk
        losses.append(lam * w.norm_squared() + h / per_step)
        w = w - lr * (vec_sum(replies) / len(counts))   # Master.scala:194,197
    return [w.get(j) for j in range(dim)], losses
