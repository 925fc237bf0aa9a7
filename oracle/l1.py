"""TEST INFRASTRUCTURE ONLY -- the sync step with an L1 penalty: calls into the checker of every model (oracle/margin.py),
and a literal restatement in plain Python that the checker is tested against.

Only tests/ and tools/ use this module; the product package never does.
"""
from __future__ import annotations

import math
from typing import Optional, Sequence

import numpy as np

from . import margin as M
from .oracle import Oracle

EPS = 1e-20   # math/Sparse.scala:104


def prox(u: float, tau: float) -> float:
    """The C checker's proximal step for one value, the one its sync steps apply."""
    return M.prox(u, tau)


def l1_norm(w) -> float:
    """||w||_1 as the device sums it."""
    return M.l1_norm(w)[0]


def sync_steps(orc: Oracle, w, idx, counts: Sequence[int], lrs, lambda1: float, logistic: bool = False,
               avg_sum: Optional[np.ndarray] = None):
    """len(lrs) sync steps of the C checker on a copy of w, with orc's rows, lambda and dimSparsity; step t at rate lrs[t].
    Returns (w_new, losses).  avg_sum (optional, modified in place) gets the weights after every step added."""
    return M.sync_steps(orc, int(logistic), w, idx, counts, lrs, lambda1=lambda1, avg_sum=avg_sum)


# ---- the literal restatement: one value at a time, Python floats, no shared code with the C checker ----------------------

def filt(v: float) -> float:
    return v if abs(v) > EPS else 0.0


def literal_prox(u: float, tau: float) -> float:
    """soft_threshold(u, tau) with the 1e-20 filter: shrink u towards 0 by tau, 0 when |u| <= tau; tau == 0 keeps u."""
    if tau == 0.0:
        return u
    if u > tau:
        return filt(u - tau)
    if u < -tau:
        return filt(u + tau)
    return 0.0


def literal_sync_steps(row_ptr, col, val, label, dim: int, lam: float, lambda1: float, d, w, idx, counts: Sequence[int],
                       lrs, logistic: bool = False):
    """The same steps as sync_steps, written out with Python floats and dicts.  ||w||_1 is math.fsum (correctly rounded).
    Returns (w_new as a list, losses as a list)."""
    w = [float(x) for x in w]
    d = [float(x) for x in d]
    rows = []
    for r in range(len(row_ptr) - 1):
        rows.append([(int(col[p]), filt(float(np.float32(val[p])))) for p in range(int(row_ptr[r]), int(row_ptr[r + 1]))])
    per_step = int(sum(counts))
    losses = []
    for t, lr in enumerate(float(x) for x in lrs):
        step = [int(i) for i in idx[t * per_step:(t + 1) * per_step]]
        c = lam * 2.0 * sum_in_order(filt(w[j] * d[j]) for j in range(dim))
        n2 = sum_in_order(w[j] * w[j] for j in range(dim))
        total = {}   # Vec.mean's running sum
        h = 0.0
        off = 0
        for k in counts:
            g = {}
            for r in step[off:off + k]:
                y = float(label[r])
                dot = sum_in_order(filt(x * w[j]) for j, x in rows[r])
                if logistic:
                    z = y * dot
                    h += max(z, 0.0) + math.log1p(math.exp(-abs(z)))
                    s = y * (1.0 / (1.0 + math.exp(-z)) if z >= 0.0 else math.exp(z) / (1.0 + math.exp(z)))
                else:
                    p = -1.0 if dot > 0.0 else (1.0 if dot < 0.0 else 0.0)
                    h += max(0.0, 1.0 - y * p)
                    if y * dot < 0.0:
                        continue
                    s = y
                for j, x in rows[r]:
                    gv = filt(x * s)
                    if gv != 0.0:
                        g[j] = filt(g.get(j, 0.0) + gv)
            off += k
            for j in sorted(g):
                v = g[j]
                if v != 0.0 and c != 0.0 and abs(c) > EPS:
                    v = filt(v + c)
                if v != 0.0:
                    total[j] = filt(total.get(j, 0.0) + v)
        losses.append(lam * n2 + lambda1 * math.fsum(abs(x) for x in w) + h / per_step)
        tau = lr * lambda1
        for j in range(dim):
            u = w[j]
            if total.get(j, 0.0) != 0.0:
                u = filt(u - filt(filt(total[j] / len(counts)) * lr))
            w[j] = literal_prox(u, tau)
    return w, losses


def sum_in_order(values) -> float:
    s = 0.0
    for v in values:
        s += v
    return s
