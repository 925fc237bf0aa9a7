"""A literal restatement of one sync step with an intercept (DESIGN.md §4.18), written from the semantics rather than from
the kernels: the independent witness of the intercept's step, as scala_semantics*.py are of the plain steps.

beta is the weight of a virtual column of value 1 in every row and is left out of every penalty:
    score  = fl(sum of filt(filt(x_j) * w_j) + filt(beta))           (the row's dot in column order, then beta)
    z      = y * score,  prediction -signum(score)
    row    SVM: s = y (weighted y * c_i), scattered when z >= 0, loss 1 - y * pred (an integer)
           logistic / squared hinge / modified Huber: s = y * scale(z) (weighted (y * scale(z)) * c_i), loss L(z)
    grad   g_j = sum_i filt(filt(x_ij) * s_i);  g_beta = sum_i filt(s_i)
    regularize  r_j = filt(g_j), then filt(r_j + c) where r_j != 0 and |c| > 1e-20, c = 2 lambda (w . d) over the weights
                only; r_beta = filt(g_beta), no c
    update r_j != 0: w_j <- filt(w_j - filt(filt(r_j / K) * lr)); then with lambda1 > 0 every w_j is soft-thresholded at
           lr * lambda1; beta <- filt(beta - filt(filt(r_beta / K) * lr)) when r_beta != 0, never thresholded
    loss   lambda ||w||^2 + lambda1 ||w||_1 + (sum of the weighted losses) / n, the norms over the weights only
intercept=False is the same step without beta: the plain step of the checker of record (oracle/margin.py).
"""
import math

import numpy as np

EPS = 1e-20


def filt(v: float) -> float:
    return v if abs(v) > EPS else 0.0


def _softplus(z):
    return max(z, 0.0) + math.log1p(math.exp(-abs(z)))


def _sigmoid(t):
    if t >= 0.0:
        return 1.0 / (1.0 + math.exp(-t))
    e = math.exp(t)
    return e / (1.0 + e)


def loss_scale(model: str, z: float):
    """(L(z), s(z)) of one sample of a model other than the SVM."""
    if model == "logistic":
        return _softplus(z), _sigmoid(z)
    if z <= -1.0:
        return 0.0, 0.0
    t = 1.0 + z
    if model == "squared_hinge" or z <= 1.0:
        return t * t, 2.0 * t
    return 4.0 * z, 4.0


def _pred(score: float) -> int:
    return -1 if score > 0.0 else (1 if score < 0.0 else 0)


def _soft(u: float, tau: float) -> float:
    if not tau > 0.0:
        return u
    return filt(u - tau) if u > tau else (filt(u + tau) if u < -tau else 0.0)


def step(rows, labels, d, w, ids, model: str, lam: float, lr: float, lambda1: float = 0.0, c=None, intercept=True):
    """One single-worker sync step.  rows: list of (cols, vals); labels: +-1 per row; d: dimSparsity (dim); w: the weights,
    dim + 1 long with beta last when `intercept`; ids: the batch; c: each row's weight (None: 1).  Returns (w_new, loss)."""
    dim = len(d)
    wv = [float(v) for v in w[:dim]]
    beta = float(w[dim]) if intercept else 0.0
    cc = lam * 2.0 * sum(filt(wv[j] * float(d[j])) for j in range(dim))
    g = [0.0] * dim
    gb, loss_sum = 0.0, 0.0
    for i in ids:
        cols, vals = rows[i]
        y = float(labels[i])
        dot = 0.0
        for j, x in zip(cols, vals):
            dot += filt(filt(float(x)) * wv[j])
        score = dot + filt(beta) if intercept else dot
        z = y * score
        ci = 1.0 if c is None else float(c[i])
        if model == "svm":
            loss_sum += ci * (1 - int(y) * _pred(score))
            if z < 0.0:
                continue
            s = y if c is None else (ci if y > 0 else -ci)
        else:
            l, sc = loss_scale(model, z)
            loss_sum += ci * l
            s = y * sc if c is None else (y * sc) * ci
        for j, x in zip(cols, vals):
            gv = filt(filt(float(x)) * s)
            if gv != 0.0:
                g[j] += gv
        gb += filt(s)
    loss = lam * sum(v * v for v in wv) + lambda1 * sum(abs(v) for v in wv) + loss_sum / len(ids)
    add_c = cc != 0.0 and abs(cc) > EPS
    out = np.zeros(len(w))
    for j in range(dim):
        v = filt(g[j])
        if v != 0.0 and add_c:
            v = filt(v + cc)
        wn = wv[j]
        if v != 0.0:
            wn = filt(wn - filt(filt(v / 1.0) * lr))
        out[j] = _soft(wn, lr * lambda1) if lambda1 > 0.0 else wn
    if intercept:
        vb = filt(gb)
        out[dim] = filt(beta - filt(filt(vb / 1.0) * lr)) if vb != 0.0 else beta
    return out, loss


def steps(rows, labels, d, w, ids, batch: int, model: str, lam: float, lrs, lambda1: float = 0.0, c=None, intercept=True):
    """len(lrs) steps of `batch` consecutive ids each; returns (w_new, losses)."""
    losses = []
    for t, lr in enumerate(lrs):
        w, l = step(rows, labels, d, w, ids[t * batch:(t + 1) * batch], model, lam, lr, lambda1, c, intercept)
        losses.append(l)
    return w, np.array(losses)


def csr_rows(row_ptr, col, val):
    """The rows of a CSR array as the list this module takes."""
    return [(col[row_ptr[r]:row_ptr[r + 1]], val[row_ptr[r]:row_ptr[r + 1]]) for r in range(len(row_ptr) - 1)]
