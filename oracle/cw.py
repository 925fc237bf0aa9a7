"""TEST INFRASTRUCTURE ONLY -- class weights: a ctypes binding of the fp64 C checker (oracle/dsgd_oracle_cw.c) for the
weighted gradient, the per-class evaluation and the weighted sync step of both models, and a literal restatement over the
Sparse vectors of oracle/scala_semantics.py that the checker is tested against.

The library is built by __graft_entry__.build(), or on first use: next to its source, or in a temporary directory if that is
read-only.  Only tests/ and tools/ use this module; the product package never does.
"""
from __future__ import annotations

import ctypes as C
import math
import os
import subprocess
import tempfile
from typing import Optional, Sequence

import numpy as np

from .oracle import Oracle, _check, _p
from .scala_semantics import Sparse, vec_sum, signum

_HERE = os.path.dirname(os.path.abspath(__file__))
_SRC = os.path.join(_HERE, "dsgd_oracle_cw.c")
_HDRS = (os.path.join(_HERE, "dsgd_oracle_cw.h"), os.path.join(_HERE, "dsgd_oracle.h"))
_NAME = "libdsgd_oracle_cw.so"
# the flags of oracle/Makefile: no fast-math, no contraction
_CFLAGS = ["-O3", "-march=x86-64-v3", "-fno-fast-math", "-ffp-contract=off", "-fPIC", "-Wall", "-Wextra", "-std=gnu11",
           "-shared"]


def _cc():
    return "/usr/bin/gcc" if os.path.exists("/usr/bin/gcc") else "gcc"


def _stale(path: str) -> bool:
    return (not os.path.exists(path)) or os.path.getmtime(path) < max(os.path.getmtime(f) for f in (_SRC, *_HDRS))


def build(force: bool = False) -> str:
    """Compile the class-weight checker (gcc only); returns the library's path."""
    path = os.path.join(_HERE, _NAME)
    if not force and not _stale(path):
        return path
    if not os.access(_HERE, os.W_OK):
        path = os.path.join(tempfile.gettempdir(), f"dsgd_oracle_cw_{os.getuid()}", _NAME)
        os.makedirs(os.path.dirname(path), exist_ok=True)
        if not force and not _stale(path):
            return path
    tmp = f"{path}.{os.getpid()}.tmp"
    subprocess.run([_cc(), *_CFLAGS, "-o", tmp, _SRC, "-lm"], check=True, capture_output=True)
    os.replace(tmp, path)
    return path


_lib = None


def lib():
    global _lib
    if _lib is None:
        _lib = C.CDLL(build())
        for f in (_lib.dsgd_oracle_cw_eval, _lib.dsgd_oracle_cw_gradient, _lib.dsgd_oracle_cw_sync_steps):
            f.restype = C.c_int
    return _lib


def eval_class(orc: Oracle, w, idx, logistic: bool = False):
    """(loss sums [L_pos, L_neg], counts [correct_pos, correct_neg, n_pos, n_neg]) of the listed rows at w."""
    idx = orc._idx(idx)
    sums, counts = np.zeros(2, dtype=np.float64), np.zeros(4, dtype=np.int64)
    _check(lib().dsgd_oracle_cw_eval(C.byref(orc._csr), C.c_int32(1 if logistic else 0), _p(orc._w(w)), _p(idx),
                                     C.c_int64(idx.size), _p(sums), _p(counts)), "cw eval")
    return sums, counts


def gradient(orc: Oracle, w, idx, w_pos: float, w_neg: float, logistic: bool = False, regularize: bool = True):
    """(gradient, loss, [L_pos, L_neg]) of one request under the class weights; regularize=False: the raw weighted sum."""
    idx = orc._idx(idx)
    g, loss, sums = np.zeros(orc.dim, dtype=np.float64), C.c_double(), np.zeros(2, dtype=np.float64)
    _check(lib().dsgd_oracle_cw_gradient(C.byref(orc._csr), C.c_int32(1 if logistic else 0), C.c_double(orc.lam), _p(orc.d),
                                         _p(orc._w(w)), _p(idx), C.c_int64(idx.size), C.c_double(w_pos), C.c_double(w_neg),
                                         C.c_int32(1 if regularize else 0), _p(g), C.byref(loss), _p(sums)), "cw gradient")
    return g, loss.value, sums


def sync_steps(orc: Oracle, w, idx, counts: Sequence[int], lrs, w_pos: float, w_neg: float, logistic: bool = False,
               lambda1: float = 0.0, avg_sum: Optional[np.ndarray] = None):
    """len(lrs) weighted sync steps of the C checker on a copy of w, with orc's rows, lambda and dimSparsity; step t at rate
    lrs[t].  Returns (w_new, losses).  avg_sum (optional, modified in place) gets the weights after every step added."""
    w = orc._w(w).copy()
    idx = orc._idx(idx)
    counts = np.ascontiguousarray(counts, dtype=np.int32)
    lrs = np.ascontiguousarray(lrs, dtype=np.float64)
    assert len(idx) == int(counts.sum()) * lrs.size
    losses = np.zeros(lrs.size, dtype=np.float64)
    if avg_sum is not None:
        assert avg_sum.dtype == np.float64 and avg_sum.flags.c_contiguous and avg_sum.size == orc.dim
    _check(lib().dsgd_oracle_cw_sync_steps(C.byref(orc._csr), C.c_int32(1 if logistic else 0), C.c_double(orc.lam),
                                           C.c_double(lambda1), _p(orc.d), _p(w), _p(idx), _p(counts), C.c_int32(len(counts)),
                                           _p(lrs), C.c_int64(lrs.size), C.c_double(w_pos), C.c_double(w_neg), _p(losses),
                                           _p(avg_sum)), "cw sync_steps")
    return w, losses


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
