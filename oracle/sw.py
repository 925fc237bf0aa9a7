"""TEST INFRASTRUCTURE ONLY -- sample weights: a ctypes binding of the fp64 C checker (oracle/dsgd_oracle_sw.c) for the
sample-weighted gradient, the weighted evaluation and the sample-weighted sync step of both models, and a literal restatement
over the Sparse vectors of oracle/scala_semantics.py that the checker is tested against.

The library is built by __graft_entry__.build(), or on first use: next to its source, or in a temporary directory if that is
read-only.  Only tests/ and tools/ use this module; the product package never does.
"""
from __future__ import annotations

import ctypes as C
import math
import os
import subprocess
import tempfile
from fractions import Fraction
from typing import Optional, Sequence

import numpy as np

from .cw import _sigmoid, _softplus
from .oracle import Oracle, _check, _p
from .scala_semantics import Sparse, signum, vec_sum

_HERE = os.path.dirname(os.path.abspath(__file__))
_SRC = os.path.join(_HERE, "dsgd_oracle_sw.c")
_HDRS = (os.path.join(_HERE, "dsgd_oracle_sw.h"), os.path.join(_HERE, "dsgd_oracle.h"))
_NAME = "libdsgd_oracle_sw.so"
# the flags of oracle/Makefile: no fast-math, no contraction
_CFLAGS = ["-O3", "-march=x86-64-v3", "-fno-fast-math", "-ffp-contract=off", "-fPIC", "-Wall", "-Wextra", "-std=gnu11",
           "-shared"]


def _cc():
    return "/usr/bin/gcc" if os.path.exists("/usr/bin/gcc") else "gcc"


def _stale(path: str) -> bool:
    return (not os.path.exists(path)) or os.path.getmtime(path) < max(os.path.getmtime(f) for f in (_SRC, *_HDRS))


def build(force: bool = False) -> str:
    """Compile the sample-weight checker (gcc only); returns the library's path."""
    path = os.path.join(_HERE, _NAME)
    if not force and not _stale(path):
        return path
    if not os.access(_HERE, os.W_OK):
        path = os.path.join(tempfile.gettempdir(), f"dsgd_oracle_sw_{os.getuid()}", _NAME)
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
        for f in (_lib.dsgd_oracle_sw_eval, _lib.dsgd_oracle_sw_gradient, _lib.dsgd_oracle_sw_sync_steps):
            f.restype = C.c_int
    return _lib


def _sw(orc: Oracle, sw):
    if sw is None:
        return None
    sw = np.ascontiguousarray(sw, dtype=np.float64)
    assert sw.size == orc.n_rows
    return sw


def eval_weighted(orc: Oracle, w, idx, w_pos: float = 1.0, w_neg: float = 1.0, sw=None, logistic: bool = False):
    """(sums [S, sum c_i [correct], sum c_i], counts [rows, correct]) of the listed rows at w."""
    idx = orc._idx(idx)
    sums, counts = np.zeros(3, dtype=np.float64), np.zeros(2, dtype=np.int64)
    _check(lib().dsgd_oracle_sw_eval(C.byref(orc._csr), C.c_int32(1 if logistic else 0), _p(orc._w(w)), _p(idx),
                                     C.c_int64(idx.size), C.c_double(w_pos), C.c_double(w_neg), _p(_sw(orc, sw)), _p(sums),
                                     _p(counts)), "sw eval")
    return sums, counts


def gradient(orc: Oracle, w, idx, sw=None, w_pos: float = 1.0, w_neg: float = 1.0, logistic: bool = False,
             regularize: bool = True):
    """(gradient, loss, S) of one request under the sample and class weights; regularize=False: the raw weighted sum."""
    idx = orc._idx(idx)
    g, loss, s = np.zeros(orc.dim, dtype=np.float64), C.c_double(), C.c_double()
    _check(lib().dsgd_oracle_sw_gradient(C.byref(orc._csr), C.c_int32(1 if logistic else 0), C.c_double(orc.lam), _p(orc.d),
                                         _p(orc._w(w)), _p(idx), C.c_int64(idx.size), C.c_double(w_pos), C.c_double(w_neg),
                                         _p(_sw(orc, sw)), C.c_int32(1 if regularize else 0), _p(g), C.byref(loss),
                                         C.byref(s)), "sw gradient")
    return g, loss.value, s.value


def sync_steps(orc: Oracle, w, idx, counts: Sequence[int], lrs, sw=None, w_pos: float = 1.0, w_neg: float = 1.0,
               logistic: bool = False, lambda1: float = 0.0, avg_sum: Optional[np.ndarray] = None):
    """len(lrs) sample-weighted sync steps of the C checker on a copy of w, with orc's rows, lambda and dimSparsity; step t at
    rate lrs[t].  Returns (w_new, losses).  avg_sum (optional, modified in place) gets the weights after every step added."""
    w = orc._w(w).copy()
    idx = orc._idx(idx)
    counts = np.ascontiguousarray(counts, dtype=np.int32)
    lrs = np.ascontiguousarray(lrs, dtype=np.float64)
    assert len(idx) == int(counts.sum()) * lrs.size
    losses = np.zeros(lrs.size, dtype=np.float64)
    if avg_sum is not None:
        assert avg_sum.dtype == np.float64 and avg_sum.flags.c_contiguous and avg_sum.size == orc.dim
    _check(lib().dsgd_oracle_sw_sync_steps(C.byref(orc._csr), C.c_int32(1 if logistic else 0), C.c_double(orc.lam),
                                           C.c_double(lambda1), _p(orc.d), _p(w), _p(idx), _p(counts), C.c_int32(len(counts)),
                                           _p(lrs), C.c_int64(lrs.size), C.c_double(w_pos), C.c_double(w_neg),
                                           _p(_sw(orc, sw)), _p(losses), _p(avg_sum)), "sw sync_steps")
    return w, losses


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
