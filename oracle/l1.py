"""TEST INFRASTRUCTURE ONLY -- the sync step with an L1 penalty: a ctypes binding of the fp64 C checker
(oracle/dsgd_oracle_l1.c) and a literal restatement in plain Python that the checker is tested against.

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

_HERE = os.path.dirname(os.path.abspath(__file__))
_SRC = os.path.join(_HERE, "dsgd_oracle_l1.c")
_HDRS = (os.path.join(_HERE, "dsgd_oracle_l1.h"), os.path.join(_HERE, "dsgd_oracle.h"))
_NAME = "libdsgd_oracle_l1.so"
# the flags of oracle/Makefile: no fast-math, no contraction
_CFLAGS = ["-O3", "-march=x86-64-v3", "-fno-fast-math", "-ffp-contract=off", "-fPIC", "-Wall", "-Wextra", "-std=gnu11",
           "-shared"]
EPS = 1e-20   # math/Sparse.scala:104


def _cc():
    return "/usr/bin/gcc" if os.path.exists("/usr/bin/gcc") else "gcc"


def _stale(path: str) -> bool:
    return (not os.path.exists(path)) or os.path.getmtime(path) < max(os.path.getmtime(f) for f in (_SRC, *_HDRS))


def build(force: bool = False) -> str:
    """Compile the L1 checker (gcc only); returns the library's path."""
    path = os.path.join(_HERE, _NAME)
    if not force and not _stale(path):
        return path
    if not os.access(_HERE, os.W_OK):
        path = os.path.join(tempfile.gettempdir(), f"dsgd_oracle_l1_{os.getuid()}", _NAME)
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
        _lib.dsgd_oracle_l1_sync_steps.restype = C.c_int
        _lib.dsgd_oracle_l1_prox.restype = C.c_double
        _lib.dsgd_oracle_l1_prox.argtypes = [C.c_double, C.c_double]
        _lib.dsgd_oracle_l1_norm.restype = C.c_double
    return _lib


def prox(u: float, tau: float) -> float:
    """The C checker's proximal step for one value."""
    return lib().dsgd_oracle_l1_prox(float(u), float(tau))


def l1_norm(w) -> float:
    w = np.ascontiguousarray(w, dtype=np.float64)
    return lib().dsgd_oracle_l1_norm(_p(w), C.c_int32(w.size), None)


def sync_steps(orc: Oracle, w, idx, counts: Sequence[int], lrs, lambda1: float, logistic: bool = False,
               avg_sum: Optional[np.ndarray] = None):
    """len(lrs) sync steps of the C checker on a copy of w, with orc's rows, lambda and dimSparsity; step t at rate lrs[t].
    Returns (w_new, losses).  avg_sum (optional, modified in place) gets the weights after every step added."""
    w = orc._w(w).copy()
    idx = orc._idx(idx)
    counts = np.ascontiguousarray(counts, dtype=np.int32)
    lrs = np.ascontiguousarray(lrs, dtype=np.float64)
    assert len(idx) == int(counts.sum()) * lrs.size
    losses = np.zeros(lrs.size, dtype=np.float64)
    if avg_sum is not None:
        assert avg_sum.dtype == np.float64 and avg_sum.flags.c_contiguous and avg_sum.size == orc.dim
    _check(lib().dsgd_oracle_l1_sync_steps(C.byref(orc._csr), C.c_int32(1 if logistic else 0), C.c_double(orc.lam),
                                           C.c_double(lambda1), _p(orc.d), _p(w), _p(idx), _p(counts),
                                           C.c_int32(len(counts)), _p(lrs), C.c_int64(lrs.size), _p(losses), _p(avg_sum)),
           "l1 sync_steps")
    return w, losses


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
