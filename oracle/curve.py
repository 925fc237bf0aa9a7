"""TEST INFRASTRUCTURE ONLY -- ctypes binding of the fp64 curve and average-precision checker (oracle/dsgd_oracle_curve.c,
linked with oracle/dsgd_oracle_metrics.c for its dots).

`curve` answers for an Oracle of oracle/oracle.py (its CSR).  The library is built by __graft_entry__.build(), or on first
use: next to its sources, or in a temporary directory if that is read-only.  Only tests/ and tools/ use it; the product
package never does.
"""
from __future__ import annotations

import ctypes as C
import math
import os
import subprocess
import tempfile
from typing import NamedTuple, Optional

import numpy as np

from .oracle import Oracle, _check, _p

_HERE = os.path.dirname(os.path.abspath(__file__))
_SRCS = (os.path.join(_HERE, "dsgd_oracle_curve.c"), os.path.join(_HERE, "dsgd_oracle_metrics.c"))
_HDRS = (os.path.join(_HERE, "dsgd_oracle.h"),)
_NAME = "libdsgd_oracle_curve.so"
# the flags of oracle/Makefile: no fast-math, no contraction
_CFLAGS = ["-O3", "-march=x86-64-v3", "-fno-fast-math", "-ffp-contract=off", "-fPIC", "-Wall", "-Wextra", "-std=gnu11",
           "-shared"]


def _cc():
    return "/usr/bin/gcc" if os.path.exists("/usr/bin/gcc") else "gcc"


def _stale(path: str) -> bool:
    return (not os.path.exists(path)) or os.path.getmtime(path) < max(os.path.getmtime(f) for f in (*_SRCS, *_HDRS))


def build(force: bool = False) -> str:
    """Compile the curve checker (gcc only); returns the library's path."""
    path = os.path.join(_HERE, _NAME)
    if not force and not _stale(path):
        return path
    if not os.access(_HERE, os.W_OK):
        path = os.path.join(tempfile.gettempdir(), f"dsgd_oracle_curve_{os.getuid()}", _NAME)
        os.makedirs(os.path.dirname(path), exist_ok=True)
        if not force and not _stale(path):
            return path
    tmp = f"{path}.{os.getpid()}.tmp"
    subprocess.run([_cc(), *_CFLAGS, "-o", tmp, *_SRCS, "-lm"], check=True, capture_output=True)
    os.replace(tmp, path)
    return path


_lib = None


def lib():
    global _lib
    if _lib is None:
        _lib = C.CDLL(build())
        _lib.dsgd_oracle_curve.restype = C.c_int
    return _lib


class Curve(NamedTuple):
    thr: np.ndarray      # distinct scores, highest first
    tp: np.ndarray       # positive rows scoring at or above thr[k]
    fp: np.ndarray       # negative rows scoring at or above thr[k]
    v: np.ndarray        # tp_i / (tp_i + fp_i) of every non-NaN positive row, at its own score
    nan: int             # rows whose margin is NaN
    ap: float            # math.fsum(v) / P; nan when a margin is NaN or there is no positive row


def curve(orc: Oracle, w, idx=None, begin: int = 0, n: Optional[int] = None, margins=None) -> Curve:
    """The curve over the listed rows of orc's data, or rows [begin, begin + n); margins (optional): the rows' margins to
    rank instead of the checker's own dots."""
    w = orc._w(w)
    if idx is not None:
        idx = orc._idx(idx)
        n = len(idx)
    elif n is None:
        n = orc.n_rows - begin
    if margins is not None:
        margins = np.ascontiguousarray(margins, dtype=np.float64)
        assert margins.shape == (n,)
    size = max(int(n), 1)
    thr, v = np.zeros(size), np.zeros(size)
    tp, fp = np.zeros(size, dtype=np.int64), np.zeros(size, dtype=np.int64)
    m, nv, nan = C.c_int64(), C.c_int64(), C.c_int64()
    _check(lib().dsgd_oracle_curve(C.byref(orc._csr), _p(w), _p(idx), C.c_int64(begin), C.c_int64(n), _p(margins),
                                   C.byref(m), _p(thr), _p(tp), _p(fp), _p(v), C.byref(nv), C.byref(nan)), "curve")
    k, nv = m.value, nv.value
    ap = math.fsum(v[:nv]) / nv if nan.value == 0 and nv else float("nan")
    return Curve(thr[:k].copy(), tp[:k].copy(), fp[:k].copy(), v[:nv].copy(), nan.value, ap)
