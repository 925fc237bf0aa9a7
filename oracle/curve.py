"""TEST INFRASTRUCTURE ONLY -- ctypes binding of the fp64 curve and average-precision checker (oracle/dsgd_oracle_curve.c,
linked with oracle/dsgd_oracle_metrics.c for its dots).

`curve` answers for an Oracle of oracle/oracle.py (its CSR).  The library is oracle/oracle.py's libdsgd_oracle.so.  Only
tests/ and tools/ use it; the product package never does.
"""
from __future__ import annotations

import ctypes as C
import math
from typing import NamedTuple, Optional

import numpy as np

from . import oracle as _oracle
from .oracle import Oracle, _check, _p


_lib = None


def lib():
    global _lib
    if _lib is None:
        _lib = _oracle.lib()
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
