"""TEST INFRASTRUCTURE ONLY -- ctypes binding of the fp64 scores and ranking-metrics checker (oracle/dsgd_oracle_metrics.c).

`margins` and `metrics` answer for an Oracle of oracle/oracle.py (its CSR).  The library is oracle/oracle.py's
libdsgd_oracle.so.  Only tests/ and tools/ use it; the product package never does.
"""
from __future__ import annotations

import ctypes as C
from typing import Optional

import numpy as np

from . import oracle as _oracle
from .oracle import Oracle, _check, _p


_lib = None


def lib():
    global _lib
    if _lib is None:
        _lib = _oracle.lib()
        for name in ("margins", "metrics"):
            getattr(_lib, "dsgd_oracle_" + name).restype = C.c_int
    return _lib


def _rows(orc: Oracle, idx, begin: int, n: Optional[int]):
    if idx is not None:
        idx = orc._idx(idx)
        return idx, len(idx)
    return None, orc.n_rows - begin if n is None else n


def margins(orc: Oracle, w, idx=None, begin: int = 0, n: Optional[int] = None) -> np.ndarray:
    """x . w (left fold) of the listed rows of orc's data, or of rows [begin, begin + n)."""
    w = orc._w(w)
    idx, n = _rows(orc, idx, begin, n)
    out = np.zeros(n, dtype=np.float64)
    _check(lib().dsgd_oracle_margins(C.byref(orc._csr), _p(w), _p(idx), C.c_int64(begin), C.c_int64(n), _p(out)), "margins")
    return out


def metrics(orc: Oracle, w, idx=None, begin: int = 0, n: Optional[int] = None, margins=None) -> np.ndarray:
    """The eight words of dsgd_eval_metrics over the listed rows, or rows [begin, begin + n); margins (optional): the rows'
    margins to rank instead of the checker's own dots."""
    w = orc._w(w)
    idx, n = _rows(orc, idx, begin, n)
    if margins is not None:
        margins = np.ascontiguousarray(margins, dtype=np.float64)
        assert margins.shape == (n,)
    out = np.zeros(8, dtype=np.int64)
    _check(lib().dsgd_oracle_metrics(C.byref(orc._csr), _p(w), _p(idx), C.c_int64(begin), C.c_int64(n), _p(margins),
                                     _p(out)), "metrics")
    return out
