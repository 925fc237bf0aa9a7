"""TEST INFRASTRUCTURE ONLY -- ctypes binding of the fp64 scores and ranking-metrics checker (oracle/dsgd_oracle_metrics.c).

`margins` and `metrics` answer for an Oracle of oracle/oracle.py (its CSR).  The library is built by
__graft_entry__.build(), or on first use: next to its source, or in a temporary directory if that is read-only.  Only
tests/ and tools/ use it; the product package never does.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess
import tempfile
from typing import Optional

import numpy as np

from .oracle import Oracle, _check, _p

_HERE = os.path.dirname(os.path.abspath(__file__))
_SRC = os.path.join(_HERE, "dsgd_oracle_metrics.c")
_HDRS = (os.path.join(_HERE, "dsgd_oracle.h"),)
_NAME = "libdsgd_oracle_metrics.so"
# the flags of oracle/Makefile: no fast-math, no contraction
_CFLAGS = ["-O3", "-march=x86-64-v3", "-fno-fast-math", "-ffp-contract=off", "-fPIC", "-Wall", "-Wextra", "-std=gnu11",
           "-shared"]


def _cc():
    return "/usr/bin/gcc" if os.path.exists("/usr/bin/gcc") else "gcc"


def _stale(path: str) -> bool:
    return (not os.path.exists(path)) or os.path.getmtime(path) < max(os.path.getmtime(f) for f in (_SRC, *_HDRS))


def build(force: bool = False) -> str:
    """Compile the metrics checker (gcc only); returns the library's path."""
    path = os.path.join(_HERE, _NAME)
    if not force and not _stale(path):
        return path
    if not os.access(_HERE, os.W_OK):
        path = os.path.join(tempfile.gettempdir(), f"dsgd_oracle_metrics_{os.getuid()}", _NAME)
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
