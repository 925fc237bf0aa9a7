"""TEST INFRASTRUCTURE ONLY -- ctypes binding of the fp64 SparseLogistic oracle (oracle/dsgd_oracle_logistic.c).

LogisticOracle is the Oracle of oracle/oracle.py with the model-dependent calls (loss_acc, gradient, sync_steps) answered by
the logistic restatement; forward and dimSparsity do not depend on the model and stay the SVM oracle's.  The library is
built by __graft_entry__.build(), or on first use: next to its source, or in a temporary directory if that is read-only.
Only tests/ and tools/ use it; the product package never does.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess
import tempfile
from typing import Optional, Sequence

import numpy as np

from .oracle import Oracle, _check, _p

_HERE = os.path.dirname(os.path.abspath(__file__))
_SRC = os.path.join(_HERE, "dsgd_oracle_logistic.c")
_HDRS = (os.path.join(_HERE, "dsgd_oracle_logistic.h"), os.path.join(_HERE, "dsgd_oracle.h"))
_NAME = "libdsgd_oracle_logistic.so"
# the flags of oracle/Makefile: no fast-math, no contraction
_CFLAGS = ["-O3", "-march=x86-64-v3", "-fno-fast-math", "-ffp-contract=off", "-fPIC", "-Wall", "-Wextra", "-std=gnu11",
           "-shared"]


def _cc():
    return "/usr/bin/gcc" if os.path.exists("/usr/bin/gcc") else "gcc"


def _stale(path: str) -> bool:
    return (not os.path.exists(path)) or os.path.getmtime(path) < max(os.path.getmtime(f) for f in (_SRC, *_HDRS))


def build(force: bool = False) -> str:
    """Compile the logistic oracle (gcc only); returns the library's path."""
    path = os.path.join(_HERE, _NAME)
    if not force and not _stale(path):
        return path
    if not os.access(_HERE, os.W_OK):
        path = os.path.join(tempfile.gettempdir(), f"dsgd_oracle_logistic_{os.getuid()}", _NAME)
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
        for name in ("loss_acc", "sample_losses", "gradient", "sync_steps"):
            getattr(_lib, "dsgd_oracle_logistic_" + name).restype = C.c_int
    return _lib


class LogisticOracle(Oracle):
    """CPU oracle of SparseLogistic over one CSR data set (the same constructor as Oracle)."""

    def loss_acc(self, w, idx=None, begin: int = 0, n: Optional[int] = None):
        w = self._w(w)
        loss, acc = C.c_double(), C.c_double()
        if idx is not None:
            idx = self._idx(idx)
            n = len(idx)
        elif n is None:
            n = self.n_rows - begin
        _check(lib().dsgd_oracle_logistic_loss_acc(C.byref(self._csr), C.c_double(self.lam), _p(w), _p(idx),
                                                   C.c_int64(begin), C.c_int64(n), C.byref(loss), C.byref(acc)),
               "logistic loss_acc")
        return loss.value, acc.value

    def sample_losses(self, w, idx=None, begin: int = 0, n: Optional[int] = None) -> np.ndarray:
        """Per-sample losses softplus(z_i) (without lambda * ||w||^2) of the listed rows, or of rows [begin, begin + n)."""
        w = self._w(w)
        if idx is not None:
            idx = self._idx(idx)
            n = len(idx)
        elif n is None:
            n = self.n_rows - begin
        out = np.zeros(n, dtype=np.float64)
        _check(lib().dsgd_oracle_logistic_sample_losses(C.byref(self._csr), _p(w), _p(idx), C.c_int64(begin),
                                                        C.c_int64(n), _p(out)), "logistic sample_losses")
        return out

    def gradient(self, w, idx):
        w, idx = self._w(w), self._idx(idx)
        out = np.zeros(self.dim, dtype=np.float64)
        c = C.c_double()
        _check(lib().dsgd_oracle_logistic_gradient(C.byref(self._csr), C.c_double(self.lam), _p(self.d), _p(w), _p(idx),
                                                   C.c_int64(len(idx)), _p(out), C.byref(c)), "logistic gradient")
        return out, c.value

    def sync_steps(self, w, idx, counts: Sequence[int], lr: float, n_steps: int = 1, threads: int = 1):
        """Runs n_steps sync steps on a copy of w; returns (w_new, losses[n_steps]).  (Serial: `threads` is ignored.)"""
        w = self._w(w).copy()
        idx = self._idx(idx)
        counts = np.ascontiguousarray(counts, dtype=np.int32)
        assert len(idx) == int(counts.sum()) * n_steps
        losses = np.zeros(n_steps, dtype=np.float64)
        _check(lib().dsgd_oracle_logistic_sync_steps(C.byref(self._csr), C.c_double(self.lam), _p(self.d), _p(w), _p(idx),
                                                     _p(counts), C.c_int32(len(counts)), C.c_double(lr),
                                                     C.c_int64(n_steps), _p(losses)), "logistic sync_steps")
        return w, losses
