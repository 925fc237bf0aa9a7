"""TEST INFRASTRUCTURE ONLY -- ctypes binding of the fp64 C oracle (oracle/dsgd_oracle.c), and the one build and load of
libdsgd_oracle.so, the library every checker of this directory is compiled into (oracle/Makefile).

Only tests/, tools/, __graft_entry__ and bench.py's cpu_baseline / --impl reference legs import this.  The product package
never does.  See oracle/dsgd_oracle.h for the parity status ("parity unpinned" beyond the VecTests known answers).
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess
import tempfile
from typing import Optional, Sequence

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_NAME = "libdsgd_oracle.so"


def _make(*args: str) -> subprocess.CompletedProcess:
    return subprocess.run(["make", "-C", _HERE, *args], capture_output=True, text=True)


def _fresh(path: str) -> bool:
    """Whether the library at `path` is newer than every source and header oracle/Makefile names."""
    return _make("-q", f"LIB={path}").returncode == 0


def build(force: bool = False) -> str:
    """Compile every checker into libdsgd_oracle.so with oracle/Makefile (gcc only, no CUDA) when it is missing or older than
    its sources; returns its path.  The library sits next to its sources, or in a per-user temporary directory when this
    directory is read-only.  It is written under a temporary name and renamed into place, so a process never loads a
    half-written file."""
    path = os.path.join(_HERE, _NAME)
    if not force and _fresh(path):
        return path
    if not os.access(_HERE, os.W_OK):
        path = os.path.join(tempfile.gettempdir(), f"dsgd_oracle_{os.getuid()}", _NAME)
        os.makedirs(os.path.dirname(path), exist_ok=True)
        if not force and _fresh(path):
            return path
    tmp = f"{path}.{os.getpid()}.tmp"
    r = _make("-B", f"LIB={tmp}")
    if r.returncode != 0:
        raise RuntimeError(f"building {_NAME} failed:\n{r.stdout}{r.stderr}")
    os.replace(tmp, path)
    return path


class _Csr(C.Structure):
    _fields_ = [("n_rows", C.c_int64), ("dim", C.c_int32), ("row_ptr", C.c_void_p), ("col", C.c_void_p),
                ("val", C.c_void_p), ("label", C.c_void_p)]


_lib = None


def lib():
    """The loaded library, built on first use.  Every module of this directory loads it through here and sets the restype /
    argtypes of its own functions."""
    global _lib
    if _lib is None:
        _lib = C.CDLL(build())
        for name in ("forward", "loss_acc", "gradient", "sync_step", "sync_steps", "sync_steps_allcores", "async_delta",
                     "async_run", "dim_sparsity"):
            getattr(_lib, "dsgd_oracle_" + name).restype = C.c_int
    return _lib


def _p(a: Optional[np.ndarray]):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


class OracleError(RuntimeError):
    pass


def _check(rc: int, what: str):
    if rc != 0:
        raise OracleError(f"oracle {what} failed with code {rc} "
                          f"({ {-1: 'alloc', -2: 'index out of range', -3: 'empty batch'}.get(rc, '?')})")


class Oracle:
    """CPU oracle over one CSR data set (the `data` array a reference Slave holds, Slave.scala:20)."""

    def __init__(self, row_ptr, col, val, label, dim: int, lam: float):
        self.row_ptr = np.ascontiguousarray(row_ptr, dtype=np.int64)
        self.col = np.ascontiguousarray(col, dtype=np.int32)
        self.val = np.ascontiguousarray(val, dtype=np.float32)
        self.label = np.ascontiguousarray(label, dtype=np.int8)
        self.dim = int(dim)
        self.lam = float(lam)
        self.n_rows = len(self.row_ptr) - 1
        assert len(self.label) == self.n_rows and len(self.col) == len(self.val) == self.row_ptr[-1]
        self._csr = _Csr(self.n_rows, self.dim, _p(self.row_ptr), _p(self.col), _p(self.val), _p(self.label))
        self.d = np.zeros(self.dim, dtype=np.float64)

    # -- helpers --
    def _w(self, w):
        w = np.ascontiguousarray(w, dtype=np.float64)
        assert w.shape == (self.dim,)
        return w

    @staticmethod
    def _idx(idx):
        return np.ascontiguousarray(idx, dtype=np.int32).reshape(-1)

    def set_dim_sparsity(self, d):
        self.d = self._w(d).copy()

    def dim_sparsity(self, n_train: int) -> np.ndarray:
        out = np.zeros(self.dim, dtype=np.float64)
        _check(lib().dsgd_oracle_dim_sparsity(C.byref(self._csr), C.c_int64(n_train), _p(out)), "dim_sparsity")
        return out

    def forward(self, w, idx) -> np.ndarray:
        w, idx = self._w(w), self._idx(idx)
        out = np.zeros(len(idx), dtype=np.float64)
        _check(lib().dsgd_oracle_forward(C.byref(self._csr), _p(w), _p(idx), C.c_int64(len(idx)), _p(out)), "forward")
        return out

    def loss_acc(self, w, idx=None, begin: int = 0, n: Optional[int] = None):
        w = self._w(w)
        loss, acc = C.c_double(), C.c_double()
        if idx is not None:
            idx = self._idx(idx)
            n = len(idx)
        elif n is None:
            n = self.n_rows - begin
        _check(lib().dsgd_oracle_loss_acc(C.byref(self._csr), C.c_double(self.lam), _p(w), _p(idx), C.c_int64(begin),
                                          C.c_int64(n), C.byref(loss), C.byref(acc)), "loss_acc")
        return loss.value, acc.value

    def gradient(self, w, idx):
        w, idx = self._w(w), self._idx(idx)
        out = np.zeros(self.dim, dtype=np.float64)
        c = C.c_double()
        _check(lib().dsgd_oracle_gradient(C.byref(self._csr), C.c_double(self.lam), _p(self.d), _p(w), _p(idx),
                                          C.c_int64(len(idx)), _p(out), C.byref(c)), "gradient")
        return out, c.value

    def sync_steps(self, w, idx, counts: Sequence[int], lr: float, n_steps: int = 1, threads: int = 1):
        """Runs n_steps sync steps in place on a copy of w; returns (w_new, losses[n_steps])."""
        w = self._w(w).copy()
        idx = self._idx(idx)
        counts = np.ascontiguousarray(counts, dtype=np.int32)
        assert len(idx) == int(counts.sum()) * n_steps
        losses = np.zeros(n_steps, dtype=np.float64)
        _check(lib().dsgd_oracle_sync_steps(C.byref(self._csr), C.c_double(self.lam), _p(self.d), _p(w), _p(idx),
                                            _p(counts), C.c_int32(len(counts)), C.c_double(lr), C.c_int64(n_steps),
                                            _p(losses), C.c_int32(threads)), "sync_steps")
        return w, losses

    def sync_steps_allcores(self, w, idx, batch: int, lr: float, n_steps: int, threads: int):
        """ONE worker, its batch split over `threads` threads (context figure, not the reference's parallelism)."""
        w = self._w(w).copy()
        idx = self._idx(idx)
        assert len(idx) == batch * n_steps
        losses = np.zeros(n_steps, dtype=np.float64)
        _check(lib().dsgd_oracle_sync_steps_allcores(C.byref(self._csr), C.c_double(self.lam), _p(self.d), _p(w), _p(idx),
                                                     C.c_int64(batch), C.c_double(lr), C.c_int64(n_steps), _p(losses),
                                                     C.c_int32(threads)), "sync_steps_allcores")
        return w, losses

    def async_delta(self, w_snapshot, idx, lr: float) -> np.ndarray:
        w, idx = self._w(w_snapshot), self._idx(idx)
        out = np.zeros(self.dim, dtype=np.float64)
        _check(lib().dsgd_oracle_async_delta(C.byref(self._csr), C.c_double(self.lam), _p(self.d), _p(w), _p(idx),
                                             C.c_int64(len(idx)), C.c_double(lr), _p(out)), "async_delta")
        return out

    def async_run(self, w, idx, batch: int, lr: float) -> np.ndarray:
        w = self._w(w).copy()
        idx = self._idx(idx)
        assert len(idx) % batch == 0
        _check(lib().dsgd_oracle_async_run(C.byref(self._csr), C.c_double(self.lam), _p(self.d), _p(w), _p(idx),
                                           C.c_int32(batch), C.c_int64(len(idx) // batch), C.c_double(lr)), "async_run")
        return w
