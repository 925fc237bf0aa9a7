"""TEST INFRASTRUCTURE ONLY -- ctypes binding of the fp64 checker of every model's sync path (oracle/dsgd_oracle_margin.c):
SparseSVM, SparseLogistic, SparseSquaredHinge and SparseModifiedHuber, in every weighting, with the L1 step, rate tables and
the averaging sum.  The class-weight, sample-weight, L1 and logistic helpers (oracle/cw.py, sw.py, l1.py, logistic.py) are
calls into this module.

`model` is a name ("svm", "logistic", "squared_hinge", "modified_huber") or its number 0-3.  The weighting of a call is
the device's: sample-weighted when `sw` is given, else class-weighted when (w_pos, w_neg) != (1, 1), else unweighted.  The
library is oracle/oracle.py's.  Only tests/ and tools/ use this module; the product package never does.
"""
from __future__ import annotations

import ctypes as C
from typing import Optional, Sequence

import numpy as np

from . import oracle as _oracle
from .oracle import Oracle, _check, _p

MODELS = ("svm", "logistic", "squared_hinge", "modified_huber")


_lib = None


def lib():
    global _lib
    if _lib is None:
        _lib = _oracle.lib()
        for name in ("row", "sample_losses", "loss_acc", "gradient", "eval", "sync_steps"):
            getattr(_lib, "dsgd_oracle_margin_" + name).restype = C.c_int
        _lib.dsgd_oracle_margin_prox.restype = C.c_double
        _lib.dsgd_oracle_margin_prox.argtypes = [C.c_double, C.c_double]
        _lib.dsgd_oracle_margin_l1_norm.restype = C.c_double
        _lib.dsgd_oracle_margin_l1_norm.argtypes = [C.c_void_p, C.c_int32, C.c_void_p]
    return _lib


def model_number(model) -> int:
    return MODELS.index(model) if isinstance(model, str) else int(model)


def _weighting(sw, w_pos: float, w_neg: float) -> int:
    return 2 if sw is not None else (1 if (w_pos, w_neg) != (1.0, 1.0) else 0)


def _sw(orc: Oracle, sw):
    if sw is None:
        return None
    sw = np.ascontiguousarray(sw, dtype=np.float64)
    assert sw.size == orc.n_rows
    return sw


def row(model, z: float):
    """(L(z), s(z)) of one sample of a model other than the SVM."""
    l, s = C.c_double(), C.c_double()
    _check(lib().dsgd_oracle_margin_row(C.c_int32(model_number(model)), C.c_double(z), C.byref(l), C.byref(s)), "margin row")
    return l.value, s.value


def prox(u: float, tau: float) -> float:
    """The L1 proximal step of one value at threshold tau, the one the sync steps apply to every column."""
    return lib().dsgd_oracle_margin_prox(float(u), float(tau))


def l1_norm(w):
    """(||w||_1 as the device's fixed-point sum, #{w_j != 0})."""
    w = np.ascontiguousarray(w, dtype=np.float64)
    nnz = C.c_int64()
    return lib().dsgd_oracle_margin_l1_norm(_p(w), w.size, C.byref(nnz)), nnz.value


def sample_losses(orc: Oracle, model, w, idx=None, begin: int = 0, n: Optional[int] = None) -> np.ndarray:
    """The per-sample losses L_i of the listed rows, or of rows [begin, begin + n)."""
    if idx is not None:
        idx = orc._idx(idx)
        n = idx.size
    elif n is None:
        n = orc.n_rows - begin
    out = np.zeros(n, dtype=np.float64)
    _check(lib().dsgd_oracle_margin_sample_losses(C.byref(orc._csr), C.c_int32(model_number(model)), _p(orc._w(w)), _p(idx),
                                                  C.c_int64(begin), C.c_int64(n), _p(out)), "margin sample_losses")
    return out


def loss_acc(orc: Oracle, model, w, idx=None, begin: int = 0, n: Optional[int] = None):
    """(loss, accuracy, S, correct) of the unweighted evaluation of the listed rows, or of rows [begin, begin + n)."""
    if idx is not None:
        idx = orc._idx(idx)
        n = idx.size
    elif n is None:
        n = orc.n_rows - begin
    loss, acc, s, correct = C.c_double(), C.c_double(), C.c_double(), C.c_int64()
    _check(lib().dsgd_oracle_margin_loss_acc(C.byref(orc._csr), C.c_int32(model_number(model)), C.c_double(orc.lam),
                                             _p(orc._w(w)), _p(idx), C.c_int64(begin), C.c_int64(n), C.byref(loss),
                                             C.byref(acc), C.byref(s), C.byref(correct)), "margin loss_acc")
    return loss.value, acc.value, s.value, correct.value


def gradient(orc: Oracle, model, w, idx, w_pos: float = 1.0, w_neg: float = 1.0, sw=None, regularize: bool = True):
    """(gradient, loss, S) of one request in the weighting of (w_pos, w_neg, sw)."""
    return _gradient(orc, model, w, idx, w_pos, w_neg, sw, regularize)[:3]


def _gradient(orc: Oracle, model, w, idx, w_pos: float = 1.0, w_neg: float = 1.0, sw=None, regularize: bool = True):
    """(gradient, loss, S, c = 2 lambda (w . d) folded in column order)"""
    idx = orc._idx(idx)
    g, loss, s, c = np.zeros(orc.dim, dtype=np.float64), C.c_double(), C.c_double(), C.c_double()
    _check(lib().dsgd_oracle_margin_gradient(C.byref(orc._csr), C.c_int32(model_number(model)),
                                             C.c_int32(_weighting(sw, w_pos, w_neg)), C.c_double(orc.lam), _p(orc.d),
                                             _p(orc._w(w)), _p(idx), C.c_int64(idx.size), C.c_double(w_pos),
                                             C.c_double(w_neg), _p(_sw(orc, sw)), C.c_int32(1 if regularize else 0), _p(g),
                                             C.byref(loss), C.byref(s), C.byref(c)), "margin gradient")
    return g, loss.value, s.value, c.value


def eval_class(orc: Oracle, model, w, idx):
    """([loss sum of the y = +1 rows, of the y = -1 rows], [correct+, correct-, rows+, rows-]), as dsgd_eval*_class."""
    idx = orc._idx(idx)
    sums, counts = np.zeros(2, dtype=np.float64), np.zeros(4, dtype=np.int64)
    _check(lib().dsgd_oracle_margin_eval(C.byref(orc._csr), C.c_int32(model_number(model)), C.c_int32(1), _p(orc._w(w)),
                                         _p(idx), C.c_int64(idx.size), C.c_double(1.0), C.c_double(1.0), None, _p(sums),
                                         _p(counts)), "margin eval_class")
    return sums, counts


def eval_weighted(orc: Oracle, model, w, idx, w_pos: float = 1.0, w_neg: float = 1.0, sw=None):
    """([S, sum c_i [correct], sum c_i], [rows, correct]), as dsgd_eval*_weighted (sw None: every s_i is 1)."""
    idx = orc._idx(idx)
    sums, counts = np.zeros(3, dtype=np.float64), np.zeros(2, dtype=np.int64)
    _check(lib().dsgd_oracle_margin_eval(C.byref(orc._csr), C.c_int32(model_number(model)), C.c_int32(2), _p(orc._w(w)),
                                         _p(idx), C.c_int64(idx.size), C.c_double(w_pos), C.c_double(w_neg),
                                         _p(_sw(orc, sw)), _p(sums), _p(counts)), "margin eval_weighted")
    return sums, counts


def sync_steps(orc: Oracle, model, w, idx, counts: Sequence[int], lrs, w_pos: float = 1.0, w_neg: float = 1.0, sw=None,
               lambda1: float = 0.0, avg_sum: Optional[np.ndarray] = None):
    """len(lrs) sync steps on a copy of w with orc's rows, lambda and dimSparsity; step t at rate lrs[t], in the weighting of
    (w_pos, w_neg, sw).  Returns (w_new, losses).  avg_sum (optional, modified in place) gets the weights after every step."""
    w = orc._w(w).copy()
    idx = orc._idx(idx)
    counts = np.ascontiguousarray(counts, dtype=np.int32)
    lrs = np.ascontiguousarray(lrs, dtype=np.float64)
    assert len(idx) == int(counts.sum()) * lrs.size
    losses = np.zeros(lrs.size, dtype=np.float64)
    if avg_sum is not None:
        assert avg_sum.dtype == np.float64 and avg_sum.flags.c_contiguous and avg_sum.size == orc.dim
    _check(lib().dsgd_oracle_margin_sync_steps(C.byref(orc._csr), C.c_int32(model_number(model)),
                                               C.c_int32(_weighting(sw, w_pos, w_neg)), C.c_double(orc.lam),
                                               C.c_double(lambda1), _p(orc.d), _p(w), _p(idx), _p(counts),
                                               C.c_int32(len(counts)), _p(lrs), C.c_int64(lrs.size), C.c_double(w_pos),
                                               C.c_double(w_neg), _p(_sw(orc, sw)), _p(losses), _p(avg_sum)),
           "margin sync_steps")
    return w, losses


class MarginOracle:
    """One model's checker with the interface of oracle.Oracle (loss_acc, sample_losses, forward, gradient, sync_steps and
    the rows, lambda and dimSparsity of `orc`), in the weighting (w_pos, w_neg, sw) and with the L1 penalty lambda1 of the
    steps, so that a test written against an Oracle can take any model of this checker."""

    def __init__(self, orc: Oracle, model, w_pos: float = 1.0, w_neg: float = 1.0, sw=None, lambda1: float = 0.0):
        self.base, self.model = orc, model
        self.w_pos, self.w_neg, self.sw, self.lambda1 = w_pos, w_neg, sw, lambda1

    def __getattr__(self, name):
        return getattr(self.base, name)

    def loss_acc(self, w, idx=None, begin: int = 0, n: Optional[int] = None):
        return loss_acc(self.base, self.model, w, idx, begin, n)[:2]

    def sample_losses(self, w, idx=None, begin: int = 0, n: Optional[int] = None) -> np.ndarray:
        return sample_losses(self.base, self.model, w, idx, begin, n)

    def gradient(self, w, idx):
        """(gradient in the weighting, c = 2 lambda (w . d))"""
        g, _, _ = gradient(self.base, self.model, w, idx, self.w_pos, self.w_neg, self.sw)
        wd = self.base._w(w) * self.base.d
        return g, self.base.lam * 2.0 * float(np.sum(np.where(np.abs(wd) > 1e-20, wd, 0.0)))

    def gradient_loss(self, w, idx) -> float:
        """The loss a gradient request reports in the weighting"""
        return gradient(self.base, self.model, w, idx, self.w_pos, self.w_neg, self.sw)[1]

    def sync_steps(self, w, idx, counts: Sequence[int], lr: float, n_steps: int = 1, lrs=None, avg_sum=None):
        lrs = np.full(n_steps, lr) if lrs is None else lrs
        return sync_steps(self.base, self.model, w, idx, counts, lrs, self.w_pos, self.w_neg, self.sw,
                          lambda1=self.lambda1, avg_sum=avg_sum)
