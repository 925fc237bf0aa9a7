"""TEST INFRASTRUCTURE ONLY -- ctypes binding of the fp64 weighted-curve checker (oracle/dsgd_oracle_wcurve.c).

`wcurve` answers for rows given by their margins (the device's own, from dsgd_margins), labels and weights c_i; `weights`
forms c_i = fl(w_y * s_i) as the device does.  The library is built by __graft_entry__.build(), or on first use: next to
its source, or in a temporary directory if that is read-only.  Only tests/ and tools/ use it; the product package never
does.
"""
from __future__ import annotations

import ctypes as C
import math
import os
import subprocess
import tempfile
from typing import NamedTuple

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_SRCS = (os.path.join(_HERE, "dsgd_oracle_wcurve.c"),)
_NAME = "libdsgd_oracle_wcurve.so"
# the flags of oracle/Makefile: no fast-math, no contraction
_CFLAGS = ["-O3", "-march=x86-64-v3", "-fno-fast-math", "-ffp-contract=off", "-fPIC", "-Wall", "-Wextra", "-std=gnu11",
           "-shared"]
WCURVE_WORDS = 13


def _cc():
    return "/usr/bin/gcc" if os.path.exists("/usr/bin/gcc") else "gcc"


def _stale(path: str) -> bool:
    return (not os.path.exists(path)) or os.path.getmtime(path) < max(os.path.getmtime(f) for f in _SRCS)


def build(force: bool = False) -> str:
    """Compile the weighted-curve checker (gcc only); returns the library's path."""
    path = os.path.join(_HERE, _NAME)
    if not force and not _stale(path):
        return path
    if not os.access(_HERE, os.W_OK):
        path = os.path.join(tempfile.gettempdir(), f"dsgd_oracle_wcurve_{os.getuid()}", _NAME)
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
        _lib.dsgd_oracle_wcurve.restype = C.c_int
        _lib.dsgd_oracle_wcurve_read.restype = C.c_double
        _lib.dsgd_oracle_wcurve_read.argtypes = [C.c_void_p, C.c_int64]
    return _lib


def _p(a):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


class WCurve(NamedTuple):
    words: np.ndarray    # the DSGD_METRICS_WORDS metrics words (counts, U2)
    wsums: np.ndarray    # the DSGD_WCURVE_WORDS weighted words of include/dsgd.h
    thr: np.ndarray      # distinct scores, highest first
    tpw: np.ndarray      # W+(>= thr[k])
    fpw: np.ndarray      # W-(>= thr[k])
    auc: float
    ap: float


def weights(label, w_pos: float = 1.0, w_neg: float = 1.0, sw=None) -> np.ndarray:
    """c_i = fl(w_y * s_i) of rows with these labels (sw None: every s_i is 1), the expression of the device."""
    label = np.asarray(label)
    wy = np.where(label > 0, w_pos, w_neg).astype(np.float64)
    return wy * (np.ones(label.size) if sw is None else np.asarray(sw, dtype=np.float64))


def auc_ap(words, wsums) -> tuple:
    """(weighted ROC AUC, weighted AP) from the words: U2w / (2 W+ W-) and S_ap / W+, with the NaN and W- = 0 rules."""
    nan, wp, wn = int(words[7]) > 0, float(wsums[11]), float(wsums[12])
    auc = math.nan if nan or wp == 0.0 or wn == 0.0 else float(wsums[6]) / (2.0 * wp * wn)
    ap = math.nan if nan or wp == 0.0 else 1.0 if wn == 0.0 else float(wsums[8]) / wp
    return auc, ap


def wcurve(margins, label, c, points: bool = True) -> WCurve:
    """The weighted curve of rows with these margins, labels (> 0: positive) and weights."""
    margins = np.ascontiguousarray(margins, dtype=np.float64)
    label = np.ascontiguousarray(np.asarray(label) > 0, dtype=np.int8)
    c = np.ascontiguousarray(c, dtype=np.float64)
    n = margins.size
    assert label.size == n and c.size == n
    words, wsums, m = np.zeros(8, dtype=np.int64), np.zeros(WCURVE_WORDS), C.c_int64()
    size = max(n, 1)
    thr, tpw, fpw = (np.zeros(size), np.zeros(size), np.zeros(size)) if points else (None, None, None)
    rc = lib().dsgd_oracle_wcurve(_p(margins), _p(label), _p(c), C.c_int64(n), _p(words), _p(wsums), C.byref(m), _p(thr),
                                  _p(tpw), _p(fpw))
    if rc:
        raise RuntimeError(f"dsgd_oracle_wcurve failed: {rc}")
    k = m.value
    auc, ap = auc_ap(words, wsums)
    if not points:
        thr = tpw = fpw = np.zeros(0)
        k = 0
    return WCurve(words, wsums, thr[:k].copy(), tpw[:k].copy(), fpw[:k].copy(), auc, ap)


def read(values) -> float:
    """read() of the exact sum of R(v) over the values, as the checker (and the device's acc_value) computes it."""
    v = np.ascontiguousarray(values, dtype=np.float64)
    return lib().dsgd_oracle_wcurve_read(_p(v), C.c_int64(v.size))


def literal(margins, label, c) -> tuple:
    """A literal restatement with fractions.Fraction: (exact AUC, exact AP) over the rows, with R(v) as
    tests/loss_sum_model.py states it and every product and division taken exactly -- no read() or fl() between the steps.  Its AUC and AP are the exact values the device's are within a few ulps of."""
    from fractions import Fraction
    R = lambda v: Fraction(round(Fraction(v) * 2 ** 160)) / 2 ** 160 if 0.0 <= v < 2.0 ** 52 else None  # noqa: E731
    rows = [(float(m), bool(y > 0), float(ci)) for m, y, ci in zip(margins, label, c)]
    ok = [(-m if m != 0.0 else 0.0, y, ci) for m, y, ci in rows if m == m]
    if len(ok) < len(rows):
        return math.nan, math.nan
    Wp = sum((R(ci) for s, y, ci in ok if y), Fraction(0))
    Wn = sum((R(ci) for s, y, ci in ok if not y), Fraction(0))
    u2 = Fraction(0)
    sap = Fraction(0)
    for s, y, ci in ok:
        if not y:
            continue
        below = sum((R(cj) for t, yj, cj in ok if not yj and t < s), Fraction(0))
        eq = sum((R(cj) for t, yj, cj in ok if not yj and t == s), Fraction(0))
        u2 += Fraction(ci) * (2 * below + eq)
        if ci > 0:
            T = sum((R(cj) for t, yj, cj in ok if yj and t >= s), Fraction(0))
            F = sum((R(cj) for t, yj, cj in ok if not yj and t >= s), Fraction(0))
            sap += Fraction(ci) * T / (T + F)
    auc = math.nan if Wp == 0 or Wn == 0 else u2 / (2 * Wp * Wn)
    ap = math.nan if Wp == 0 else Fraction(1) if Wn == 0 else sap / Wp
    return auc, ap
