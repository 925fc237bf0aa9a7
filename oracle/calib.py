"""TEST INFRASTRUCTURE ONLY -- the checker of the calibration calls (DESIGN.md §4.11): a ctypes binding of
oracle/dsgd_oracle_calib.c, and beside it a literal Python restatement (math.fsum sums) that the C checker is tested against.

Both work on an array of scores f = x . w (the device's own dsgd_margins in the GPU tests) and labels.  The library is
oracle/oracle.py's libdsgd_oracle.so.  Only tests/ and tools/ use it; the product package never does.
"""
from __future__ import annotations

import ctypes as C
import math
from typing import NamedTuple

import numpy as np

from . import oracle as _oracle

CONVERGED, ITERATION_LIMIT, LINE_SEARCH_FAILED, NON_FINITE = 0, 1, 2, 3
MAX_ITER, RIDGE, GRAD_EPS, MIN_STEP, ARMIJO = 100, 1e-12, 1e-5, 1e-10, 1e-4


_lib = None


def lib():
    global _lib
    if _lib is None:
        _lib = _oracle.lib()
        _lib.dsgd_oracle_calib_fit.restype = C.c_int
        _lib.dsgd_oracle_calib_sums.restype = None
        _lib.dsgd_oracle_calib_probs.restype = None
        _lib.dsgd_oracle_calib_quality.restype = None
    return _lib


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def _fy(f, y):
    f = np.ascontiguousarray(f, dtype=np.float64).reshape(-1)
    y = np.ascontiguousarray(np.where(np.asarray(y).reshape(-1) > 0, 1, -1), dtype=np.int8)
    assert f.size == y.size
    return f, y


class Fit(NamedTuple):
    a: float
    b: float
    objective: float
    iterations: int
    status: int
    rows: int
    nan_rows: int
    evaluations: int


class Quality(NamedTuple):
    brier_sum: float
    log_loss_sum: float
    bin_rows: np.ndarray
    bin_pos: np.ndarray
    bin_psum: np.ndarray
    rows: int
    left_out: int
    edge_rows: int      # rows whose p * n_bins is within 4 ulp of an integer: another exp could bin them next door


def targets(f, y):
    """(t_pos, t_neg, B0, N+, N-, NaN rows) of the rows with a score."""
    f, y = _fy(f, y)
    ok = ~np.isnan(f)
    n_pos, n_neg = int(np.sum(ok & (y > 0))), int(np.sum(ok & (y < 0)))
    return ((n_pos + 1.0) / (n_pos + 2.0), 1.0 / (n_neg + 2.0), math.log((n_neg + 1.0) / (n_pos + 1.0)), n_pos, n_neg,
            int(np.sum(~ok)))


# ---- the C checker ---------------------------------------------------------------------------------------------------

def sums(f, y, t_pos: float, t_neg: float, a: float, b: float) -> np.ndarray:
    """{F, dF/dA, dF/dB, H_AA, H_AB, H_BB} at (a, b), without the ridge."""
    f, y = _fy(f, y)
    out = np.zeros(6)
    lib().dsgd_oracle_calib_sums(_p(f), _p(y), C.c_int64(f.size), C.c_double(t_pos), C.c_double(t_neg), C.c_double(a),
                                 C.c_double(b), _p(out))
    return out


def fit(f, y) -> Fit:
    """The Platt fit; raises ValueError when a class is missing (the library's DSGD_ERR_EMPTY)."""
    f, y = _fy(f, y)
    ab, obj, info = np.zeros(2), C.c_double(), np.zeros(5, dtype=np.int64)
    rc = lib().dsgd_oracle_calib_fit(_p(f), _p(y), C.c_int64(f.size), _p(ab), C.byref(obj), _p(info))
    if rc:
        raise ValueError("a sigmoid needs rows of both classes")
    return Fit(float(ab[0]), float(ab[1]), obj.value, *[int(v) for v in info])


def probs(f, a: float, b: float) -> np.ndarray:
    f = np.ascontiguousarray(f, dtype=np.float64).reshape(-1)
    out = np.zeros(f.size)
    lib().dsgd_oracle_calib_probs(_p(f), C.c_int64(f.size), C.c_double(a), C.c_double(b), _p(out))
    return out


def quality(f, y, a: float, b: float, n_bins: int) -> Quality:
    f, y = _fy(f, y)
    s, words, edge = np.zeros(2), np.zeros(2, dtype=np.int64), C.c_int64()
    rows, pos, psum = np.zeros(n_bins, dtype=np.int64), np.zeros(n_bins, dtype=np.int64), np.zeros(n_bins)
    lib().dsgd_oracle_calib_quality(_p(f), _p(y), C.c_int64(f.size), C.c_double(a), C.c_double(b), C.c_int32(n_bins), _p(s),
                                    _p(rows), _p(pos), _p(psum), _p(words), C.byref(edge))
    return Quality(float(s[0]), float(s[1]), rows, pos, psum, int(words[0]), int(words[1]), edge.value)


# ---- the literal restatement -------------------------------------------------------------------------------------------

def _terms(fi: float, t: float, a: float, b: float):
    z = a * fi + b
    if z >= 0.0:
        e = math.exp(-z)
        den = 1.0 + e
        return t * z + math.log1p(e), e / den, 1.0 / den
    e = math.exp(z)
    den = 1.0 + e
    return (t - 1.0) * z + math.log1p(e), 1.0 / den, e / den


def sums_literal(f, y, t_pos: float, t_neg: float, a: float, b: float) -> np.ndarray:
    cols = [[] for _ in range(6)]
    for fi, yi in zip(np.asarray(f, dtype=np.float64).tolist(), np.asarray(y).tolist()):
        if math.isnan(fi):
            continue
        t = t_pos if yi > 0 else t_neg
        term, p, q = _terms(fi, t, a, b)
        d1, d2 = t - p, p * q
        for c, v in zip(cols, (term, fi * d1, d1, (fi * fi) * d2, fi * d2, d2)):
            c.append(v)

    def total(c):
        return math.fsum(c) if all(abs(v) < 2.0 ** 52 for v in c) else float("nan")   # NaN fails the test too
    return np.array([total(c) for c in cols])


def fit_literal(f, y) -> Fit:
    t_pos, t_neg, b0, n_pos, n_neg, n_nan = targets(f, y)
    if n_pos == 0 or n_neg == 0:
        raise ValueError("a sigmoid needs rows of both classes")
    A, B, it, evals = 0.0, b0, 0, 1
    S = sums_literal(f, y, t_pos, t_neg, A, B)
    F = S[0]
    while True:
        if not np.all(np.isfinite(S)):
            return Fit(math.nan, math.nan, math.nan, it, NON_FINITE, n_pos + n_neg, n_nan, evals)
        g1, g2, h11, h21, h22 = S[1], S[2], S[3] + RIDGE, S[4], S[5] + RIDGE
        if abs(g1) < GRAD_EPS and abs(g2) < GRAD_EPS:
            status = CONVERGED
            break
        if it >= MAX_ITER:
            status = ITERATION_LIMIT
            break
        det = h11 * h22 - h21 * h21
        dA, dB = -(h22 * g1 - h21 * g2) / det, -(h11 * g2 - h21 * g1) / det
        gd = g1 * dA + g2 * dB
        step, moved = 1.0, False
        while step >= MIN_STEP:
            na, nb = A + step * dA, B + step * dB
            S = sums_literal(f, y, t_pos, t_neg, na, nb)
            evals += 1
            if not np.all(np.isfinite(S)):
                break
            if S[0] < F + ARMIJO * step * gd:
                A, B, F, moved = na, nb, S[0], True
                break
            step = step / 2.0
        if not moved:
            if np.all(np.isfinite(S)):
                status = LINE_SEARCH_FAILED
                break
            continue
        it += 1
    return Fit(float(A), float(B), float(F), it, status, n_pos + n_neg, n_nan, evals)


def summary(q: Quality) -> dict:
    """Brier score, log loss, ECE and MCE from the sums and bins, as Master.local_calibration derives them."""
    n = q.rows
    with np.errstate(invalid="ignore", divide="ignore"):
        mean_p = np.where(q.bin_rows > 0, q.bin_psum / q.bin_rows, np.nan)
        freq = np.where(q.bin_rows > 0, q.bin_pos / q.bin_rows, np.nan)
    gap = np.abs(mean_p - freq)
    filled = q.bin_rows > 0
    return {"brier": q.brier_sum / n, "log_loss": q.log_loss_sum / n,
            "ece": float(np.sum(q.bin_rows[filled] / n * gap[filled])), "mce": float(np.max(gap[filled])),
            "mean_predicted": mean_p, "observed": freq}
