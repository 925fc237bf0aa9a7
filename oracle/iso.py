"""TEST INFRASTRUCTURE ONLY -- the checker of the isotonic calibration calls (DESIGN.md §4.16): a ctypes binding of
oracle/dsgd_oracle_iso.c (qsort, the monotone chain in int64, numpy's interpolation and the quality sums), and beside it the
fit restated literally as pool-adjacent-violators over fractions.Fraction, which the C checker is tested against.

Both work on an array of margins f = x . w (the device's own dsgd_margins in the GPU tests) and labels; the score is s = -f.
The library is oracle/oracle.py's libdsgd_oracle.so.  Only tests/ and tools/ use it; the product package never does.
"""
from __future__ import annotations

import ctypes as C
import math
from fractions import Fraction
from typing import NamedTuple

import numpy as np

from . import oracle as _oracle


_lib = None


def lib():
    global _lib
    if _lib is None:
        _lib = _oracle.lib()
        _lib.dsgd_oracle_iso_fit.restype = C.c_int
        _lib.dsgd_oracle_iso_probs.restype = None
        _lib.dsgd_oracle_iso_quality.restype = None
    return _lib


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def _fy(f, y):
    f = np.ascontiguousarray(f, dtype=np.float64).reshape(-1)
    y = np.ascontiguousarray(np.where(np.asarray(y).reshape(-1) > 0, 1, -1), dtype=np.int8)
    assert f.size == y.size
    return f, y


class Fit(NamedTuple):
    x: np.ndarray          # thresholds, ascending score
    y: np.ndarray          # the block value at each
    block_rows: np.ndarray
    block_pos: np.ndarray
    info: np.ndarray       # blocks, points, rows used, NaN rows, distinct scores


class Quality(NamedTuple):
    brier_sum: float
    log_loss_sum: float    # over the rows whose term is finite
    bin_rows: np.ndarray
    bin_pos: np.ndarray
    bin_psum: np.ndarray
    rows: int
    left_out: int
    infinite: int          # rows whose log-loss term is infinite


# ---- the C checker ---------------------------------------------------------------------------------------------------

def fit(f, y) -> Fit:
    """The isotonic fit over margins f; raises ValueError when no margin is a number (the library's DSGD_ERR_EMPTY)."""
    f, y = _fy(f, y)
    size = max(f.size, 1)
    x, yy = np.zeros(size), np.zeros(size)
    br, bp = np.zeros(size, dtype=np.int64), np.zeros(size, dtype=np.int64)
    info, k = np.zeros(5, dtype=np.int64), C.c_int64()
    if lib().dsgd_oracle_iso_fit(_p(f), _p(y), C.c_int64(f.size), C.byref(k), _p(x), _p(yy), _p(br), _p(bp), _p(info)):
        raise ValueError("no row with a non-NaN score")
    nb = int(info[0])
    return Fit(x[:k.value].copy(), yy[:k.value].copy(), br[:nb].copy(), bp[:nb].copy(), info)


def probs(f, x, y) -> np.ndarray:
    """interp(-f, x, y) as the library computes it (numpy.interp, NaN for a NaN score)."""
    f = np.ascontiguousarray(f, dtype=np.float64).reshape(-1)
    x, y = np.ascontiguousarray(x, dtype=np.float64), np.ascontiguousarray(y, dtype=np.float64)
    out = np.zeros(f.size)
    lib().dsgd_oracle_iso_probs(_p(f), C.c_int64(f.size), _p(x), _p(y), C.c_int64(x.size), _p(out))
    return out


def quality(f, y, x, yv, n_bins: int) -> Quality:
    f, y = _fy(f, y)
    x, yv = np.ascontiguousarray(x, dtype=np.float64), np.ascontiguousarray(yv, dtype=np.float64)
    s, words = np.zeros(2), np.zeros(3, dtype=np.int64)
    rows, pos, psum = np.zeros(n_bins, dtype=np.int64), np.zeros(n_bins, dtype=np.int64), np.zeros(n_bins)
    lib().dsgd_oracle_iso_quality(_p(f), _p(y), C.c_int64(f.size), _p(x), _p(yv), C.c_int64(x.size), C.c_int32(n_bins),
                                  _p(s), _p(rows), _p(pos), _p(psum), _p(words))
    return Quality(float(s[0]), float(s[1]), rows, pos, psum, int(words[0]), int(words[1]), int(words[2]))


# ---- the literal restatement: pool-adjacent-violators in exact rationals ----------------------------------------------

def fit_literal(f, y) -> Fit:
    """Isotonic regression of o = [y > 0] on s = -f, increasing in s, by pool-adjacent-violators: the distinct scores in
    ascending order start as one block each (value = positives / rows, a Fraction); a block whose value is not below its
    successor's is pooled with it, and pooling repeats backwards while the new block is not below its predecessor.  Pooling
    equal values too makes adjacent blocks differ, the hull's vertex rule.  Each block's value is then rounded once."""
    f = np.asarray(f, dtype=np.float64).reshape(-1)
    lab = np.asarray(y).reshape(-1) > 0
    ok = ~np.isnan(f)
    s = -f[ok]
    s = np.where(s == 0.0, 0.0, s)
    o = lab[ok]
    if s.size == 0:
        raise ValueError("no row with a non-NaN score")
    uniq, inv = np.unique(s, return_inverse=True)                   # ascending; -0 and +0 are one score
    rows = np.bincount(inv, minlength=uniq.size)
    pos = np.bincount(inv, weights=o.astype(np.float64), minlength=uniq.size).astype(np.int64)
    blocks = []                                                     # [first score index, last, rows, positives]
    for i in range(uniq.size):
        blocks.append([i, i, int(rows[i]), int(pos[i])])
        while len(blocks) >= 2 and Fraction(blocks[-2][3], blocks[-2][2]) >= Fraction(blocks[-1][3], blocks[-1][2]):
            b = blocks.pop()
            blocks[-1][1] = b[1]
            blocks[-1][2] += b[2]
            blocks[-1][3] += b[3]
    xs, ys = [], []
    for first, last, r, p in blocks:
        v = float(np.float64(p) / np.float64(r))                    # one IEEE division of the exact counts
        xs.append(float(uniq[first]))
        ys.append(v)
        if last != first:
            xs.append(float(uniq[last]))
            ys.append(v)
    info = np.array([len(blocks), len(xs), int(s.size), int(f.size - s.size), int(uniq.size)], dtype=np.int64)
    return Fit(np.array(xs), np.array(ys), np.array([b[2] for b in blocks], dtype=np.int64),
               np.array([b[3] for b in blocks], dtype=np.int64), info)


def summary(q: Quality) -> dict:
    """Brier score, log loss (+inf when a term is infinite), ECE and MCE, as Master.local_calibration derives them."""
    n = q.rows
    with np.errstate(invalid="ignore", divide="ignore"):
        mean_p = np.where(q.bin_rows > 0, q.bin_psum / q.bin_rows, np.nan)
        freq = np.where(q.bin_rows > 0, q.bin_pos / q.bin_rows, np.nan)
    gap = np.abs(mean_p - freq)
    filled = q.bin_rows > 0
    return {"brier": q.brier_sum / n, "log_loss": math.inf if q.infinite else q.log_loss_sum / n,
            "ece": float(np.sum(q.bin_rows[filled] / n * gap[filled])), "mce": float(np.max(gap[filled]))}
