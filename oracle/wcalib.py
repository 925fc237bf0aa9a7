"""TEST INFRASTRUCTURE ONLY -- the checker of the weighted calibration calls (DESIGN.md §4.17): a ctypes binding of
oracle/dsgd_oracle_wcalib.c, and beside it a literal Python restatement of R(v), read() and the weighted quality sums over
`fractions.Fraction`, which the C checker is tested against.

Both work on an array of scores f = x . w (the device's own dsgd_margins in the GPU tests), labels and row weights c.
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
        _lib.dsgd_oracle_wcalib_fit.restype = C.c_int
        _lib.dsgd_oracle_wcalib_sums.restype = None
        _lib.dsgd_oracle_wcalib_targets.restype = None
        _lib.dsgd_oracle_wcalib_quality.restype = None
    return _lib


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def _fyc(f, y, c):
    f = np.ascontiguousarray(f, dtype=np.float64).reshape(-1)
    y = np.ascontiguousarray(np.where(np.asarray(y).reshape(-1) > 0, 1, -1), dtype=np.int8)
    c = np.ascontiguousarray(c, dtype=np.float64).reshape(-1)
    assert f.size == y.size == c.size
    return f, y, c


class Fit(NamedTuple):
    a: float
    b: float
    objective: float
    iterations: int
    status: int
    rows: int
    nan_rows: int
    evaluations: int
    w_pos: float
    w_neg: float
    nan_weight: float


class Quality(NamedTuple):
    sums: np.ndarray         # {Brier sum, log-loss sum, weight used, infinite-term weight (0)}
    bin_weight: np.ndarray
    bin_pos_weight: np.ndarray
    bin_psum: np.ndarray
    rows: int
    left_out: int
    edge_rows: int           # rows of positive weight whose p * n_bins is within 4 ulp of an integer


# ---- the C checker ---------------------------------------------------------------------------------------------------

def targets(f, y, c):
    """({W+, W-, NaN weight}, (t+, t-, B0)) with the library's read() of each weight."""
    f, y, c = _fyc(f, y, c)
    ws, tg = np.zeros(3), np.zeros(3)
    lib().dsgd_oracle_wcalib_targets(_p(f), _p(y), _p(c), C.c_int64(f.size), _p(ws), _p(tg))
    return ws, tg


def sums(f, y, c, t_pos: float, t_neg: float, a: float, b: float) -> np.ndarray:
    f, y, c = _fyc(f, y, c)
    out = np.zeros(6)
    lib().dsgd_oracle_wcalib_sums(_p(f), _p(y), _p(c), C.c_int64(f.size), C.c_double(t_pos), C.c_double(t_neg),
                                  C.c_double(a), C.c_double(b), _p(out))
    return out


def fit(f, y, c) -> Fit:
    """The weighted Platt fit; raises ValueError when W+ or W- is 0 (the library's DSGD_ERR_EMPTY)."""
    f, y, c = _fyc(f, y, c)
    ab, obj, info, ws = np.zeros(2), C.c_double(), np.zeros(5, dtype=np.int64), np.zeros(3)
    rc = lib().dsgd_oracle_wcalib_fit(_p(f), _p(y), _p(c), C.c_int64(f.size), _p(ab), C.byref(obj), _p(info), _p(ws))
    if rc:
        raise ValueError("a sigmoid needs positive weight in both classes")
    return Fit(float(ab[0]), float(ab[1]), obj.value, *[int(v) for v in info], *[float(v) for v in ws])


def quality(f, y, c, a: float, b: float, n_bins: int) -> Quality:
    f, y, c = _fyc(f, y, c)
    s, words, edge = np.zeros(4), np.zeros(2, dtype=np.int64), C.c_int64()
    bw, bp, bs = np.zeros(n_bins), np.zeros(n_bins), np.zeros(n_bins)
    lib().dsgd_oracle_wcalib_quality(_p(f), _p(y), _p(c), C.c_int64(f.size), C.c_double(a), C.c_double(b),
                                     C.c_int32(n_bins), _p(s), _p(bw), _p(bp), _p(bs), _p(words), C.byref(edge))
    return Quality(s, bw, bp, bs, int(words[0]), int(words[1]), edge.value)


# ---- the literal restatement -------------------------------------------------------------------------------------------

def r_int(v: float) -> int:
    """R(v) in units of 2^-160: v 2^160 rounded half to even (exact: the scaling of a double by 2^160 is exact, and
    Python rounds a float to an int half to even)."""
    return round(v * 2.0 ** 160)


def read(total: int) -> float:
    """read() of an exact non-negative sum of R values given in units of 2^-160: its six 40-bit limbs converted from the
    top down, each limb a double and each step one IEEE addition."""
    mask = (1 << 40) - 1
    q = [(total >> (40 * i)) & mask for i in range(5)] + [total >> 200]
    s = float(q[5]) * 2.0 ** 40
    for i in range(4, -1, -1):
        s += float(q[i]) * 2.0 ** (40 * i - 160)
    return s


def _rsum(values) -> float:
    values = list(values)
    if not all(0.0 <= v < 2.0 ** 52 for v in values):
        return math.nan
    return read(sum(r_int(v) for v in values))


def _sigmoid(t: float) -> float:
    if t >= 0.0:
        return 1.0 / (1.0 + math.exp(-t))
    e = math.exp(t)
    return e / (1.0 + e)


def _softplus(z: float) -> float:
    return (z if z > 0.0 else 0.0) + math.log1p(math.exp(-abs(z)))


def quality_literal(f, y, c, a: float, b: float, n_bins: int):
    """(sums, bin_weight, bin_pos_weight, bin_psum, rows, left_out) of the weighted quality pass, literally."""
    brier, ll, wt = [], [], []
    bins = [([], [], []) for _ in range(n_bins)]
    rows = out = 0
    for fi, yi, ci in zip(np.asarray(f, dtype=np.float64).tolist(), np.asarray(y).tolist(),
                          np.asarray(c, dtype=np.float64).tolist()):
        z = a * fi + b
        if math.isnan(z):
            out += 1
            continue
        rows += 1
        if r_int(ci) == 0:
            continue
        pos = yi > 0
        p = _sigmoid(-z)
        d = p - (1.0 if pos else 0.0)
        brier.append(ci * (d * d))
        ll.append(ci * _softplus(z if pos else -z))
        wt.append(ci)
        k = min(int(math.floor(p * n_bins)), n_bins - 1)
        bins[k][0].append(ci)
        if pos:
            bins[k][1].append(ci)
        bins[k][2].append(ci * p)
    sums_ = np.array([_rsum(brier), _rsum(ll), _rsum(wt), 0.0])
    bw, bp, bs = (np.array([_rsum(bins[k][j]) for k in range(n_bins)]) for j in range(3))
    return sums_, bw, bp, bs, rows, out


def targets_literal(f, y, c):
    """({W+, W-, NaN weight}, (t+, t-, B0)), literally."""
    f, y, c = _fyc(f, y, c)
    nan = np.isnan(f)
    wp = _rsum(c[~nan & (y > 0)].tolist())
    wn = _rsum(c[~nan & (y < 0)].tolist())
    wnan = _rsum(c[nan].tolist())
    return np.array([wp, wn, wnan]), ((wp + 1.0) / (wp + 2.0), 1.0 / (wn + 2.0), math.log((wn + 1.0) / (wp + 1.0)))


# ---- the weighted isotonic fit ------------------------------------------------------------------------------------------

class IsoFit(NamedTuple):
    x: np.ndarray
    y: np.ndarray
    block_weight: np.ndarray
    block_pos_weight: np.ndarray
    info: tuple          # blocks, points, rows of positive weight, NaN rows, scores of positive weight
    wsums: tuple         # W+, W- of the non-NaN rows


class RangeError(ValueError):
    """The library's DSGD_ERR_RANGE: a total weight of 2^96 or more, or a weight of 2^52 or more."""


def _points(f, y, c):
    """Distinct non-NaN scores s = -f, highest first, with the exact R sums of their positive and negative rows"""
    f, y, c = _fyc(f, y, c)
    by = {}
    for fi, yi, ci in zip(f.tolist(), y.tolist(), c.tolist()):
        if math.isnan(fi):
            continue
        if not ci < 2.0 ** 52:
            raise RangeError("a weight of 2^52 or more")
        s = -fi
        s = 0.0 if s == 0.0 else s
        p, q = by.get(s, (0, 0))
        by[s] = (p + r_int(ci), q) if yi > 0 else (p, q + r_int(ci))
    return sorted(by.items(), key=lambda kv: -kv[0]), int(np.sum(np.isnan(f))), \
        int(np.sum(~np.isnan(f) & (np.round(c * 2.0 ** 160) != 0)))


def fit_isotonic(f, y, c) -> IsoFit:
    """The weighted isotonic fit as the library states it: points of non-zero weight increment, the upper concave hull of
    them and the origin with exact integer turn tests, p = fl(read(dY) / read(dX)).  Raises ValueError (DSGD_ERR_EMPTY)
    with no non-NaN row of positive weight, RangeError above the turn test's bound."""
    pts, n_nan, n_wrows = _points(f, y, c)
    wp, wn = sum(p for _, (p, _) in pts), sum(q for _, (_, q) in pts)
    if wp + wn >= 2 ** 256:
        raise RangeError("total weight 2^96 or more")
    if wp + wn == 0:
        raise ValueError("no non-NaN row of positive weight")
    xs, ys, thr, X, Y = [0], [0], [], 0, 0
    for s, (p, q) in pts:
        if p + q == 0:
            continue
        X, Y = X + p + q, Y + p
        xs.append(X)
        ys.append(Y)
        thr.append(s)
    hull = []
    for j in range(len(xs)):
        while len(hull) >= 2:
            o, a = hull[-2], hull[-1]
            if (xs[a] - xs[o]) * (ys[j] - ys[o]) - (ys[a] - ys[o]) * (xs[j] - xs[o]) >= 0:
                hull.pop()
            else:
                break
        hull.append(j)
    X_out, Y_out, bw, bp = [], [], [], []
    for b in range(len(hull) - 2, -1, -1):          # ascending in s
        i0, i1 = hull[b], hull[b + 1]
        dw, dp = read(xs[i1] - xs[i0]), read(ys[i1] - ys[i0])
        v = dp / dw
        bw.append(dw)
        bp.append(dp)
        X_out.append(thr[i1 - 1])
        Y_out.append(v)
        if i1 - i0 >= 2:
            X_out.append(thr[i0])
            Y_out.append(v)
    return IsoFit(np.array(X_out), np.array(Y_out), np.array(bw), np.array(bp),
                  (len(hull) - 1, len(X_out), n_wrows, n_nan, len(thr)), (read(wp), read(wn)))


def fit_isotonic_pav(f, y, c):
    """The same fit restated literally: weighted pool-adjacent-violators over the distinct scores (ascending), every
    weight the Fraction R(c_i), rows of zero weight dropped first, adjacent blocks pooled while the left one's mean is not
    below the right one's.  (x, y, block weights, block positive weights) with read() of each block's exact sums."""
    pts, _, _ = _points(f, y, c)
    blocks = []                                       # [W, W+, lowest score, highest score]
    for s, (p, q) in reversed(pts):
        if p + q == 0:
            continue
        blocks.append([Fraction(p + q), Fraction(p), s, s])
        while len(blocks) >= 2 and blocks[-2][1] / blocks[-2][0] >= blocks[-1][1] / blocks[-1][0]:
            w2, p2, _, hi = blocks.pop()
            blocks[-1][0] += w2
            blocks[-1][1] += p2
            blocks[-1][3] = hi
    X, Y, bw, bp = [], [], [], []
    for w_, p_, lo, hi in blocks:
        dw, dp = read(int(w_)), read(int(p_))
        X.append(lo)
        Y.append(dp / dw)
        if hi != lo:
            X.append(hi)
            Y.append(dp / dw)
        bw.append(dw)
        bp.append(dp)
    return np.array(X), np.array(Y), np.array(bw), np.array(bp)


def _interp(s, X, Y):
    return float(np.interp(s, X, Y))


def quality_isotonic(f, y, c, X, Y, n_bins: int):
    """The weighted quality pass at the map (X, Y): (sums, bin_weight, bin_pos_weight, bin_psum, words); the sums and bins
    in the library's exact R sums, p by numpy.interp as the library applies it."""
    f, y, c = _fyc(f, y, c)
    X, Y = np.asarray(X, dtype=np.float64), np.asarray(Y, dtype=np.float64)
    br, ll, wt, inf = [], [], [], []
    bins = [([], [], []) for _ in range(n_bins)]
    rows = out = n_inf = 0
    for fi, yi, ci in zip(f.tolist(), y.tolist(), c.tolist()):
        s = -fi
        if math.isnan(s):
            out += 1
            continue
        rows += 1
        if r_int(ci) == 0:
            continue
        pos = yi > 0
        p = _interp(s, X, Y)
        d = p - (1.0 if pos else 0.0)
        with np.errstate(divide="ignore"):
            term = float(-np.log(p)) if pos else float(-np.log1p(-p))
        br.append(ci * (d * d))
        if math.isinf(term):
            n_inf += 1
            inf.append(ci)
        else:
            ll.append(ci * term)
        wt.append(ci)
        k = min(int(math.floor(p * n_bins)), n_bins - 1)
        bins[k][0].append(ci)
        if pos:
            bins[k][1].append(ci)
        bins[k][2].append(ci * p)
    sums_ = np.array([_rsum(br), _rsum(ll), _rsum(wt), _rsum(inf)])
    bw, bp, bs = (np.array([_rsum(bins[k][j]) for k in range(n_bins)]) for j in range(3))
    return sums_, bw, bp, bs, (rows, out, n_inf)
