"""A CPU model of how the streaming pass (k_stream_rows, csrc/dsgd_stream.cuh) decides one row: the fp32 dot against the
fp32 shadow of the weights, bit for bit, and the rounding band that sends the row to the fp64 row fold.

The model restates the kernel's arithmetic for a row whose first unit sits at virtual position `start` of its block (lane
start mod 32; start 0: the row is the first non-empty row of its block):
  * k_repack: a value |x| <= 1e-20 is stored as 0; a row of L pairs is padded to ceil(L / 2) 16-byte units with
    (last column, 0); yabs is sum |x| in fp64 (pair k on lane k mod 32, lane sums in order, xor butterfly), rounded up to fp32;
  * w32 = (float)w for every column, and max|w32| over all of them with fmaxf (a NaN weight is skipped);
  * unit u = (c0, x0, c1, x1): pp = fma(x1, w32[c1], x0 * w32[c0]) in fp32, the fma rounded once;
  * unit u is added to the running sum of lane (start + u) mod 32, in order, from +0; the row's dot is the xor butterfly
    over offsets 16, 8, 4, 2, 1 of the 32 lane sums (lanes without a unit of the row hold +0);
  * the decision, with the kernel's own operations and types (numpy float32 / float64 operations round like the device's,
    which is built with --fmad=false and without flush-to-zero).

decide() returns, per row, +1 or -1 (the pass takes x.w > 0 or < 0 from the fp32 dot; its prediction is the negation) or
0 (the row goes to the fp64 row fold).  fp32_band=True restates the earlier rule, before non-finite dots and subnormal
weights were handled: an fp32 threshold 1.5 * 2^-24 * max|w32| * yabs * (units/32 + 10) + 2e-20 * units, and any |dot|
above it decided.
"""
from fractions import Fraction
import math

import numpy as np

EPS = 1e-20                                    # the reference's filter (Sparse constructor)
FLT_MAX = float(np.finfo(np.float32).max)
TWO_M24 = 2.0 ** -24
TWO_M126 = 2.0 ** -126                         # smallest normal fp32
RECOMPUTE = 0


def shadow(w):
    """The fp32 shadow of fp64 weights (k_to_f32): round to nearest, |w| beyond FLT_MAX + half an ulp to +-inf."""
    with np.errstate(over="ignore", invalid="ignore"):
        return np.asarray(w, np.float64).astype(np.float32)


def shadow_max(w32):
    """max|w32| as the kernel's staging takes it: fmaxf from +0, which skips NaN."""
    a = np.abs(np.asarray(w32, np.float32))
    a = a[~np.isnan(a)]
    return np.float32(a.max()) if a.size else np.float32(0.0)


def _fma32(a, b, c):
    """fp32 fma(a, b, c) rounded once: a * b is exact in fp64, the fp64 sum with c is rounded to odd, and rounding to odd
    in 53 bits then to nearest in 24 bits is the correctly rounded result."""
    with np.errstate(all="ignore"):
        p = a.astype(np.float64) * b.astype(np.float64)
        cc = c.astype(np.float64)
        s = p + cc
        bp = s - p
        e = (p - (s - bp)) + (cc - bp)                              # exact error of s (TwoSum), when everything is finite
        fix = np.isfinite(s) & np.isfinite(e) & (e != 0) & ((s.view(np.int64) & 1) == 0)
        s[fix] = np.nextafter(s[fix], np.where(e[fix] > 0, np.inf, -np.inf))
        return s.astype(np.float32)


def _round_up_f32(a):
    """__double2float_ru"""
    with np.errstate(over="ignore"):
        f = a.astype(np.float32)
    lo = f.astype(np.float64) < a
    f[lo] = np.nextafter(f[lo], np.float32(np.inf))
    return f


def _units(rows):
    """Per row (cols, filtered values) of its padded pair window."""
    out = []
    for cols, vals in rows:
        c = np.asarray(cols, np.int64)
        v = np.asarray(vals, np.float32)
        v = np.where(np.abs(v.astype(np.float64)) > EPS, v, np.float32(0.0)).astype(np.float32)
        if c.size % 2:
            c = np.append(c, c[-1])
            v = np.append(v, np.float32(0.0))
        out.append((c, v))
    return out


def yabs(rows):
    """|yabs| of each row as k_repack stores it."""
    res = np.zeros(len(rows), np.float32)
    for i, (c, v) in enumerate(_units(rows)):
        if c.size == 0:
            continue
        k = c.size
        lanes = np.zeros(32)
        a = np.abs(v.astype(np.float64))
        for j in range(0, k, 32):                                 # lane l adds pairs l, l + 32, ... in order
            seg = a[j:j + 32]
            lanes[:seg.size] = lanes[:seg.size] + seg
        for o in (16, 8, 4, 2, 1):
            lanes = lanes + lanes[np.arange(32) ^ o]
        res[i] = _round_up_f32(np.array([lanes[0]]))[0]
    return res


def dot32(rows, w32, start=None):
    """The fp32 dot of each row at virtual start position start[i] (default 0), bit for bit."""
    R = len(rows)
    start = np.zeros(R, np.int64) if start is None else np.asarray(start, np.int64) % 32
    units = _units(rows)
    n_units = np.array([c.size // 2 for c, _ in units], np.int64)
    M = max(32, int(((start + n_units).max() + 31) // 32 * 32)) if R else 32
    X0, X1 = np.zeros((R, M), np.float32), np.zeros((R, M), np.float32)
    C0, C1 = np.zeros((R, M), np.int64), np.zeros((R, M), np.int64)
    live = np.zeros((R, M), bool)
    for i, (c, v) in enumerate(units):
        u = n_units[i]
        sl = slice(int(start[i]), int(start[i] + u))
        X0[i, sl], X1[i, sl] = v[0::2], v[1::2]
        C0[i, sl], C1[i, sl] = c[0::2], c[1::2]
        live[i, sl] = True
    w32 = np.asarray(w32, np.float32)
    with np.errstate(all="ignore"):
        pp = _fma32(X1, w32[C1], X0 * w32[C0])
        pp[~live] = np.float32(0.0)
        lanes = np.zeros((R, 32), np.float32)
        for j in range(0, M, 32):                                # each lane's running sum, unit by unit
            lanes = lanes + pp[:, j:j + 32]
        for o in (16, 8, 4, 2, 1):
            lanes = lanes + lanes[:, np.arange(32) ^ o]
    return lanes[:, 0], n_units


def thresholds(ya, n_units, wmax, fp32_band=False):
    """The band of each row, in the kernel's types and order of operations."""
    ya = np.abs(np.asarray(ya, np.float32))
    k = (np.asarray(n_units, np.int64) >> 5) + 10
    with np.errstate(all="ignore"):
        if fp32_band:
            band_scale = np.float32(1.5) * np.float32(TWO_M24) * np.float32(wmax)
            return band_scale * ya * k.astype(np.float32) + np.float32(2e-20) * np.asarray(n_units).astype(np.float32)
        band_scale = 1.5 * TWO_M24 * max(float(wmax), TWO_M126)
        return band_scale * ya.astype(np.float64) * k.astype(np.float64) + 2e-20 * np.asarray(n_units).astype(np.float64)


def decide(rows, w, start=None, fp32_band=False):
    """(decision, dot32, threshold) of each row (cols, vals) at the fp64 weights w: decision +1 / -1 is the sign the pass
    takes from the fp32 dot, 0 (RECOMPUTE) sends the row to the fp64 row fold.  An empty row (no pairs) is never streamed
    through the band (the pass scores it 0 itself); its decision here is RECOMPUTE and callers skip it."""
    w32 = shadow(w)
    d, n_units = dot32(rows, w32, start)
    t = thresholds(yabs(rows), n_units, shadow_max(w32), fp32_band)
    with np.errstate(invalid="ignore"):
        a = np.abs(d)
        if fp32_band:
            ok = a > t
        else:
            ok = (a <= np.float32(FLT_MAX)) & (a.astype(np.float64) > t)
    dec = np.where(ok, np.where(d > 0, 1, -1), RECOMPUTE).astype(np.int64)
    dec[n_units == 0] = RECOMPUTE
    return dec, d, t


def decide_starts(rows, w, fp32_band=False):
    """decide() of every row at each of the 32 start lanes: an (R, 32) array."""
    w32 = shadow(w)
    t = None
    out = np.zeros((len(rows), 32), np.int64)
    for s in range(32):
        d, n_units = dot32(rows, w32, np.full(len(rows), s))
        if t is None:
            t = thresholds(yabs(rows), n_units, shadow_max(w32), fp32_band)
        with np.errstate(invalid="ignore"):
            a = np.abs(d)
            ok = (a > t) if fp32_band else ((a <= np.float32(FLT_MAX)) & (a.astype(np.float64) > t))
        out[:, s] = np.where(ok, np.where(d > 0, 1, -1), RECOMPUTE)
        out[n_units == 0, s] = RECOMPUTE
    return out


def exact_sign(cols, vals, w):
    """Sign of sum filt(filt(x) * w) over the fp64 products, summed exactly (Fraction); a product that is NaN is dropped
    by the filter (fabs(NaN) > 1e-20 is false), infinite products follow IEEE: +inf and -inf together give 0 (the fp64 sum
    is NaN, which predicts 0)."""
    s, pinf, ninf = Fraction(0), False, False
    for c, x in zip(cols, vals):
        xv = float(np.float32(x))
        xv = xv if abs(xv) > EPS else 0.0
        with np.errstate(all="ignore"):
            p = float(np.float64(xv) * np.float64(w[c]))
        if not abs(p) > EPS:
            continue
        if math.isinf(p):
            pinf, ninf = pinf or p > 0, ninf or p < 0
        else:
            s += Fraction(p)
    if pinf or ninf:
        return 0 if (pinf and ninf) else (1 if pinf else -1)
    return (s > 0) - (s < 0)


def block_starts(n, sm_count):
    """Virtual start positions are counted from the first row of each block: the first pass position of the block that
    holds each position, as stream_launch (csrc/dsgd_api.cu) splits a pass of n rows over sm_count SMs."""
    W = 32 * sm_count
    rlog = 5
    while rlog > 3 and ((n + (1 << rlog) - 1) >> rlog) < 6 * W:
        rlog -= 1
    tlog = max(3, rlog - 1)
    n_big = ((n - n // 5) >> rlog) if tlog < rlog else ((n + (1 << rlog) - 1) >> rlog)
    pos = np.arange(n, dtype=np.int64)
    tail0 = n_big << rlog
    return np.where(pos < tail0, (pos >> rlog) << rlog, tail0 + (((pos - tail0) >> tlog) << tlog))


def pass_starts(n_units_of_pass, sm_count):
    """The virtual start position of each row of a pass (its units, in pass order): the units of the rows before it in
    its block (empty rows take none)."""
    u = np.asarray(n_units_of_pass, np.int64)
    first = block_starts(u.size, sm_count)
    cs = np.concatenate([[0], np.cumsum(u)])
    return cs[:-1] - cs[first]
