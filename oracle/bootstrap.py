"""TEST INFRASTRUCTURE ONLY -- the Poisson bootstrap of dsgd_eval_*bootstrap (DESIGN.md §4.19) restated in Python.

* `mix`, `stream`, `multiplicity`, `multiplicities`: the draw of distributed_sgd_b200/csrc/dsgd_bootstrap.h.
* `thresholds`: the T_k = floor(F(k) 2^64) rebuilt exactly with fractions (e^-1 as an alternating rational series), and
  `header_thresholds` the literals the header commits.
* `replicate`: one replicate as its definition states it -- the existing checkers (oracle/metrics.py, curve.py, margin.py)
  over the expanded list, position i repeated m_i times.
* `grouped`: the same replicate from the sorted tie groups and the multiplicities, the arithmetic of k_boot_rep, in exact
  integers and fractions.
Only tests/ and tools/ use it; the product package never does.
"""
from __future__ import annotations

import math
import os
import re
from fractions import Fraction
from typing import NamedTuple

import numpy as np

from . import curve as _curve
from . import margin as _margin
from . import metrics as _metrics

M64 = (1 << 64) - 1
PHI = 0x9E3779B97F4A7C15
MAX_M = 20
HEADER = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "distributed_sgd_b200", "csrc",
                      "dsgd_bootstrap.h")


def thresholds(terms: int = 60) -> list:
    """T_k = floor(F(k) 2^64), k = 0..19, F the Poisson(1) CDF.  e^-1 = sum (-1)^j / j! is bracketed by its partial sum and
    the next term (below 2^-270 at 60 terms); both ends of the bracket must give the same floor."""
    s = sum(Fraction((-1) ** j, math.factorial(j)) for j in range(terms + 1))
    err = Fraction(1, math.factorial(terms + 1))
    out, cdf = [], Fraction(0)
    for k in range(MAX_M):
        cdf += Fraction(1, math.factorial(k))
        lo, hi = math.floor((s - err) * cdf * 2 ** 64), math.floor((s + err) * cdf * 2 ** 64)
        assert lo == hi, "the bracket of e^-1 is too wide"
        out.append(lo)
    return out


def header_thresholds() -> list:
    """The T_k literals of dsgd_bootstrap.h, in order."""
    text = open(HEADER).read()
    body = re.search(r"t\[DSGD_BOOT_MAX_M\]\s*=\s*\{(.*?)\};", text, re.S).group(1)
    return [int(x, 16) for x in re.findall(r"0x([0-9A-Fa-f]+)ull", body)]


def mix(z: int) -> int:
    z &= M64
    z = ((z ^ (z >> 30)) * 0xBF58476D1CE4E5B9) & M64
    z = ((z ^ (z >> 27)) * 0x94D049BB133111EB) & M64
    return z ^ (z >> 31)


def stream(key: int, b: int) -> int:
    return mix(int(key) + PHI * (int(b) + 1))


def multiplicity(key: int, b: int, i: int) -> int:
    u = mix(stream(key, b) + PHI * (int(i) + 1))
    return sum(1 for t in thresholds_cached() if u >= t)


_T = None


def thresholds_cached() -> list:
    global _T
    if _T is None:
        _T = thresholds()
    return _T


def multiplicities(key: int, b: int, n: int) -> np.ndarray:
    """m_i(b) of positions 0..n-1, vectorised (uint64 arithmetic wraps as the C code does)."""
    zb = np.uint64(stream(key, b))
    with np.errstate(over="ignore"):
        z = zb + np.uint64(PHI) * (np.arange(n, dtype=np.uint64) + np.uint64(1))
        z = (z ^ (z >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)
        z = (z ^ (z >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)
        u = z ^ (z >> np.uint64(31))
    return np.searchsorted(np.array(thresholds_cached(), dtype=np.uint64), u, side="right").astype(np.int64)


def expand(ids, m) -> np.ndarray:
    """The expanded list: ids[i] repeated m[i] times, in position order."""
    return np.repeat(np.asarray(ids, dtype=np.int32), np.asarray(m, dtype=np.int64))


class Replicate(NamedTuple):
    words: np.ndarray   # the 8 metrics words and the size
    ap: float
    loss: float         # the SVM's hinge sum, or the exact sum of R(L_i) of the other models (nan if an L_i is not finite)


def _r(v: float) -> Fraction:
    """R(v): v to the 2^-160 grid of the device's fixed-point sums."""
    return Fraction(round(Fraction(v) * 2 ** 160), 2 ** 160)


def row_losses(model, margins, labels) -> np.ndarray:
    """Each row's loss from its margin: the SVM's hinge 1 - y p (p = -signum(margin), 0 for NaN), else L(y margin)."""
    out = []
    for x, y in zip(margins, labels):
        if model in (None, "svm"):
            p = 0 if math.isnan(x) or x == 0 else (-1 if x > 0 else 1)
            out.append(float(1 - int(y) * p))
        else:
            out.append(_margin.row(model, float(y) * float(x))[0])
    return np.array(out, dtype=np.float64)


def _loss_sum(model, losses, m) -> float:
    """The replicate's loss sum over positions drawn at least once: a position with m = 0 adds nothing, whatever its loss
    (NaN included), as on the device."""
    drawn = [(l, int(k)) for l, k in zip(losses, m) if k > 0]
    if any(not (0.0 <= l < 2.0 ** 52) for l, _ in drawn):
        return float("nan")
    if model in (None, "svm"):
        return float(sum(int(l) * k for l, k in drawn))
    return float(sum((_r(l) * k for l, k in drawn), Fraction(0)))


def replicate(orc, model, w, ids, m, margins) -> Replicate:
    """One replicate literally: the metrics and curve checkers over the expanded list (each copy ranked by its row's margin,
    margins[i] of position i), and its loss sum."""
    ex = expand(np.arange(len(ids)), m)
    idx = np.asarray(ids, dtype=np.int32)[ex]
    mex = np.asarray(margins, dtype=np.float64)[ex]
    labels = np.asarray(orc.label)[idx] if len(idx) else np.zeros(0)
    if len(idx) == 0:
        return Replicate(np.zeros(9, np.int64), float("nan"), 0.0)
    words = _metrics.metrics(orc, w, idx=idx, margins=mex)
    ap = _curve.curve(orc, w, idx=idx, margins=mex).ap
    losses = row_losses(model, mex, labels)
    return Replicate(np.concatenate([words, [len(idx)]]).astype(np.int64), ap, _loss_sum(model, losses, np.ones(len(idx))))


def grouped(model, margins, labels, m) -> Replicate:
    """The same replicate from tie groups, as k_boot_rep forms it: scores s = -margin, highest first; per group the masses
    above (A) and through (E); U2 += N_g (2 A_P + P_g); S += P_g v, v = E_P / (E_P + E_N) one IEEE division."""
    margins = np.asarray(margins, dtype=np.float64)
    labels = np.asarray(labels)
    m = np.asarray(m, dtype=np.int64)
    words = [0] * 9
    for x, y, k in zip(margins, labels, m):
        p = 0 if math.isnan(x) or x == 0 else (-1 if x > 0 else 1)
        words[(0 if p == 1 else 1 if p == -1 else 2) + (0 if y > 0 else 3)] += int(k)
        words[7] += int(k) if math.isnan(x) else 0
        words[8] += int(k)
    groups = {}
    for x, y, k in zip(margins, labels, m):
        if not math.isnan(x):
            g = groups.setdefault(-x + 0.0, [0, 0])
            g[0 if y > 0 else 1] += int(k)
    pa = na = u2 = 0
    s = Fraction(0)
    for score in sorted(groups, reverse=True):
        pg, ng = groups[score]
        u2 += ng * (2 * pa + pg)
        pt, nt = pa + pg, na + ng
        if pg:
            s += pg * _r(float(pt) / float(pt + nt))
        pa, na = pt, nt
    words[6] = u2
    P = words[0] + words[1] + words[2]
    ap = float("nan") if words[7] or P == 0 else float(s) / P
    return Replicate(np.array(words, np.int64), ap, _loss_sum(model, row_losses(model, margins, labels), m))
