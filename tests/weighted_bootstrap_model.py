"""TEST INFRASTRUCTURE ONLY -- the weighted bootstrap replicate restated from tie groups, in exact fractions.

`grouped` forms one replicate as k_wboot_rep does, from the rows (not the expanded list) and their multiplicities m: scores
s = -margin, highest first; per tie group the masses through it (E) and above it (A-) as exact sums of m R(c); at the
group's end T = read(E+), F = read(E-), B = read(2 (W- - E-) + (E- - A-)), and every non-NaN positive of the group adds
m R(fl(c B)) to U2w and, when c > 0, m R(fl(c fl(T / (T + F)))) to S_ap.  The confusion, NaN and class weights and the loss
are exact sums of m R(c) and m R(fl(c L)).  tests/test_oracle_weighted_bootstrap.py pins it against the weighted-curve
checker (oracle/wcurve.py) over the expanded list; the device is pinned against the expanded list on the GPU.
"""
from __future__ import annotations

import math
from fractions import Fraction
from typing import NamedTuple

import numpy as np

NAN = float("nan")


class XSum(NamedTuple):
    """An exact sum of R values and the number of values that could not be cut (2^52 or more, inf, NaN, negative)."""
    v: Fraction = Fraction(0)
    ovf: int = 0

    def add(self, x: float, m: int = 1) -> "XSum":
        if m == 0:
            return self
        if not (0.0 <= x < 2.0 ** 52):
            return XSum(self.v, self.ovf + m)
        return XSum(self.v + m * Fraction(round(Fraction(x) * 2 ** 160), 2 ** 160), self.ovf)

    def __add__(self, o: "XSum") -> "XSum":
        return XSum(self.v + o.v, self.ovf + o.ovf)

    def __sub__(self, o: "XSum") -> "XSum":
        return XSum(self.v - o.v, self.ovf - o.ovf)

    def read(self) -> float:
        """read(): the limbs of the exact value converted from the top down in fp64, as acc_value does; NaN on overflow."""
        if self.ovf:
            return NAN
        q = self.v * 2 ** 160
        assert q.denominator == 1 and q >= 0
        q = int(q)
        s = float(q >> 200) * 2.0 ** 40
        for i in range(4, -1, -1):
            s += float((q >> (40 * i)) & ((1 << 40) - 1)) * 2.0 ** (40 * i - 160)
        return s


def _div(a: float, b: float) -> float:
    with np.errstate(divide="ignore", invalid="ignore"):
        return float(np.float64(a) / np.float64(b))


def _mul(a: float, b: float) -> float:
    with np.errstate(over="ignore", invalid="ignore"):
        return float(np.float64(a) * np.float64(b))


class WReplicate(NamedTuple):
    size: int
    nan_rows: int
    wsums: np.ndarray   # the DSGD_WCURVE_WORDS words
    loss: float         # read() of sum m R(fl(c L))


def grouped(margins, labels, c, cl, m) -> WReplicate:
    """One weighted replicate of rows with these margins, labels (> 0: positive), weights c, terms cl = fl(c L) and
    multiplicities m."""
    margins = np.asarray(margins, np.float64)
    pos = np.asarray(labels) > 0
    c, cl, m = np.asarray(c, np.float64), np.asarray(cl, np.float64), np.asarray(m, np.int64)
    Z = XSum()
    size, nan_rows, loss = int(m.sum()), 0, Z
    conf = {k: Z for k in ("tp", "fn", "pz", "fp", "tn", "nz", "pnan", "nnan")}
    groups = {}
    for x, p, ci, li, k in zip(margins, pos, c, cl, m):
        k = int(k)
        loss = loss.add(li, k)
        if math.isnan(x):
            nan_rows += k
            conf["pnan" if p else "nnan"] = conf["pnan" if p else "nnan"].add(ci, k)
            continue
        s = -x + 0.0
        key = ("tp" if s > 0 else "fn" if s < 0 else "pz") if p else ("fp" if s > 0 else "tn" if s < 0 else "nz")
        conf[key] = conf[key].add(ci, k)
        groups.setdefault(s, []).append((p, ci, k))
    w_neg = conf["fp"] + conf["tn"] + conf["nz"]
    above_p, above_n = Z, Z
    u2, sap = Z, Z
    for s in sorted(groups, reverse=True):
        gp, gn = Z, Z
        for p, ci, k in groups[s]:
            if p:
                gp = gp.add(ci, k)
            else:
                gn = gn.add(ci, k)
        ep, en = above_p + gp, above_n + gn
        t, f = ep.read(), en.read()
        b = (w_neg + w_neg - en - en + gn).read()
        for p, ci, k in groups[s]:
            if p and k:
                u2 = u2.add(_mul(ci, b), k)
                if ci > 0.0:
                    sap = sap.add(_mul(ci, _div(t, t + f)), k)
        above_p, above_n = ep, en
    wp = conf["tp"] + conf["fn"] + conf["pz"] + conf["pnan"]
    wn = w_neg + conf["nnan"]
    words = [conf["tp"], conf["fn"], conf["pz"] + conf["pnan"], conf["fp"], conf["tn"], conf["nz"] + conf["nnan"], u2,
             conf["pnan"] + conf["nnan"], sap, conf["tp"] + conf["tn"], wp + wn, wp, wn]
    return WReplicate(size, nan_rows, np.array([x.read() for x in words]), loss.read())
