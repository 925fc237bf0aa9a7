"""Exact model of the logistic loss sum of csrc/dsgd_fixed.cuh (test infrastructure only).

A value v in [0, 2^52) contributes R(v) = rint(v * 2^160) * 2^-160 (ties to even, like CUDA's rint): the sum's resolution is
2^-160, so a value below 2^-161 contributes exactly 0.  A pass reports a double within one ulp of the exact sum of the R(v_i),
and that sum itself whenever it is a double.  A pass with a NaN, an infinity or a value of 2^52 or more reports NaN.
"""
from __future__ import annotations

import math
from fractions import Fraction
from typing import Iterable, Optional

RES_BITS = 160
MAX_VALUE = 2.0 ** 52          # the first value that is not summed
LIMB_BITS = 40


def r_units(v: float) -> Optional[int]:
    """rint(v * 2^160) as an integer, or None if v is not summed (NaN, inf, negative, >= 2^52)."""
    v = float(v)
    if not (0.0 <= v < MAX_VALUE):
        return None
    num, den = v.as_integer_ratio()            # den is a power of two
    q, r = divmod(num << RES_BITS, den)
    if 2 * r > den or (2 * r == den and q & 1):
        q += 1
    return q


def R(v: float) -> Optional[Fraction]:
    """The value one sample contributes, exactly."""
    u = r_units(v)
    return None if u is None else Fraction(u, 1 << RES_BITS)


def exact_sum(values: Iterable[float], repeat: int = 1) -> Optional[Fraction]:
    """sum_i R(v_i) over every value (each counted `repeat` times), or None (the pass reads NaN)."""
    total = 0
    for v in values:
        u = r_units(v)
        if u is None:
            return None
        total += u
    return Fraction(total * repeat, 1 << RES_BITS)


def within_one_ulp(device: float, exact: Optional[Fraction]) -> bool:
    """Whether a reported sum meets the semantics: NaN for None; the exact sum itself when it is a double; otherwise one of
    the two doubles around it, or at most one ulp of the nearest one away."""
    if exact is None:
        return math.isnan(device)
    if not math.isfinite(device):
        return False
    nearest = float(exact)                     # correctly rounded
    if Fraction(nearest) == exact:
        return device == nearest
    return abs(Fraction(device) - exact) <= Fraction(math.ulp(nearest))


def describe(device: float, exact: Optional[Fraction]) -> str:
    """Failure message: the reported and the exact sum, and their distance in ulps."""
    if exact is None:
        return f"device {device!r}, expected NaN"
    nearest = float(exact)
    ulps = float((Fraction(device) - exact) / Fraction(math.ulp(nearest))) if math.isfinite(device) else math.inf
    return f"device {device!r} ({device:.6e}), exact {nearest!r} ({nearest:.6e}), {ulps:+.3g} ulp"


def device_model(values: Iterable[float]) -> float:
    """What the device's reader computes from the limbs of `values`: six 40-bit limbs summed as integers, the carries
    propagated, then converted from the top limb down in fp64 (acc_value)."""
    q = [0] * 6
    for v in values:
        u = r_units(v)
        if u is None:
            return math.nan
        for k in range(6):
            q[k] += (u >> (LIMB_BITS * k)) & ((1 << LIMB_BITS) - 1) if k < 5 else u >> (LIMB_BITS * 5)
    for k in range(5):
        q[k + 1] += q[k] >> LIMB_BITS
        q[k] &= (1 << LIMB_BITS) - 1
    s = float(q[5]) * 2.0 ** 40
    for k in range(4, -1, -1):
        s += float(q[k]) * 2.0 ** (LIMB_BITS * k - RES_BITS)
    return s
