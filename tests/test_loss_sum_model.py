"""Known answers of the exact loss-sum model (tests/loss_sum_model.py) that the GPU tests of the logistic loss sum measure
the device against, and of the six-limb reader it stands for.  CPU only."""
import math
from fractions import Fraction

import numpy as np
import pytest

from loss_sum_model import MAX_VALUE, R, device_model, exact_sum, r_units, within_one_ulp

TINY = 2.0 ** -161


def test_log2_is_kept_exactly():
    # log 2 has bits down to 2^-53: far above the resolution
    assert R(math.log(2.0)) == Fraction(math.log(2.0))
    assert exact_sum([math.log(2.0)] * 3) == 3 * Fraction(math.log(2.0))
    assert exact_sum([math.log(2.0)], repeat=1 << 25) == (1 << 25) * Fraction(math.log(2.0))


def test_resolution_edges():
    assert r_units(0.0) == 0
    assert r_units(2.0 ** -160) == 1
    assert r_units(TINY) == 0                                    # a tie, to even
    assert r_units(3 * 2.0 ** -162) == 1                         # 0.75 units
    assert r_units(float(np.nextafter(TINY, 1.0))) == 1          # just above half a unit
    assert r_units(float(np.nextafter(TINY, 0.0))) == 0
    assert r_units(3 * TINY) == 2                                # 1.5 units: a tie, to even
    assert r_units(5 * TINY) == 2                                # 2.5 units: a tie, to even
    assert r_units(math.exp(-200.0)) == 0                        # softplus(-200) ~ 1.4e-87
    assert exact_sum([math.exp(-200.0)] * 1000) == 0
    assert r_units(math.exp(-100.0)) == round(Fraction(math.exp(-100.0)) * 2 ** 160)


def test_limb_boundaries():
    # limb 3 (2^-40 .. 2^-1) all ones and limb 4 zero; then the sum that carries across every limb
    v = 1.0 - 2.0 ** -40
    assert R(v) == Fraction(v)
    assert exact_sum([v, 2.0 ** -40]) == 1
    full = Fraction((1 << 200) - 1, 1 << 160)                    # limbs 0..3 all ones, limb 4 = 2^40 - 1
    assert exact_sum([2.0 ** 40 - 1.0, 1.0 - 2.0 ** -40, 2.0 ** -40 - 2.0 ** -80, 2.0 ** -80 - 2.0 ** -120,
                      2.0 ** -120 - 2.0 ** -160]) == full
    assert exact_sum([2.0 ** 40 - 1.0, 1.0 - 2.0 ** -40, 2.0 ** -40 - 2.0 ** -80, 2.0 ** -80 - 2.0 ** -120,
                      2.0 ** -120 - 2.0 ** -160, 2.0 ** -160]) == 2 ** 40


def test_not_summed():
    big = float(np.nextafter(MAX_VALUE, 0.0))
    assert big == MAX_VALUE - 0.5 and R(big) == Fraction(big)
    for v in (MAX_VALUE, math.inf, math.nan, -1.0, 1e300):
        assert r_units(v) is None
        assert exact_sum([1.0, v, 2.0]) is None


def test_within_one_ulp():
    # an exact sum that is a double must be reported exactly
    assert within_one_ulp(3.0, Fraction(3))
    assert not within_one_ulp(float(np.nextafter(3.0, 4.0)), Fraction(3))
    # otherwise within one ulp of the nearest double
    x = Fraction(1) + Fraction(1, 3 << 53)
    assert within_one_ulp(1.0, x) and within_one_ulp(1.0 + 2.0 ** -52, x)
    assert not within_one_ulp(1.0 + 2.0 ** -51, x) and not within_one_ulp(1.0 - 2.0 ** -52, x)
    assert within_one_ulp(math.nan, None) and not within_one_ulp(0.0, None)
    assert not within_one_ulp(math.nan, Fraction(1)) and not within_one_ulp(math.inf, Fraction(1))


@pytest.mark.parametrize("seed", range(6))
def test_reader_model_is_within_one_ulp(seed):
    """The limb layout and top-down conversion the device uses meet the semantics on values spread over every limb."""
    rng = np.random.default_rng(seed)
    for _ in range(40):
        n = int(rng.integers(1, 300))
        vals = np.exp(rng.uniform(-110.0, 36.0, size=n)).tolist()
        if seed % 2:
            vals += [float(rng.integers(1, 1 << 52)) - 0.5 for _ in range(int(rng.integers(0, 3)))]
        ex = exact_sum(vals)
        assert within_one_ulp(device_model(vals), ex)
    dy = [2.0 ** -40, 1.0 - 2.0 ** -40, 2.0 ** 40 - 1.0, 3.0 * 2.0 ** -160, MAX_VALUE - 0.5]
    ex = exact_sum(dy)
    assert float(ex) == ex or within_one_ulp(device_model(dy), ex)
    assert device_model([MAX_VALUE - 0.5] * 4097) == float(exact_sum([MAX_VALUE - 0.5], repeat=4097))
    assert math.isnan(device_model([1.0, MAX_VALUE]))
