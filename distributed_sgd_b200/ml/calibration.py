"""Fitted probability links for a trained model: P(y = +1 | x) = 1 / (1 + exp(a x.w + b)) (Platt scaling), or the
isotonic map numpy.interp(-x.w, x, y) (IsotonicCalibration)."""
from __future__ import annotations

from dataclasses import dataclass, field

import numpy as np

CONVERGED, ITERATION_LIMIT, LINE_SEARCH_FAILED, NON_FINITE = 0, 1, 2, 3


@dataclass(frozen=True)
class Calibration:
    """(a, b) and how the fit that produced them ended.  x.w is the margin as Slave.margins returns it: a positive row has
    a negative x.w, so a fitted `a` is normally positive."""
    a: float
    b: float
    objective: float = float("nan")   # F(a, b), the regularised cross-entropy the fit minimised
    iterations: int = 0               # accepted Newton steps
    status: int = CONVERGED           # CONVERGED, ITERATION_LIMIT, LINE_SEARCH_FAILED or NON_FINITE
    rows: int = 0                     # rows the fit used
    nan_rows: int = 0                 # rows left out because their margin was NaN
    # a weighted fit (Master.calibrate(weighted=True)): every row counted by its weight c_i; W+ and W- of the rows used and
    # the weight of the NaN rows.  Left out of repr, so that an unweighted Calibration prints as it always has.
    weighted: bool = field(default=False, repr=False)
    weight_pos: float = field(default=0.0, repr=False)
    weight_neg: float = field(default=0.0, repr=False)
    nan_weight: float = field(default=0.0, repr=False)

    @staticmethod
    def identity() -> "Calibration":
        """(1, 0): the SparseLogistic model's own probability sigmoid(-x.w)."""
        return Calibration(1.0, 0.0)


METHODS = ("sigmoid", "isotonic")


@dataclass(frozen=True, eq=False)
class IsotonicCalibration:
    """An isotonic map from the score s = -x.w to P(y = +1 | x) = numpy.interp(s, x, y): x the thresholds ascending (the
    lowest and highest score of every block), y the block's value at each, and per block (ascending) its rows and positive
    rows, so that each value is positives / rows.  Compared by identity (it holds arrays)."""
    x: np.ndarray
    y: np.ndarray
    block_rows: np.ndarray
    block_pos: np.ndarray
    blocks: int = 0
    rows: int = 0                     # rows the fit used
    nan_rows: int = 0                 # rows left out because their margin was NaN
    distinct_scores: int = 0
    # a weighted fit (Master.calibrate(method="isotonic", weighted=True)): block_rows / block_pos then hold each block's
    # weight and positive weight (doubles), rows and distinct_scores count the rows and scores of positive weight, and
    # weight_pos / weight_neg are W+ and W- of the non-NaN rows.  Left out of repr.
    weighted: bool = field(default=False, repr=False)
    weight_pos: float = field(default=0.0, repr=False)
    weight_neg: float = field(default=0.0, repr=False)

    @property
    def points(self) -> int:
        return int(self.x.size)
