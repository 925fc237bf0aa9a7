"""Decaying learning rate of the sync steps: eta_t = lr0 / (1 + decay * t)^power, t the global step index of a fit.

power = 1 is the schedule of Bottou's svmsgd, power = 0.75 that of svmasgd (averaged SGD); decay = 0 is the reference's
constant rate.  The table is computed on the host in fp64 and handed to the device as it is (dsgd_sync_steps_lr): every
rank computes the same table from the same inputs, so nothing is exchanged, and the oracle replays the same bits."""
from __future__ import annotations

import math

import numpy as np


def check_schedule(decay: float, power: float) -> None:
    if not decay >= 0.0:
        raise ValueError(f"learning_rate_decay must be >= 0, got {decay}")
    if not power > 0.0:
        raise ValueError(f"learning_rate_power must be > 0, got {power}")


def learning_rates(lr0: float, decay: float, power: float, t_begin: int, n: int) -> np.ndarray:
    """eta_t = lr0 / (1 + decay * t)^power for t in [t_begin, t_begin + n), fp64.  Each entry depends on t alone, so a
    slice of a longer table equals the table of the slice.  decay = 0 gives lr0 exactly."""
    check_schedule(decay, power)
    lr0, decay, power = float(lr0), float(decay), float(power)
    # the C library's pow one entry at a time: the value of an entry cannot depend on where it sits in the array (a
    # vectorised power may take another code path for an array's tail)
    return np.array([lr0 / math.pow(1.0 + decay * float(t), power) for t in range(t_begin, t_begin + n)],
                    dtype=np.float64).reshape(n)
