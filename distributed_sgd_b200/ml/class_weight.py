"""Class weights of a model: one weight per label, acting on the model's backward and loss in sync training.

A model's `class_weight` field is None (every row weighs 1), a pair (w_pos, w_neg) for the rows labelled +1 and -1, or
"balanced": w_c = n / (2 n_c) from the label counts of the train rows, so that both classes carry the same total weight
and the weights average to 1 over the rows.
"""
from __future__ import annotations

import math
from typing import Tuple

import numpy as np


def parse_class_weight(raw: str):
    """The configuration value: `none`, `balanced` or `w_pos,w_neg`."""
    raw = raw.strip().strip('"').strip().lower()
    if raw in ("", "none"):
        return None
    if raw == "balanced":
        return "balanced"
    parts = raw.split(",")
    if len(parts) != 2:
        raise ValueError(f"class-weight: expected none, balanced or w_pos,w_neg, got {raw!r}")
    return _checked((float(parts[0]), float(parts[1])))


def _checked(pair) -> Tuple[float, float]:
    w_pos, w_neg = float(pair[0]), float(pair[1])
    if not (math.isfinite(w_pos) and w_pos >= 0.0 and math.isfinite(w_neg) and w_neg >= 0.0):
        raise ValueError(f"class_weight: both weights must be finite and >= 0, got ({w_pos}, {w_neg})")
    return w_pos, w_neg


def resolve_class_weight(class_weight, train_labels) -> Tuple[float, float]:
    """(w_pos, w_neg) of a model's class_weight over the train rows' labels; (1.0, 1.0) for None."""
    if class_weight is None:
        return 1.0, 1.0
    if isinstance(class_weight, str):
        if class_weight != "balanced":
            raise ValueError(f"class_weight: expected None, a pair or 'balanced', got {class_weight!r}")
        labels = np.asarray(train_labels)
        n_pos, n_neg = int(np.count_nonzero(labels > 0)), int(np.count_nonzero(labels < 0))
        if n_pos == 0 or n_neg == 0:
            raise ValueError(f"class_weight='balanced': the train rows hold {n_pos} positive and {n_neg} negative labels; "
                             "both classes are needed")
        n = n_pos + n_neg
        return n / (2.0 * n_pos), n / (2.0 * n_neg)
    if len(class_weight) != 2:
        raise ValueError(f"class_weight: expected None, a pair or 'balanced', got {class_weight!r}")
    return _checked(class_weight)
