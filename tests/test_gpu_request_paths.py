"""Every request entry point of the C ABI: forward, gradient, margins, probabilities, and the 46 evaluation entry points --
dsgd_eval and fifteen families in three row forms each (a range, a device-drawn sample, a list of ids): counts, sums, the
per-class and weighted tallies, metrics, curves and weighted curves, the Platt and isotonic fits and their quality passes,
counted and weighted.

* The kernels one call launches (the dsgd_launch_count delta), on an SVM and a logistic context, over fewer and more ids than
  kStreamMinRows (2048, csrc/dsgd_api.cu) where the SVM's streaming pass takes over; with the resident weights and with the
  same weights passed in, which must give the same bits.  The logistic gradient adds to g with fp64 atomics in the order the
  rows arrive, so its gradient agrees to rounding and its loss (a fixed-point sum) to the bit.
* The error each bad argument gets on its own, a message that names the entry point that was called, and no launch: every
  check before a pass runs before its first kernel.
* A list of more ids than rows is refused while an async loop is started, even after the loop ended by itself: growing a
  buffer then would wait for every kernel on the device, and a loop that runs until stopped never ends."""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LAM = 1e-4
N_ROWS = 6000
KEY = 0x9E3779B97F4A7C15
SIZES = {"small": 300, "large": 4000}          # ids (or rows) of one call: below and above kStreamMinRows
SIGMOID = (1.5, -0.25)                         # (a, b) of the Platt quality calls
MAP = (np.array([-2.0, 0.0, 2.0]), np.array([0.2, 0.5, 0.8]))   # a valid map (X, Y) for the isotonic quality calls
MAX_BINS = 64                                  # DSGD_CALIBRATION_MAX_BINS

# The evaluation families: dsgd_<family> over a range, and its drawn-sample and id-list forms (dsgd_eval has only the
# range form), with the arguments each wrapper takes after the rows
EVAL_FAMILIES = {"eval_counts": (), "eval_sums": (), "eval_class": (), "eval_weighted": (), "eval_metrics": (),
                 "eval_curve": (), "eval_weighted_curve": (), "calibrate": (), "calibrate_weighted": (),
                 "eval_calibration": SIGMOID, "eval_weighted_calibration": SIGMOID, "calibrate_isotonic": (),
                 "eval_isotonic_calibration": MAP, "calibrate_isotonic_weighted": (),
                 "eval_weighted_isotonic_calibration": MAP}


def row_forms(family):
    """{entry point: its form} of one evaluation family"""
    if family.startswith("calibrate"):
        return {family: "range", family + "_sampled": "drawn", family + "_samples": "list"}
    rest = family[len("eval_"):]
    return {family: "range", "eval_sampled_" + rest: "drawn", "eval_samples_" + rest: "list"}


FORM = {"forward": "list", "gradient": "list", "eval": "range", "margins": "list", "probabilities": "list"}
FAMILY = {name: name for name in FORM}
for _f in EVAL_FAMILIES:
    FORM.update(row_forms(_f))
    FAMILY.update({name: _f for name in row_forms(_f)})


def _request(name):
    """one call of entry point `name` over the rows that `ids` stands for, with weights w (None: the resident ones)"""
    extra, form = EVAL_FAMILIES.get(FAMILY[name], ()), FORM[name]
    if name in ("forward", "margins", "probabilities"):
        return lambda c, ids, w: getattr(c, name)(ids, w)
    if name == "gradient":
        return lambda c, ids, w: c.gradient(ids, w, want_loss=True)
    if form == "range":
        return lambda c, ids, w: getattr(c, name)(7, 7 + ids.size, *extra, w=w)
    if form == "drawn":
        return lambda c, ids, w: getattr(c, name)(7, N_ROWS, KEY, 5, 5 + ids.size, *extra, w=w)
    return lambda c, ids, w: getattr(c, name)(ids, *extra, w=w)


REQUESTS = {name: _request(name) for name in FORM}
SVM_ONLY = {"eval_counts", "eval_sampled_counts", "eval_samples_counts"}
LOGISTIC_ONLY = {"probabilities"}

# (model, size, entry point) -> launch_count() delta of one call (resident weights, weights passed in)
LAUNCHES = {
    ('svm', 'large', 'forward'): (1, 3),
    ('svm', 'large', 'gradient'): (3, 5),
    ('svm', 'large', 'eval'): (2, 4),
    ('svm', 'large', 'margins'): (1, 3),
    ('svm', 'large', 'eval_counts'): (2, 4),
    ('svm', 'large', 'eval_sampled_counts'): (3, 5),
    ('svm', 'large', 'eval_samples_counts'): (2, 4),
    ('svm', 'large', 'eval_sums'): (2, 4),
    ('svm', 'large', 'eval_sampled_sums'): (3, 5),
    ('svm', 'large', 'eval_samples_sums'): (2, 4),
    ('svm', 'large', 'eval_class'): (2, 4),
    ('svm', 'large', 'eval_sampled_class'): (3, 5),
    ('svm', 'large', 'eval_samples_class'): (2, 4),
    ('svm', 'large', 'eval_weighted'): (2, 4),
    ('svm', 'large', 'eval_sampled_weighted'): (3, 5),
    ('svm', 'large', 'eval_samples_weighted'): (2, 4),
    ('svm', 'large', 'eval_metrics'): (2, 4),
    ('svm', 'large', 'eval_sampled_metrics'): (3, 5),
    ('svm', 'large', 'eval_samples_metrics'): (2, 4),
    ('svm', 'large', 'eval_curve'): (4, 6),
    ('svm', 'large', 'eval_sampled_curve'): (5, 7),
    ('svm', 'large', 'eval_samples_curve'): (4, 6),
    ('svm', 'large', 'eval_weighted_curve'): (4, 6),
    ('svm', 'large', 'eval_sampled_weighted_curve'): (5, 7),
    ('svm', 'large', 'eval_samples_weighted_curve'): (4, 6),
    ('svm', 'large', 'calibrate'): (2, 4),
    ('svm', 'large', 'calibrate_sampled'): (3, 5),
    ('svm', 'large', 'calibrate_samples'): (2, 4),
    ('svm', 'large', 'calibrate_weighted'): (2, 4),
    ('svm', 'large', 'calibrate_weighted_sampled'): (3, 5),
    ('svm', 'large', 'calibrate_weighted_samples'): (2, 4),
    ('svm', 'large', 'eval_calibration'): (2, 4),
    ('svm', 'large', 'eval_sampled_calibration'): (3, 5),
    ('svm', 'large', 'eval_samples_calibration'): (2, 4),
    ('svm', 'large', 'eval_weighted_calibration'): (1, 3),
    ('svm', 'large', 'eval_sampled_weighted_calibration'): (2, 4),
    ('svm', 'large', 'eval_samples_weighted_calibration'): (1, 3),
    ('svm', 'large', 'calibrate_isotonic'): (7, 9),
    ('svm', 'large', 'calibrate_isotonic_sampled'): (8, 10),
    ('svm', 'large', 'calibrate_isotonic_samples'): (7, 9),
    ('svm', 'large', 'eval_isotonic_calibration'): (2, 4),
    ('svm', 'large', 'eval_sampled_isotonic_calibration'): (3, 5),
    ('svm', 'large', 'eval_samples_isotonic_calibration'): (2, 4),
    ('svm', 'large', 'calibrate_isotonic_weighted'): (9, 11),
    ('svm', 'large', 'calibrate_isotonic_weighted_sampled'): (10, 12),
    ('svm', 'large', 'calibrate_isotonic_weighted_samples'): (9, 11),
    ('svm', 'large', 'eval_weighted_isotonic_calibration'): (1, 3),
    ('svm', 'large', 'eval_sampled_weighted_isotonic_calibration'): (2, 4),
    ('svm', 'large', 'eval_samples_weighted_isotonic_calibration'): (1, 3),
    ('svm', 'small', 'forward'): (1, 3),
    ('svm', 'small', 'gradient'): (3, 5),
    ('svm', 'small', 'eval'): (2, 4),
    ('svm', 'small', 'margins'): (1, 3),
    ('svm', 'small', 'eval_counts'): (2, 4),
    ('svm', 'small', 'eval_sampled_counts'): (3, 5),
    ('svm', 'small', 'eval_samples_counts'): (2, 4),
    ('svm', 'small', 'eval_sums'): (2, 4),
    ('svm', 'small', 'eval_sampled_sums'): (3, 5),
    ('svm', 'small', 'eval_samples_sums'): (2, 4),
    ('svm', 'small', 'eval_class'): (2, 4),
    ('svm', 'small', 'eval_sampled_class'): (3, 5),
    ('svm', 'small', 'eval_samples_class'): (2, 4),
    ('svm', 'small', 'eval_weighted'): (2, 4),
    ('svm', 'small', 'eval_sampled_weighted'): (3, 5),
    ('svm', 'small', 'eval_samples_weighted'): (2, 4),
    ('svm', 'small', 'eval_metrics'): (2, 4),
    ('svm', 'small', 'eval_sampled_metrics'): (3, 5),
    ('svm', 'small', 'eval_samples_metrics'): (2, 4),
    ('svm', 'small', 'eval_curve'): (4, 6),
    ('svm', 'small', 'eval_sampled_curve'): (5, 7),
    ('svm', 'small', 'eval_samples_curve'): (4, 6),
    ('svm', 'small', 'eval_weighted_curve'): (4, 6),
    ('svm', 'small', 'eval_sampled_weighted_curve'): (5, 7),
    ('svm', 'small', 'eval_samples_weighted_curve'): (4, 6),
    ('svm', 'small', 'calibrate'): (2, 4),
    ('svm', 'small', 'calibrate_sampled'): (3, 5),
    ('svm', 'small', 'calibrate_samples'): (2, 4),
    ('svm', 'small', 'calibrate_weighted'): (2, 4),
    ('svm', 'small', 'calibrate_weighted_sampled'): (3, 5),
    ('svm', 'small', 'calibrate_weighted_samples'): (2, 4),
    ('svm', 'small', 'eval_calibration'): (2, 4),
    ('svm', 'small', 'eval_sampled_calibration'): (3, 5),
    ('svm', 'small', 'eval_samples_calibration'): (2, 4),
    ('svm', 'small', 'eval_weighted_calibration'): (1, 3),
    ('svm', 'small', 'eval_sampled_weighted_calibration'): (2, 4),
    ('svm', 'small', 'eval_samples_weighted_calibration'): (1, 3),
    ('svm', 'small', 'calibrate_isotonic'): (6, 8),
    ('svm', 'small', 'calibrate_isotonic_sampled'): (7, 9),
    ('svm', 'small', 'calibrate_isotonic_samples'): (6, 8),
    ('svm', 'small', 'eval_isotonic_calibration'): (2, 4),
    ('svm', 'small', 'eval_sampled_isotonic_calibration'): (3, 5),
    ('svm', 'small', 'eval_samples_isotonic_calibration'): (2, 4),
    ('svm', 'small', 'calibrate_isotonic_weighted'): (8, 10),
    ('svm', 'small', 'calibrate_isotonic_weighted_sampled'): (9, 11),
    ('svm', 'small', 'calibrate_isotonic_weighted_samples'): (8, 10),
    ('svm', 'small', 'eval_weighted_isotonic_calibration'): (1, 3),
    ('svm', 'small', 'eval_sampled_weighted_isotonic_calibration'): (2, 4),
    ('svm', 'small', 'eval_samples_weighted_isotonic_calibration'): (1, 3),
    ('logistic', 'large', 'forward'): (1, 3),
    ('logistic', 'large', 'gradient'): (3, 5),
    ('logistic', 'large', 'eval'): (2, 4),
    ('logistic', 'large', 'margins'): (1, 3),
    ('logistic', 'large', 'probabilities'): (1, 3),
    ('logistic', 'large', 'eval_sums'): (2, 4),
    ('logistic', 'large', 'eval_sampled_sums'): (3, 5),
    ('logistic', 'large', 'eval_samples_sums'): (2, 4),
    ('logistic', 'large', 'eval_class'): (2, 4),
    ('logistic', 'large', 'eval_sampled_class'): (3, 5),
    ('logistic', 'large', 'eval_samples_class'): (2, 4),
    ('logistic', 'large', 'eval_weighted'): (2, 4),
    ('logistic', 'large', 'eval_sampled_weighted'): (3, 5),
    ('logistic', 'large', 'eval_samples_weighted'): (2, 4),
    ('logistic', 'large', 'eval_metrics'): (2, 4),
    ('logistic', 'large', 'eval_sampled_metrics'): (3, 5),
    ('logistic', 'large', 'eval_samples_metrics'): (2, 4),
    ('logistic', 'large', 'eval_curve'): (4, 6),
    ('logistic', 'large', 'eval_sampled_curve'): (5, 7),
    ('logistic', 'large', 'eval_samples_curve'): (4, 6),
    ('logistic', 'large', 'eval_weighted_curve'): (4, 6),
    ('logistic', 'large', 'eval_sampled_weighted_curve'): (5, 7),
    ('logistic', 'large', 'eval_samples_weighted_curve'): (4, 6),
    ('logistic', 'large', 'calibrate'): (2, 4),
    ('logistic', 'large', 'calibrate_sampled'): (3, 5),
    ('logistic', 'large', 'calibrate_samples'): (2, 4),
    ('logistic', 'large', 'calibrate_weighted'): (2, 4),
    ('logistic', 'large', 'calibrate_weighted_sampled'): (3, 5),
    ('logistic', 'large', 'calibrate_weighted_samples'): (2, 4),
    ('logistic', 'large', 'eval_calibration'): (2, 4),
    ('logistic', 'large', 'eval_sampled_calibration'): (3, 5),
    ('logistic', 'large', 'eval_samples_calibration'): (2, 4),
    ('logistic', 'large', 'eval_weighted_calibration'): (1, 3),
    ('logistic', 'large', 'eval_sampled_weighted_calibration'): (2, 4),
    ('logistic', 'large', 'eval_samples_weighted_calibration'): (1, 3),
    ('logistic', 'large', 'calibrate_isotonic'): (7, 9),
    ('logistic', 'large', 'calibrate_isotonic_sampled'): (8, 10),
    ('logistic', 'large', 'calibrate_isotonic_samples'): (7, 9),
    ('logistic', 'large', 'eval_isotonic_calibration'): (2, 4),
    ('logistic', 'large', 'eval_sampled_isotonic_calibration'): (3, 5),
    ('logistic', 'large', 'eval_samples_isotonic_calibration'): (2, 4),
    ('logistic', 'large', 'calibrate_isotonic_weighted'): (9, 11),
    ('logistic', 'large', 'calibrate_isotonic_weighted_sampled'): (10, 12),
    ('logistic', 'large', 'calibrate_isotonic_weighted_samples'): (9, 11),
    ('logistic', 'large', 'eval_weighted_isotonic_calibration'): (1, 3),
    ('logistic', 'large', 'eval_sampled_weighted_isotonic_calibration'): (2, 4),
    ('logistic', 'large', 'eval_samples_weighted_isotonic_calibration'): (1, 3),
    ('logistic', 'small', 'forward'): (1, 3),
    ('logistic', 'small', 'gradient'): (3, 5),
    ('logistic', 'small', 'eval'): (2, 4),
    ('logistic', 'small', 'margins'): (1, 3),
    ('logistic', 'small', 'probabilities'): (1, 3),
    ('logistic', 'small', 'eval_sums'): (2, 4),
    ('logistic', 'small', 'eval_sampled_sums'): (3, 5),
    ('logistic', 'small', 'eval_samples_sums'): (2, 4),
    ('logistic', 'small', 'eval_class'): (2, 4),
    ('logistic', 'small', 'eval_sampled_class'): (3, 5),
    ('logistic', 'small', 'eval_samples_class'): (2, 4),
    ('logistic', 'small', 'eval_weighted'): (2, 4),
    ('logistic', 'small', 'eval_sampled_weighted'): (3, 5),
    ('logistic', 'small', 'eval_samples_weighted'): (2, 4),
    ('logistic', 'small', 'eval_metrics'): (2, 4),
    ('logistic', 'small', 'eval_sampled_metrics'): (3, 5),
    ('logistic', 'small', 'eval_samples_metrics'): (2, 4),
    ('logistic', 'small', 'eval_curve'): (4, 6),
    ('logistic', 'small', 'eval_sampled_curve'): (5, 7),
    ('logistic', 'small', 'eval_samples_curve'): (4, 6),
    ('logistic', 'small', 'eval_weighted_curve'): (4, 6),
    ('logistic', 'small', 'eval_sampled_weighted_curve'): (5, 7),
    ('logistic', 'small', 'eval_samples_weighted_curve'): (4, 6),
    ('logistic', 'small', 'calibrate'): (2, 4),
    ('logistic', 'small', 'calibrate_sampled'): (3, 5),
    ('logistic', 'small', 'calibrate_samples'): (2, 4),
    ('logistic', 'small', 'calibrate_weighted'): (2, 4),
    ('logistic', 'small', 'calibrate_weighted_sampled'): (3, 5),
    ('logistic', 'small', 'calibrate_weighted_samples'): (2, 4),
    ('logistic', 'small', 'eval_calibration'): (2, 4),
    ('logistic', 'small', 'eval_sampled_calibration'): (3, 5),
    ('logistic', 'small', 'eval_samples_calibration'): (2, 4),
    ('logistic', 'small', 'eval_weighted_calibration'): (1, 3),
    ('logistic', 'small', 'eval_sampled_weighted_calibration'): (2, 4),
    ('logistic', 'small', 'eval_samples_weighted_calibration'): (1, 3),
    ('logistic', 'small', 'calibrate_isotonic'): (6, 8),
    ('logistic', 'small', 'calibrate_isotonic_sampled'): (7, 9),
    ('logistic', 'small', 'calibrate_isotonic_samples'): (6, 8),
    ('logistic', 'small', 'eval_isotonic_calibration'): (2, 4),
    ('logistic', 'small', 'eval_sampled_isotonic_calibration'): (3, 5),
    ('logistic', 'small', 'eval_samples_isotonic_calibration'): (2, 4),
    ('logistic', 'small', 'calibrate_isotonic_weighted'): (8, 10),
    ('logistic', 'small', 'calibrate_isotonic_weighted_sampled'): (9, 11),
    ('logistic', 'small', 'calibrate_isotonic_weighted_samples'): (8, 10),
    ('logistic', 'small', 'eval_weighted_isotonic_calibration'): (1, 3),
    ('logistic', 'small', 'eval_sampled_weighted_isotonic_calibration'): (2, 4),
    ('logistic', 'small', 'eval_samples_weighted_isotonic_calibration'): (1, 3),
}

# the refusals of each row form, one bad argument at a time, and the exception each gets
BAD_ROWS = {
    "list": [([0, N_ROWS], "DsgdRange"), ([-1, 3], "DsgdRange"), ([], "DsgdEmpty"), ("NULL", "DsgdInvalid")],
    "range": [((0, N_ROWS + 1), "DsgdRange"), ((-1, 5), "DsgdRange"), ((9, 8), "DsgdRange"), ((4, 4), "DsgdEmpty")],
    "drawn": [((0, N_ROWS + 1, 1, 0, 5), "DsgdRange"), ((-1, 10, 1, 0, 5), "DsgdRange"), ((5, 5, 1, 0, 0), "DsgdEmpty"),
              ((10, 20, 1, -1, 3), "DsgdInvalid"), ((10, 20, 1, 0, 11), "DsgdInvalid"), ((10, 20, 1, 4, 12), "DsgdInvalid"),
              ((10, 20, 1, 3, 3), "DsgdEmpty"), ((10, 20, 1, 5, 4), "DsgdEmpty")],
}
GOOD_ROWS = {"list": [1, 2, 3], "range": (10, 20), "drawn": (10, 20, 1, 0, 5)}

# family -> the arguments of its entry points after the rows: OUT an output that must not be NULL, None an output that may
# be (and is left) NULL, else the value passed
OUT = "out"
TAIL = {
    "forward": [OUT], "gradient": [OUT, None], "margins": [OUT], "probabilities": [OUT], "eval": [None, None],
    "eval_counts": [None] * 3, "eval_sums": [None] * 3, "eval_class": [None] * 3, "eval_weighted": [None] * 3,
    "eval_metrics": [OUT],
    "eval_curve": [OUT] * 6, "eval_weighted_curve": [OUT] * 6,         # words, AP or sums, points; thr, tp, fp
    "calibrate": [OUT] * 3, "calibrate_weighted": [OUT] * 4,
    "eval_calibration": [*SIGMOID, 10] + [OUT] * 5, "eval_weighted_calibration": [*SIGMOID, 10] + [OUT] * 5,
    "calibrate_isotonic": [OUT] * 6, "calibrate_isotonic_weighted": [OUT] * 7,
    "eval_isotonic_calibration": [*MAP, 3, 10] + [OUT] * 5, "eval_weighted_isotonic_calibration": [*MAP, 3, 10] + [OUT] * 5,
}
# family -> its bad non-pointer arguments, (position after the rows, value): a non-finite a or b, 0 or too many bins
_SIGMOID_BAD = [(0, float("inf")), (1, float("nan")), (2, 0), (2, MAX_BINS + 1)]
_MAP_BAD = [(3, 0), (3, MAX_BINS + 1)]
BAD_VALUES = {"eval_calibration": _SIGMOID_BAD, "eval_weighted_calibration": _SIGMOID_BAD,
              "eval_isotonic_calibration": _MAP_BAD, "eval_weighted_isotonic_calibration": _MAP_BAD}
# families whose row weights belong to the sync paths: an async context is refused (dsgd_eval*_weighted takes one)
ASYNC_REFUSED = {"eval_weighted_curve", "calibrate_weighted", "eval_weighted_calibration", "calibrate_isotonic_weighted",
                 "eval_weighted_isotonic_calibration"}


def error_cases():
    """(entry point, context, rows (None: GOOD_ROWS of its form), bad argument (None, or (position after the rows,
    value)), expected exception class name or None): each bad argument on its own."""
    cases = []
    for name in REQUESTS:
        fam, own = FAMILY[name], "logistic" if name in LOGISTIC_ONLY else "svm"
        cases += [(name, own, rows, None, None if (name, rows) == ("forward", []) else exc)     # forward of no ids: a no-op
                  for rows, exc in BAD_ROWS[FORM[name]]]
        cases.append((name, "empty_" + own, None, None, "DsgdState"))
        cases += [(name, own, None, (i, None), "DsgdInvalid") for i, v in enumerate(TAIL[fam]) if v is OUT]
        cases += [(name, own, None, bad, "DsgdInvalid") for bad in BAD_VALUES.get(fam, ())]
        if fam in ASYNC_REFUSED:
            cases.append((name, "async", None, None, "DsgdState"))
        if name in SVM_ONLY:
            cases.append((name, "logistic", None, None, "DsgdState"))
        if name in LOGISTIC_ONLY:
            cases.append((name, "svm", None, None, "DsgdState"))
    cases.append(("gradient", "no_d", None, None, "DsgdState"))
    return cases


def request_ids(n):
    return np.random.default_rng(n).integers(0, N_ROWS, size=n).astype(np.int32)


def bits(x):
    if isinstance(x, tuple):
        return tuple(bits(v) for v in x)
    if isinstance(x, np.ndarray):
        return x.dtype.str, x.tobytes()
    return float(x).hex() if isinstance(x, float) else x


def entry_points(model):
    return [n for n in REQUESTS if n not in (LOGISTIC_ONLY if model == "svm" else SVM_ONLY)]


def make_contexts():
    """model -> (ctx with N_ROWS rows, dimSparsity and resident weights w, w); plus the contexts of the error table:
    `empty_*` without rows, `no_d` with rows and no dimSparsity, `async` an async-mode context with rows."""
    from distributed_sgd_b200.native import NativeCtx
    from distributed_sgd_b200.utils import synthetic_rcv1
    data = synthetic_rcv1(n_rows=N_ROWS, seed=31)
    rng = np.random.default_rng(31)
    w = np.where(rng.random(data.dim) < 0.6, rng.standard_normal(data.dim) * 0.1, 0.0)
    out = {}
    for model in ("svm", "logistic"):
        ctx = NativeCtx(0, data.dim, LAM, logistic=model == "logistic")
        ctx.load_csr(data.row_ptr, data.col, data.val, data.label)
        ctx.compute_dim_sparsity(N_ROWS)
        ctx.set_weights(w)
        out[model] = ctx
        out["empty_" + model] = NativeCtx(0, data.dim, LAM, logistic=model == "logistic")
    out["no_d"] = NativeCtx(0, data.dim, LAM)
    out["no_d"].load_csr(data.row_ptr, data.col, data.val, data.label)
    out["async"] = NativeCtx(0, data.dim, LAM, is_async=True)
    out["async"].load_csr(data.row_ptr, data.col, data.val, data.label)
    return out, w


def observe_launches(ctxs, w, model, size):
    """entry point -> ((delta, delta), (result, result)): one call with the resident weights and one with w passed in."""
    ctx, ids, out = ctxs[model], request_ids(SIZES[size]), {}
    for name in entry_points(model):
        deltas, results = [], []
        for wa in (None, w):
            before = ctx.launch_count()
            results.append(REQUESTS[name](ctx, ids, wa))
            deltas.append(ctx.launch_count() - before)
        out[name] = (tuple(deltas), tuple(results))
    return out


def raw_call(ctx, name, rows, bad):
    """dsgd_<name> through ctypes with `rows` in its form, no weights, and the arguments of TAIL with `bad` in its place:
    (exception class name or None, message, launch_count() delta)."""
    from distributed_sgd_b200.native import _EXC
    if FORM[name] == "list":
        ids = None if rows == "NULL" else np.asarray(rows, np.int32)
        args = (None if ids is None else ids.ctypes.data, 3 if ids is None else ids.size)
    else:
        args = tuple(rows)
    fn, tail, keep = getattr(ctx._l, "dsgd_" + name), list(TAIL[FAMILY[name]]), []
    if bad is not None:
        tail[bad[0]] = bad[1]
    for i, (v, t) in enumerate(zip(tail, fn.argtypes[-len(tail):])):
        if v is OUT:                    # room for every output: at most one value per row, of 8 bytes
            keep.append(np.zeros(max(N_ROWS, ctx.dim) + 8))
            v = keep[-1]
        if isinstance(v, np.ndarray):
            tail[i] = v.ctypes.data if t is C.c_void_p else v.ctypes.data_as(t)
    before = ctx.launch_count()
    rc = fn(ctx._h, None, *args, *tail)
    launched = ctx.launch_count() - before
    return (None if rc == 0 else _EXC[rc].__name__), (ctx._l.dsgd_last_error(ctx._h) or b"").decode(), launched


@pytest.fixture(scope="module")
def ctxs():
    out, w = make_contexts()
    yield out, w
    for c in out.values():
        c.close()


@pytest.mark.parametrize("size", sorted(SIZES))
@pytest.mark.parametrize("model", ["svm", "logistic"])
def test_launches_and_resident_weights(ctxs, model, size):
    got = observe_launches(*ctxs, model, size)
    assert {name: d for name, (d, _) in got.items()} == {k[2]: v for k, v in LAUNCHES.items() if k[:2] == (model, size)}
    (g0, loss0), (g1, loss1) = got.pop("gradient")[1] if model == "logistic" else ((0.0, 0.0), (0.0, 0.0))
    np.testing.assert_allclose(g0, g1, rtol=1e-12, atol=1e-18)
    assert bits(loss0) == bits(loss1)
    assert [name for name, (_, (a, b)) in got.items() if bits(a) != bits(b)] == []


def test_errors(ctxs):
    cases = error_cases()
    assert len(REQUESTS) == 50 and len(cases) == 529
    for name, kind, rows, bad, expected in cases:
        ctx = ctxs[0][kind]
        got, msg, launched = raw_call(ctx, name, GOOD_ROWS[FORM[name]] if rows is None else rows, bad)
        assert got == expected, (name, kind, rows, bad, msg)
        if expected is not None:
            assert msg.startswith(f"dsgd_{name}: "), (name, kind, rows, bad, msg)
        assert launched == 0, (name, kind, rows, bad, msg, launched)
    w = ctxs[1]                                       # the contexts still answer after the refusals
    assert bits(ctxs[0]["svm"].eval_sums(0, N_ROWS)) == bits(ctxs[0]["svm"].eval_sums(0, N_ROWS, w))


_LOOP = r"""
import sys, time
sys.path.insert(0, {root!r})
import numpy as np
from distributed_sgd_b200.native import DsgdState, NativeCtx
from distributed_sgd_b200.utils import synthetic_rcv1
data = synthetic_rcv1(n_rows=3000, seed=8)
ctx = NativeCtx(0, data.dim, 1e-4, is_async=True)
ctx.load_csr(data.row_ptr, data.col, data.val, data.label)
ctx.compute_dim_sparsity(3000)
ctx.start_async(np.zeros(data.dim), np.arange(3000, dtype=np.int32), 8, 0.1, concurrency=1, max_updates=64, seed=1)
try:
    t0 = time.time()
    while ctx.async_running():
        if time.time() - t0 > 60:
            raise SystemExit("the loop did not end by itself")
        time.sleep(0.01)
    ids = np.zeros(3001, np.int32)
    extra = {{"eval_samples_calibration": (1.5, -0.25),
             "eval_samples_isotonic_calibration": (np.array([-2.0, 0.0, 2.0]), np.array([0.2, 0.5, 0.8]))}}
    refused = []
    for name in {names!r}:
        try:
            getattr(ctx, name)(ids, *extra.get(name, ()))
        except DsgdState as e:
            refused.append(name if str(e).split("] ", 1)[1].startswith("dsgd_" + name + ": ") else name + "?")
    print("REFUSED", " ".join(refused))
finally:
    ctx.stop_async()
print("AFTER", len(ctx.forward(ids)))
ctx.close()
"""
# the list forms an async context takes
LOOP_LISTS = ("forward", "gradient", "eval_samples_counts", "eval_samples_sums", "margins", "eval_samples_metrics",
              "eval_samples_class", "eval_samples_weighted", "eval_samples_curve", "calibrate_samples",
              "eval_samples_calibration", "calibrate_isotonic_samples", "eval_samples_isotonic_calibration")


def test_longer_list_than_rows_is_refused_while_a_loop_is_started():
    """The loop ends by itself on max_updates; the context still counts as running until stop_async, so the list requests
    refuse a list their buffers cannot hold, and take it once the loop is stopped.  The subprocess has a timeout."""
    r = subprocess.run([sys.executable, "-s", "-c", _LOOP.format(root=ROOT, names=LOOP_LISTS)], cwd=ROOT,
                       capture_output=True, text=True, timeout=180)
    assert r.returncode == 0, r.stdout + r.stderr
    assert ("REFUSED " + " ".join(LOOP_LISTS) + "\nAFTER 3001") in r.stdout, r.stdout + r.stderr
