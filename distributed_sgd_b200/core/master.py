"""core/Master.scala, MasterSync.scala, MasterAsync.scala -- the coordination loop.

The reference master is a separate process that shuffles index ranges, fans `gradient` RPCs out to K
slaves, averages the replies and updates the weights (core/Master.scala:120-218).  Here the master
logic runs SPMD: every rank executes the same loop with the same seed, so all ranks draw the same
batches; each rank feeds ITS slice to its GPU and the replies are summed on the devices (NCCL over
NVLink inside libdsgd.so).  Weights never leave the GPUs during `fit`.  What remains on the host is
control flow over a handful of scalars per epoch (losses, accuracies, the stopping rule).
"""
from __future__ import annotations

import dataclasses
from typing import Callable, List, NamedTuple, Optional, Sequence, Union

import numpy as np

from ..ml import split_strategy as SplitStrategy  # noqa: N812
from ..ml.calibration import METHODS as CALIBRATION_METHODS, Calibration, IsotonicCalibration
from ..ml.class_weight import resolve_class_weight
from ..ml.grad_state import GradState
from ..ml.lr_schedule import check_schedule, learning_rates
from ..ml.one_vs_rest import OneVsRest, threshold_report, topic_ranking_report, topic_report
from ..ml.sparse_logistic import SparseLogistic
from ..ml.sparse_margin import SparseModifiedHuber, SparseSquaredHinge
from ..ml.sparse_svm import SparseSVM
from ..native import ERR_EMPTY, DsgdEmpty, NativeCtx, row_methods, topic_rank_words, topic_words
from ..utils.dataset import SAMPLE_WEIGHT_ASYNC, Data, has_sample_weights
from .group import Group
from .slave import Slave

EarlyStopping = Callable[[Sequence[float]], bool]
Split = Callable[[int, int], List[range]]

_M64 = (1 << 64) - 1


def sampled_key(seed: int, t: int) -> int:
    """Key of the t-th device-drawn sample of a Master seeded with `seed` (Master.local_sampled_*).  splitmix64's finaliser
    over seed * phi + (t + 1) * c (mod 2^64, c odd): for one seed it maps different t to different keys, and every rank
    computes the same key from the same (seed, t)."""
    z = (int(seed) * 0x9E3779B97F4A7C15 + (int(t) + 1) * 0xD1B54A32D192ED03) & _M64
    z = ((z ^ (z >> 30)) * 0xBF58476D1CE4E5B9) & _M64
    z = ((z ^ (z >> 27)) * 0x94D049BB133111EB) & _M64
    return z ^ (z >> 31)


def bootstrap_key(seed: int) -> int:
    """The bootstrap key of a Master seeded with `seed` (Master.local_bootstrap with key=None): sampled_key at t = 2^64 - 1,
    which no sample draw reaches."""
    return sampled_key(seed, _M64)


# the metrics a bootstrap reports, and whether a larger value is better
BOOTSTRAP_METRICS = {"accuracy": True, "loss": False, "auc": True, "ap": True, "precision": True, "recall": True, "f1": True}


def bootstrap_values(words, ap, loss_sum, penalty: float) -> dict:
    """Each BOOTSTRAP_METRICS value of every replicate from its native.BOOTSTRAP_WORDS words, AP and loss sum, as
    metrics_dict forms them from the counts (nan where undefined); loss = penalty + loss sum / replicate size."""
    w = np.asarray(words, dtype=np.int64).reshape(-1, 9).astype(np.float64)
    tp, fn, pos_none, fp, tn, neg_none, u2, nan, size = w.T
    P, N = tp + fn + pos_none, fp + tn + neg_none

    def ratio(a, b):
        with np.errstate(divide="ignore", invalid="ignore"):
            return np.where(b > 0, a / np.where(b > 0, b, 1.0), np.nan)

    auc = np.where((nan == 0) & (P > 0) & (N > 0), u2 / np.where(P * N > 0, 2.0 * P * N, 1.0), np.nan)
    return {"accuracy": ratio(tp + tn, P + N), "loss": penalty + ratio(np.asarray(loss_sum, np.float64), size),
            "auc": auc, "ap": np.asarray(ap, dtype=np.float64), "precision": ratio(tp, tp + fp), "recall": ratio(tp, P),
            "f1": ratio(2 * tp, 2 * tp + fp + fn + pos_none)}


def weighted_bootstrap_values(words, wsums, loss_sum, penalty: float) -> dict:
    """Each BOOTSTRAP_METRICS value of every weighted replicate from its two words (size, NaN-score rows), its
    native.WCURVE_WORDS weighted words and its weighted loss sum, by the formulas of weighted_curve_dict and
    native.weighted_auc_ap (nan where undefined); loss = penalty + loss sum / replicate size, as in local_weighted_report."""
    size, nan = np.asarray(words, dtype=np.int64).reshape(-1, 2).astype(np.float64).T
    tp, fn, pos_none, fp, _, _, u2w, _, s_ap, correct, total, wp, wn = np.asarray(wsums, np.float64).reshape(-1, 13).T

    def ratio(a, b):
        with np.errstate(divide="ignore", invalid="ignore"):
            return np.where(b > 0, a / np.where(b > 0, b, 1.0), np.nan)

    with np.errstate(divide="ignore", invalid="ignore"):
        auc = np.where((nan == 0) & (wp != 0) & (wn != 0), u2w / (2.0 * wp * wn), np.nan)
        ap = np.where((nan == 0) & (wp != 0), np.where(wn == 0, 1.0, s_ap / wp), np.nan)
    return {"accuracy": ratio(correct, total), "loss": penalty + ratio(np.asarray(loss_sum, np.float64), size),
            "auc": auc, "ap": ap, "precision": ratio(tp, tp + fp), "recall": ratio(tp, wp),
            "f1": ratio(2.0 * tp, 2.0 * tp + fp + fn + pos_none)}


# The replicate layout of a bootstrap call, as (int64 words, doubles) per replicate: the unweighted calls return
# BOOTSTRAP_WORDS words and the AP, the weighted ones the size and NaN rows and the WCURVE_WORDS words; both then a loss sum.
BOOTSTRAP_LAYOUT = {False: (9, 1), True: (2, 13)}


def bootstrap_pack(words, mid, loss) -> np.ndarray:
    """One rank's replicates as one float64 array: the words' bits, then the middle doubles (AP or the weighted words), then
    the loss sums, each block replicate-major."""
    return np.concatenate([np.asarray(words, np.int64).reshape(-1).view(np.float64),
                           np.asarray(mid, np.float64).reshape(-1), np.asarray(loss, np.float64).reshape(-1)])


def bootstrap_unpack(parts, weighted: bool = False):
    """bootstrap_pack's arrays of every rank, in rank order, back into (words[k, nw], mid, loss[k]) over all replicates:
    mid is ap[k] (unweighted) or wsums[k, 13] (weighted)."""
    nw, nm = BOOTSTRAP_LAYOUT[bool(weighted)]
    words, mid, loss = [], [], []
    for p in parts:
        p = np.asarray(p, np.float64)
        k = p.size // (nw + nm + 1)
        words.append(p[:nw * k].view(np.int64).reshape(k, nw))
        mid.append(p[nw * k:(nw + nm) * k].reshape(k, nm) if weighted else p[nw * k:(nw + nm) * k])
        loss.append(p[(nw + nm) * k:])
    return np.concatenate(words), np.concatenate(mid), np.concatenate(loss)


def bootstrap_summary(estimate: float, reps, level: float) -> dict:
    """One metric's bootstrap: the full-sample estimate, the percentile interval at `level` (numpy.quantile's default method)
    over the replicates where the metric is defined and how many those are, the standard error (their standard deviation),
    and the replicates (nan where undefined)."""
    reps = np.asarray(reps, dtype=np.float64)
    ok = reps[~np.isnan(reps)]
    a = (1.0 - level) / 2.0
    lo, hi = (float(x) for x in np.quantile(ok, [a, 1.0 - a])) if ok.size else (float("nan"), float("nan"))
    se = float(np.std(ok, ddof=1)) if ok.size > 1 else float("nan")
    return {"estimate": float(estimate), "lo": lo, "hi": hi, "se": se, "n_defined": int(ok.size), "replicates": reps}


def bootstrap_share(n_boot: int, world: int, rank: int):
    """Replicates [lo, hi) that rank `rank` of `world` computes: contiguous, disjoint, covering [0, n_boot)."""
    return (n_boot * rank) // world, (n_boot * (rank + 1)) // world


def sample_shard(k: int, world: int, rank: int):
    """Positions [lo, hi) of a k-row sample that rank `rank` of `world` evaluates: the shards are disjoint and cover
    [0, k), and their sizes differ by at most one."""
    return (k * rank) // world, (k * (rank + 1)) // world


class Rows(NamedTuple):
    """The rows of one evaluation request, in the form of the entry point that takes them: rows [lo, hi) (key and ids
    None); positions [lo, hi) of the sample the device draws from rows [b, e) with `key`; or positions [lo, hi) of the row
    ids `ids`."""
    lo: int
    hi: int
    b: int = 0
    e: int = 0
    key: Optional[int] = None
    ids: Optional[np.ndarray] = None

    def call(self, ctx, family: str, *args, **kw):
        """ctx's method of `family` (native.row_methods) for this form, over these rows, with the family's arguments."""
        if self.ids is not None:
            form, rows = "list", (self.ids[self.lo:self.hi],)
        elif self.key is not None:
            form, rows = "drawn", (self.b, self.e, self.key, self.lo, self.hi)
        else:
            form, rows = "range", (self.lo, self.hi)
        return getattr(ctx, row_methods(family)[form])(*rows, *args, **kw)

    def shard(self, world: int, rank: int) -> Optional["Rows"]:
        """The contiguous share of these rows that rank `rank` of `world` evaluates (sample_shard of the positions), or
        None when it is empty."""
        lo, hi = sample_shard(self.hi - self.lo, world, rank)
        return self._replace(lo=self.lo + lo, hi=self.lo + hi) if hi > lo else None


def metrics_dict(words) -> dict:
    """The result of Master.local_metrics from the native.METRICS_WORDS counts of a dsgd_eval_*metrics call: the eight counts
    (tp, fn, pos_no_pred, fp, tn, neg_no_pred, u2, nan_scores), precision = TP / (TP + FP), recall = TP / P, f1 = 2 TP /
    (2 TP + FP + FN + pos_no_pred) -- the harmonic mean of the two where both are defined --, auc = U2 / (2 P N) and accuracy
    = (TP + TN) / (P + N), with P and N the positive and negative rows.  A ratio whose denominator is 0 is nan, and so is auc
    when a score is NaN or a class is empty."""
    tp, fn, pos_none, fp, tn, neg_none, u2, nan = (int(x) for x in words)
    P, N = tp + fn + pos_none, fp + tn + neg_none

    def ratio(a: int, b: int) -> float:
        return a / b if b else float("nan")

    auc = float(u2) / float(2 * P * N) if nan == 0 and P and N else float("nan")   # one IEEE division
    return {"tp": tp, "fn": fn, "pos_no_pred": pos_none, "fp": fp, "tn": tn, "neg_no_pred": neg_none, "u2": u2,
            "nan_scores": nan, "precision": ratio(tp, tp + fp), "recall": ratio(tp, P),
            "f1": ratio(2 * tp, 2 * tp + fp + fn + pos_none), "auc": auc, "accuracy": ratio(tp + tn, P + N)}


def _calibration(result) -> Calibration:
    """A NativeCtx.calibrate* result as a Calibration."""
    a, b, objective, info = result
    return Calibration(a, b, objective, int(info[0]), int(info[1]), int(info[2]), int(info[3]))


def _weighted_calibration(result) -> Calibration:
    """A NativeCtx.calibrate_weighted* result as a weighted Calibration."""
    a, b, objective, info, wsums = result
    return Calibration(a, b, objective, int(info[0]), int(info[1]), int(info[2]), int(info[3]), True, float(wsums[0]),
                       float(wsums[1]), float(wsums[2]))


def _weighted_isotonic(result) -> IsotonicCalibration:
    """A NativeCtx.calibrate_isotonic_weighted* result as a weighted IsotonicCalibration."""
    x, y, block_w, block_pw, info, wsums = result
    return IsotonicCalibration(x, y, block_w, block_pw, int(info[0]), int(info[2]), int(info[3]), int(info[4]), True,
                               float(wsums[0]), float(wsums[1]))


def _isotonic(result) -> IsotonicCalibration:
    """A NativeCtx.calibrate_isotonic* result as an IsotonicCalibration."""
    x, y, block_rows, block_pos, info = result
    return IsotonicCalibration(x, y, block_rows, block_pos, int(info[0]), int(info[2]), int(info[3]), int(info[4]))


def _method(method: str) -> str:
    if method not in CALIBRATION_METHODS:
        raise ValueError(f"calibration method: expected one of {', '.join(CALIBRATION_METHODS)}, got {method!r}")
    return method


def isotonic_calibration_dict(result) -> dict:
    """calibration_dict of a NativeCtx.eval_*isotonic_calibration result, plus infinite_log_loss_rows: the rows whose term
    -log p (o = 1) or -log(1 - p) (o = 0) is infinite; any such row makes log_loss +inf."""
    sums, bin_rows, bin_pos, bin_psum, words = result
    out = calibration_dict((sums, bin_rows, bin_pos, bin_psum, words[:2]))
    out["infinite_log_loss_rows"] = int(words[2])
    if words[2]:
        out["log_loss"] = float("inf")
    return out


def calibration_dict(result) -> dict:
    """The result of Master.local_calibration from a NativeCtx.eval_*calibration result: brier and log_loss (means over the
    rows used), ece = sum over the bins of (rows_b / rows) |mean predicted_b - observed frequency_b|, mce = the largest such
    gap, rows, nan_rows, and bins: edges (n_bins + 1), rows, positives, mean_predicted and observed (NaN for an empty bin)."""
    sums, bin_rows, bin_pos, bin_psum, words = result
    n, m = int(words[0]), len(bin_rows)
    filled = bin_rows > 0
    den = np.where(filled, bin_rows, 1)
    mean_p = np.where(filled, bin_psum / den, np.nan)
    freq = np.where(filled, bin_pos / den, np.nan)
    gap = np.abs(mean_p - freq)[filled]
    nan = float("nan")
    return {"brier": float(sums[0]) / n if n else nan, "log_loss": float(sums[1]) / n if n else nan,
            "ece": float(np.sum(bin_rows[filled] / n * gap)) if n else nan, "mce": float(np.max(gap)) if n else nan,
            "rows": n, "nan_rows": int(words[1]),
            "bins": {"edges": np.arange(m + 1) / m, "rows": bin_rows, "positives": bin_pos, "mean_predicted": mean_p,
                     "observed": freq}}


def weighted_calibration_dict(result) -> dict:
    """The result of Master.local_calibration(weighted=True) from a NativeCtx.eval_*weighted_calibration result, every row
    counted by its weight: with W = sums[2] the weight of the rows used, brier = S_brier / W, log_loss = S_ll / W (+inf when a
    row of positive weight has an infinite term, sums[3] > 0), ece = sum over the bins of (W_b / W) |psum_b / W_b - pos_b /
    W_b|, mce = the largest such gap, rows and nan_rows (counts), weight = W, and bins: edges, weight, positive_weight,
    mean_predicted and observed (NaN for a bin of zero weight); at an isotonic map also infinite_log_loss_rows."""
    sums, bin_w, bin_pw, bin_psum, words = result
    W, m = float(sums[2]), len(bin_w)
    filled = bin_w > 0
    den = np.where(filled, bin_w, 1.0)
    mean_p = np.where(filled, bin_psum / den, np.nan)
    freq = np.where(filled, bin_pw / den, np.nan)
    gap = np.abs(mean_p - freq)[filled]
    nan = float("nan")
    log_loss = float("inf") if sums[3] > 0 else (float(sums[1]) / W if W else nan)
    extra = {"infinite_log_loss_rows": int(words[2])} if len(words) > 2 else {}
    return {**extra, "brier": float(sums[0]) / W if W else nan, "log_loss": log_loss,
            "ece": float(np.sum(bin_w[filled] / W * gap)) if W else nan, "mce": float(np.max(gap)) if gap.size else nan,
            "rows": int(words[0]), "nan_rows": int(words[1]), "weight": W,
            "bins": {"edges": np.arange(m + 1) / m, "weight": bin_w, "positive_weight": bin_pw, "mean_predicted": mean_p,
                     "observed": freq}}


# (weighted, isotonic) -> the fit family and its result's converter (Master.calibrate), and the quality family and its
# result's converter (Master.local_calibration)
_FITS = {(False, False): ("calibrate", _calibration), (True, False): ("calibrate_weighted", _weighted_calibration),
         (False, True): ("calibrate_isotonic", _isotonic), (True, True): ("calibrate_isotonic_weighted", _weighted_isotonic)}
_QUALITY = {(False, False): ("eval_calibration", calibration_dict),
            (True, False): ("eval_weighted_calibration", weighted_calibration_dict),
            (False, True): ("eval_isotonic_calibration", isotonic_calibration_dict),
            (True, True): ("eval_weighted_isotonic_calibration", weighted_calibration_dict)}


def curve_dict(result) -> dict:
    """The result of Master.local_curve from a NativeCtx.eval_*curve result: metrics_dict(words) plus average_precision and
    n_points, and for a full curve pass the points under "curve", highest score first (the scalar counts and rates of
    metrics_dict keep their keys): thresholds, tp and fp (the rows at or above each threshold) and the derived precision =
    tp / (tp + fp), recall = tpr = tp / P and fpr = fp / N, with P and N the non-NaN positive and negative rows; a rate whose
    denominator is 0 is nan."""
    words, ap = result[0], result[1]
    out = metrics_dict(words)
    out["average_precision"] = float(ap)
    out["n_points"] = int(result[2]) if len(result) == 3 else len(result[2])   # distinct scores
    if len(result) == 5:
        thr, tp, fp = result[2], np.asarray(result[3], dtype=np.int64), np.asarray(result[4], dtype=np.int64)
        P, N = (int(tp[-1]), int(fp[-1])) if len(tp) else (0, 0)
        nan = float("nan")
        with np.errstate(divide="ignore", invalid="ignore"):
            precision = np.where(tp + fp > 0, tp / np.maximum(tp + fp, 1), nan)
            recall = tp / P if P else np.full(len(tp), nan)
            fpr = fp / N if N else np.full(len(fp), nan)
        out["curve"] = {"thresholds": [float(x) for x in thr], "tp": [int(x) for x in tp], "fp": [int(x) for x in fp],
                        "precision": [float(x) for x in precision], "recall": [float(x) for x in recall],
                        "tpr": [float(x) for x in recall], "fpr": [float(x) for x in fpr]}
    return out


def weighted_curve_dict(result, curve: bool = True) -> dict:
    """The result of Master.local_weighted_curve from a NativeCtx.eval_*weighted_curve result (include/dsgd.h): the weighted
    confusion sums tp, fn, pos_no_pred, fp, tn, neg_no_pred (each row counted by its weight c_i), nan_weight, and with the
    formulas of metrics_dict on the weights precision = TP / (TP + FP), recall = TP / W+, f1 = 2 TP / (2 TP + FP + FN +
    pos_no_pred); auc = U2w / (2 W+ W-), average_precision = S_ap / W+, accuracy = the correct rows' weight / weight_sum,
    weight_sum, n_points and nan_scores (rows).  With `curve` (a result with its points), "curve": thresholds, tp_weight and fp_weight (W+ and W- at
    or above each threshold), precision, recall and fpr.  A ratio whose denominator is 0 is nan."""
    tp, fn, pos_none, fp, tn, neg_none, _, nan_w, _, correct, total, wp, wn = (float(x) for x in result.wsums)
    nan = float("nan")

    def ratio(a: float, b: float) -> float:
        return a / b if b else nan

    out = {"tp": tp, "fn": fn, "pos_no_pred": pos_none, "fp": fp, "tn": tn, "neg_no_pred": neg_none, "nan_weight": nan_w,
           "nan_scores": int(result.words[7]), "precision": ratio(tp, tp + fp), "recall": ratio(tp, wp),
           "f1": ratio(2.0 * tp, 2.0 * tp + fp + fn + pos_none), "auc": float(result.auc),
           "average_precision": float(result.ap), "accuracy": ratio(correct, total), "weight_sum": total,
           "n_points": int(result.n_points)}
    if curve:
        tpw, fpw = np.asarray(result.tpw, dtype=np.float64), np.asarray(result.fpw, dtype=np.float64)
        P, N = (float(tpw[-1]), float(fpw[-1])) if len(tpw) else (0.0, 0.0)
        with np.errstate(divide="ignore", invalid="ignore"):
            precision = np.where(tpw + fpw > 0, tpw / np.where(tpw + fpw > 0, tpw + fpw, 1.0), nan)
            recall = tpw / P if P else np.full(len(tpw), nan)
            fpr = fpw / N if N else np.full(len(fpw), nan)
        out["curve"] = {"thresholds": [float(x) for x in result.thr], "tp_weight": [float(x) for x in tpw],
                        "fp_weight": [float(x) for x in fpw], "precision": [float(x) for x in precision],
                        "recall": [float(x) for x in recall], "fpr": [float(x) for x in fpr]}
    return out


class EpochDraw(list):
    """The batch draws of one epoch: `self[s][k]` = row ids of worker k at step s (a list of lists of int32 arrays, the
    shape the tests and the oracle replay), backed by ONE array `ids[steps, K, batch]` (-1 beyond a short slice) and
    `counts[steps, K]` so that `fit` can hand whole runs of steps to the device without per-step Python work."""

    ids: np.ndarray
    counts: np.ndarray

    @classmethod
    def _wrap(cls, ids: np.ndarray, counts: np.ndarray) -> "EpochDraw":
        self = cls([[ids[s, k, :counts[s, k]] for k in range(ids.shape[1])] for s in range(ids.shape[0])])
        self.ids, self.counts = ids, counts
        return self

    @classmethod
    def draw(cls, seed: int, epoch: int, groups: List[range], batch_size: int) -> "EpochDraw":
        import ctypes as C
        from .. import native
        K = len(groups)
        g_start = np.array([g.start for g in groups], dtype=np.int64)
        g_len = np.array([len(g) for g in groups], dtype=np.int64)
        steps = -(-int(g_len.max()) // batch_size) if K else 0
        ids = np.empty((steps, K, batch_size), dtype=np.int32)
        counts = np.empty((steps, K), dtype=np.int32)
        h = native.host_lib()
        rc = h.dsgd_draw_epoch(C.c_uint64(seed & 0xFFFFFFFFFFFFFFFF), epoch, K, g_start.ctypes.data_as(C.c_void_p),
                               g_len.ctypes.data_as(C.c_void_p), batch_size, ids.ctypes.data_as(C.c_void_p),
                               counts.ctypes.data_as(C.c_void_p), ids.size)
        if rc != steps:
            raise ValueError(f"draw_epoch failed ({rc})")
        return cls._wrap(ids, counts)

    @classmethod
    def from_steps(cls, steps_list) -> "EpochDraw":
        steps, K = len(steps_list), len(steps_list[0]) if steps_list else 0
        B = max((len(b) for st in steps_list for b in st), default=0)
        ids = np.full((steps, K, B), -1, dtype=np.int32)
        counts = np.zeros((steps, K), dtype=np.int32)
        for s, st in enumerate(steps_list):
            for k, b in enumerate(st):
                ids[s, k, :len(b)] = b
                counts[s, k] = len(b)
        return cls._wrap(ids, counts)


class Master:
    """core/Master.scala:19-255 (abstract).  `Master.apply` (Master.scala:259-271) is `Master.create`."""

    def __init__(self, node: int, data: Data, test_data: Data, model: Union[SparseSVM, SparseLogistic, SparseSquaredHinge, SparseModifiedHuber],
                 expected_node_count: int, *,
                 slave: Slave, group: Optional[Group] = None, seed: int = 0, log: Optional[Callable[[str], None]] = None,
                 jvm_exact: bool = False, attach: bool = True):
        self.node, self.model, self.expected_node_count = node, model, expected_node_count
        # every model but SparseSVM has non-integer loss sums: the float *_sums evaluations, gathered in rank order
        self.logistic = not isinstance(model, SparseSVM)
        # (w_pos, w_neg) as the Slave resolved and installed them; (1, 1): every evaluation makes the calls it made before
        self.class_weight = getattr(slave, "class_weight", (1.0, 1.0))
        # the Slave loaded per-row sample weights: every loss evaluation makes the *_weighted calls, whose loss sums already
        # carry the class weights, so the per-class split below is not used
        self.sample_weighted = bool(getattr(slave, "sample_weighted", False))
        self.weighted = self.class_weight != (1.0, 1.0) and not self.sample_weighted
        self.n_train, self.n_test = data.n_rows, test_data.n_rows
        self.dim = data.dim
        # the model fits an intercept (fit_intercept): every weight vector in or out is dim + 1 long, the intercept last
        self.intercept = bool(getattr(slave, "intercept", False))
        self.wdim = self.dim + (1 if self.intercept else 0)
        self.slave = slave
        self.ctx: NativeCtx = slave.ctx
        self.group = group or Group()
        if self.group.world != slave.world:
            raise ValueError("process group size and Slave world size differ")
        if slave.n_test != self.n_test or slave.n_train != self.n_train:
            raise ValueError("the Slave must hold the same train/test rows as the Master")
        # Random.setSeed(0) (Main.scala:32): one stream, identical on every rank
        self.seed = int(seed)
        self.rng = np.random.default_rng(seed)
        self._epochs_drawn = 0
        self._draw_cache = None   # fit_one_vs_rest: {(epoch, batch, groups): EpochDraw}, the draws every topic's fit shares
        # the Slave's topics (train rows, then test rows), None without any
        self.topics = getattr(slave, "topics", None)
        self._sampled_draws = 0   # t of sampled_key: device-drawn evaluation samples so far (apart from the epoch draws)
        # jvm_exact: draw the batches with java.util.Random(seed) + Scala 2.12's Random.shuffle, the stream a reference
        # run consumes (SURVEY.md 8f N4); default: numpy's generator (statistically the same draws, much faster)
        self.jvm = None
        if jvm_exact:
            from ..utils.jvm_random import JvmRandom
            self.jvm = JvmRandom(seed)
        self.log = log or (lambda s: None)
        # attach=False: the Slave's device context already carries its communicator / peer exchange
        if attach and self.group.world > 1 and not slave.is_async:
            # NCCL communicator (general path: several logical workers per GPU) ...
            uid = NativeCtx.comm_unique_id() if self.group.rank == 0 else b""
            self.ctx.comm_init(self.group.broadcast_bytes(uid, 0))
            # ... and the peer-memory exchange of the fused persistent kernel (one worker per GPU)
            if hasattr(self.ctx, "setup_peer_exchange"):
                self.ctx.setup_peer_exchange(self.group)

    @staticmethod
    def create(node, data, test_data, model, is_async, node_count, **kw) -> "Master":
        """Master.apply (core/Master.scala:259-271)."""
        return (MasterAsync if is_async else MasterSync)(node, data, test_data, model, node_count, **kw)

    # ---- evaluation ------------------------------------------------------------------------------------
    def _split(self, test_data: bool):
        """(b, e): the train rows [0, n_train) or the test rows [n_train, n_train + n_test)."""
        return (self.n_train, self.n_train + self.n_test) if test_data else (0, self.n_train)

    def _rows(self, test_data: bool, samples_count: Optional[int] = None, empty: Optional[str] = None) -> Optional[Rows]:
        """The rows of a request over the train (or test) rows: all of them (samples_count None), or a fresh sample of
        min(samples_count, n) of them (_draw_sample).  An empty sample raises DsgdEmpty with the message `empty`, or gives
        None when `empty` is None."""
        if samples_count is None:
            return Rows(*self._split(test_data))
        b, e, k, key, ids = self._draw_sample(samples_count, test_data)
        if k <= 0:
            if empty is None:
                return None
            raise DsgdEmpty(ERR_EMPTY, empty)
        return Rows(0, k, b, e, key, ids)

    def _local_eval(self, rows: Rows, weights):
        """(loss sum, correct count, ||w||^2) of `rows`: the eval_counts family for the SVM (its loss sum is the integer
        hinge sum), eval_sums for every other model.  With class weights eval_class, and a fourth value: (loss sum of the
        positive rows, correct count, ||w||^2, loss sum of the negative rows), unweighted.  With sample weights
        eval_weighted: (S = sum c_i L_i, correct count, ||w||^2)."""
        if self.sample_weighted:
            we = rows.call(self.ctx, "eval_weighted", weights)
            return we.loss_sum, we.correct, we.norm_squared
        if self.weighted:
            ce = rows.call(self.ctx, "eval_class", weights)
            as_sum = float if self.logistic else int   # the SVM's sums are integers: all-reduced exactly
            return as_sum(ce.loss_pos), ce.correct_pos + ce.correct_neg, ce.norm_squared, as_sum(ce.loss_neg)
        return rows.call(self.ctx, "eval_sums" if self.logistic else "eval_counts", weights)

    def _loss_sum(self, h, *h_neg):
        """The loss sum of an evaluation from its combined totals: h itself, or with class weights w_pos * h + w_neg * h_neg,
        formed once from the totals of all ranks."""
        return self.class_weight[0] * h + self.class_weight[1] * h_neg[0] if h_neg else h

    def _combine(self, h, c, n2, *rows):
        """(loss sum, correct[, rows], ||w||^2) over all ranks; ||w||^2 is identical on every rank that evaluated and 0 on idle
        ranks: its maximum.  SVM: the sums are integers below 2^53, exact in any order (all-reduce).  Logistic: the loss
        sums are not integers, so the partials are gathered and added in rank order and every rank gets the same bits --
        ranks whose stopping rule saw different losses would leave `fit` at different epochs and hang the next collective.
        Sample-weighted loss sums are not integers either: they take the logistic path."""
        if not (self.logistic or self.sample_weighted):
            return (*self.group.all_reduce_sum([h, c, *rows]), self.group.all_reduce_max(n2))
        mine = np.array([h, c, *rows, n2], dtype=np.float64)
        parts = [np.frombuffer(b, dtype=np.float64) for b in self.group.all_gather_bytes(mine.tobytes())]
        sums = [0.0] * (mine.size - 1)
        for p in parts:
            sums = [s + float(v) for s, v in zip(sums, p[:-1])]
        return (*sums, max(float(p[-1]) for p in parts))

    def _penalty(self, n2: float, weights, want_loss: bool) -> float:
        """lambda * ||w||^2, plus l1 * ||w||_1 of the same weights (weights None: the resident ones) when the model has an L1
        penalty.  ||w||_1 is an order-free device sum: the same bits on every rank.  want_loss False (an accuracy query): the
        loss is not used, so no device pass is made for ||w||_1."""
        if not self.model.l1:
            return self.model.lam * n2
        if not want_loss:
            return float("nan")
        return self.model.lam * n2 + self.model.l1 * self.ctx.weights_l1(weights)[0]

    def _loss_accuracy(self, weights, rows: Optional[Rows], want_loss: bool = True, grouped: bool = False):
        """(loss, accuracy) of a row-sharded pass over `rows`: rank r of W evaluates rows.shard(W, r), and the loss sums and
        counters are combined over ranks.  grouped (distributed_*): `rows` is already this rank's group of a split strategy
        (None: it has none), and the groups' row counts are combined with the sums."""
        share = rows if grouped else rows.shard(self.group.world, self.group.rank)
        if share is None:
            h, c, n2, *h_neg = (0, 0, 0.0, 0) if self.weighted else (0, 0, 0.0)
        else:
            h, c, n2, *h_neg = self._local_eval(share, weights)
        if grouped:
            hs, cs, n, *h_neg, n2 = self._combine(h, c, n2, 0 if share is None else share.hi - share.lo, *h_neg)
        else:
            hs, cs, *h_neg, n2 = self._combine(h, c, n2, *h_neg)
            n = rows.hi - rows.lo
        return self._penalty(n2, weights, want_loss) + self._loss_sum(hs, *h_neg) / n, cs / n

    def local_loss(self, weights=None, test_data: bool = False) -> float:
        """Master.localLoss (core/Master.scala:105-107)."""
        return self._loss_accuracy(weights, self._rows(test_data))[0]

    def local_accuracy(self, weights=None, test_data: bool = False) -> float:
        """Master.localAccuracy (core/Master.scala:100-103)."""
        return self._loss_accuracy(weights, self._rows(test_data), want_loss=False)[1]

    def local_loss_accuracy(self, weights=None, test_data: bool = False):
        return self._loss_accuracy(weights, self._rows(test_data))

    def _draw_sample(self, samples_count: int, test_data: bool):
        """(b, e, k, key, ids): a fresh sample of k = min(samples_count, n) of the working rows [b, e).  Every call draws anew,
        as every reference call reshuffles.  Default: the sample is drawn on the device with key = sampled_key(seed, t), t
        counting this Master's draws (the epoch draws of `fit` are separate); k <= 0 consumes no draw.  jvm_exact: ids =
        `Random.shuffle(indices) take k` from the java.util.Random stream `fit` also draws from (key is None)."""
        b, e = self._split(test_data)
        n = e - b
        k = min(int(samples_count), n)
        key = ids = None
        if self.jvm is not None:
            # the reference shuffles every index before `take`: the stream moves by one shuffle whatever k is
            ids = self.jvm.shuffle(np.arange(n, dtype=np.int32))[:max(k, 0)] + np.int32(b)
        elif k > 0:
            key = sampled_key(self.seed, self._sampled_draws)
            self._sampled_draws += 1
        return b, e, k, key, ids

    def local_sampled_loss(self, weights, samples_count: int, test_data: bool = False) -> float:
        """Master.localSampledLoss (core/Master.scala:109-112).  An empty sample raises DsgdEmpty, as the reference's
        `reduce` on an empty list throws."""
        return self.local_sampled_loss_accuracy(weights, samples_count, test_data)[0]

    def local_sampled_accuracy(self, weights, samples_count: int, test_data: bool = False) -> float:
        """Master.localSampledAccuracy (core/Master.scala:114-118).  An empty sample gives nan (the reference's 0.0 / 0)."""
        rows = self._rows(test_data, samples_count)
        return float("nan") if rows is None else self._loss_accuracy(weights, rows, want_loss=False)[1]

    def local_sampled_loss_accuracy(self, weights, samples_count: int, test_data: bool = False):
        """(loss, accuracy) on ONE sample, drawn once for both numbers; rank r of W evaluates positions sample_shard(k, W,
        r).  An empty sample raises DsgdEmpty."""
        return self._loss_accuracy(weights, self._rows(
            test_data, samples_count, f"sampled evaluation of {samples_count} rows: reduce on an empty collection"))

    # ---- per-class report (extension) -------------------------------------------------------------------------------------
    # Like the ranking metrics below it is not sharded: every rank holds every row and evaluates the whole range or sample,
    # and the counts are exact integers, so every rank returns the same numbers without a collective.
    def _class_report(self, ce, weights) -> dict:
        nan = float("nan")
        n = ce.n_pos + ce.n_neg
        rec_pos = ce.correct_pos / ce.n_pos if ce.n_pos else nan
        rec_neg = ce.correct_neg / ce.n_neg if ce.n_neg else nan
        pen = self._penalty(ce.norm_squared, weights, True)
        return {"n_pos": ce.n_pos, "n_neg": ce.n_neg, "correct_pos": ce.correct_pos, "correct_neg": ce.correct_neg,
                "recall_pos": rec_pos, "recall_neg": rec_neg, "balanced_accuracy": (rec_pos + rec_neg) / 2.0,
                "accuracy": (ce.correct_pos + ce.correct_neg) / n, "class_weight": self.class_weight,
                "loss": pen + (ce.loss_pos + ce.loss_neg) / n,
                "weighted_loss": pen + ce.weighted_loss_sum(*self.class_weight) / n}

    def local_class_report(self, weights=None, test_data: bool = False) -> dict:
        """Rows, correct predictions and recall per class, balanced accuracy, accuracy, and the loss both unweighted and
        under the model's class weights, over the train (or test) rows; works whatever the weights are."""
        return self._class_report(self._rows(test_data).call(self.ctx, "eval_class", weights), weights)

    def local_sampled_class_report(self, weights, samples_count: int, test_data: bool = False) -> dict:
        """local_class_report on a fresh sample (_draw_sample).  An empty sample raises DsgdEmpty."""
        rows = self._rows(test_data, samples_count, f"sampled evaluation of {samples_count} rows: reduce on an empty collection")
        return self._class_report(rows.call(self.ctx, "eval_class", weights), weights)

    # ---- sample-weighted report (extension) -------------------------------------------------------------------------------
    # Not sharded, like the per-class report: every rank evaluates the whole range or sample, and the fixed-point sums have
    # the same bits on every rank.
    def _weighted_report(self, we, weights) -> dict:
        nan = float("nan")
        pen = self._penalty(we.norm_squared, weights, True)
        return {"n": we.n, "weight_sum": we.weight_sum, "weighted_loss": pen + we.loss_sum / we.n,
                "weighted_accuracy": we.correct_weight / we.weight_sum if we.weight_sum > 0.0 else nan}

    def local_weighted_report(self, weights=None, test_data: bool = False) -> dict:
        """Rows, the sum of their combined weights c_i = class weight x sample weight, the weighted loss penalty + S / n and
        the weighted accuracy sum c_i [correct] / sum c_i over the train (or test) rows.  Without sample weights c_i is the
        class weight."""
        return self._weighted_report(self._rows(test_data).call(self.ctx, "eval_weighted", weights), weights)

    def local_sampled_weighted_report(self, weights, samples_count: int, test_data: bool = False) -> dict:
        """local_weighted_report on a fresh sample (_draw_sample).  An empty sample raises DsgdEmpty."""
        rows = self._rows(test_data, samples_count, f"sampled evaluation of {samples_count} rows: reduce on an empty collection")
        return self._weighted_report(rows.call(self.ctx, "eval_weighted", weights), weights)

    # ---- one-vs-rest topics (extension) ----------------------------------------------------------------------------------
    def _topic_weights(self, weights) -> np.ndarray:
        """[T, wdim] weights of every loaded topic, from an OneVsRest (its topics must be the loaded ones, in order) or an
        array."""
        if self.topics is None:
            raise ValueError("topic report: the Slave holds no topics")
        if isinstance(weights, OneVsRest):
            if tuple(weights.topics) != self.topics.names:
                raise ValueError("topic report: the model must hold one weight vector per loaded topic, in their order")
            weights = weights.weights
        W = np.ascontiguousarray(weights, dtype=np.float64)
        if W.shape != (self.topics.n_topics, self.wdim):
            raise ValueError(f"topic report: weights must be [{self.topics.n_topics}, {self.wdim}], got {W.shape}")
        return W

    def _topic_thresholds(self, weights, thresholds) -> Optional[np.ndarray]:
        """The margin thresholds of a topic report: `thresholds` when given, else an OneVsRest's own; None for neither (the
        binary rule, every tau 0)."""
        if thresholds is None and isinstance(weights, OneVsRest):
            thresholds = weights.thresholds
        if thresholds is None:
            return None
        thr = np.ascontiguousarray(thresholds, dtype=np.float64).reshape(-1)
        if thr.size != self.topics.n_topics or np.isnan(thr).any():
            raise ValueError(f"topic report: expected {self.topics.n_topics} thresholds, none NaN, got {thr.size}")
        return thr

    def _topic_report(self, W: np.ndarray, rows: Rows, k: Optional[int] = None, thr: Optional[np.ndarray] = None) -> dict:
        """The topic report (k None; at the margin thresholds thr when given) or the topic ranking report at k of the T
        weight vectors W over `rows`.  Rank r of R evaluates rows.shard(R, r), and the words are summed over ranks: integers
        and limbs below 2^40, so the float64 sum is exact, every rank gets the same bits and merged limbs convert once
        (topic_ranking_report)."""
        share = rows.shard(self.group.world, self.group.rank)
        if k is None and thr is not None:
            words = (np.zeros(topic_words(len(W)), np.int64) if share is None
                     else share.call(self.ctx, "eval_thresholded_topics", W, thr))
        elif k is None:
            words = np.zeros(topic_words(len(W)), np.int64) if share is None else share.call(self.ctx, "eval_topics", W)
        else:
            words = (np.zeros(topic_rank_words(k), np.int64) if share is None
                     else share.call(self.ctx, "eval_topic_ranking", W, k)[0])
        total = np.rint(self.group.all_reduce_sum([float(x) for x in words])).astype(np.int64)
        return topic_report(total, self.topics.names) if k is None else topic_ranking_report(total, k)

    def local_topic_report(self, weights, test_data: bool = True, thresholds=None) -> dict:
        """Multi-label quality of one-vs-rest weights (an OneVsRest or a [T, wdim] array) over the test (or train) rows, all
        topics in one device pass (dsgd_eval_topics): per topic the counts, precision, recall and F1; micro precision,
        recall and F1, macro F1, subset accuracy, Hamming loss and top-1 accuracy (ml/one_vs_rest.py: topic_report).  Each
        rank evaluates a contiguous share of the rows, as local_loss splits them.  With margin thresholds (`thresholds`, or
        an OneVsRest's own) topic t is predicted present below tau_t (dsgd_eval_thresholded_topics)."""
        W = self._topic_weights(weights)
        return self._topic_report(W, self._rows(test_data), thr=self._topic_thresholds(weights, thresholds))

    def local_sampled_topic_report(self, weights, samples_count: int, test_data: bool = True, thresholds=None) -> dict:
        """local_topic_report on a fresh sample of min(samples_count, n) rows, drawn as local_sampled_loss draws it once the
        weights are checked; rank r of R evaluates positions sample_shard(k, R, r).  An empty sample raises DsgdEmpty."""
        W = self._topic_weights(weights)
        thr = self._topic_thresholds(weights, thresholds)
        return self._topic_report(W, self._rows(test_data, samples_count,
                                                f"sampled topic report of {samples_count} rows: the sample is empty"),
                                  thr=thr)

    def _tune_topic_thresholds(self, weights, W: np.ndarray, rows: Rows, fbr: float):
        """(OneVsRest with the tuned thresholds, threshold_report) over `rows`.  Not sharded: the rows are replicated on
        every rank, and every rank tunes over the whole request and gets the same bits."""
        thr, words = rows.call(self.ctx, "tune_topic_thresholds", W, float(fbr))
        if isinstance(weights, OneVsRest):
            model = dataclasses.replace(weights, thresholds=thr)
        else:
            model = OneVsRest(W.copy(), self.topics.names, [], thr)
        return model, threshold_report(words, thr, self.topics.names)

    def tune_topic_thresholds(self, weights, test_data: bool = False, fbr: float = 0.0):
        """Each topic's F1-optimal margin threshold (SCut with the fbr fallback, dsgd_tune_topic_thresholds) for one-vs-rest
        weights (an OneVsRest or a [T, wdim] array) over the train (or test) rows: (an OneVsRest with those thresholds,
        its threshold_report).  Thresholds tuned on the rows the model was fitted on are optimistic: they fit the training
        margins, which separate better than new rows' do.  To tune on a list of held-out rows, call
        NativeCtx.tune_topic_thresholds_samples and put the thresholds into the OneVsRest."""
        W = self._topic_weights(weights)
        return self._tune_topic_thresholds(weights, W, self._rows(test_data), fbr)

    def sampled_tune_topic_thresholds(self, weights, samples_count: int, test_data: bool = False, fbr: float = 0.0):
        """tune_topic_thresholds on a fresh sample of min(samples_count, n) rows, drawn as local_sampled_loss draws it once
        the weights are checked.  An empty sample raises DsgdEmpty."""
        W = self._topic_weights(weights)
        return self._tune_topic_thresholds(weights, W, self._rows(
            test_data, samples_count, f"sampled threshold tuning of {samples_count} rows: the sample is empty"), fbr)

    def local_topic_ranking_report(self, weights, k: int, test_data: bool = True) -> dict:
        """Multi-label ranking quality of one-vs-rest weights (an OneVsRest or a [T, wdim] array) over the test (or train)
        rows in one device pass (dsgd_eval_topic_ranking): precision@j and recall@j for j = 1..k, label ranking average
        precision, coverage error and ranking loss (ml/one_vs_rest.py: topic_ranking_report).  Each rank evaluates a
        contiguous share of the rows, as local_topic_report splits them."""
        return self._topic_report(self._topic_weights(weights), self._rows(test_data), k)

    def local_sampled_topic_ranking_report(self, weights, k: int, samples_count: int, test_data: bool = True) -> dict:
        """local_topic_ranking_report on a fresh sample of min(samples_count, n) rows, drawn as local_sampled_loss draws it
        once the weights are checked; rank r of R evaluates positions sample_shard(m, R, r) of the m drawn rows.  An empty
        sample raises DsgdEmpty."""
        W = self._topic_weights(weights)
        return self._topic_report(W, self._rows(test_data, samples_count,
                                                f"sampled topic ranking report of {samples_count} rows: the sample is empty"), k)

    # ---- ranking metrics (extension) -------------------------------------------------------------------------------------
    # AUC is not a sum over rows, so these are not sharded: rows are replicated on every rank (quirk Q13) and every rank
    # evaluates the whole range or sample itself.  The counts are exact integers, so every rank returns the same bits without
    # a collective.
    def local_metrics(self, weights=None, test_data: bool = False) -> dict:
        """Confusion counts, precision, recall, F1, ROC AUC and accuracy over the train (or test) rows (metrics_dict).
        weights None: the resident weights -- in `fit` the last iterate, not the average of average_from."""
        return metrics_dict(self._rows(test_data).call(self.ctx, "eval_metrics", weights))

    def local_sampled_metrics(self, weights, samples_count: int, test_data: bool = False) -> dict:
        """local_metrics on a fresh sample of min(samples_count, n) rows, drawn as local_sampled_loss draws it (one draw of
        sampled_key, or the jvm_exact shuffle).  An empty sample raises DsgdEmpty."""
        rows = self._rows(test_data, samples_count, f"sampled metrics of {samples_count} rows: the sample is empty")
        return metrics_dict(rows.call(self.ctx, "eval_metrics", weights))

    def local_curve(self, weights=None, test_data: bool = False, curve: bool = True) -> dict:
        """local_metrics plus average precision, and with `curve` the ROC and precision-recall points over the train (or test)
        rows (curve_dict).  Like local_metrics, every rank evaluates the whole range."""
        return curve_dict(self._rows(test_data).call(self.ctx, "eval_curve", weights, curve=curve))

    def local_sampled_curve(self, weights, samples_count: int, test_data: bool = False, curve: bool = True) -> dict:
        """local_curve on a fresh sample of min(samples_count, n) rows, drawn as local_sampled_metrics draws it.  An empty
        sample raises DsgdEmpty."""
        rows = self._rows(test_data, samples_count, f"sampled curve of {samples_count} rows: the sample is empty")
        return curve_dict(rows.call(self.ctx, "eval_curve", weights, curve=curve))

    def local_weighted_curve(self, weights=None, test_data: bool = False, curve: bool = True) -> dict:
        """local_curve with every row counted by its weight c_i = class weight x sample weight (weighted_curve_dict).  Not
        sharded either: every rank evaluates the whole range, and every word is an order-free fixed-point sum, so every
        rank gets the same bits."""
        return weighted_curve_dict(self._rows(test_data).call(self.ctx, "eval_weighted_curve", weights, curve=curve), curve)

    def local_sampled_weighted_curve(self, weights, samples_count: int, test_data: bool = False, curve: bool = True) -> dict:
        """local_weighted_curve on a fresh sample of min(samples_count, n) rows, drawn as local_sampled_curve draws it.  An
        empty sample raises DsgdEmpty."""
        rows = self._rows(test_data, samples_count, f"sampled weighted curve of {samples_count} rows: the sample is empty")
        return weighted_curve_dict(rows.call(self.ctx, "eval_weighted_curve", weights, curve=curve), curve)

    # ---- bootstrap (extension) -------------------------------------------------------------------------------------------
    # Poisson-bootstrap intervals of the ranking metrics, accuracy and loss (dsgd_eval_*bootstrap).  Every rank holds every
    # row; rank r computes the replicates bootstrap_share(n_boot, W, r) and all are gathered in rank order, so every rank
    # returns the same bits -- a replicate's bits do not depend on which rank computed it.
    # weighted=True counts every row by its weight c_i = class weight x sample weight (dsgd_eval_*weighted_bootstrap): the
    # same seven metrics by weighted_curve_dict's formulas, the estimates from the weighted curve and evaluation calls.
    def _estimates(self, cw, sums, weights):
        """(estimates, penalty) of an unweighted bootstrap from the curve words and the *_sums of its rows."""
        penalty = self._penalty(sums[2], weights, True)
        words, ap = cw[0], cw[1]
        n = int(np.sum(np.asarray(words)[[0, 1, 2, 3, 4, 5]]))
        est = {k: float(v[0]) for k, v in bootstrap_values(np.concatenate([words, [n]]), [ap], [sums[0]], penalty).items()}
        return est, penalty

    def _weighted_estimates(self, wc, we, weights):
        """(estimates, penalty) of a weighted bootstrap, as local_weighted_curve and local_weighted_report form them."""
        curve, report = weighted_curve_dict(wc, curve=False), self._weighted_report(we, weights)
        est = {"accuracy": curve["accuracy"], "loss": report["weighted_loss"], "auc": curve["auc"],
               "ap": curve["average_precision"], "precision": curve["precision"], "recall": curve["recall"],
               "f1": curve["f1"]}
        return est, self._penalty(we.norm_squared, weights, True)

    # weighted -> (curve family, evaluation family, estimates, replicate family, replicate values)
    _BOOTSTRAP = {False: ("eval_curve", "eval_sums", _estimates, "eval_bootstrap", bootstrap_values),
                  True: ("eval_weighted_curve", "eval_weighted", _weighted_estimates, "eval_weighted_bootstrap",
                         weighted_bootstrap_values)}

    def _bootstrap_case(self, weights, rows: Rows, n_boot: int, key: Optional[int], weighted: bool):
        """(estimates, replicates) of one bootstrap over `rows`: the estimates from the curve and evaluation calls over the
        same rows, and every BOOTSTRAP_METRICS value of replicates [0, n_boot) with `key` (None: bootstrap_key(seed)), rank r
        computing bootstrap_share(n_boot, W, r), gathered in rank order."""
        weighted = bool(weighted)
        curve_family, eval_family, estimates, family, values = self._BOOTSTRAP[weighted]
        est, penalty = estimates(self, rows.call(self.ctx, curve_family, weights, curve=False),
                                 rows.call(self.ctx, eval_family, weights), weights)
        key = bootstrap_key(self.seed) if key is None else int(key)
        if n_boot <= 0:
            raise ValueError(f"n_boot: expected a number of replicates > 0, got {n_boot}")
        lo, hi = bootstrap_share(int(n_boot), self.group.world, self.group.rank)
        mine = bootstrap_pack(*rows.call(self.ctx, family, key, lo, hi, weights)) if hi > lo else np.zeros(0)
        parts = [np.frombuffer(b, dtype=np.float64) for b in self.group.all_gather_bytes(mine.tobytes())]
        return est, values(*bootstrap_unpack(parts, weighted), penalty)

    def _bootstrap(self, weights, rows: Rows, n_boot, key, level, weighted) -> dict:
        est, reps = self._bootstrap_case(weights, rows, n_boot, key, weighted)
        return {m: bootstrap_summary(est[m], reps[m], level) for m in BOOTSTRAP_METRICS}

    def local_bootstrap(self, weights=None, test_data: bool = True, n_boot: int = 1000, key: Optional[int] = None,
                        level: float = 0.95, weighted: bool = False) -> dict:
        """Poisson-bootstrap intervals over the test (or train) rows: for each of accuracy, loss (penalty + S / n, the
        unweighted loss of the *_sums calls), auc, ap, precision, recall and f1 (BOOTSTRAP_METRICS) a dict of the full-sample
        estimate, the percentile interval [lo, hi] at `level` over the replicates where the metric is defined, n_defined,
        the standard error se and the raw replicates.  key None: bootstrap_key(seed).  weighted: every row counted by its
        weight c_i = class weight x sample weight -- the metrics of local_weighted_curve and the loss of
        local_weighted_report, resampled with the same multiplicities as the unweighted bootstrap of the same key."""
        return self._bootstrap(weights, self._rows(test_data), n_boot, key, level, weighted)

    def local_sampled_bootstrap(self, weights, samples_count: int, test_data: bool = True, n_boot: int = 1000,
                                key: Optional[int] = None, level: float = 0.95, weighted: bool = False) -> dict:
        """local_bootstrap over a fresh sample of min(samples_count, n) rows (_draw_sample).  An empty sample raises
        DsgdEmpty."""
        rows = self._rows(test_data, samples_count, f"sampled bootstrap of {samples_count} rows: the sample is empty")
        return self._bootstrap(weights, rows, n_boot, key, level, weighted)

    def compare_bootstrap(self, weights_a, weights_b, test_data: bool = True, n_boot: int = 1000, key: Optional[int] = None,
                          level: float = 0.95, weighted: bool = False) -> dict:
        """Paired comparison of two weight vectors over the same rows: both are scored with the same bootstrap key, so
        replicate b resamples the same rows for both.  Per metric: the difference b - a of the estimates, its percentile
        interval, standard error and defined-replicate count (replicates where the metric is defined for both), and
        p_better, the share of those replicates in which b is better (higher, or lower for the loss).  weighted: as in
        local_bootstrap."""
        key = bootstrap_key(self.seed) if key is None else int(key)
        rows = self._rows(test_data)
        (ea, ra), (eb, rb) = [self._bootstrap_case(w, rows, n_boot, key, weighted) for w in (weights_a, weights_b)]
        out = {}
        for m, higher in BOOTSTRAP_METRICS.items():
            d = rb[m] - ra[m]
            s = bootstrap_summary(eb[m] - ea[m], d, level)
            ok = d[~np.isnan(d)]
            s["p_better"] = float(np.mean(ok > 0 if higher else ok < 0)) if ok.size else float("nan")
            out[m] = s
        return out

    # ---- calibration (extension) -----------------------------------------------------------------------------------------
    # Like the ranking metrics, these are not sharded: rows are replicated on every rank and every rank fits or evaluates
    # the whole range or sample itself.  Every sum over the rows is an order-free fixed-point sum and the arithmetic between
    # the sums is one fixed sequence, so every rank gets the same bits without a collective.  None of them touches the
    # weights or the step state: they can be called from `fit`'s on_epoch hook.
    def calibrate(self, weights=None, test_data: bool = False, method: str = "sigmoid", weighted: bool = False):
        """A calibration of the margins over the train (or test) rows.  method "sigmoid": Platt scaling, the Calibration
        (a, b) that makes 1 / (1 + exp(a x.w + b)) a probability; "isotonic": isotonic regression, an IsotonicCalibration.
        weights None: the resident weights, as in local_metrics.  weighted: fitted with every row counted by its weight
        c_i = class weight x sample weight (dsgd_calibrate_weighted, dsgd_calibrate_isotonic_weighted)."""
        family, convert = _FITS[bool(weighted), _method(method) == "isotonic"]
        return convert(self._rows(test_data).call(self.ctx, family, weights))

    def sampled_calibrate(self, weights, samples_count: int, test_data: bool = False, method: str = "sigmoid",
                          weighted: bool = False):
        """calibrate on a fresh sample of min(samples_count, n) rows, drawn as local_sampled_metrics draws it once the method
        is checked.  An empty sample raises DsgdEmpty."""
        family, convert = _FITS[bool(weighted), _method(method) == "isotonic"]
        rows = self._rows(test_data, samples_count, f"sampled calibration of {samples_count} rows: the sample is empty")
        return convert(rows.call(self.ctx, family, weights))

    def _calibration_quality(self, calibration, weights, rows: Rows, n_bins: int, weighted: bool) -> dict:
        """local_calibration over `rows`: the quality family of the calibration's kind and of `weighted` (_QUALITY)."""
        isotonic = isinstance(calibration, IsotonicCalibration)
        family, convert = _QUALITY[bool(weighted), isotonic]
        params = (calibration.x, calibration.y) if isotonic else (calibration.a, calibration.b)
        return convert(rows.call(self.ctx, family, *params, n_bins, weights))

    def local_calibration(self, calibration, weights=None, test_data: bool = False, n_bins: int = 10,
                          weighted: bool = False) -> dict:
        """How well `calibration` (a Calibration or an IsotonicCalibration) fits the train (or test) rows: Brier score, log
        loss, expected and maximum calibration error and the reliability bins (calibration_dict; isotonic_calibration_dict
        for an isotonic map).  Every rank evaluates the whole range itself.  weighted: every row counted by its weight c_i
        (weighted_calibration_dict)."""
        return self._calibration_quality(calibration, weights, self._rows(test_data), n_bins, weighted)

    def local_sampled_calibration(self, calibration: Calibration, weights, samples_count: int, test_data: bool = False,
                                  n_bins: int = 10, weighted: bool = False) -> dict:
        """local_calibration on a fresh sample of min(samples_count, n) rows.  An empty sample raises DsgdEmpty."""
        rows = self._rows(test_data, samples_count,
                          f"sampled calibration quality of {samples_count} rows: the sample is empty")
        return self._calibration_quality(calibration, weights, rows, n_bins, weighted)

    def predict(self, weights, split_strategy: Split = SplitStrategy.vanilla) -> dict:
        """Master.predict (core/Master.scala:61-75): idx -> prediction over the training rows; each worker
        answers for its split group."""
        groups = split_strategy(self.n_train, self.group.world)
        mine = groups[self.group.rank] if self.group.rank < len(groups) else range(0)
        idx = np.fromiter(mine, dtype=np.int32, count=len(mine))
        preds = self.slave.forward(idx, weights) if len(idx) else np.zeros(0)
        import pickle
        parts = self.group.all_gather_bytes(pickle.dumps((idx, preds)))
        out = {}
        for blob in parts:
            i, p = pickle.loads(blob)
            out.update(zip(i.tolist(), p.tolist()))
        return out

    def distributed_accuracy(self, weights, split_strategy: Split = SplitStrategy.vanilla) -> float:
        """Master.distributedAccuracy (core/Master.scala:77-85)."""
        return self._loss_accuracy(weights, self._group_rows(split_strategy), want_loss=False, grouped=True)[1]

    def distributed_loss(self, weights, split_strategy: Split = SplitStrategy.vanilla) -> float:
        """Master.distributedLoss (core/Master.scala:87-98)."""
        return self._loss_accuracy(weights, self._group_rows(split_strategy), grouped=True)[0]

    def _group_rows(self, split_strategy: Split) -> Optional[Rows]:
        """This rank's group of split_strategy over the train rows, None when it has none: the same numbers as predict +
        host-side counting, without shipping N predictions around."""
        groups = split_strategy(self.n_train, self.group.world)
        mine = groups[self.group.rank] if self.group.rank < len(groups) else range(0)
        return Rows(mine.start, mine.stop) if len(mine) else None


class MasterSync(Master):
    """core/MasterSync.scala + the sync `fit` of core/Master.scala:120-218."""

    def update_grad(self, grad_update):  # MasterSync.scala:16-17
        raise NotImplementedError("Synchronous master cannot perform async operation update grad")

    def draw_epoch(self, groups: List[range], batch_size: int, epoch: Optional[int] = None):
        """Sample ids of one epoch: for every step (`0 until maxSamples by batchSize`, Master.scala:179) and
        every worker a fresh shuffle of its range, sliced at [batch, batch + batchSize) (Master.scala:
        184-187, quirk Q5).  A slice of a fresh permutation is a uniform draw without replacement of
        min(batchSize, len - batch) elements -- drawn directly (csrc/dsgd_host.c: dsgd_draw_epoch) from a counter-based
        generator keyed by (seed, epoch, step, worker), identical on every rank.  Returns an EpochDraw: a list of steps,
        each a list of per-worker arrays (what the oracle replays), plus the same ids as one array for the device."""
        if epoch is None:
            epoch = self._epochs_drawn
        self._epochs_drawn = epoch + 1
        if self.jvm is not None:
            n, size = groups[-1].stop, len(groups[0])
            if [(g.start, g.stop) for g in groups] != [(a, min(a + size, n)) for a in range(0, n, size)]:
                raise ValueError("jvm_exact draws are defined for SplitStrategy.vanilla groups")
            return EpochDraw.from_steps(self.jvm.sync_epoch(n, len(groups), batch_size, group_size=size))
        if self._draw_cache is not None:   # the draws do not depend on the labels: one draw per epoch for every topic
            key = (epoch, batch_size, tuple((g.start, g.stop) for g in groups))
            if key not in self._draw_cache:
                self._draw_cache[key] = EpochDraw.draw(self.seed, epoch, groups, batch_size)
            return self._draw_cache[key]
        return EpochDraw.draw(self.seed, epoch, groups, batch_size)

    def fit_one_vs_rest(self, initial_weights: np.ndarray, max_epochs: int, batch_size: int, learning_rate: float,
                        stopping_criterion: EarlyStopping, topics=None, **fit_kwargs) -> OneVsRest:
        """One-vs-rest training of the Slave's topics: for each chosen topic t (topics None: every loaded topic, else their
        names or indices, in that order) the device labels become "has topic t" (ctx.select_topic), a "balanced"
        class_weight is resolved again from topic t's train labels, and `fit` runs with the given arguments.  Each fit
        draws exactly the batches of a fresh MasterSync of the same seed (epoch numbering restarts at 0); the draws do not
        depend on the labels, so every epoch is drawn once and shared by all topics.  Every rank runs the same sequence.
        A topic without a positive or without a negative train row, and jvm_exact (its stream is one reference run), are
        refused before any fit.  The loaded labels and the Slave's class weights are restored afterwards, also when a fit
        raises."""
        if self.topics is None:
            raise ValueError("fit_one_vs_rest: the Slave holds no topics")
        if self.jvm is not None:
            raise ValueError("fit_one_vs_rest: jvm_exact draws are one reference run's stream; one-vs-rest fits cannot share it")
        names = self.topics.names
        chosen = list(range(len(names))) if topics is None else [names.index(t) if t in names else -1 if isinstance(t, str)
                                                                  else int(t) for t in topics]
        if not chosen or any(not 0 <= t < len(names) for t in chosen):
            raise ValueError(f"fit_one_vs_rest: topics must name loaded topics, got {topics!r}")
        train = self.topics.rows(0, self.n_train)
        labels = {t: train.labels(t) for t in chosen}
        for t in chosen:
            n_pos = int(np.count_nonzero(labels[t] > 0))
            if n_pos == 0 or n_pos == self.n_train:
                raise ValueError(f"fit_one_vs_rest: topic {names[t]!r} has {n_pos} positive train rows of {self.n_train}; "
                                 "both classes are needed")
        balanced = getattr(self.model, "class_weight", None) == "balanced"
        saved = (self.class_weight, self.weighted, getattr(self.slave, "class_weight", self.class_weight))
        weights, histories = [], []
        self._draw_cache = {}
        try:
            for t in chosen:
                self.ctx.select_topic(t)
                if balanced:
                    cw = resolve_class_weight("balanced", labels[t])
                    self.ctx.set_class_weights(*cw)
                    self.class_weight, self.slave.class_weight = cw, cw
                    self.weighted = cw != (1.0, 1.0) and not self.sample_weighted
                self._epochs_drawn = 0
                state = self.fit(initial_weights, max_epochs, batch_size, learning_rate, stopping_criterion, **fit_kwargs)
                weights.append(np.array(state.grad, dtype=np.float64))
                histories.append(self.history)
        finally:
            self._draw_cache = None
            self._epochs_drawn = 0
            self.ctx.select_topic(-1)
            self.class_weight, self.weighted, self.slave.class_weight = saved
            if balanced:
                self.ctx.set_class_weights(*saved[0])
        return OneVsRest(np.stack(weights), tuple(names[t] for t in chosen), histories)

    def fit(self, initial_weights: np.ndarray, max_epochs: int, batch_size: int, learning_rate: float,
            stopping_criterion: EarlyStopping, split_strategy: Split = SplitStrategy.vanilla, *,
            virtual_workers: int = 1, on_epoch: Optional[Callable[[int, dict], None]] = None,
            average_from: Optional[int] = None, learning_rate_decay: float = 0.0,
            learning_rate_power: float = 1.0) -> GradState:
        """Master.fit (core/Master.scala:120-218).

        virtual_workers (extension): logical reference workers per GPU, so that `node-count` can exceed the
        number of GPUs (K = world * virtual_workers).
        average_from (extension): averaged SGD from epoch `average_from` (0-based) on.  The device adds the weights after
        every step of that epoch and of the later ones to a running sum (ctx.average_begin); the per-epoch evaluations, and
        so the stopping rule, then see the mean of those weights, and `fit` returns it.  history["averaged_steps"] holds
        the number of steps averaged.  None: the last weights, as in the reference.
        learning_rate_decay, learning_rate_power (extension): step t of the fit (counted from 0 over every epoch) uses
        learning_rate / (1 + decay * t)^power (ml/lr_schedule.py), handed to the device as a per-step table
        (ctx.sync_steps_lr).  decay = 0: the constant learning_rate of the reference, through the scalar calls of before.
        Together with average_from this is Bottou's averaged SGD (power 0.75 in svmasgd).
        A model with l1 > 0 (the Slave set it on the device) soft-thresholds every weight in every step; the losses then
        include l1 * ||w||_1 and history["nnz"] holds the non-zero weights of each epoch's evaluated weights.
        """
        if average_from is not None and not 0 <= average_from < max_epochs:
            raise ValueError(f"average_from must lie in [0, max_epochs = {max_epochs}), got {average_from}")
        if np.asarray(initial_weights).size != self.wdim:
            raise ValueError(f"initial_weights: expected {self.wdim} values (dim = {self.dim}"
                             f"{' and the intercept last' if self.intercept else ''}), got {np.asarray(initial_weights).size}")
        check_schedule(learning_rate_decay, learning_rate_power)
        decaying = learning_rate_decay > 0.0
        t_global = 0   # global index of the next step: the schedule's t
        W, r, V = self.group.world, self.group.rank, virtual_workers
        K = W * V
        groups = split_strategy(self.n_train, K)             # Master.scala:136 (may hold fewer than K groups)
        k_total = len(groups)                                 # workers.zip(split): extra workers get no request
        my_groups = [k for k in range(r * V, (r + 1) * V) if k < k_total]
        self.ctx.set_weights(initial_weights)
        state = GradState.start_state(np.asarray(initial_weights, dtype=np.float64))
        losses: List[float] = []
        accs: List[float] = []
        test_losses: List[float] = []
        test_accs: List[float] = []
        nnz: List[int] = []
        self.step_losses: List[np.ndarray] = []
        epoch = 0
        # a one-thread pool overlaps the next epoch's draw with the current epoch's kernel (not with jvm_exact: that
        # stream is sequential and must not run ahead of an early stop)
        from concurrent.futures import ThreadPoolExecutor
        prefetch = ThreadPoolExecutor(1) if self.jvm is None else None
        pending = None
        averaging, n_averaged = False, 0   # averaging: average_begin was called, so average_end on every way out
        try:
            while True:
                if losses:
                    self.log(f"loss after epoch {epoch}: {losses[0]}")
                    self.log(f"acc after epoch {epoch}: {accs[0]}")
                if epoch >= max_epochs or stopping_criterion(test_losses):   # Master.scala:154,166
                    self.log("Reached max number of epochs: stopping computation" if epoch >= max_epochs
                             else "Converged to target: stopping computation")
                    self.history = {"losses": losses[::-1], "test_losses": test_losses[::-1], "accs": accs[::-1],
                                    "test_accs": test_accs[::-1]}
                    if average_from is not None:
                        self.history["averaged_steps"] = n_averaged
                    if self.model.l1:
                        self.history["nnz"] = nnz[::-1]
                    if prefetch is not None:
                        prefetch.shutdown(wait=True)
                    # `losses.head` throws on an empty list in the reference (max_epochs == 0)
                    return state.finish(losses[0])
                if epoch == average_from:
                    self.ctx.average_begin()    # the steps of this epoch and of every later one are averaged
                    averaging = True
                steps = pending.result() if pending is not None else self.draw_epoch(groups, batch_size)
                pending = None
                if not isinstance(steps, EpochDraw):
                    steps = EpochDraw.from_steps(steps)
                if prefetch is not None and epoch + 1 < max_epochs:
                    # the draws of epoch e + 1 do not depend on epoch e: make them while the GPU runs epoch e
                    pending = prefetch.submit(self.draw_epoch, groups, batch_size, self._epochs_drawn)
                counts = steps.counts                                                 # [steps, k_total]
                if counts.size and (counts[:, :k_total] == 0).any():
                    raise ValueError("Cannot sum an empty list of vectors")  # Vec.scala:129 via Master.scala:187 (Q7)
                # consecutive steps with identical counts for ALL workers go to the device in one call; the boundaries come
                # from the global shape so that every rank issues the same sequence of calls (the fused multi-GPU kernel
                # numbers its exchange tags by call)
                n_steps = counts.shape[0]
                change = np.flatnonzero((counts[1:] != counts[:-1]).any(axis=1)) + 1 if n_steps > 1 else np.zeros(0, dtype=np.int64)
                bounds = [0, *change.tolist(), n_steps]
                for i, j in zip(bounds[:-1], bounds[1:]):
                    if j == i:
                        continue
                    shape = [int(counts[i, k]) for k in my_groups]
                    if my_groups:
                        g0, g1 = my_groups[0], my_groups[-1] + 1
                        if all(c == steps.ids.shape[2] for c in shape):
                            flat = np.ascontiguousarray(steps.ids[i:j, g0:g1, :]).reshape(-1)
                        else:
                            flat = np.concatenate([steps.ids[s, k, :counts[s, k]] for s in range(i, j) for k in my_groups])
                    else:
                        flat = np.zeros(0, dtype=np.int32)
                    self.ctx.set_workers(shape, k_total)
                    if decaying:   # this call's slice of the fit's table: the same on every rank
                        lrs = learning_rates(learning_rate, learning_rate_decay, learning_rate_power, t_global, j - i)
                        ls = self.ctx.sync_steps_lr(flat, int(sum(shape)), lrs, want_losses=True)
                    else:
                        ls = self.ctx.sync_steps(flat, int(sum(shape)), j - i, learning_rate, want_losses=True)
                    t_global += j - i
                    self.step_losses.append(ls)
                # evaluate the resident weights, or while averaging the mean of the averaged steps' weights
                w = None
                if averaging:
                    w, n_averaged = self.ctx.average_weights()
                tl, ta = self.local_loss_accuracy(w, test_data=False)        # Master.scala:206-207
                vl, va = self.local_loss_accuracy(w, test_data=True)         # Master.scala:208-209
                losses.insert(0, tl); accs.insert(0, ta); test_losses.insert(0, vl); test_accs.insert(0, va)
                if self.model.l1:
                    nnz.insert(0, self.ctx.weights_l1(w)[1])
                epoch += 1
                state = state.replace_grad(self.ctx.get_weights() if w is None else w)   # Master.scala:205
                if on_epoch:
                    on_epoch(epoch, {"loss": tl, "acc": ta, "test_loss": vl, "test_acc": va})
        finally:
            if averaging:
                self.ctx.average_end()


class MasterAsync(Master):
    """core/MasterAsync.scala -- Hogwild: every worker runs its loop on its GPU and pushes deltas into every peer
    replica and into the master replica (hosted on rank 0's GPU) over NVLink; the master logic polls the update
    counter, evaluates the master replica on the test rows every `check_every` updates with a leaky average, keeps
    the best weights, and stops on `n_train * max_epoch` updates or the early-stopping rule.  SparseSVM only."""

    def __init__(self, node, data, test_data, model, expected_node_count, **kw):
        if isinstance(model, (SparseLogistic, SparseSquaredHinge, SparseModifiedHuber)):
            raise ValueError(f"{type(model).__name__}: asynchronous (Hogwild) training supports SparseSVM only")
        if model.l1:
            raise ValueError("l1: the L1 penalty is a step of sync training; asynchronous (Hogwild) training has none")
        if getattr(model, "fit_intercept", False):
            raise ValueError("fit_intercept: the intercept is fitted by sync training; asynchronous (Hogwild) training has none")
        from ..ml.class_weight import resolve_class_weight
        if resolve_class_weight(getattr(model, "class_weight", None), data.label) != (1.0, 1.0):   # as the Slave decides
            raise ValueError("class_weight: class weights belong to sync training; asynchronous (Hogwild) training has none")
        if has_sample_weights(data, test_data):   # as the Slave decides
            raise ValueError(SAMPLE_WEIGHT_ASYNC)
        super().__init__(node, data, test_data, model, expected_node_count, **kw)

    def _attach_replicas(self):
        from ..native import REPLICA_MASTER, REPLICA_SELF
        W, r = self.group.world, self.group.rank
        mine = self.ctx.ipc_export(REPLICA_SELF)
        master = self.ctx.ipc_export(REPLICA_MASTER) if r == 0 else b""
        handles = self.group.all_gather_bytes(mine)
        master = self.group.broadcast_bytes(master, 0)
        for k, h in enumerate(handles):
            if k != r:
                self.ctx.ipc_import(k, h)
        if r != 0:
            self.ctx.ipc_import(W, master)
        self.group.barrier()

    def fit(self, initial_weights: np.ndarray, max_epoch: int, batch_size: int, learning_rate: float,
            stopping_criterion: EarlyStopping, split_strategy: Split = SplitStrategy.vanilla, check_every: int = 100,
            leak_loss_coef: float = 0.9, *, concurrency: int = 1, poll_seconds: float = 0.05, seed: int = 0,
            on_check: Optional[Callable[[int, dict], None]] = None) -> GradState:
        """MasterAsync.fit (core/MasterAsync.scala:32-62) + startLossChecking (96-162) + updateGrad's stop rule
        (164-177) + endComputation (87-94).  concurrency (extension): Hogwild lanes per GPU."""
        import time
        if not (0 <= leak_loss_coef <= 1):
            raise ValueError("leaking coefficient must be between 0 and 1")      # MasterAsync.scala:97
        if getattr(self, "_running", False):
            raise RuntimeError("Cannot start async computation: a computation is already running")
        W, r = self.group.world, self.group.rank
        w0 = np.asarray(initial_weights, dtype=np.float64)
        groups = split_strategy(self.n_train, W)
        max_steps = self.n_train * max_epoch                                      # MasterAsync.scala:83
        self.ctx.set_weights(w0)                     # every replica first, then the loops (no start-up race)
        if r == 0:
            self.ctx.async_host_master(w0)
        if W > 1:
            self._attach_replicas()
        self._running = True
        mine = groups[r] if r < len(groups) else range(0)
        if len(mine):
            self.slave.start_async(None, np.fromiter(mine, dtype=np.int32, count=len(mine)), batch_size, learning_rate,
                                   concurrency=concurrency, max_updates=0, seed=seed + 1000 * r)
        state = GradState.start_state(w0)
        test_losses: List[float] = []
        test_accs: List[float] = []
        best_loss, best_w = float("inf"), None
        last_step = -check_every                                                  # MasterAsync.scala:161
        # polls: every look at the update counter (updates, computed?); raw_*: the unsmoothed numbers of the computed polls --
        # what a replay of core/MasterAsync.scala:96-162 over the same stream needs (tests/test_host_logic.py)
        self.history = {"test_losses": test_losses, "test_accs": test_accs, "checks_at": [], "polls": [],
                        "raw_test_losses": [], "raw_test_accs": [], "best_check": None, "ended_by": None}
        try:
            while True:
                updates = self.ctx.async_updates() if r == 0 else 0
                updates = int(self.group.all_reduce_max(float(updates)))
                if updates >= max_steps:                                          # MasterAsync.scala:171-174
                    self.log("max number of steps reached: stopping computation")
                    self.history["polls"].append((updates, False))
                    self.history["ended_by"] = "max_steps"
                    break
                if updates - last_step < check_every:                             # latest computation was too close
                    self.history["polls"].append((updates, False))
                    time.sleep(poll_seconds)                                      # (the reference waits 2.5 s)
                    continue
                # innerGradState.grad: ONE snapshot (rank 0 hosts the master replica), evaluated row-sharded by everybody
                blob = self.ctx.async_master_weights().tobytes() if r == 0 else b""
                w = np.frombuffer(self.group.broadcast_bytes(blob, 0), dtype=np.float64).copy()
                loss, acc = self.local_loss_accuracy(w, test_data=True)           # MasterAsync.scala:118-120
                loss_s = leak_loss_coef * loss + (1 - leak_loss_coef) * (test_losses[0] if test_losses else loss)
                acc_s = leak_loss_coef * acc + (1 - leak_loss_coef) * (test_accs[0] if test_accs else acc)
                if best_loss > loss_s:                                            # MasterAsync.scala:130-139
                    best_loss, best_w = loss_s, w
                    self.history["best_check"] = len(self.history["checks_at"])
                test_losses.insert(0, loss_s)
                test_accs.insert(0, acc_s)
                self.history["checks_at"].append(updates)
                self.history["polls"].append((updates, True))
                self.history["raw_test_losses"].append(loss)
                self.history["raw_test_accs"].append(acc)
                if on_check:
                    on_check(updates, {"test_loss": loss_s, "test_acc": acc_s, "weights": w})
                if stopping_criterion(test_losses):                               # MasterAsync.scala:146-152
                    self.log("converged to target: stopping computation")
                    self.history["ended_by"] = "converged"
                    break
                last_step = updates
        finally:
            if len(mine):
                self.slave.stop_async()                                           # endComputation: stopAsync to all
            self._running = False
            self.group.barrier()
        if best_w is None:
            # the reference would hand back its initial bestGrad (Vec.zeros(1)) here; we return what the master holds
            blob = self.ctx.async_master_weights().tobytes() if r == 0 else b""
            best_w = np.frombuffer(self.group.broadcast_bytes(blob, 0), dtype=np.float64).copy()
            best_loss = self.local_loss_accuracy(best_w, test_data=True)[0]
        return state.replace_grad(best_w).finish(best_loss)                       # MasterAsync.scala:91
