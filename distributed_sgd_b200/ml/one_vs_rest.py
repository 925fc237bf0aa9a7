"""One-vs-rest (OvR) models of a multi-label set: one binary model per topic, "has topic t" against the rest.

`MasterSync.fit_one_vs_rest` trains them one topic after another on one device context (dsgd_select_topic switches the
labels on the device), and `Master.local_topic_report` judges them all in one pass (dsgd_eval_*topics).  The ranking of a
row's topics by their scores is one more pass: `OneVsRest.predict_topk` (dsgd_topics_topk) and
`Master.local_topic_ranking_report` (dsgd_eval_*topic_ranking, read by `topic_ranking_report`).  `Master.tune_topic_thresholds`
places each topic's F1-optimal margin threshold (SCut, dsgd_tune_topic_thresholds*, read by `threshold_report`), which
`OneVsRest.predict` and the topic reports then apply.
"""
from __future__ import annotations

from dataclasses import dataclass
from typing import List, Optional, Sequence

import numpy as np


@dataclass
class OneVsRest:
    """weights[t] is topic topics[t]'s weight vector (wdim values: dim, then the intercept on an intercept model),
    histories[t] the `fit` history of that topic, and thresholds[t] its margin threshold tau_t (None: every tau is 0, the
    binary rule)."""
    weights: np.ndarray      # float64[T', wdim]
    topics: tuple            # the topic names, in the order of weights
    histories: List[dict]
    thresholds: Optional[np.ndarray] = None   # float64[T'] (Master.tune_topic_thresholds)

    def predict(self, slave, idx: Sequence[int]) -> np.ndarray:
        """bool[n, T']: topic t predicted present for row idx[i], i.e. p = +1: its margin x . w_t below tau_t (0 without
        thresholds), from slave.margins per topic."""
        idx = np.asarray(idx, dtype=np.int32).reshape(-1)
        out = np.zeros((idx.size, len(self.topics)), dtype=bool)
        for t in range(len(self.topics)):
            tau = 0.0 if self.thresholds is None else float(self.thresholds[t])
            out[:, t] = slave.margins(idx, self.weights[t]) < tau
        return out

    def predict_topk(self, slave, idx: Sequence[int], k: int):
        """(ids int32[n, k], margins float64[n, k]): row idx[i]'s k highest-scored topics (score -x . w_t; ties to the lower
        index), as indices into `topics`, and their margins, in one device pass (Slave.topics_topk, dsgd_topics_topk).
        Topics with a NaN score are left out; their slots hold -1 and NaN."""
        return slave.topics_topk(idx, self.weights, k)


def parse_topics(raw: str):
    """The configuration value `topics`: empty (off) -> None, `all` -> "all", else the list of comma-separated names."""
    raw = raw.strip().strip('"').strip()
    if not raw:
        return None
    if raw.lower() == "all":
        return "all"
    names = [x.strip() for x in raw.split(",")]
    if any(not x for x in names) or len(set(names)) != len(names):
        raise ValueError(f"topics: expected all or distinct comma-separated topic names, got {raw!r}")
    return names


def topic_report(words, names) -> dict:
    """The report of a dsgd_eval_*topics call from its DSGD_TOPIC_WORDS(T) words (T = len(names)).
    Per topic: the counts, precision = TP / (TP + FP), recall = TP / P and f1 = 2 TP / (2 TP + FP + FN + pos_no_pred)
    (metrics_dict's formulas; nan where the denominator is 0).  Micro precision, recall and F1: the same formulas over the
    counts summed over the topics.  Macro F1: the mean of the topics' F1 where it is defined, with that topic count.
    Subset accuracy: rows right for every topic / rows.  Hamming loss: sum over topics of (FN + pos_no_pred + FP +
    neg_no_pred) / (rows T).  Top-1 accuracy: rows whose top-scored topic is theirs / rows with a topic."""
    names = tuple(names)
    T = len(names)
    w = np.asarray(words, dtype=np.int64).reshape(-1)
    if w.size != 8 * T + 8:
        raise ValueError(f"topic_report: {w.size} words for {T} topics, expected {8 * T + 8}")

    def ratio(a, b) -> float:
        return a / b if b else float("nan")

    per = {}
    tot = np.zeros(8, dtype=np.int64)
    f1s = []
    for t, name in enumerate(names):
        tp, fn, pos_none, fp, tn, neg_none, _, nan = (int(x) for x in w[8 * t:8 * t + 8])
        tot += w[8 * t:8 * t + 8]
        f1 = ratio(2 * tp, 2 * tp + fp + fn + pos_none)
        per[name] = {"tp": tp, "fn": fn, "pos_no_pred": pos_none, "fp": fp, "tn": tn, "neg_no_pred": neg_none,
                     "nan_scores": nan, "precision": ratio(tp, tp + fp), "recall": ratio(tp, tp + fn + pos_none), "f1": f1}
        if f1 == f1:
            f1s.append(f1)
    rows, exact, top1, no_topic, no_score = (int(x) for x in w[8 * T:8 * T + 5])
    tp, fn, pos_none, fp, _, neg_none = (int(x) for x in tot[:6])
    return {"topics": per, "rows": rows, "rows_without_topic": no_topic, "rows_without_score": no_score,
            "micro_precision": ratio(tp, tp + fp), "micro_recall": ratio(tp, tp + fn + pos_none),
            "micro_f1": ratio(2 * tp, 2 * tp + fp + fn + pos_none),
            "macro_f1": float(np.mean(f1s)) if f1s else float("nan"), "macro_f1_topics": len(f1s),
            "subset_accuracy": ratio(exact, rows), "hamming_loss": ratio(fn + pos_none + fp + neg_none, rows * T),
            "top1_accuracy": ratio(top1, rows - no_topic)}


TOPIC_RANK_MAX_K = 32   # DSGD_TOPIC_RANK_MAX_K
LIMB_BITS, RES_BITS = 40, 160


def parse_topic_rank_k(k: int, topics) -> int:
    """The configuration value `topic-rank-k`: 0 (off) or 1..32, and only with `topics` set (the parsed value)."""
    k = int(k)
    if not 0 <= k <= TOPIC_RANK_MAX_K:
        raise ValueError(f"topic-rank-k: expected 0 (off) or 1 .. {TOPIC_RANK_MAX_K}, got {k}")
    if k and topics is None:
        raise ValueError("topic-rank-k: ranks the topics of a one-vs-rest model; set `topics` too")
    return k


def limbs_value(block) -> float:
    """The value of one fixed-point sum of seven words (limbs 0..5, limb i worth 2^(40 i - 160), then the overflow count),
    converted exactly as the device's reader acc_value converts it: NaN with an overflow, else the carries propagated, then
    the limbs added as doubles from the top down.  The limbs may be sums of several calls' limbs."""
    q = [int(x) for x in np.asarray(block).reshape(-1)[:7]]
    if q[6]:
        return float("nan")
    mask = (1 << LIMB_BITS) - 1
    for i in range(5):
        q[i + 1] += q[i] >> LIMB_BITS
        q[i] &= mask
    s = float(q[5]) * 2.0 ** LIMB_BITS
    for i in range(4, -1, -1):
        s += float(q[i]) * 2.0 ** (LIMB_BITS * i - RES_BITS)
    return s


def topic_ranking_report(words, k: int) -> dict:
    """The report of a dsgd_eval_*topic_ranking call (or of several, their words added) from its DSGD_TOPIC_RANK_WORDS(k)
    words.  Over the N ranked rows (a topic and no NaN score): precision@j = hits in the top j / (j N), recall@j = C_j / N,
    label ranking average precision = A / N, coverage error = coverage / N and ranking loss = B / (N - rows with every
    topic); NaN where a denominator is 0.  A, B and C_j are the values of their limbs (limbs_value)."""
    k = int(k)
    w = np.asarray(words, dtype=np.int64).reshape(-1)
    if w.size != 8 + k + 7 * (2 + k):
        raise ValueError(f"topic_ranking_report: {w.size} words for k = {k}, expected {8 + k + 7 * (2 + k)}")

    def ratio(a, b) -> float:
        return a / b if b else float("nan")

    rows, N, nan_rows, no_topic, every, coverage = (int(x) for x in w[:6])
    sums = [limbs_value(w[8 + k + 7 * s:8 + k + 7 * s + 7]) for s in range(2 + k)]
    return {"k": k, "rows": rows, "ranked_rows": N, "rows_with_nan_score": nan_rows, "rows_without_topic": no_topic,
            "rows_with_every_topic": every,
            "precision_at": {j: ratio(int(w[8 + j - 1]), j * N) for j in range(1, k + 1)},
            "recall_at": {j: ratio(sums[2 + j - 1], N) for j in range(1, k + 1)},
            "lrap": ratio(sums[0], N), "coverage_error": ratio(coverage, N), "ranking_loss": ratio(sums[1], N - every)}


TOPIC_THRESHOLD_MODES = ("none", "scut")
THRESHOLD_STATUS = ("tuned", "no positive row", "below fbr", "no margin")   # word 6 of DSGD_TOPIC_TUNE_WORDS


def parse_topic_thresholds(mode: str, fbr: float, topics):
    """The configuration values `topic-thresholds` (none or scut, only with `topics` set) and `topic-threshold-fbr` (in
    [0, 1], non-zero only with scut): (mode, fbr)."""
    mode = str(mode).strip().strip('"').strip().lower()
    if mode not in TOPIC_THRESHOLD_MODES:
        raise ValueError(f"topic-thresholds: expected one of {', '.join(TOPIC_THRESHOLD_MODES)}, got {mode!r}")
    if mode != "none" and topics is None:
        raise ValueError("topic-thresholds: tunes the thresholds of a one-vs-rest model; set `topics` too")
    fbr = float(fbr)
    if not 0.0 <= fbr <= 1.0:
        raise ValueError(f"topic-threshold-fbr: expected a value in [0, 1], got {fbr}")
    if fbr != 0.0 and mode != "scut":
        raise ValueError("topic-threshold-fbr: the fallback of SCut tuning; set topic-thresholds = scut too")
    return mode, fbr


def threshold_report(words, thresholds, names) -> dict:
    """The report of a dsgd_tune_topic_thresholds* call from its thresholds and DSGD_TOPIC_TUNE_WORDS(T) words
    (T = len(names)).  Per topic: the threshold tau, the status and the chosen candidate j, the distinct non-NaN margins D,
    the positive rows P, the NaN margins, and tp and the rows predicted present at tau with the tuned F1 = 2 tp / (P +
    predicted) (nan where that is 0 / 0).  Then the rows and the topic count of each status."""
    names = tuple(names)
    T = len(names)
    w = np.asarray(words, dtype=np.int64).reshape(-1)
    thr = np.asarray(thresholds, dtype=np.float64).reshape(-1)
    if w.size != 8 * T or thr.size != T:
        raise ValueError(f"threshold_report: {w.size} words and {thr.size} thresholds for {T} topics, expected {8 * T} "
                         f"and {T}")
    per = {}
    for t, name in enumerate(names):
        rows, P, nan, D, tp, pred, status, j = (int(x) for x in w[8 * t:8 * t + 8])
        per[name] = {"threshold": float(thr[t]), "status": THRESHOLD_STATUS[status], "candidate": j, "distinct_margins": D,
                     "positives": P, "nan_margins": nan, "tp": tp, "predicted": pred,
                     "f1": 2 * tp / (P + pred) if P + pred else float("nan")}
    return {"topics": per, "rows": int(w[0]) if T else 0,
            "status_counts": {s: sum(v["status"] == s for v in per.values()) for s in THRESHOLD_STATUS}}
