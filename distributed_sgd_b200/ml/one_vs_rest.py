"""One-vs-rest (OvR) models of a multi-label set: one binary model per topic, "has topic t" against the rest.

`MasterSync.fit_one_vs_rest` trains them one topic after another on one device context (dsgd_select_topic switches the
labels on the device), and `Master.local_topic_report` judges them all in one pass (dsgd_eval_*topics).
"""
from __future__ import annotations

from dataclasses import dataclass
from typing import List, Sequence

import numpy as np


@dataclass
class OneVsRest:
    """weights[t] is topic topics[t]'s weight vector (wdim values: dim, then the intercept on an intercept model), and
    histories[t] the `fit` history of that topic."""
    weights: np.ndarray      # float64[T', wdim]
    topics: tuple            # the topic names, in the order of weights
    histories: List[dict]

    def predict(self, slave, idx: Sequence[int]) -> np.ndarray:
        """bool[n, T']: topic t predicted present for row idx[i], i.e. p = +1 (x . w_t < 0), from slave.margins per topic."""
        idx = np.asarray(idx, dtype=np.int32).reshape(-1)
        out = np.zeros((idx.size, len(self.topics)), dtype=bool)
        for t in range(len(self.topics)):
            out[:, t] = slave.margins(idx, self.weights[t]) < 0.0
        return out


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
