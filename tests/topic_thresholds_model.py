"""A literal numpy restatement of per-topic threshold tuning (dsgd_tune_topic_thresholds*, include/dsgd.h) and of the
thresholded topic words (dsgd_eval*_thresholded_topics), the independent witness of the C checker
(oracle/dsgd_oracle_topic_thresh.c): from a [T, n] array of margins and a bool [n, T] topic indicator.  Every candidate is
counted by brute force and its F1 kept as a Fraction; no sort, no scan."""
from fractions import Fraction

import numpy as np

from topics_model import topic_words

TUNED, NO_POSITIVE, BELOW_FBR, NO_MARGIN = 0, 1, 2, 3


def midpoint(c: float, c1: float) -> float:
    """tau_j of candidate j < D - 1: fl(c_j / 2 + c_(j+1) / 2) when it lies in (c_j, c_(j+1)], else c_(j+1) (two adjacent
    doubles, whose midpoint rounds to c_j, or an infinite end)"""
    mid = float(c) / 2.0 + float(c1) / 2.0
    return mid if c < mid <= c1 else float(c1)


def counts_at(m, y, tau: float):
    """(tp, predicted): rows the thresholded rule predicts present at tau (m < tau), and those with the topic"""
    below = np.asarray(m) < tau
    return int(np.sum(below & y)), int(np.sum(below))


def tune_topic(m, y, fbr: float = 0.0):
    """(tau, words[8]) of one topic over margins m[n] and topic flags y[n]"""
    m = np.asarray(m, dtype=np.float64)
    y = np.asarray(y, dtype=bool)
    n, P = m.size, int(np.sum(y))
    nan = np.isnan(m)
    c = sorted({float(v) + 0.0 for v in m[~nan]})          # + 0.0: -0 becomes +0, one margin
    D = len(c)
    if D == 0:
        status, j, tau = NO_MARGIN, -1, 0.0
    elif P == 0:
        status, j, tau = NO_POSITIVE, -1, 0.0
    else:
        best, best_f1 = 0, None
        for k in range(D):
            sel = m <= c[k]
            f1 = Fraction(2 * int(np.sum(sel & y)), P + int(np.sum(sel)))
            if best_f1 is None or f1 > best_f1:
                best, best_f1 = k, f1
        tp, pp = int(np.sum((m <= c[best]) & y)), int(np.sum(m <= c[best]))
        status, j = (BELOW_FBR, 0) if (2 * tp) / (P + pp) < fbr else (TUNED, best)
        tau = float("inf") if j == D - 1 else midpoint(c[j], c[j + 1])
    tp, pp = counts_at(m, y, tau)
    return tau, np.array([n, P, int(np.sum(nan)), D, tp, pp, status, j], dtype=np.int64)


def tune(margins, has, fbr: float = 0.0):
    """(thresholds float64[T], words int64[8 T]) of dsgd_tune_topic_thresholds over margins[T, n] and has[n, T]"""
    m = np.asarray(margins, dtype=np.float64)
    has = np.asarray(has, dtype=bool)
    T = m.shape[0]
    thr = np.zeros(T, dtype=np.float64)
    words = np.zeros(8 * T, dtype=np.int64)
    for t in range(T):
        thr[t], words[8 * t:8 * t + 8] = tune_topic(m[t], has[:, t], fbr)
    return thr, words


def candidate_counts(m, y, j: int):
    """(tp_j, pp_j): rows with m <= c_j, and those with the topic"""
    m = np.asarray(m, dtype=np.float64)
    c = sorted({float(v) + 0.0 for v in m[~np.isnan(m)]})
    sel = m <= c[j]
    return int(np.sum(sel & np.asarray(y, dtype=bool))), int(np.sum(sel))


def thresholded_words(margins, has, thresholds) -> np.ndarray:
    """The DSGD_TOPIC_WORDS(T) words of dsgd_eval_thresholded_topics: topic_words with margins shifted so that the
    thresholded rule at tau_t becomes the sign rule, except the top-1 word, which ranks the raw margins"""
    m = np.asarray(margins, dtype=np.float64)
    has = np.asarray(has, dtype=bool)
    thr = np.asarray(thresholds, dtype=np.float64).reshape(-1, 1)
    # p = +1 for m < tau, -1 for m > tau, none at tau or NaN: the sign rule of a stand-in array -1 / +1 / 0 / NaN
    stand = np.where(m < thr, -1.0, np.where(m > thr, 1.0, np.where(np.isnan(m), np.nan, 0.0)))
    out = topic_words(stand, has)
    out[8 * m.shape[0] + 2] = topic_words(m, has)[8 * m.shape[0] + 2]
    return out
