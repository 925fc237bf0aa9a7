"""A literal numpy restatement of the words of dsgd_eval_*topics (include/dsgd.h), the independent witness of the C
checker (oracle/dsgd_oracle_topics.c): from a [T, n] array of margins and a bool [n, T] topic indicator, with no sort and
no search."""
import numpy as np


def topic_words(margins: np.ndarray, has: np.ndarray) -> np.ndarray:
    m = np.asarray(margins, dtype=np.float64)
    has = np.asarray(has, dtype=bool)
    T, n = m.shape
    out = np.zeros(8 * T + 8, dtype=np.int64)
    pred = np.where(m < 0.0, 1, np.where(m > 0.0, -1, 0))          # -signum; none for 0 and NaN
    nan = np.isnan(m)
    for t in range(T):
        y = has[:, t]
        p = pred[t]
        out[8 * t:8 * t + 8] = [np.sum(y & (p == 1)), np.sum(y & (p == -1)), np.sum(y & (p == 0)),
                                np.sum(~y & (p == 1)), np.sum(~y & (p == -1)), np.sum(~y & (p == 0)), 0, np.sum(nan[t])]
    rw = out[8 * T:]
    for i in range(n):
        rw[0] += 1
        rw[1] += all(pred[t, i] == (1 if has[i, t] else -1) for t in range(T))
        best = None
        for t in range(T):                                          # the lowest margin; ties to the lowest t
            if not nan[t, i] and (best is None or m[t, i] < m[best, i]):
                best = t
        rw[2] += bool(has[i].any() and best is not None and has[i, best])
        rw[3] += not has[i].any()
        rw[4] += best is None
    return out
