"""A literal numpy restatement of the words and sums of dsgd_eval_*topic_ranking (include/dsgd.h), the independent witness
of the C checker (oracle/dsgd_oracle_topic_rank.c): from a [T, n] array of margins and a bool [n, T] topic indicator.  The
fixed-point sums go through tests/loss_sum_model.py: their limbs are the base-2^40 digits of the exact integer sum of the
terms' units, and their values that model's device reader."""
import numpy as np

from loss_sum_model import LIMB_BITS, device_model, r_units


def ranks(s: np.ndarray) -> np.ndarray:
    """rank_l = #{u : s_u >= s_l} of one row's scores s (the "max" rank: ties count against the row)"""
    s = np.asarray(s, dtype=np.float64)
    return (s[None, :] >= s[:, None]).sum(axis=1).astype(np.int64)    # row l: the u with s_u >= s_l


def order(m: np.ndarray) -> list:
    """the topics by score -m descending, ties to the lower t (+0 and -0 are one score), over the non-NaN margins"""
    return sorted((t for t in range(len(m)) if not np.isnan(m[t])), key=lambda t: (float(m[t]), t))


def limbs(values) -> list:
    """the seven words of a fixed-point sum of `values`: limbs 0..4 in [0, 2^40), limb 5, the overflow count"""
    units = [r_units(v) for v in values]
    if any(u is None for u in units):
        raise ValueError("every ranking term lies in [0, 1]")
    total = sum(units)
    mask = (1 << LIMB_BITS) - 1
    return [(total >> (LIMB_BITS * i)) & mask for i in range(5)] + [total >> (LIMB_BITS * 5), 0]


def topic_ranking(margins: np.ndarray, has: np.ndarray, k: int):
    """(words int64[8 + k + 7 (2 + k)], sums float64[2 + k])"""
    m = np.asarray(margins, dtype=np.float64)
    has = np.asarray(has, dtype=bool)
    T, n = m.shape
    w = np.zeros(8 + k, dtype=np.int64)
    terms = [[] for _ in range(2 + k)]                              # A, B, C_1 .. C_k
    for i in range(n):
        s = -m[:, i]
        Y = [t for t in range(T) if has[i, t]]
        nY = len(Y)
        w[0] += 1
        if np.isnan(s).any():
            w[2] += 1
            continue
        if nY == 0:
            w[3] += 1
            continue
        w[1] += 1
        w[4] += nY == T
        rank = ranks(s)
        L = {l: sum(1 for u in Y if s[u] >= s[l]) for l in Y}
        w[5] += max(int(rank[l]) for l in Y)
        p = sum(int(rank[l]) - L[l] for l in Y)
        w[6] += p
        for l in Y:
            terms[0].append(L[l] / (int(rank[l]) * nY))
        if nY < T:
            terms[1].append(p / (nY * (T - nY)))
        top = order(m[:, i])
        for j in range(1, k + 1):
            hits = sum(1 for t in top[:j] if has[i, t])
            w[8 + j - 1] += hits
            terms[2 + j - 1].append(hits / nY)
    words = np.concatenate([w] + [np.array(limbs(v), dtype=np.int64) for v in terms])
    sums = np.array([device_model(v) for v in terms], dtype=np.float64)
    return words, sums


def topk(margins: np.ndarray, k: int):
    """(ids int32[n, k], margins float64[n, k]) of dsgd_topics_topk from [T, n] margins: -1 and NaN past the non-NaN ones"""
    m = np.asarray(margins, dtype=np.float64)
    T, n = m.shape
    ids = np.full((n, k), -1, dtype=np.int32)
    top = np.full((n, k), np.nan)
    for i in range(n):
        o = order(m[:, i])[:k]
        ids[i, :len(o)] = o
        top[i, :len(o)] = m[o, i]
    return ids, top
