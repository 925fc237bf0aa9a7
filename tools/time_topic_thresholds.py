"""Dev tool: time the per-topic threshold calls on a full-size synthetic RCV1-shaped set (560 000 train and 140 000 test
rows) with about 100 planted topics (utils.synthetic_topics), alternated:

  * dsgd_tune_topic_thresholds over the 140 000 test rows and over the 560 000 train rows, each against the two ways of
    getting the same thresholds without it: T x (dsgd_select_topic + dsgd_eval_curve) with a host argmax over each curve,
    and T x dsgd_margins to the host with a numpy sort and scan;
  * dsgd_eval_thresholded_topics at the tuned thresholds against dsgd_eval_topics over the test rows.

Before timing, both alternatives' thresholds equal the device's bit for bit on the test rows.  With --profile the tuner's
three kernels (score pass, segmented sort, scan) are read apart with torch.profiler (CUDA activity), in a run of its own.

Every call is timed on the host clock between two device synchronisations (the calls end in one themselves); medians with
the 10th and 90th percentiles.  The card's name and power limit are read in the same run with a read-only nvidia-smi query.

    python tools/time_topic_thresholds.py [--topics 103] [--reps 5] [--warmup 1] [--profile] [--json out.json]
"""
import argparse
import dataclasses
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import numpy as np  # noqa: E402

from distributed_sgd_b200.native import NativeCtx  # noqa: E402
from distributed_sgd_b200.utils import synthetic_rcv1, synthetic_topics  # noqa: E402
from tools.time_metrics import N_TEST, N_TRAIN, alternated, card  # noqa: E402


def tau_of(c, j):
    """the threshold of candidate j over the distinct margins c (ascending): the midpoint rule, +inf for the last"""
    if j == len(c) - 1:
        return float("inf")
    mid = float(c[j]) / 2.0 + float(c[j + 1]) / 2.0
    return mid if c[j] < mid <= c[j + 1] else float(c[j + 1])


def best_candidate(tp, pp, P):
    """j of the highest 2 tp / (P + pp), exactly (integers), ties to the lowest j"""
    num, den = 2 * np.asarray(tp, dtype=object), P + np.asarray(pp, dtype=object)
    j = 0
    for k in range(1, len(num)):
        if num[k] * den[j] > num[j] * den[k]:
            j = k
    return j


def numpy_scut(m, y):
    """tau of one topic with a NaN-free margin array m and flags y, P > 0: sort, cumulative sums, argmax"""
    order = np.argsort(m, kind="stable")
    ms, ys = m[order] + 0.0, y[order]
    ends = np.flatnonzero(np.append(ms[1:] != ms[:-1], True))
    tp, pp = np.cumsum(ys)[ends], ends + 1
    P = int(y.sum())
    f = 2.0 * tp / (P + pp)                                            # exact argmax among the float ties below
    cand = np.flatnonzero(f == f.max())
    j = int(cand[0]) if cand.size == 1 else int(cand[best_candidate(tp[cand], pp[cand], P)])
    return tau_of(ms[ends], j)


def curve_scut(ctx, b, e, W, t, P):
    """tau of topic t from dsgd_eval_curve after dsgd_select_topic(t): the points are the candidates in order"""
    ctx.select_topic(t)
    _, _, thr, tp, fp = ctx.eval_curve(b, e, W[t])
    j = best_candidate(tp, tp + fp, P)
    return tau_of(-np.asarray(thr) + 0.0, j)                            # + 0.0: a zero margin as +0, as the device has it


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--topics", type=int, default=103)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--profile", action="store_true", help="read the tuner's kernels apart with torch.profiler instead")
    ap.add_argument("--json", default=None, help="also write the results to this file")
    a = ap.parse_args()
    gpu = card()
    T = a.topics
    data = synthetic_rcv1(n_rows=N_TRAIN + N_TEST, seed=0)
    data = dataclasses.replace(data, topics=synthetic_topics(data, T, seed=0))
    ctx = NativeCtx(0, data.dim, 1e-5)
    ctx.load_csr(data.row_ptr, data.col, data.val, data.label)
    ctx.compute_dim_sparsity(N_TRAIN)
    ctx.load_topics(data.topics.ptr, data.topics.ids, T)
    rng = np.random.default_rng(0)
    W = np.where(rng.random((T, data.dim)) < 0.6, rng.standard_normal((T, data.dim)) * 0.05, 0.0)
    has = data.topics.indicator()
    splits = {"test": (N_TRAIN, N_TRAIN + N_TEST), "train": (0, N_TRAIN)}

    if a.profile:
        import torch
        from torch.profiler import ProfilerActivity, profile
        torch.cuda.init()
        out = {}
        for split, (b, e) in splits.items():
            ctx.tune_topic_thresholds(b, e, W)
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                for _ in range(a.reps):
                    ctx.tune_topic_thresholds(b, e, W)
            for name, key in (("score pass (k_topic_keys)", "k_topic_keys"), ("segmented sort", "SegmentedRadixSort"),
                              ("scan (k_topic_tune)", "k_topic_tune")):
                ts = [ev.device_time for ev in prof.events() if key in ev.name]
                # the sort is several kernels per call: their sum per call
                per_call = float(np.sum(ts)) / a.reps / 1000.0 if ts else float("nan")
                out[f"{split}: {name}"] = per_call
        ctx.close()
        print(f"card: {gpu}")
        for k, v in out.items():
            print(f"{k:48s} {v:10.3f} ms per call (torch.profiler)")
        if a.json:
            with open(a.json, "w") as f:
                json.dump({"card": gpu, "topics": T, "reps": a.reps, "kernel_ms_per_call": out}, f, indent=1)
        return

    b, e = splits["test"]
    ids = np.arange(b, e, dtype=np.int32)
    thr, words = ctx.tune_topic_thresholds(b, e, W)
    tuned = np.flatnonzero(words[6::8] == 0)                           # the alternatives assume a positive row
    P = has[b:e].sum(axis=0)
    ref_np = np.array([numpy_scut(ctx.margins(ids, W[t]), has[b:e, t]) for t in tuned])
    ref_curve = np.array([curve_scut(ctx, b, e, W, t, int(P[t])) for t in tuned])
    ctx.select_topic(-1)
    assert np.array_equal(thr[tuned].view(np.int64), ref_np.view(np.int64)), "numpy SCut disagrees with the device"
    assert np.array_equal(thr[tuned].view(np.int64), ref_curve.view(np.int64)), "curve SCut disagrees with the device"
    print(f"{tuned.size} of {T} topics tuned on the test rows; both alternatives give the device's thresholds")
    tw = ctx.eval_thresholded_topics(b, e, W, thr)
    assert np.array_equal(tw[0:8 * T:8], words[4::8]), "thresholded counts disagree with the tuner's words"

    fns = {}
    for split, (sb, se) in splits.items():
        sids = np.arange(sb, se, dtype=np.int32)
        Ps = has[sb:se].sum(axis=0)
        fns[f"dsgd_tune_topic_thresholds, {split} rows"] = lambda sb=sb, se=se: ctx.tune_topic_thresholds(sb, se, W)
        fns[f"{T} x (select_topic + eval_curve) + argmax, {split}"] = (
            lambda sb=sb, se=se, Ps=Ps: [curve_scut(ctx, sb, se, W, t, int(Ps[t])) for t in range(T)])
        fns[f"{T} x dsgd_margins + numpy SCut, {split}"] = (
            lambda sids=sids, sb=sb, se=se: [numpy_scut(ctx.margins(sids, W[t]), has[sb:se, t]) for t in range(T)])
    fns["dsgd_eval_thresholded_topics, test rows"] = lambda: ctx.eval_thresholded_topics(b, e, W, thr)
    fns["dsgd_eval_topics, test rows"] = lambda: ctx.eval_topics(b, e, W)
    r = alternated(ctx, fns, a.warmup, a.reps)
    ctx.select_topic(-1)
    ctx.close()
    rows = [{"case": c, **v} for c, v in r.items()]
    print(f"card: {gpu}")
    print(f"{'case (test: 140 000 rows, train: 560 000 rows)':64s} {'median ms':>10s} {'p10':>10s} {'p90':>10s}")
    for x in rows:
        print(f"{x['case']:64s} {x['median_ms']:10.2f} {x['p10_ms']:10.2f} {x['p90_ms']:10.2f}")
    if a.json:
        with open(a.json, "w") as f:
            json.dump({"card": gpu, "topics": T, "reps": a.reps, "warmup": a.warmup, "rows": rows}, f, indent=1)


if __name__ == "__main__":
    main()
