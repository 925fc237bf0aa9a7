"""Dev tool: time the topic ranking calls on a full-size synthetic RCV1-shaped set (560 000 train and 140 000 test rows)
with about 100 planted topics (utils.synthetic_topics).  Over the 140 000 test rows, alternated:

  * dsgd_eval_topic_ranking at k (the whole call: the W copy, the pass, the words back) against dsgd_eval_topics;
  * dsgd_topics_topk at k against OneVsRest.predict's way of getting the same answer: T x dsgd_margins to the host, then a
    numpy ordering of the margins with the tie rule.

The two kernels' times are read apart with torch.profiler (CUDA activity) in a run of their own.  Before timing, the
device's top k equals the numpy ordering and hits@1 equals dsgd_eval_topics' top-1 word.

Every call is timed on the host clock between two device synchronisations (the calls end in one themselves); medians with
the 10th and 90th percentiles.  The card's name and power limit are read in the same run with a read-only nvidia-smi query.

    python tools/time_topic_ranking.py [--topics 103] [--k 5] [--reps 7] [--warmup 2] [--json out.json]
"""
import argparse
import dataclasses
import json
import os
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import numpy as np  # noqa: E402

from distributed_sgd_b200.native import NativeCtx  # noqa: E402
from distributed_sgd_b200.utils import synthetic_rcv1, synthetic_topics  # noqa: E402
from tools.time_metrics import N_TEST, N_TRAIN, alternated, card  # noqa: E402


def numpy_topk(margins, k):
    """ids [n, k] of the k lowest margins of each row (the highest scores), ties to the lower t; NaN margins last"""
    key = np.where(np.isnan(margins), np.inf, margins).T                 # [n, T]
    order = np.argsort(key, axis=1, kind="stable")[:, :k]              # stable: equal margins keep the lower t first
    return order.astype(np.int32)


def kernel_ms(fn, name, reps):
    """median time of the kernels whose name contains `name` (torch.profiler, CUDA activity)"""
    import torch
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.init()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(reps):
            fn()
    ts = [ev.device_time for ev in prof.events() if name in ev.name]
    return float(np.median(ts)) / 1000.0 if ts else float("nan")


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--topics", type=int, default=103)
    ap.add_argument("--k", type=int, default=5)
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--json", default=None, help="also write the results to this file")
    a = ap.parse_args()
    gpu = card()
    T, k = a.topics, a.k
    data = synthetic_rcv1(n_rows=N_TRAIN + N_TEST, seed=0)
    data = dataclasses.replace(data, topics=synthetic_topics(data, T, seed=0))
    ctx = NativeCtx(0, data.dim, 1e-5)
    ctx.load_csr(data.row_ptr, data.col, data.val, data.label)
    ctx.compute_dim_sparsity(N_TRAIN)
    ctx.load_topics(data.topics.ptr, data.topics.ids, T)
    rng = np.random.default_rng(0)
    W = np.where(rng.random((T, data.dim)) < 0.6, rng.standard_normal((T, data.dim)) * 0.05, 0.0)
    b, e = N_TRAIN, N_TRAIN + N_TEST
    ids = np.arange(b, e, dtype=np.int32)

    margins = np.stack([ctx.margins(ids, W[t]) for t in range(T)])
    top_ids, _ = ctx.topics_topk(ids, W, k)
    assert np.array_equal(top_ids, numpy_topk(margins, k)), "the timed top k disagrees with numpy"
    words, sums = ctx.eval_topic_ranking(b, e, W, k)
    tw = ctx.eval_topics(b, e, W)
    assert words[2] == 0 and words[8] == tw[8 * T + 2], "hits@1 disagrees with the top-1 word"

    def margins_numpy():
        numpy_topk(np.stack([ctx.margins(ids, W[t]) for t in range(T)]), k)

    r = alternated(ctx, {
        f"dsgd_eval_topic_ranking, T = {T}, k = {k}": lambda: ctx.eval_topic_ranking(b, e, W, k),
        f"dsgd_eval_topics, T = {T}": lambda: ctx.eval_topics(b, e, W),
        f"dsgd_topics_topk, k = {k}": lambda: ctx.topics_topk(ids, W, k),
        f"{T} x dsgd_margins to the host + numpy top {k}": margins_numpy}, a.warmup, a.reps)
    rows = [{"case": c, **v} for c, v in r.items()]
    kern = {"k_topic_rank (ranking)": kernel_ms(lambda: ctx.eval_topic_ranking(b, e, W, k), "k_topic_rank", a.reps),
            "k_topic_eval": kernel_ms(lambda: ctx.eval_topics(b, e, W), "k_topic_eval", a.reps),
            "k_topic_rank (top k)": kernel_ms(lambda: ctx.topics_topk(ids, W, k), "k_topic_rank", a.reps)}
    ctx.close()

    from distributed_sgd_b200.ml.one_vs_rest import topic_ranking_report
    rep = topic_ranking_report(words, k)
    print(f"card: {gpu}")
    print(f"ranked test rows {rep['ranked_rows']}, precision@{k} {rep['precision_at'][k]:.4f}, LRAP {rep['lrap']:.4f} "
          "(random weights: a check of the words, not a model)")
    print(f"{'case (over the 140 000 test rows)':64s} {'median ms':>10s} {'p10':>8s} {'p90':>8s}")
    for x in rows:
        print(f"{x['case']:64s} {x['median_ms']:10.3f} {x['p10_ms']:8.3f} {x['p90_ms']:8.3f}")
    for name, ms in kern.items():
        print(f"{name} kernel (torch.profiler), median: {ms:.3f} ms")
    if a.json:
        with open(a.json, "w") as f:
            json.dump({"card": gpu, "topics": T, "k": k, "reps": a.reps, "warmup": a.warmup, "rows": rows,
                       "kernel_ms": kern}, f, indent=1)


if __name__ == "__main__":
    main()
