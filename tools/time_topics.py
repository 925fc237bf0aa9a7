"""Dev tool: time the one-vs-rest topic calls on a full-size synthetic RCV1-shaped set (560 000 train and 140 000 test rows)
with about 100 planted topics (utils.synthetic_topics).  Over the 140 000 test rows, alternated:

  * dsgd_eval_topics with the T weight vectors (the whole call: the W copy, the pass and the words back);
  * the W copy alone (T * dim doubles, pageable host memory to the device, as the call makes it);
  * T x dsgd_eval_metrics, the per-topic words without the row words (the labels already those of each topic would be one
    more dsgd_select_topic per topic);
  * T x (dsgd_select_topic + dsgd_eval_metrics), the same words for the right labels;
  * T x dsgd_margins to the host plus numpy forming every word (the alternative without the new pass);
  * dsgd_select_topic.

The k_topic_eval kernel time is read apart with torch.profiler (CUDA activity) in a run of its own.  Then one
fit_one_vs_rest over the first topics times one topic's fit, and its host share: the wall time outside the library calls.

Every call is timed on the host clock between two device synchronisations (the calls end in one themselves); medians with
the 10th and 90th percentiles.  The card's name and power limit are read in the same run with a read-only nvidia-smi query.

    python tools/time_topics.py [--topics 103] [--reps 7] [--warmup 2] [--json out.json]
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


def numpy_words(margins, has):
    """The words of dsgd_eval_topics from [T, n] margins and a bool [n, T] indicator, vectorised"""
    T, n = margins.shape
    out = np.zeros(8 * T + 8, dtype=np.int64)
    p = np.where(margins < 0.0, 1, np.where(margins > 0.0, -1, 0))
    y = has.T
    for k, (cls, pred) in enumerate([(y, 1), (y, -1), (y, 0), (~y, 1), (~y, -1), (~y, 0)]):
        out[k:8 * T:8] = np.sum(cls & (p == pred), axis=1)
    nan = np.isnan(margins)
    out[7:8 * T:8] = nan.sum(axis=1)
    out[8 * T] = n
    out[8 * T + 1] = np.sum(np.all(p == np.where(y, 1, -1), axis=0))
    best = np.argmin(np.where(nan, np.inf, margins), axis=0)     # the first lowest: ties to the lowest t
    scored = ~nan.all(axis=0)
    some = has.any(axis=1)
    out[8 * T + 2] = np.sum(some & scored & has[np.arange(n), best])
    out[8 * T + 3] = np.sum(~some)
    out[8 * T + 4] = np.sum(~scored)
    return out


def kernel_ms(ctx, b, e, W, reps):
    """median k_topic_eval kernel time (torch.profiler, CUDA activity)"""
    import torch
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.init()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(reps):
            ctx.eval_topics(b, e, W)
    ts = [ev.device_time for ev in prof.events() if "k_topic_eval" in ev.name]
    return float(np.median(ts)) / 1000.0 if ts else float("nan")


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--topics", type=int, default=103)
    ap.add_argument("--fit-topics", type=int, default=3, help="topics of the timed fit_one_vs_rest")
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--json", default=None, help="also write the results to this file")
    a = ap.parse_args()
    gpu = card()
    T = a.topics
    t0 = time.perf_counter()
    data = synthetic_rcv1(n_rows=N_TRAIN + N_TEST, seed=0)
    data = dataclasses.replace(data, topics=synthetic_topics(data, T, seed=0))
    plant_s = time.perf_counter() - t0
    ctx = NativeCtx(0, data.dim, 1e-5)
    ctx.load_csr(data.row_ptr, data.col, data.val, data.label)
    ctx.compute_dim_sparsity(N_TRAIN)
    ctx.load_topics(data.topics.ptr, data.topics.ids, T)
    rng = np.random.default_rng(0)
    W = np.where(rng.random((T, data.dim)) < 0.6, rng.standard_normal((T, data.dim)) * 0.05, 0.0)
    b, e = N_TRAIN, N_TRAIN + N_TEST
    ids = np.arange(b, e, dtype=np.int32)
    has = data.topics.indicator()[b:e]
    words = ctx.eval_topics(b, e, W)
    margins = np.stack([ctx.margins(ids, W[t]) for t in range(T)])
    assert np.array_equal(words, numpy_words(margins, has)), "the timed pass disagrees with numpy"
    import torch
    dev = torch.device("cuda", 0)
    buf = torch.empty(W.shape, dtype=torch.float64, device=dev)
    Wt = torch.from_numpy(W)

    def w_copy():
        buf.copy_(Wt)
        torch.cuda.synchronize()

    def per_topic_metrics(select):
        for t in range(T):
            if select:
                ctx.select_topic(t)
            ctx.eval_metrics(b, e, W[t])
        if select:
            ctx.select_topic(-1)

    def margins_numpy():
        numpy_words(np.stack([ctx.margins(ids, W[t]) for t in range(T)]), has)

    r = alternated(ctx, {
        f"dsgd_eval_topics, T = {T}": lambda: ctx.eval_topics(b, e, W),
        f"W copy alone ({W.nbytes / 2**20:.1f} MiB, pageable)": w_copy,
        f"{T} x dsgd_eval_metrics": lambda: per_topic_metrics(False),
        f"{T} x (dsgd_select_topic + dsgd_eval_metrics)": lambda: per_topic_metrics(True),
        f"{T} x dsgd_margins to the host + numpy": margins_numpy,
        "dsgd_select_topic": lambda: ctx.select_topic(1)}, a.warmup, a.reps)
    ctx.select_topic(-1)
    k_ms = kernel_ms(ctx, b, e, W, a.reps)
    rows = [{"case": k, **v} for k, v in r.items()]

    # one topic's fit inside fit_one_vs_rest: the wall time, and the time outside the library calls (the host's share)
    from distributed_sgd_b200 import MasterSync, Slave, SparseSVM
    ctx.close()
    train, test = data.split_at(N_TRAIN)
    model = SparseSVM(1e-5)
    slave = Slave(0, 0, train, model, False, test_data=test)
    in_lib = [0.0]

    class Timed:   # the Slave's context with every call's wall time summed
        def __init__(self, c):
            self._c = c

        def __getattr__(self, name):
            f = getattr(self._c, name)
            if not callable(f):
                return f

            def g(*args, **kw):
                s = time.perf_counter()
                try:
                    return f(*args, **kw)
                finally:
                    in_lib[0] += time.perf_counter() - s
            return g

    slave.ctx = Timed(slave.ctx)
    m = MasterSync(0, train, test, model, 1, slave=slave, seed=0)
    stop = lambda tl: False   # noqa: E731
    topics = list(data.topics.names[1:1 + a.fit_topics])
    s = time.perf_counter()
    m.fit_one_vs_rest(np.zeros(data.dim), 1, 100, 0.5, stop, topics=topics)
    wall = time.perf_counter() - s
    fit = {"topics": topics, "epochs": 1, "batch": 100, "steps_per_topic": -(-N_TRAIN // 100),
           "ms_per_topic": 1000.0 * wall / len(topics), "host_share": 1.0 - in_lib[0] / wall}
    slave.stop()

    print(f"card: {gpu}")
    print(f"planting {T} topics on {N_TRAIN + N_TEST} rows: {plant_s:.1f} s; {int(words[8 * T + 3])} test rows without a topic")
    print(f"{'case (over the 140 000 test rows)':64s} {'median ms':>10s} {'p10':>8s} {'p90':>8s}")
    for x in rows:
        print(f"{x['case']:64s} {x['median_ms']:10.3f} {x['p10_ms']:8.3f} {x['p90_ms']:8.3f}")
    print(f"k_topic_eval kernel (torch.profiler), median: {k_ms:.3f} ms")
    print(f"fit_one_vs_rest: {fit['ms_per_topic']:.1f} ms per topic ({fit['steps_per_topic']} steps of {fit['batch']}, "
          f"1 epoch), host share {100 * fit['host_share']:.1f} %")
    if a.json:
        with open(a.json, "w") as f:
            json.dump({"card": gpu, "topics": T, "reps": a.reps, "warmup": a.warmup, "rows": rows, "kernel_ms": k_ms,
                       "fit": fit}, f, indent=1)


if __name__ == "__main__":
    main()
