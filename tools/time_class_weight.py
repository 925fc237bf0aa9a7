"""Dev tool: the cost of class weights (dsgd_set_class_weights) on the full-size synthetic RCV1-shaped set (700 000 rows, the
first 560 000 of them train rows), and one quality figure.  Every timing case runs the same work with the weights off,
(1, 1), and on, (2, 0.5), alternated on one context:

    persistent kernel and its weighted form, batch 64, 256 and 1024 (2 188 steps per call)
    fallback (k_rows + k_update against
        k_rows<svm, kClassWeighted, …> + k_class_fold + k_update<kCw>), batch 32 G + 1 (200 steps per call)
    SparseLogistic, batch 256 (k_rows<logistic, kUnweighted, …> against
        k_rows<logistic, kClassWeighted, …>, 200 steps per call)
    dsgd_eval_class against dsgd_eval_counts over the 140 000 test rows and the 560 000 train rows
    dsgd_gradient over 262 144 ids, unweighted and weighted

Each case runs `--warmup` untimed calls per arm, then `--reps` rounds of one timed call per arm (off first, then on), each on
the host clock between two device synchronisations; every step call starts from the same weights.  The card's name and
power limit are read in the same run with a read-only nvidia-smi query; prints one JSON line.

--quality: MasterSync.fit on the same rows with the positives thinned to about 10 %, class_weight None against "balanced"
(one worker, batch 256, rate 0.5, lambda 1e-5, at most 10 epochs, the default stopping rule): test accuracy, recall of the
positive class, F1 and average precision.

    python tools/time_class_weight.py [--reps 7] [--warmup 1] [--quality] [--json out.json]
"""
import argparse
import json
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import numpy as np  # noqa: E402

from distributed_sgd_b200.native import NativeCtx  # noqa: E402
from distributed_sgd_b200.utils import synthetic_rcv1  # noqa: E402

N_ROWS, N_TRAIN = 700_000, 560_000
STEPS, SHORT_STEPS = 2188, 200
LAM, LR = 1e-5, 0.5
ON = (2.0, 0.5)


def card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True, check=True)
    return r.stdout.strip().splitlines()[0]


def new_ctx(data, logistic=False):
    c = NativeCtx(0, data.dim, LAM, logistic=logistic)
    c.load_csr(data.row_ptr, data.col, data.val, data.label)
    c.compute_dim_sparsity(N_TRAIN)
    return c


def draw(seed, steps, batch):
    rng = np.random.default_rng(seed)
    return np.concatenate([rng.choice(N_TRAIN, size=batch, replace=False) for _ in range(steps)]).astype(np.int32)


def clock(c, fn):
    """Host milliseconds of fn() between two device synchronisations."""
    c.synchronize()
    t0 = time.perf_counter()
    fn()
    c.synchronize()
    return (time.perf_counter() - t0) * 1e3


def alternate(c, arms, reps, warmup):
    """Medians (ms) and samples of the two arms, alternated."""
    for _ in range(warmup):
        for f in arms:
            clock(c, f)
    t = [[], []]
    for _ in range(reps):
        for k, f in enumerate(arms):
            t[k].append(clock(c, f))
    return float(np.median(t[0])), float(np.median(t[1])), t


def thinned(data, share, seed):
    """`data` with positives dropped at random until about `share` of the rows are positive."""
    from distributed_sgd_b200.utils.dataset import Data
    rng = np.random.default_rng(seed)
    pos, neg = np.flatnonzero(data.label > 0), np.flatnonzero(data.label < 0)
    keep = np.sort(np.concatenate([neg, rng.choice(pos, size=int(len(neg) * share / (1.0 - share)), replace=False)]))
    lens = np.diff(data.row_ptr)[keep]
    rp = np.concatenate([[0], np.cumsum(lens)]).astype(np.int64)
    take = np.repeat(data.row_ptr[keep] - rp[:-1], lens) + np.arange(rp[-1])
    return Data(rp, data.col[take], data.val[take], data.label[keep], data.dim)


def quality(data):
    from distributed_sgd_b200 import EarlyStopping, Master, Slave, SparseSVM
    from distributed_sgd_b200.core import Group
    d = thinned(data, 0.10, 1)
    train, test = d.split_at(int(d.n_rows * 0.8))
    out = {"rows": {"train": train.n_rows, "test": test.n_rows},
           "train_positive_share": float(np.mean(train.label > 0))}
    for name, cw in (("none", None), ("balanced", "balanced")):
        model = SparseSVM(LAM, class_weight=cw)
        slave = Slave(0, 0, train, model, False, test_data=test)
        try:
            m = Master.create(0, train, test, model, False, 1, slave=slave, group=Group(), seed=0)
            t0 = time.perf_counter()
            state = m.fit(np.zeros(d.dim), 10, 256, LR, EarlyStopping.no_improvement(patience=5, min_delta=0.01, min_steps=None))
            secs = time.perf_counter() - t0
            cur = m.local_curve(state.grad, test_data=True, curve=False)
            rep = m.local_class_report(state.grad, test_data=True)
            out[name] = {"class_weight": list(slave.class_weight), "fit_seconds": secs, "epochs": len(m.history["losses"]),
                         "test_accuracy": rep["accuracy"], "recall_pos": rep["recall_pos"], "recall_neg": rep["recall_neg"],
                         "balanced_accuracy": rep["balanced_accuracy"], "precision": cur["precision"], "f1": cur["f1"],
                         "average_precision": cur["average_precision"]}
        finally:
            slave.stop()
    return out


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--quality", action="store_true")
    ap.add_argument("--json", default=None, help="also write the results to this file")
    a = ap.parse_args()
    gpu = card()
    data = synthetic_rcv1(n_rows=N_ROWS, seed=0)
    w0 = np.zeros(data.dim)
    svm = new_ctx(data)
    S = int(svm.info()["sm_count"])
    logistic = new_ctx(data, logistic=True)
    cases = [(f"persistent, batch {b}", svm, b, STEPS) for b in (64, 256, 1024)]
    cases.append((f"fallback, batch {32 * S + 1} (32 G + 1)", svm, 32 * S + 1, SHORT_STEPS))
    cases.append(("logistic, batch 256", logistic, 256, SHORT_STEPS))

    def steps_call(c, b, steps, cw):
        def f():
            c.set_class_weights(*cw)
            c.set_weights(w0)
            c.sync_steps_staged(0, b, steps, LR)
        return f

    rows = []
    for label, c, b, steps in cases:
        c.stage_samples(draw(b, steps, b))
        off, on, t = alternate(c, [steps_call(c, b, steps, (1.0, 1.0)), steps_call(c, b, steps, ON)], a.reps, a.warmup)
        c.set_class_weights(1.0, 1.0)
        rows.append({"case": label, "steps": steps, "off_us_per_step": off * 1e3 / steps, "on_us_per_step": on * 1e3 / steps,
                     "on_over_off": on / off, "off_ms": t[0], "on_ms": t[1]})
    # evaluation and gradient requests at trained weights (the resident ones after a persistent run)
    svm.stage_samples(draw(256, STEPS, 256))
    svm.set_weights(w0)
    svm.sync_steps_staged(0, 256, STEPS, LR)
    svm.synchronize()
    for label, (lo, hi) in (("eval, 140 000 test rows", (N_TRAIN, N_ROWS)), ("eval, 560 000 train rows", (0, N_TRAIN))):
        off, on, t = alternate(svm, [lambda: svm.eval_counts(lo, hi), lambda: svm.eval_class(lo, hi)], a.reps, a.warmup)
        rows.append({"case": label + ": dsgd_eval_counts (off) / dsgd_eval_class (on)", "off_ms_median": off,
                     "on_ms_median": on, "on_over_off": on / off, "off_ms": t[0], "on_ms": t[1]})
    ids = draw(7, 1, 262144)

    def grad(cw):
        def f():
            svm.set_class_weights(*cw)
            svm.gradient(ids)
        return f
    off, on, t = alternate(svm, [grad((1.0, 1.0)), grad(ON)], a.reps, a.warmup)
    svm.set_class_weights(1.0, 1.0)
    rows.append({"case": "dsgd_gradient, 262 144 ids", "off_ms_median": off, "on_ms_median": on, "on_over_off": on / off,
                 "off_ms": t[0], "on_ms": t[1]})
    for c in (svm, logistic):
        c.close()
    out = {"card": gpu, "sm_count": S, "weights_on": list(ON), "reps": a.reps, "warmup": a.warmup, "rows": rows}
    if a.quality:
        out["quality"] = quality(data)
    print(json.dumps(out))
    if a.json:
        with open(a.json, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
