"""Dev tool: the cost of an intercept (DSGD_FLAG_INTERCEPT, fit_intercept) on the full-size synthetic RCV1-shaped set
(700 000 rows, the first 560 000 of them train rows), and one quality figure.  Every timing case runs the same work on a
plain context and on an intercept context holding the same rows, alternated:

    SVM sync steps, batch 64, 256 and 1024 (2 188 steps per call): the persistent kernel against the intercept's
        per-step path (k_rows<svm, …, kIcpt> + k_update<…, kIcpt>)
    SparseLogistic sync steps, batch 64, 256 and 1024 (200 steps per call): per-step path against per-step path
    one evaluation pass over the 560 000 train rows (SVM: the fp32 streaming pass against the fp64 row kernel)
    dsgd_eval_metrics and dsgd_calibrate over the 140 000 test rows (SVM)

Each case runs `--warmup` untimed calls per arm, then `--reps` rounds of one timed call per arm (plain first), each on the
host clock between two device synchronisations; every step call starts from the same weights (the intercept 0).  The
card's name and power limit are read in the same run with a read-only nvidia-smi query; prints one JSON line.

--quality: MasterSync.fit on the same rows with the positives thinned to about 10 %, without and with fit_intercept (SVM,
one worker, batch 256, rate 0.5, lambda 1e-5, at most 10 epochs, the default stopping rule): test accuracy, balanced
accuracy, average precision and the learned intercept.

    python tools/time_intercept.py [--reps 7] [--warmup 1] [--quality] [--json out.json]
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


def card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True, check=True)
    return r.stdout.strip().splitlines()[0]


def new_ctx(data, model, intercept):
    c = NativeCtx(0, data.dim, LAM, model=model, intercept=intercept)
    c.load_csr(data.row_ptr, data.col, data.val, data.label)
    c.compute_dim_sparsity(N_TRAIN)
    return c


def draw(seed, steps, batch):
    rng = np.random.default_rng(seed)
    return np.concatenate([rng.choice(N_TRAIN, size=batch, replace=False) for _ in range(steps)]).astype(np.int32)


def clock(ctxs, fn):
    """Host milliseconds of fn() between two synchronisations of the device the contexts share."""
    for c in ctxs:
        c.synchronize()
    t0 = time.perf_counter()
    fn()
    for c in ctxs:
        c.synchronize()
    return (time.perf_counter() - t0) * 1e3


def alternate(ctxs, arms, reps, warmup):
    """Medians (ms) and samples of the two arms, alternated."""
    for _ in range(warmup):
        for f in arms:
            clock(ctxs, f)
    t = [[], []]
    for _ in range(reps):
        for k, f in enumerate(arms):
            t[k].append(clock(ctxs, f))
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
    for name, fi in (("no_intercept", False), ("fit_intercept", True)):
        model = SparseSVM(LAM, fit_intercept=fi)
        slave = Slave(0, 0, train, model, False, test_data=test)
        try:
            m = Master.create(0, train, test, model, False, 1, slave=slave, group=Group(), seed=0)
            t0 = time.perf_counter()
            state = m.fit(np.zeros(d.dim + fi), 10, 256, LR,
                          EarlyStopping.no_improvement(patience=5, min_delta=0.01, min_steps=None))
            secs = time.perf_counter() - t0
            cur = m.local_curve(state.grad, test_data=True, curve=False)
            rep = m.local_class_report(state.grad, test_data=True)
            out[name] = {"fit_seconds": secs, "epochs": len(m.history["losses"]), "test_accuracy": rep["accuracy"],
                         "balanced_accuracy": rep["balanced_accuracy"], "recall_pos": rep["recall_pos"],
                         "average_precision": cur["average_precision"],
                         "intercept": float(state.grad[d.dim]) if fi else None}
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
    pairs = {m: (new_ctx(data, m, False), new_ctx(data, m, True)) for m in ("svm", "logistic")}
    w0 = {False: np.zeros(data.dim), True: np.zeros(data.dim + 1)}

    def steps_call(c, b, steps):
        def f():
            c.set_weights(w0[c.intercept])
            c.sync_steps_staged(0, b, steps, LR)
        return f

    rows = []
    for model, steps in (("svm", STEPS), ("logistic", SHORT_STEPS)):
        plain, icpt = pairs[model]
        for b in (64, 256, 1024):
            ids = draw(b, steps, b)
            plain.stage_samples(ids)
            icpt.stage_samples(ids)
            off, on, t = alternate((plain, icpt), [steps_call(plain, b, steps), steps_call(icpt, b, steps)], a.reps, a.warmup)
            rows.append({"case": f"{model} sync steps, batch {b}", "steps": steps, "plain_us_per_step": off * 1e3 / steps,
                         "intercept_us_per_step": on * 1e3 / steps, "intercept_over_plain": on / off, "plain_ms": t[0],
                         "intercept_ms": t[1]})
    # the readers at trained weights: the resident ones after a run of 256-row steps, the intercept 0 on both contexts so
    # that both score the same rows the same way
    plain, icpt = pairs["svm"]
    plain.stage_samples(draw(256, STEPS, 256))
    plain.set_weights(w0[False])
    plain.sync_steps_staged(0, 256, STEPS, LR)
    w = plain.get_weights()
    icpt.set_weights(np.append(w, 0.0))
    readers = (("eval, 560 000 train rows", lambda c: c.eval_counts(0, N_TRAIN)),
               ("dsgd_eval_metrics, 140 000 test rows", lambda c: c.eval_metrics(N_TRAIN, N_ROWS)),
               ("dsgd_calibrate, 140 000 test rows", lambda c: c.calibrate(N_TRAIN, N_ROWS)))
    for label, fn in readers:
        off, on, t = alternate((plain, icpt), [lambda: fn(plain), lambda: fn(icpt)], a.reps, a.warmup)
        rows.append({"case": label, "plain_ms_median": off, "intercept_ms_median": on, "intercept_over_plain": on / off,
                     "plain_ms": t[0], "intercept_ms": t[1]})
    S = int(plain.info()["sm_count"])
    for p in pairs.values():
        for c in p:
            c.close()
    out = {"card": gpu, "sm_count": S, "reps": a.reps, "warmup": a.warmup, "rows": rows}
    if a.quality:
        out["quality"] = quality(data)
    print(json.dumps(out))
    if a.json:
        with open(a.json, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
