"""Dev tool: the cost of per-row sample weights (dsgd_set_sample_weights) on the full-size synthetic RCV1-shaped set (700 000
rows, the first 560 000 of them train rows).  Every case runs the same work in three arms alternated on one context: no
weights, all ones, and random weights (uniform in [0, 2)):

    one-GPU step, batch 64, 256 and 1024 (2 188 steps per call): the persistent kernel without weights, the per-step path
        (k_rows<…, kSampleWeighted, …> + k_sw_fold + k_update<kCw>) with them
    per-step path, batch 32 G + 1 (200 steps per call): k_rows + k_update against the sample-weighted pass
    SparseLogistic, batch 256 (200 steps per call)
    dsgd_gradient over 262 144 ids: the streaming pass without weights, k_rows<…, kSampleWeighted, …> with them
    dsgd_eval_weighted over the 140 000 test rows and the 560 000 train rows (dsgd_eval_counts in the no-weights arm)

Each case runs `--warmup` untimed rounds, then `--reps` rounds of one timed call per arm, each on the host clock between two
device synchronisations (loading an arm's weights happens before the clock starts); every step call starts from the same
weights.  Reports medians, minima and maxima.  The card's name
and power limit are read in the same run with a read-only nvidia-smi query.  Prints one JSON line; writes a file only with
--out.

    python tools/time_sample_weight.py [--reps 7] [--warmup 1] [--out result.json]
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
ARMS = ("none", "ones", "random")


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
    """{arm: {median, min, max, ms}} of the arms, alternated round by round.  An arm is (setup, fn): setup (loading the arm's
    weights) runs before the clock starts."""
    for _ in range(warmup):
        for setup, f in arms:
            setup()
            clock(c, f)
    t = [[] for _ in arms]
    for _ in range(reps):
        for k, (setup, f) in enumerate(arms):
            setup()
            t[k].append(clock(c, f))
    return {name: {"median_ms": float(np.median(x)), "min_ms": float(np.min(x)), "max_ms": float(np.max(x)), "ms": x}
            for name, x in zip(ARMS, t)}


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--out", default=None, help="also write the result to this file")
    a = ap.parse_args()
    gpu = card()
    data = synthetic_rcv1(n_rows=N_ROWS, seed=0)
    weights = {"none": None, "ones": np.ones(N_ROWS), "random": np.random.default_rng(5).random(N_ROWS) * 2.0}
    w0 = np.zeros(data.dim)
    svm = new_ctx(data)
    S = int(svm.info()["sm_count"])
    logistic = new_ctx(data, logistic=True)
    cases = [(f"one-GPU step, batch {b}", svm, b, STEPS) for b in (64, 256, 1024)]
    cases.append((f"per-step path, batch {32 * S + 1} (32 G + 1)", svm, 32 * S + 1, SHORT_STEPS))
    cases.append(("logistic, batch 256", logistic, 256, SHORT_STEPS))

    def with_weights(c, arm, fn):
        return (lambda: c.set_sample_weights(weights[arm])), fn

    def steps_call(c, b, steps):
        def f():
            c.set_weights(w0)
            c.sync_steps_staged(0, b, steps, LR)
        return f

    rows = []
    for label, c, b, steps in cases:
        c.stage_samples(draw(b, steps, b))
        r = alternate(c, [with_weights(c, arm, steps_call(c, b, steps)) for arm in ARMS], a.reps, a.warmup)
        rows.append({"case": label, "steps": steps,
                     **{f"{k}_us_per_step": v["median_ms"] * 1e3 / steps for k, v in r.items()}, "arms": r})
    svm.set_sample_weights(None)
    # requests at trained weights (the resident ones after a run without weights)
    svm.stage_samples(draw(256, STEPS, 256))
    svm.set_weights(w0)
    svm.sync_steps_staged(0, 256, STEPS, LR)
    svm.synchronize()
    ids = draw(7, 1, 262144)
    r = alternate(svm, [with_weights(svm, arm, lambda: svm.gradient(ids)) for arm in ARMS], a.reps, a.warmup)
    rows.append({"case": "dsgd_gradient, 262 144 ids", **{f"{k}_ms": v["median_ms"] for k, v in r.items()}, "arms": r})
    for label, (lo, hi) in (("eval, 140 000 test rows", (N_TRAIN, N_ROWS)), ("eval, 560 000 train rows", (0, N_TRAIN))):
        arms = [with_weights(svm, "none", lambda: svm.eval_counts(lo, hi))]
        arms += [with_weights(svm, arm, lambda: svm.eval_weighted(lo, hi)) for arm in ARMS[1:]]
        r = alternate(svm, arms, a.reps, a.warmup)
        rows.append({"case": label + ": dsgd_eval_counts (none) / dsgd_eval_weighted (ones, random)",
                     **{f"{k}_ms": v["median_ms"] for k, v in r.items()}, "arms": r})
    for c in (svm, logistic):
        c.close()
    out = {"card": gpu, "sm_count": S, "reps": a.reps, "warmup": a.warmup, "rows": rows}
    print(json.dumps(out))
    if a.out:
        with open(a.out, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
