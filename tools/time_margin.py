"""Dev tool: time all four models (SparseSVM, SparseLogistic, SparseSquaredHinge, SparseModifiedHuber) in the same process,
alternated, on the full-size synthetic RCV1-shaped set (700 000 rows, the first 560 000 of them train rows): sync steps at
batch 64, 256 and 1024 (2 188 steps per call), a full evaluation pass over the train rows, and a gradient request over
262 144 rows.

Each case runs `--warmup` untimed calls per model, then `--reps` rounds of one timed call per model (in the order above),
each on the host clock between two device synchronisations; a row reports the median of each model's calls.  Every context
starts every step call from the same weights.  The card's name and power limit are read in the same run with a read-only
nvidia-smi query; prints one JSON line.

    python tools/time_margin.py [--reps 7] [--warmup 1] [--json out.json]
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
STEPS = 2188
BATCHES = (64, 256, 1024)
GRAD_ROWS = 262_144
MODELS = ("svm", "logistic", "squared_hinge", "modified_huber")
LR = 0.1


def card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True, check=True)
    return r.stdout.strip().splitlines()[0]


def host_ms(ctx, fn):
    ctx.synchronize()
    t0 = time.perf_counter()
    fn()
    ctx.synchronize()
    return (time.perf_counter() - t0) * 1e3


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--json", default=None, help="also write the results to this file")
    a = ap.parse_args()
    gpu = card()
    data = synthetic_rcv1(n_rows=N_ROWS, seed=0)
    ctxs = {}
    for name in MODELS:
        c = NativeCtx(0, data.dim, 1e-5, model=name)
        c.load_csr(data.row_ptr, data.col, data.val, data.label)
        c.compute_dim_sparsity(N_TRAIN)
        ctxs[name] = c
    rng = np.random.default_rng(0)
    w_eval = np.where(rng.random(data.dim) < 0.6, rng.standard_normal(data.dim) * 0.05, 0.0)
    w0 = np.zeros(data.dim)
    grad_ids = rng.choice(N_TRAIN, size=GRAD_ROWS, replace=False).astype(np.int32)

    cases = []
    for b in BATCHES:
        def steps(c, b=b):   # from the same weights every call (the timed call includes this dsgd_set_weights)
            c.set_weights(w0)
            c.sync_steps_staged(0, b, STEPS, LR, want_losses=True)
        cases.append((f"sync steps, batch {b}", STEPS, steps))
    cases.append(("eval pass, train rows", 1, lambda c: c.eval(0, N_TRAIN)))
    cases.append((f"gradient, {GRAD_ROWS} rows", 1, lambda c: c.gradient(grad_ids)))

    rows = []
    for label, per, fn in cases:
        if label.startswith("sync"):   # the staged ids of this batch size
            b = int(label.split()[-1])
            ids = np.concatenate([np.random.default_rng(b).choice(N_TRAIN, size=b, replace=False) for _ in range(STEPS)])
            for c in ctxs.values():
                c.stage_samples(ids.astype(np.int32))
        else:
            for c in ctxs.values():
                c.set_weights(w_eval)
        for _ in range(a.warmup):
            for c in ctxs.values():
                fn(c)
        t = {k: [] for k in ctxs}
        for _ in range(a.reps):
            for k, c in ctxs.items():
                t[k].append(host_ms(c, lambda: fn(c)))
        row = {"case": label}
        for k in ctxs:
            med = float(np.median(t[k]))
            row[f"{k}_ms"] = med
            row[f"{k}_us_per_step" if per > 1 else f"{k}_us"] = med * 1e3 / per
        for k in MODELS[1:]:
            row[f"{k}_over_svm"] = row[f"{k}_ms"] / row["svm_ms"]
        rows.append(row)
    out = {"card": gpu, "reps": a.reps, "warmup": a.warmup, "rows": rows}
    print(json.dumps(out))
    if a.json:
        with open(a.json, "w") as f:
            json.dump(out, f, indent=1)
    for c in ctxs.values():
        c.close()


if __name__ == "__main__":
    main()
