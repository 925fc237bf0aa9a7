"""Dev tool: the cost of the L1 penalty (dsgd_set_l1) per sync step, on the full-size synthetic RCV1-shaped set (700 000 rows,
the first 560 000 of them train rows).  Every case runs the same staged steps with the penalty off and on, alternated on one
context:

    persistent kernel and its L1 form, batch 64, 256 and 1024 (2 188 steps per call)
    fallback (k_rows + k_update against k_rows + k_update<..., kL1>), batch 32 G + 1, G = SM count (200 steps per call)
    SparseLogistic, batch 256 (k_rows<logistic, …> + k_update against k_update<..., kL1>, 200 steps per call)

Each case runs `--warmup` untimed calls per arm, then `--reps` rounds of one timed call per arm (off first, then on), each on
the host clock between two device synchronisations; every call starts from the same weights.  The card's name and power
limit are read in the same run with a read-only nvidia-smi query; prints one JSON line.

    python tools/time_l1.py [--reps 7] [--warmup 1] [--lambda1 1e-5] [--json out.json]
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


def new_ctx(data, logistic=False):
    c = NativeCtx(0, data.dim, LAM, logistic=logistic)
    c.load_csr(data.row_ptr, data.col, data.val, data.label)
    c.compute_dim_sparsity(N_TRAIN)
    return c


def draw(seed, steps, batch):
    rng = np.random.default_rng(seed)
    return np.concatenate([rng.choice(N_TRAIN, size=batch, replace=False) for _ in range(steps)]).astype(np.int32)


def timed(c, batch, steps, w0, lambda1):
    """One call of `steps` staged steps from w0 with the penalty lambda1.  Host milliseconds between synchronisations."""
    c.synchronize()
    t0 = time.perf_counter()
    c.set_l1(lambda1)
    c.set_weights(w0)
    c.sync_steps_staged(0, batch, steps, LR)
    c.synchronize()
    return (time.perf_counter() - t0) * 1e3


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--lambda1", type=float, default=1e-5)
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

    rows = []
    for label, c, b, steps in cases:
        c.stage_samples(draw(b, steps, b))
        for _ in range(a.warmup):
            for lam1 in (0.0, a.lambda1):
                timed(c, b, steps, w0, lam1)
        t = {0: [], 1: []}
        for _ in range(a.reps):
            for k, lam1 in enumerate((0.0, a.lambda1)):
                t[k].append(timed(c, b, steps, w0, lam1))
        c.set_l1(0.0)
        c.set_l1(a.lambda1)
        c.set_weights(w0)
        c.sync_steps_staged(0, b, steps, LR)
        nnz = c.weights_l1()[1]
        c.set_l1(0.0)
        off, on = float(np.median(t[0])), float(np.median(t[1]))
        rows.append({"case": label, "steps": steps, "off_us_per_step": off * 1e3 / steps, "on_us_per_step": on * 1e3 / steps,
                     "on_over_off": on / off, "nnz_after_on": nnz, "off_ms": t[0], "on_ms": t[1]})
    out = {"card": gpu, "sm_count": S, "lambda1": a.lambda1, "reps": a.reps, "warmup": a.warmup, "rows": rows}
    print(json.dumps(out))
    if a.json:
        with open(a.json, "w") as f:
            json.dump(out, f, indent=1)
    for c in (svm, logistic):
        c.close()


if __name__ == "__main__":
    main()
