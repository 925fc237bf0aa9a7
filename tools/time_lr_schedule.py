"""Dev tool: the cost of a per-step learning-rate table (dsgd_sync_steps_lr) against the scalar rate (dsgd_sync_steps), on the
full-size synthetic RCV1-shaped set (700 000 rows, the first 560 000 of them train rows).  Every case runs the same steps
through both calls, alternated on one context (fused: on both ranks' contexts):

    persistent kernel, batch 64, 256 and 1024 (2 188 steps per call)
    fallback (k_rows + k_update), batch 32 G + 1, G = SM count (200 steps per call)
    SparseLogistic, batch 256 (k_rows<logistic, …> + k_update, 200 steps per call)
    fused K = 2 on one GPU: two contexts of S / 2 CTAs each, batch 256 per rank (2 188 steps per call).  A CTA of the fused
    kernel owns at most 448 columns, so this case runs on a synthetic set of the same shape at dim 448 (S / 2) - 1.

The table holds the scalar rate at every step, so both arms compute the same trajectory and the difference is the table's
cost alone (its copy to the device and, on the persistent and fused kernels, one 8-byte load per thread and interval).  Both
calls copy their samples to the device, the same bytes.  Each case runs `--warmup` untimed calls per arm, then `--reps` rounds
of one timed call per arm (scalar first in even rounds, table first in odd ones), each on the host clock around the call,
which synchronises; every
call starts from the same weights.  The card's name and power limit are read in the same run with a read-only nvidia-smi
query; prints one JSON line.

    python tools/time_lr_schedule.py [--reps 7] [--warmup 1] [--json out.json]
"""
import argparse
import json
import os
import subprocess
import sys
import threading
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


def new_ctx(data, logistic=False, rank=0, world=1):
    c = NativeCtx(0, data.dim, LAM, rank=rank, world=world, logistic=logistic)
    c.load_csr(data.row_ptr, data.col, data.val, data.label)
    c.compute_dim_sparsity(N_TRAIN)
    return c


def draw(seed, steps, batch):
    rng = np.random.default_rng(seed)
    return np.concatenate([rng.choice(N_TRAIN, size=batch, replace=False) for _ in range(steps)]).astype(np.int32)


def timed(ctxs, samples, batch, steps, w0, use_table):
    """One call of `steps` steps on every context (one host thread each when there are several), from w0, with the scalar
    rate or with a table of it.  Host milliseconds from the start to the last context's return."""
    lrs = np.full(steps, LR)

    def run(i):
        c = ctxs[i]
        c.set_weights(w0)
        if use_table:
            c.sync_steps_lr(samples[i], batch, lrs, want_losses=False)
        else:
            c.sync_steps(samples[i], batch, steps, LR, want_losses=False)

    for c in ctxs:
        c.synchronize()
    t0 = time.perf_counter()
    if len(ctxs) == 1:
        run(0)
    else:
        th = [threading.Thread(target=run, args=(i,)) for i in range(len(ctxs))]
        for t in th:
            t.start()
        for t in th:
            t.join()
    return (time.perf_counter() - t0) * 1e3


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--json", default=None, help="also write the results to this file")
    a = ap.parse_args()
    gpu = card()
    data = synthetic_rcv1(n_rows=N_ROWS, seed=0)
    w0 = np.zeros(data.dim)
    svm = new_ctx(data)
    S = int(svm.info()["sm_count"])
    logistic = new_ctx(data, logistic=True)
    # the fused pair: each rank on half the SMs; every buffer (the table's included) reserved before the threads start
    G = S // 2
    fused_data = synthetic_rcv1(n_rows=N_ROWS, dim=448 * G - 1, seed=0)
    pair = [new_ctx(fused_data, rank=r, world=2) for r in range(2)]
    for c in pair:
        c.set_grid_limit(G)
        c.reserve(STEPS * 256, STEPS)
    pair[0].xchg_attach(1, pair[1])
    pair[1].xchg_attach(0, pair[0])
    for c in (svm, logistic):
        c.reserve(STEPS * 1024, STEPS)

    cases = [(f"persistent, batch {b}", [svm], b, STEPS, w0) for b in (64, 256, 1024)]
    cases.append((f"fallback, batch {32 * S + 1} (32 G + 1)", [svm], 32 * S + 1, SHORT_STEPS, w0))
    cases.append(("logistic, batch 256", [logistic], 256, SHORT_STEPS, w0))
    cases.append((f"fused K = 2 on one GPU, {G} CTAs per rank, dim {fused_data.dim}, batch 256 per rank", pair, 256, STEPS,
                  np.zeros(fused_data.dim)))

    rows = []
    for label, ctxs, b, steps, w0 in cases:
        samples = [draw(b + 7919 * r, steps, b) for r in range(len(ctxs))]
        for _ in range(a.warmup):
            for use_table in (False, True):
                timed(ctxs, samples, b, steps, w0, use_table)
        t = {False: [], True: []}
        for i in range(a.reps):
            for use_table in ((False, True) if i % 2 == 0 else (True, False)):   # neither arm always runs second
                t[use_table].append(timed(ctxs, samples, b, steps, w0, use_table))
        off, on = float(np.median(t[False])), float(np.median(t[True]))
        rows.append({"case": label, "steps": steps, "scalar_us_per_step": off * 1e3 / steps,
                     "table_us_per_step": on * 1e3 / steps, "table_over_scalar": on / off, "scalar_ms": t[False],
                     "table_ms": t[True]})
    out = {"card": gpu, "sm_count": S, "reps": a.reps, "warmup": a.warmup, "rows": rows}
    print(json.dumps(out))
    if a.json:
        with open(a.json, "w") as f:
            json.dump(out, f, indent=1)
    for c in (svm, logistic, *pair):
        c.close()


if __name__ == "__main__":
    main()
