"""Dev tool: time the sampled evaluation (dsgd_eval_sampled_counts, dsgd_eval_samples_counts) against the full
evaluation pass (dsgd_eval_counts) over the test rows of a full-size synthetic RCV1-shaped set (560 000 train and
140 000 test rows), with non-zero weights resident on the device.

Per case: `--warmup` calls, then `--reps` calls, each timed on the host clock between two device synchronisations (the
call itself ends in one); the list pass includes its host-to-device copy of the ids.  For the streaming kernel, CUDA
events around its launches give the kernel time alone (passes below 2048 rows run k_rows, which is not bracketed).
The card's name and power limit are read in the same run with a read-only nvidia-smi query.

    python tools/time_sampled_eval.py [--reps 200] [--warmup 20] [--json out.json]
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

N_TRAIN, N_TEST = 560_000, 140_000
KS = (1_000, 10_000, 14_000, 100_000, 140_000)   # 14 000 = 10 % of the test rows


def card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True, check=True)
    return r.stdout.strip().splitlines()[0]


def timed(ctx, fn, warmup, reps):
    for _ in range(warmup):
        fn()
    ctx.synchronize()
    t = np.empty(reps)
    for i in range(reps):
        ctx.synchronize()
        t0 = time.perf_counter()
        fn()
        ctx.synchronize()
        t[i] = (time.perf_counter() - t0) * 1e3
    ctx.profile_begin(1)
    for _ in range(min(reps, 50)):
        fn()
    kern_ms, n_sampled = ctx.profile_end()
    return {"median_ms": float(np.median(t)), "p10_ms": float(np.percentile(t, 10)), "p90_ms": float(np.percentile(t, 90)),
            "kernel_ms": float(kern_ms) if n_sampled else None}


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--reps", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--json", default=None, help="also write the results to this file")
    a = ap.parse_args()
    gpu = card()
    data = synthetic_rcv1(n_rows=N_TRAIN + N_TEST, seed=0)
    ctx = NativeCtx(0, data.dim, 1e-5)
    ctx.load_csr(data.row_ptr, data.col, data.val, data.label)
    ctx.compute_dim_sparsity(N_TRAIN)
    rng = np.random.default_rng(0)
    ctx.set_weights(np.where(rng.random(data.dim) < 0.6, rng.standard_normal(data.dim) * 0.05, 0.0))
    b, e = N_TRAIN, N_TRAIN + N_TEST
    rows = []
    keys = iter(range(1, 1 << 30))
    r = timed(ctx, lambda: ctx.eval_counts(b, e), a.warmup, a.reps)
    rows.append({"pass": "full dsgd_eval_counts", "k": N_TEST, **r})
    for k in KS:
        r = timed(ctx, lambda: ctx.eval_sampled_counts(b, e, next(keys), 0, k), a.warmup, a.reps)
        rows.append({"pass": "device-drawn dsgd_eval_sampled_counts", "k": k, **r})
        ids = (b + rng.choice(N_TEST, size=k, replace=False)).astype(np.int32)
        r = timed(ctx, lambda: ctx.eval_samples_counts(ids), a.warmup, a.reps)
        rows.append({"pass": "list dsgd_eval_samples_counts (H2D incl.)", "k": k, **r})
    print(f"card: {gpu}")
    print(f"{'pass':44s} {'k':>7s} {'median ms':>10s} {'p10':>8s} {'p90':>8s} {'kernel ms':>10s}")
    for x in rows:
        kern = f"{x['kernel_ms']:.4f}" if x["kernel_ms"] is not None else "n/a"
        print(f"{x['pass']:44s} {x['k']:7d} {x['median_ms']:10.4f} {x['p10_ms']:8.4f} {x['p90_ms']:8.4f} {kern:>10s}")
    if a.json:
        with open(a.json, "w") as f:
            json.dump({"card": gpu, "reps": a.reps, "warmup": a.warmup, "rows": rows}, f, indent=1)
    ctx.close()


if __name__ == "__main__":
    main()
