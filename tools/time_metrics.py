"""Dev tool: time the ranking-metrics pass (dsgd_eval_metrics: score, sort, count) against the evaluation pass
(dsgd_eval_sums) over the same rows of a full-size synthetic RCV1-shaped set (560 000 train and 140 000 test rows), and
dsgd_margins over 262 144 ids, with non-zero weights resident on the device.

The two passes over one range are called alternately, `--warmup` times each and then `--reps` times each; every call is
timed on the host clock between two device synchronisations (the calls end in one themselves), and the medians are
reported with the 10th and 90th percentiles.  The margins include the ids' host-to-device copy and the values' copy back.
The card's name and power limit are read in the same run with a read-only nvidia-smi query.

    python tools/time_metrics.py [--reps 15] [--warmup 3] [--json out.json]
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
N_MARGINS = 262_144


def card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True, check=True)
    return r.stdout.strip().splitlines()[0]


def one(ctx, fn):
    ctx.synchronize()
    t0 = time.perf_counter()
    fn()
    ctx.synchronize()
    return (time.perf_counter() - t0) * 1e3


def alternated(ctx, fns, warmup, reps):
    """{name: ms of each call} with the calls of the named functions interleaved."""
    for _ in range(warmup):
        for fn in fns.values():
            fn()
    t = {k: [] for k in fns}
    for _ in range(reps):
        for k, fn in fns.items():
            t[k].append(one(ctx, fn))
    return {k: {"median_ms": float(np.median(v)), "p10_ms": float(np.percentile(v, 10)),
                "p90_ms": float(np.percentile(v, 90)), "calls": len(v)} for k, v in t.items()}


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--reps", type=int, default=15)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--json", default=None, help="also write the results to this file")
    a = ap.parse_args()
    if a.reps < 7:
        ap.error("--reps must be at least 7")
    gpu = card()
    data = synthetic_rcv1(n_rows=N_TRAIN + N_TEST, seed=0)
    ctx = NativeCtx(0, data.dim, 1e-5)
    ctx.load_csr(data.row_ptr, data.col, data.val, data.label)
    ctx.compute_dim_sparsity(N_TRAIN)
    rng = np.random.default_rng(0)
    ctx.set_weights(np.where(rng.random(data.dim) < 0.6, rng.standard_normal(data.dim) * 0.05, 0.0))
    rows = []
    for name, b, e in (("test rows", N_TRAIN, N_TRAIN + N_TEST), ("train rows", 0, N_TRAIN)):
        r = alternated(ctx, {"dsgd_eval_metrics": lambda: ctx.eval_metrics(b, e),
                             "dsgd_eval_sums": lambda: ctx.eval_sums(b, e)}, a.warmup, a.reps)
        rows += [{"case": f"{k} over the {name}", "rows": e - b, **v} for k, v in r.items()]
    ids = rng.integers(0, N_TRAIN + N_TEST, size=N_MARGINS).astype(np.int32)
    r = alternated(ctx, {"dsgd_margins": lambda: ctx.margins(ids)}, a.warmup, a.reps)
    rows += [{"case": "dsgd_margins (H2D ids, D2H values incl.)", "rows": N_MARGINS, **r["dsgd_margins"]}]
    print(f"card: {gpu}")
    print(f"{'case':44s} {'rows':>7s} {'median ms':>10s} {'p10':>8s} {'p90':>8s}")
    for x in rows:
        print(f"{x['case']:44s} {x['rows']:7d} {x['median_ms']:10.4f} {x['p10_ms']:8.4f} {x['p90_ms']:8.4f}")
    if a.json:
        with open(a.json, "w") as f:
            json.dump({"card": gpu, "reps": a.reps, "warmup": a.warmup, "rows": rows}, f, indent=1)
    ctx.close()


if __name__ == "__main__":
    main()
