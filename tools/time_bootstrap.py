"""Dev tool: time the Poisson bootstrap (dsgd_eval_bootstrap) at 100 and 1000 replicates over the 140 000 test rows and the
560 000 train rows of a full-size synthetic RCV1-shaped set, against one average-precision pass (dsgd_eval_curve with
curve=False) over the same rows, with non-zero weights resident on the device.

The calls over one range are alternated, `--warmup` times each and then `--reps` times each; every call is timed on the host
clock between two device synchronisations (the calls end in one themselves), and the medians are reported with the 10th and
90th percentiles.  For context, a host bootstrap of the same size is timed too: dsgd_margins of the rows, then per replicate
numpy's Poisson draw, a weighted sort-based ROC AUC and average precision -- over `--host-reps` replicates only, and
extrapolated to 1000 (labelled as such).  The card's name and power limit are read in the same run with a read-only
nvidia-smi query.

    python tools/time_bootstrap.py [--reps 9] [--warmup 2] [--host-reps 5] [--json out.json]
"""
import argparse
import json
import os
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import numpy as np  # noqa: E402

from distributed_sgd_b200.native import NativeCtx  # noqa: E402
from distributed_sgd_b200.utils import synthetic_rcv1  # noqa: E402
from tools.time_metrics import N_TEST, N_TRAIN, alternated, card  # noqa: E402


def host_replicate(rng, margins, labels):
    """One host replicate: Poisson(1) multiplicities, then AUC and AP of the weighted rows by one sort."""
    m = rng.poisson(1.0, size=margins.size)
    order = np.argsort(margins, kind="stable")            # score -margin, highest first
    w, y = m[order], labels[order] > 0
    tp, fp = np.cumsum(w * y), np.cumsum(w * ~y)
    P, N = tp[-1], fp[-1]
    ap = float(np.sum((w * y) * tp / np.maximum(tp + fp, 1))) / max(P, 1)
    auc = float(np.sum((w * ~y) * (2 * tp - w * y))) / max(2 * P * N, 1)
    return auc, ap


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--reps", type=int, default=9)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--host-reps", type=int, default=5)
    ap.add_argument("--json", default=None, help="also write the results to this file")
    a = ap.parse_args()
    if a.reps < 5:
        ap.error("--reps must be at least 5")
    gpu = card()
    data = synthetic_rcv1(n_rows=N_TRAIN + N_TEST, seed=0)
    ctx = NativeCtx(0, data.dim, 1e-5)
    ctx.load_csr(data.row_ptr, data.col, data.val, data.label)
    ctx.compute_dim_sparsity(N_TRAIN)
    rng = np.random.default_rng(0)
    ctx.set_weights(np.where(rng.random(data.dim) < 0.6, rng.standard_normal(data.dim) * 0.05, 0.0))
    rows = []
    for name, b, e in (("test rows", N_TRAIN, N_TRAIN + N_TEST), ("train rows", 0, N_TRAIN)):
        r = alternated(ctx, {"dsgd_eval_curve, AP only": lambda: ctx.eval_curve(b, e, curve=False),
                             "dsgd_eval_bootstrap, 100 replicates": lambda: ctx.eval_bootstrap(b, e, 1, 0, 100),
                             "dsgd_eval_bootstrap, 1000 replicates": lambda: ctx.eval_bootstrap(b, e, 1, 0, 1000)},
                       a.warmup, a.reps)
        rows += [{"case": f"{k} over the {name}", "rows": e - b, **v} for k, v in r.items()]
        t0 = time.perf_counter()
        ids = np.arange(b, e, dtype=np.int32)
        margins = ctx.margins(ids)
        labels = data.label[b:e]
        hr = np.random.default_rng(1)
        for _ in range(a.host_reps):
            host_replicate(hr, margins, labels)
        t = (time.perf_counter() - t0) / a.host_reps * 1000.0 * 1000.0
        rows.append({"case": f"host bootstrap (margins + numpy), {name}, {a.host_reps} replicates extrapolated to 1000",
                     "rows": e - b, "median_ms": t, "p10_ms": float("nan"), "p90_ms": float("nan")})
    print(f"card: {gpu}")
    print(f"{'case':80s} {'rows':>7s} {'median ms':>10s} {'p10':>8s} {'p90':>8s}")
    for x in rows:
        print(f"{x['case']:80s} {x['rows']:7d} {x['median_ms']:10.3f} {x['p10_ms']:8.3f} {x['p90_ms']:8.3f}")
    if a.json:
        with open(a.json, "w") as f:
            json.dump({"card": gpu, "reps": a.reps, "warmup": a.warmup, "rows": rows}, f, indent=1)
    ctx.close()


if __name__ == "__main__":
    main()
