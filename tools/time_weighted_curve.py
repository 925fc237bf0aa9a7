"""Dev tool: time the weighted curve passes (dsgd_eval_weighted_curve, words only and with its points) against the unweighted
curve passes (dsgd_eval_curve, AP only and with its points) over the same rows of a full-size synthetic RCV1-shaped set
(560 000 train and 140 000 test rows), with non-zero weights resident on the device and sample and class weights loaded.

The four passes over one range are called alternately, `--warmup` times each and then `--reps` times each; every call is
timed on the host clock between two device synchronisations (the calls end in one themselves), and the medians are
reported with the 10th and 90th percentiles.  The card's name and power limit are read in the same run with a read-only
nvidia-smi query.

    python tools/time_weighted_curve.py [--reps 15] [--warmup 3] [--json out.json]
"""
import argparse
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import numpy as np  # noqa: E402

from distributed_sgd_b200.native import NativeCtx  # noqa: E402
from distributed_sgd_b200.utils import synthetic_rcv1  # noqa: E402
from tools.time_metrics import N_TEST, N_TRAIN, alternated, card  # noqa: E402


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
    ctx.set_sample_weights(rng.random(data.n_rows) * 2.0)
    ctx.set_class_weights(2.0, 0.5)
    rows = []
    for name, b, e in (("test rows", N_TRAIN, N_TRAIN + N_TEST), ("train rows", 0, N_TRAIN)):
        points = ctx.eval_weighted_curve(b, e).n_points
        r = alternated(ctx, {"dsgd_eval_curve, AP only": lambda: ctx.eval_curve(b, e, curve=False),
                             "dsgd_eval_weighted_curve, words only": lambda: ctx.eval_weighted_curve(b, e, curve=False),
                             "dsgd_eval_curve, points": lambda: ctx.eval_curve(b, e),
                             "dsgd_eval_weighted_curve, points": lambda: ctx.eval_weighted_curve(b, e)}, a.warmup, a.reps)
        rows += [{"case": f"{k} over the {name}", "rows": e - b, "points": points, **v} for k, v in r.items()]
    print(f"card: {gpu}")
    print(f"{'case':56s} {'rows':>7s} {'points':>7s} {'median ms':>10s} {'p10':>8s} {'p90':>8s}")
    for x in rows:
        print(f"{x['case']:56s} {x['rows']:7d} {x['points']:7d} {x['median_ms']:10.4f} {x['p10_ms']:8.4f} {x['p90_ms']:8.4f}")
    if a.json:
        with open(a.json, "w") as f:
            json.dump({"card": gpu, "reps": a.reps, "warmup": a.warmup, "rows": rows}, f, indent=1)
    ctx.close()


if __name__ == "__main__":
    main()
