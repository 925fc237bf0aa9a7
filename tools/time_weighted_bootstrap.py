"""Dev tool: time the weighted Poisson bootstrap (dsgd_eval_weighted_bootstrap) at 100 and 1000 replicates over the 140 000
test rows and the 560 000 train rows of a full-size synthetic RCV1-shaped set, alternated with the unweighted bootstrap
(dsgd_eval_bootstrap) of the same replicates and one weighted curve pass (dsgd_eval_weighted_curve with curve=False), with
non-zero weights resident on the device, balanced class weights and random sample weights.

The calls over one range are alternated, `--warmup` times each and then `--reps` times each; every call is timed on the host
clock between two device synchronisations (the calls end in one themselves), and the medians are reported with the 10th and
90th percentiles.  The card's name and power limit are read in the same run with a read-only nvidia-smi query.

    python tools/time_weighted_bootstrap.py [--reps 7] [--warmup 2] [--json out.json]
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
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--warmup", type=int, default=2)
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
    n_pos = int(np.sum(data.label > 0))
    n = data.label.size
    ctx.set_class_weights(n / (2.0 * n_pos), n / (2.0 * (n - n_pos)))
    ctx.set_sample_weights(rng.random(n) * 2.0)
    rows = []
    for name, b, e in (("test rows", N_TRAIN, N_TRAIN + N_TEST), ("train rows", 0, N_TRAIN)):
        r = alternated(ctx, {
            "dsgd_eval_weighted_curve, words only": lambda: ctx.eval_weighted_curve(b, e, curve=False),
            "dsgd_eval_bootstrap, 100 replicates": lambda: ctx.eval_bootstrap(b, e, 1, 0, 100),
            "dsgd_eval_weighted_bootstrap, 100 replicates": lambda: ctx.eval_weighted_bootstrap(b, e, 1, 0, 100),
            "dsgd_eval_bootstrap, 1000 replicates": lambda: ctx.eval_bootstrap(b, e, 1, 0, 1000),
            "dsgd_eval_weighted_bootstrap, 1000 replicates": lambda: ctx.eval_weighted_bootstrap(b, e, 1, 0, 1000)},
            a.warmup, a.reps)
        rows += [{"case": f"{k} over the {name}", "rows": e - b, **v} for k, v in r.items()]
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
