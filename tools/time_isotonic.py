"""Dev tool: time the isotonic fit (dsgd_calibrate_isotonic: the curve pass with its points left on the device, then the
hull and the emit) against the Platt fit (dsgd_calibrate) and the curve with its points (dsgd_eval_curve), and against the
path a user had before: dsgd_margins of the rows to the host and scikit-learn's IsotonicRegression fit.  Also the map
applied (dsgd_isotonic_probabilities) against the sigmoid (dsgd_calibrated_probabilities), and the device time of every
kernel of one fit from the profiler's own events: scoring, sort, merge, scans, emit and the hull rounds.  Full-size
synthetic RCV1-shaped set (560 000 train and 140 000 test rows) with trained resident weights.  Calls are alternated; every
timed call ends in a device synchronise, and the host clock is read around it (medians of --reps).  The card's name and
power limit are read in the same run.

    python tools/time_isotonic.py [--rows 700000] [--reps 15] [--out FILE]
"""
import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from time_calibration import alternated, card  # noqa: E402


def kernel_group(name: str) -> str:
    for key, group in (("k_metrics_score", "score"), ("RadixSort", "sort"), ("Merge", "merge"), ("Scan", "scans"),
                       ("k_curve_count", "curve count"), ("k_curve_sum", "curve count"), ("k_curve_emit", "curve emit"),
                       ("k_iso_tile", "hull tiles"), ("k_iso_merge", "hull merge rounds"), ("k_iso_emit", "iso emit")):
        if key in name:
            return group
    return "other"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=700_000)
    ap.add_argument("--reps", type=int, default=15)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--out", default=None, help="also write the JSON result to this file")
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("time_isotonic: no GPU; a CPU run gives no time")
    from sklearn.isotonic import IsotonicRegression

    from distributed_sgd_b200.native import NativeCtx
    from distributed_sgd_b200.utils import synthetic_rcv1

    data = synthetic_rcv1(n_rows=a.rows, seed=0)
    n_train = int(a.rows * 0.8)
    ctx = NativeCtx(0, data.dim, 1e-5)
    ctx.load_csr(data.row_ptr, data.col, data.val, data.label)
    ctx.compute_dim_sparsity(n_train)
    rng = np.random.default_rng(0)
    ctx.set_weights(np.zeros(data.dim))
    ctx.sync_steps(rng.integers(0, n_train, size=2000 * 100).astype(np.int32), 100, 2000, 0.5, want_losses=False)
    out = {"card": card(), "rows": a.rows, "cases": []}
    for name, (b, e) in {"test": (n_train, a.rows), "train": (0, n_train)}.items():
        ids = np.arange(b, e, dtype=np.int32)
        y = (np.asarray(data.label)[ids] > 0).astype(np.float64)
        fit = ctx.calibrate_isotonic(b, e)
        ab = ctx.calibrate(b, e)
        before = ctx.launch_count()
        ctx.calibrate_isotonic(b, e)
        launches = ctx.launch_count() - before

        def host_path():
            IsotonicRegression(increasing=True, out_of_bounds="clip").fit(-ctx.margins(ids), y)

        r = alternated({"dsgd_calibrate_isotonic": lambda: ctx.calibrate_isotonic(b, e),
                        "dsgd_calibrate": lambda: ctx.calibrate(b, e),
                        "dsgd_eval_curve with points": lambda: ctx.eval_curve(b, e),
                        "dsgd_margins to the host + scikit-learn fit": host_path,
                        "dsgd_isotonic_probabilities": lambda: ctx.isotonic_probabilities(ids, fit[0], fit[1]),
                        "dsgd_calibrated_probabilities": lambda: ctx.calibrated_probabilities(ids, ab[0], ab[1])},
                       a.warmup, a.reps)
        split = {}
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            for _ in range(5):
                ctx.calibrate_isotonic(b, e)
        for ev in prof.key_averages():
            g = split.setdefault(kernel_group(ev.key), {"us_per_fit": 0.0, "launches_per_fit": 0.0})
            g["us_per_fit"] += float(ev.device_time_total) / 5
            g["launches_per_fit"] += ev.count / 5
        out["cases"].append({"rows_set": name, "n": int(e - b), "blocks": int(fit[4][0]), "points": int(fit[4][1]),
                             "distinct_scores": int(fit[4][4]), "counted_launches": int(launches), "timings": r,
                             "kernel_split": split})
    ctx.close()
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(out, f, indent=1)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
