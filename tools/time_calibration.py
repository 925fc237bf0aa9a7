"""Dev tool: time the calibration fit (dsgd_calibrate: score, then the whole Newton fit in one cooperative launch) against
the ranking-metrics pass (dsgd_eval_metrics) over the same rows, and against the path a user had before: dsgd_margins of the
rows to the host and the C checker's fit on one core.  Full-size synthetic RCV1-shaped set (560 000 train and 140 000 test
rows) with trained resident weights.  Calls are alternated; every timed call ends in a device synchronise, and the host clock
is read around it.  The card's name and power limit are read in the same run.

    python tools/time_calibration.py [--rows 700000] [--reps 15] [--out FILE]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def stats(ms):
    ms = np.asarray(ms)
    return {"median_ms": float(np.median(ms)), "p10_ms": float(np.percentile(ms, 10)), "p90_ms": float(np.percentile(ms, 90)),
            "n": int(ms.size)}


def alternated(calls: dict, warmup: int, reps: int) -> dict:
    for _ in range(warmup):
        for f in calls.values():
            f()
    t = {k: [] for k in calls}
    for _ in range(reps):
        for k, f in calls.items():
            t0 = time.perf_counter()
            f()
            t[k].append((time.perf_counter() - t0) * 1e3)
    return {k: stats(v) for k, v in t.items()}


def card():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30)
        return r.stdout.strip().splitlines()[0]
    except Exception as e:  # noqa: BLE001 -- reported, not hidden
        return f"unknown ({e})"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=700_000)
    ap.add_argument("--reps", type=int, default=15)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--out", default=None, help="also write the JSON result to this file")
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("time_calibration: no GPU; a CPU run gives no time")
    from distributed_sgd_b200.native import NativeCtx
    from distributed_sgd_b200.utils import synthetic_rcv1
    from oracle import calib

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
        y = np.asarray(data.label)[ids]
        fit = ctx.calibrate(b, e)
        rev = ctx.calibrate_samples(ids[::-1].copy())
        order_free = fit[:3] == rev[:3] and fit[3].tolist() == rev[3].tolist()
        ref = calib.fit(ctx.margins(ids), y)

        def host_path():
            calib.fit(ctx.margins(ids), y)

        def margins_only():
            ctx.margins(ids)

        r = alternated({"dsgd_calibrate": lambda: ctx.calibrate(b, e), "dsgd_eval_metrics": lambda: ctx.eval_metrics(b, e),
                        "dsgd_eval_calibration (10 bins)": lambda: ctx.eval_calibration(b, e, fit[0], fit[1], 10),
                        "dsgd_margins to the host + checker fit on one core": host_path,
                        "dsgd_margins to the host alone": margins_only}, a.warmup, a.reps)
        # the split of the call: device time of each kernel of one fit from the profiler's own events
        split = {}
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            for _ in range(5):
                ctx.calibrate(b, e)
        for ev in prof.key_averages():
            if "k_calib" in ev.key:
                split[ev.key.split("(")[0]] = {"mean_us": float(ev.device_time_total) / max(ev.count, 1), "count": int(ev.count)}
        out["cases"].append({"rows_set": name, "n": int(e - b), "A": fit[0], "B": fit[1], "iterations": int(fit[3][0]),
                             "status": int(fit[3][1]), "barriers": int(fit[3][4]), "order_free": bool(order_free),
                             "checker": {"A": ref.a, "B": ref.b, "iterations": ref.iterations, "points": ref.evaluations},
                             "timings": r, "kernel_split": split})
    ctx.close()
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(out, f, indent=1)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
