"""Dev tool: the one-GPU persistent sync step of two builds of libdsgd.so side by side -- microseconds per step at batch 64, 256
and 1024, and the per-step timeline of each build (stamps of tools/timeline.py, DSGD_PERSIST_TIMELINE), in one run.

    python tools/time_sync_chain.py --base OLD/libdsgd.so [--new distributed_sgd_b200/libdsgd.so] [--rounds 3] [--json out.json]

Every build runs in a process of its own (a library is loaded once per process), on the full-size synthetic RCV1-shaped set
(700 000 rows, the first 560 000 train rows) with the same staged samples: per batch, one untimed call, then `--reps` calls of
2 188 steps with losses on (bench.py's workload), each timed with CUDA events.  The builds alternate, `--rounds` times each.
The card's name and power limit come from a read-only nvidia-smi query, and its SM clock from queries taken while the timed
calls run.  Timeline: cycles from a grid barrier's pass (stamp 7 of the step before) to CTA 0's stamps of the next step,
averaged over steps 50..250 at each batch; whether the slowest update warp reached the CTA barrier after the slowest consumer
warp; CTA 0's place among the arrivals of steps 100..103, and in each of those steps whether the CTAs that arrived last held
a row of more than one 128-pair chunk.  Prints one JSON line.
"""
import argparse
import json
import os
import subprocess
import sys
import threading

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

N_ROWS, N_TRAIN, STEPS, TL_STEPS = 700_000, 560_000, 2188, 300
LAM, LR = 1e-5, 0.5
BATCHES = (64, 256, 1024)
STAMPS = {9: "update warp 0: c handed over", 10: "update warp 0: columns updated", 13: "slowest consumer warp at CTA barrier",
          14: "slowest update warp at CTA barrier", 6: "CTA arriving at grid barrier", 7: "next grid barrier passed"}


def smi(fields):
    r = subprocess.run(["nvidia-smi", f"--query-gpu={fields}", "--format=csv,noheader,nounits"], capture_output=True,
                       text=True, check=True)
    return [v.strip() for v in r.stdout.strip().splitlines()[0].split(",")]


def timeline_stats(tl):
    import numpy as np
    t = tl[:4096].reshape(256, 16)
    per = tl[4096:].reshape(4, 160, 4)
    ok = [s for s in range(51, 250) if t[s - 1, 7] > 0 and all(t[s, k] > 0 for k in STAMPS)]
    passed = np.array([t[s - 1, 7] for s in ok])
    d = {k: np.array([t[s, k] for s in ok]) - passed for k in STAMPS}
    out = {"steps": len(ok), "cycles_after_barrier_pass": {STAMPS[k]: round(float(d[k].mean())) for k in STAMPS},
           "update_after_consumers_share": float(np.mean(d[14] > d[13]))}
    ranks, order = [], []
    for k in range(4):
        a = per[k, :, 0]
        G = int(np.count_nonzero(a))
        if G:
            ranks.append(int(np.sum(a[:G] > a[0])))   # CTAs that arrived after CTA 0
            order.append(arrival_order(a[:G], per[k, :G, 3]))
    out["cta0_arrivals_after_it"] = ranks
    out["arrival_order_by_multi_chunk_row"] = order
    return out


def arrival_order(arrive_ns, chunk_word):
    """One step's grid-barrier arrivals against whether the CTA held a row of more than one chunk (record word 3: chunks in
    the low 32 bits, rows of several chunks in the high 32): the share of such CTAs among all, among the latest tenth and
    as the last to arrive, and the mean arrival rank (0 first, 1 last) of the CTAs with and without one."""
    import numpy as np
    G = len(arrive_ns)
    multi = (chunk_word >> 32) > 0
    chunks = chunk_word & 0xffffffff
    rank = np.argsort(np.argsort(arrive_ns, kind="stable"), kind="stable") / max(G - 1, 1)
    late = np.argsort(arrive_ns, kind="stable")[-max(G // 10, 1):]
    mean = lambda m: round(float(rank[m].mean()), 3) if m.any() else None
    return {"ctas": G, "multi_share": round(float(multi.mean()), 3), "multi_share_latest_tenth": round(float(multi[late].mean()), 3),
            "last_holds_multi": bool(multi[late[-1]]), "mean_rank_multi": mean(multi), "mean_rank_single": mean(~multi),
            "chunks_latest_tenth": chunks[late].astype(int).tolist(), "max_chunks": int(chunks.max())}


def worker(lib_path, reps, timeline):
    import numpy as np
    from distributed_sgd_b200 import native
    native.LIB_PATH = lib_path
    from distributed_sgd_b200.native import NativeCtx
    from distributed_sgd_b200.utils import synthetic_rcv1
    data = synthetic_rcv1(n_rows=N_ROWS, seed=0)
    ctx = NativeCtx(0, data.dim, LAM)
    ctx.load_csr(data.row_ptr, data.col, data.val, data.label)
    ctx.compute_dim_sparsity(N_TRAIN)
    res = {}
    for B in BATCHES:
        steps = TL_STEPS if timeline else STEPS
        rng = np.random.default_rng(B)
        ctx.stage_samples(np.concatenate([rng.choice(N_TRAIN, size=B, replace=False) for _ in range(steps)]).astype(np.int32))
        ctx.set_weights(np.zeros(data.dim))
        ctx.sync_steps_staged(0, B, steps, LR, want_losses=True)
        ctx.synchronize()
        if timeline:
            res[B] = timeline_stats(ctx.debug_timeline())
            continue
        clocks = []
        sampler = threading.Thread(target=lambda: clocks.append(int(smi("clocks.sm")[0])))
        ms = []
        for i in range(reps):
            if i == reps // 2:
                sampler.start()
            ctx.set_weights(np.zeros(data.dim))
            ctx.timer_start()
            ctx.sync_steps_staged(0, B, steps, LR, want_losses=True)
            ms.append(ctx.timer_stop())
        sampler.join()
        res[B] = {"us_per_step": [m * 1e3 / steps for m in ms], "sm_clock_mhz": clocks}
    ctx.close()
    print(json.dumps(res))


def run_worker(lib_path, reps, timeline):
    env = dict(os.environ)
    if timeline:
        env["DSGD_PERSIST_TIMELINE"] = "1"
    r = subprocess.run([sys.executable, os.path.abspath(__file__), "--worker", lib_path, "--reps", str(reps)]
                       + (["--timeline"] if timeline else []), capture_output=True, text=True, env=env)
    if r.returncode != 0:
        sys.stderr.write(r.stderr)
        raise RuntimeError(f"worker for {lib_path} failed")
    return {int(k): v for k, v in json.loads(r.stdout.strip().splitlines()[-1]).items()}


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--base", help="libdsgd.so of the build to compare against")
    ap.add_argument("--new", default=os.path.join(ROOT, "distributed_sgd_b200", "libdsgd.so"))
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--json", default=None, help="also write the results to this file")
    ap.add_argument("--worker", default=None, help=argparse.SUPPRESS)
    ap.add_argument("--timeline", action="store_true", help=argparse.SUPPRESS)
    a = ap.parse_args()
    if a.worker:
        return worker(a.worker, a.reps, a.timeline)
    if not a.base:
        ap.error("--base is required")
    import numpy as np
    name, power_limit, max_clock = smi("name,power.limit,clocks.max.sm")
    builds = {"base": os.path.abspath(a.base), "new": os.path.abspath(a.new)}
    runs = {k: [] for k in builds}
    for _ in range(a.rounds):
        for k, path in builds.items():
            runs[k].append(run_worker(path, a.reps, False))
    out = {"card": name, "power_limit_w": power_limit, "max_sm_clock_mhz": max_clock, "rounds": a.rounds, "reps": a.reps,
           "steps_per_call": STEPS, "batches": {}}
    for B in BATCHES:
        row = {}
        for k in builds:
            per_round = [float(np.median(r[B]["us_per_step"])) for r in runs[k]]
            row[k] = {"median_us_per_step_by_round": per_round, "min": min(per_round), "max": max(per_round),
                      "sm_clock_mhz": [c for r in runs[k] for c in r[B]["sm_clock_mhz"]]}
        row["new_slowest_beats_base_fastest"] = row["new"]["max"] < row["base"]["min"]
        row["speedup_median"] = float(np.median(row["base"]["median_us_per_step_by_round"]) /
                                      np.median(row["new"]["median_us_per_step_by_round"]))
        out["batches"][B] = row
    out["timeline"] = {k: run_worker(path, 1, True) for k, path in builds.items()}
    print(json.dumps(out))
    if a.json:
        with open(a.json, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
