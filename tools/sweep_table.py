"""BASELINE.json configs[4] as a table: reads bench.py JSON lines (one file per GPU count; each carries the `sweep` and `async`
sub-records measured in that run) and prints markdown.
    python tools/sweep_table.py bench_n1.json bench_n2.json ... > sweep.md"""
import json
import sys

rows = []
for path in sys.argv[1:]:
    try:
        j = json.loads(open(path).read().strip().splitlines()[-1])
    except Exception as e:  # noqa: BLE001
        print(f"<!-- {path}: unreadable ({e}) -->")
        continue
    n = j["n_gpus"]
    for r in j.get("sweep") or []:
        rows.append((n, "sync", r["batch_per_gpu"], "-", r["value"], r["us_per_step"], r["roofline_frac"], path))
    a = j.get("async")
    for r in a if isinstance(a, list) else []:
        rows.append((n, "async", r["batch"], r["lanes_per_gpu"], r["value"], r["us_per_update_per_lane"], r["roofline_frac"], path))
rows.sort(key=lambda r: (r[1], r[2], r[3] if r[3] != "-" else 0, r[0]))
print("| mode | batch per GPU | Hogwild lanes per GPU | GPUs | samples/s (all GPUs) | us per step (sync) / per update and lane (async) | "
      "fraction of the HBM roofline (algorithmic bytes / time / measured peak, per GPU) |")
print("|---|---|---|---|---|---|---|")
for n, mode, b, lanes, v, us, frac, _ in rows:
    print(f"| {mode} | {b} | {lanes} | {n} | {v:.4g} | {us:.2f} | {frac:.5f} |")
