"""Dev tool: per-phase clock64 timeline of the persistent sync kernel (CTA 0), averaged over steps 50..250, plus the
per-CTA barrier arrivals of steps 100..103 against each CTA's non-zeros (is the arrival skew the row lengths?).
  python tools/timeline.py [batch]                      one GPU
  python tools/timeline.py [batch] --world N            N GPUs (one process each over gloo), stamps of rank 0"""
import os, socket, sys
os.environ["DSGD_PERSIST_TIMELINE"] = "1"
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np

NAMES = {0: "interval start (consumer warp 0)", 11: "K GPUs: push of g_{T-1} issued", 12: "K GPUs: column updated, W_T word published",
         1: "stage full (TMA landed)", 2: "first chunk: weights gathered, products done", 4: "first chunk: dot reduced",
         3: "rows done (scatter issued)", 13: "slowest consumer warp at the CTA barrier", 14: "slowest update warp at the CTA barrier", 6: "CTA synced, arriving at grid barrier",
         7: "grid barrier passed", 10: "update warp 0: its columns updated",
         9: "c_{t-1} summed from the barrier's partials, handed over"}


def report(tl_all, B, ms, S, world):
    tl = tl_all[:4096].reshape(256, 16)
    per_cta = tl_all[4096:].reshape(4, 160, 4)
    t = tl[50:250]
    print(f"world {world} batch {B}: {ms * 1e3 / S:.3f} us/step; step period {np.mean(np.diff(t[:, 0])):.0f} cycles")
    for k in sorted(NAMES, key=lambda k: np.mean((t[:, k] - t[:, 0])[t[:, k] > 0]) if (t[:, k] > 0).any() else 1e18):
        v = (t[:, k] - t[:, 0])[t[:, k] > 0]
        if len(v):
            print(f"  {NAMES[k]:48s} +{np.mean(v):8.0f} cycles (min {v.min()}, max {v.max()})")
    G = 132   # one CTA per SM of an H100
    for k in range(4):
        a, b, nz = per_cta[k, :G, 0], per_cta[k, :G, 1], per_cta[k, :G, 2]
        if not a.any():
            continue
        a0 = a.min()
        corr = float(np.corrcoef(a - a0, nz)[0, 1]) if nz.std() > 0 else float("nan")
        late = np.argsort(a)[-5:]
        print(f"step {100 + k} (ns): arrivals spread {a.max() - a0} (p50 {int(np.median(a - a0))}, p90 {int(np.percentile(a - a0, 90))}); "
              f"last arrival -> first exit {b.min() - a.max()}, -> last exit {b.max() - a.max()}; corr(arrival, pairs) {corr:.2f}; "
              f"pairs mean {nz.mean():.0f} max {nz.max()}; 5 latest CTAs pairs {nz[late].tolist()}")


def run(rank, world, port, B):
    from distributed_sgd_b200.native import NativeCtx
    from distributed_sgd_b200.utils import synthetic_rcv1
    group = None
    if world > 1:
        import torch, torch.distributed as dist
        from distributed_sgd_b200.core import Group
        torch.cuda.set_device(rank)
        dist.init_process_group("gloo", init_method=f"tcp://127.0.0.1:{port}", rank=rank, world_size=world)
        group = Group()
    S = 300
    data = synthetic_rcv1(n_rows=200000, seed=0)
    ctx = NativeCtx(rank, data.dim, 1e-5, rank=rank, world=world)
    ctx.load_csr(data.row_ptr, data.col, data.val, data.label)
    ctx.compute_dim_sparsity(160000)
    if world > 1:
        ctx.setup_peer_exchange(group)
    per = 160000 // world
    rng = np.random.default_rng(rank)
    idx = np.stack([rank * per + rng.choice(per, size=B, replace=False) for _ in range(S)]).astype(np.int32).reshape(-1)
    ctx.stage_samples(idx)
    ctx.set_weights(np.zeros(data.dim))
    ms = 0.0
    for _ in range(3):
        if group:
            group.barrier()
        ctx.timer_start()
        ctx.sync_steps_staged(0, B, S, 0.5, want_losses=True)
        ms = ctx.timer_stop()
    if rank == 0:
        tl = ctx.debug_timeline()
        report(tl, B, ms, S, world)
        if os.environ.get("TIMELINE_DUMP"):
            np.save(os.environ["TIMELINE_DUMP"], tl)
        if world > 1:
            v, b, n = ctx.xchg_stats()
            print(f"  pushed per peer and step: {v / max(n, 1):.0f} value words (16 B) + {b / max(n, 1):.0f} bitmap words (8 B) "
                  f"= {(16 * v + 8 * b) / max(n, 1) / 1e3:.1f} KB")
    if group:
        group.barrier()
    ctx.close()
    if world > 1:
        import torch.distributed as dist
        dist.destroy_process_group()


if __name__ == "__main__":
    args = [a for a in sys.argv[1:] if not a.startswith("--")]
    B = int(args[0]) if args else 256
    world = int(sys.argv[sys.argv.index("--world") + 1]) if "--world" in sys.argv else 1
    if world == 1:
        run(0, 1, 0, B)
    else:
        import torch.multiprocessing as mp
        with socket.socket() as s:
            s.bind(("127.0.0.1", 0)); port = s.getsockname()[1]
        mp.start_processes(run, args=(world, port, B), nprocs=world, start_method="spawn")
