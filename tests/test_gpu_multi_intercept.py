"""Two-GPU sync steps with an intercept: one process per GPU, two workers per rank, gradients and the intercept's slot summed
by the NCCL allreduce (dim + 3 words).  At lambda = 0 on dyadic rows the run equals, bit for bit, the same run of plain
contexts of dimension dim + 1 whose rows end in (dim, 1.0), and the replicas are identical.  Skipped on a single-GPU box."""
import os
import socket
import sys

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _free_port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def _worker(rank, world, port, q):
    sys.path.insert(0, ROOT)
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    import torch
    import torch.distributed as dist
    from distributed_sgd_b200.core import Group
    from distributed_sgd_b200.native import NativeCtx
    from helpers import data_from_csr
    from test_gpu_intercept import DIM, _augment, _rows, _weights

    torch.cuda.set_device(rank)
    dist.init_process_group("gloo", init_method=f"tcp://127.0.0.1:{port}", rank=rank, world_size=world)
    group = Group()
    rp, col, val, lab = _rows(21, n=4000)
    d = np.random.default_rng(3).integers(0, 65, size=DIM) / 64.0
    runs = []
    for intercept in (True, False):
        data = (data_from_csr(rp, col, val, lab, DIM) if intercept
                else data_from_csr(*_augment(rp, col, val, DIM), lab, DIM + 1))
        ctx = NativeCtx(rank, data.dim, 0.0, rank=rank, world=world, intercept=intercept)
        ctx.load_csr(data.row_ptr, data.col, data.val, data.label)
        ctx.set_dim_sparsity(d if intercept else np.append(d, 0.0))
        uid = NativeCtx.comm_unique_id() if rank == 0 else b""
        ctx.comm_init(group.broadcast_bytes(uid, 0))
        V, batch, steps = 2, 24, 8
        rng = np.random.default_rng(5)
        idx = rng.integers(0, 4000, size=(steps, world * V, batch)).astype(np.int32)
        mine = idx[:, rank * V:(rank + 1) * V, :].reshape(-1)
        ctx.set_weights(_weights(1, 0.25))
        ctx.set_workers([batch] * V, world * V)
        losses = ctx.sync_steps(mine, V * batch, steps, 0.0625)
        runs.append((losses, ctx.get_weights()))
        ctx.close()
    (li, wi), (la, wa) = runs
    same_aug = bool(np.array_equal(li.view(np.int64), la.view(np.int64)) and np.array_equal(wi.view(np.int64), wa.view(np.int64)))
    blobs = group.all_gather_bytes(wi.tobytes())
    q.put((rank, same_aug, all(b == blobs[0] for b in blobs), float(wi[DIM])))
    dist.destroy_process_group()


def test_two_gpu_intercept_step_equals_the_augmented_context():
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    import torch.multiprocessing as mp
    ctxmp = mp.get_context("spawn")
    q = ctxmp.Queue()
    port = _free_port()
    procs = [ctxmp.Process(target=_worker, args=(r, 2, port, q)) for r in range(2)]
    for p in procs:
        p.start()
    res = [q.get(timeout=300) for _ in procs]
    for p in procs:
        p.join(timeout=60)
    for rank, same_aug, same, beta in res:
        assert same_aug, f"rank {rank}: the intercept run differs from the augmented run"
        assert same, "weight replicas differ across GPUs"
        assert beta != 0.25
