"""A destroyed context gives back every byte of device memory it took.

Contexts are created and destroyed over and over, in every mode (one-GPU sync on the persistent kernel with its debug
timeline, async with an outbox and a hosted master, and a K = 2 pair of fused ranks on one GPU), and the device's free
memory must come back to where it was.  The cycles run in a child process: DSGD_PERSIST_TIMELINE is read once per process,
and the free-memory figure then belongs to this workload alone.
"""
import os
import subprocess
import sys

import pytest

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

_CHILD = r"""
import sys
import threading
sys.path.insert(0, sys.argv[1])
import numpy as np
import torch
from distributed_sgd_b200.native import NativeCtx
from distributed_sgd_b200.utils import synthetic_rcv1

data = synthetic_rcv1(n_rows=3000, dim=5000, seed=3, mean_nnz=20.0)
n_train, lam, lr, batch, steps = 2400, 1e-4, 0.5, 64, 8
rng = np.random.default_rng(0)
idx = rng.integers(0, n_train, size=batch * steps).astype(np.int32)
w_host = rng.standard_normal(data.dim) * 0.01
sms = torch.cuda.get_device_properties(0).multi_processor_count


def loaded(**kw):
    ctx = NativeCtx(0, data.dim, lam, **kw)
    ctx.load_csr(data.row_ptr, data.col, data.val, data.label)
    ctx.compute_dim_sparsity(n_train)
    return ctx


def sync_cycle():
    ctx = loaded()
    ctx.profile_begin(1)
    ctx.sync_steps(idx, batch, steps, lr)                      # one persistent launch
    assert ctx.profile_end()[1] == 1
    assert ctx.debug_timeline().any()
    ctx.eval(n_train, data.n_rows)
    ctx.gradient(idx[:batch], w=w_host)
    ctx.forward(idx[:batch], w=w_host)
    ctx.eval_sampled_counts(0, data.n_rows, 7, 0, 2500)        # >= 2048 rows: the streaming pass
    ctx.close()


def async_cycle():
    ctx = loaded(is_async=True)
    ctx.async_outbox_enable()
    ctx.async_host_master(w_host)
    ctx.start_async(w_host, np.arange(n_train, dtype=np.int32), batch=8, lr=lr, concurrency=16, max_updates=200)
    ctx.stop_async()
    ctx.update_grad(np.arange(5000, dtype=np.int32), np.full(5000, 1e-3))
    ctx.close()


def pair_cycle():
    ctxs = [loaded(rank=r, world=2) for r in range(2)]
    for c in ctxs:
        c.set_grid_limit(sms // 2)
        c.reserve(batch * steps, steps)
    ctxs[0].xchg_attach(1, ctxs[1])
    ctxs[1].xchg_attach(0, ctxs[0])
    errs = []

    def run(c):
        try:
            c.set_weights(w_host)
            c.sync_steps(idx, batch, steps, lr)
        except Exception as e:  # noqa: BLE001 -- reported below
            errs.append(e)

    th = [threading.Thread(target=run, args=(c,)) for c in ctxs]
    for t in th:
        t.start()
    for t in th:
        t.join(timeout=120)
    for c in ctxs:
        c.close()
    assert not errs, errs


sync_cycle(); async_cycle(); pair_cycle()                        # modules loaded, allocator warm
free0 = torch.cuda.mem_get_info()[0]
for _ in range(200):
    sync_cycle()
for _ in range(5):
    async_cycle()
for _ in range(3):
    pair_cycle()
free1 = torch.cuda.mem_get_info()[0]
print(f"free device memory: {free0} before, {free1} after, {free0 - free1} bytes not returned")
assert free0 - free1 <= 2 << 20, free0 - free1
"""


def test_destroyed_contexts_return_their_device_memory():
    env = dict(os.environ, DSGD_PERSIST_TIMELINE="1")
    cmd = [sys.executable] + (["-s"] if sys.flags.no_user_site else []) + ["-c", _CHILD, ROOT]
    r = subprocess.run(cmd, env=env, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stdout + r.stderr
