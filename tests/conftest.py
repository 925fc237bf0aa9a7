import os
import sys

import numpy as np
import pytest

# K ranks share one GPU in tests/test_gpu_fused_one_gpu.py and their kernels must run concurrently: give the device more
# hardware queues than streams (the default is 8; must be set before CUDA initialises)
os.environ.setdefault("CUDA_DEVICE_MAX_CONNECTIONS", "32")

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs an H100 (sm_90a); select with -m gpu")


def random_csr(rng, n_rows, dim, max_nnz=12, min_nnz=1, allow_empty=False, dup_values=False):
    """Small random CSR problem (sorted unique 0-based columns, fp32 values, +/-1 labels)."""
    row_ptr = [0]
    cols, vals = [], []
    for _ in range(n_rows):
        k = int(rng.integers(0 if allow_empty else min_nnz, max_nnz + 1))
        k = min(k, dim)
        c = np.sort(rng.choice(dim, size=k, replace=False))
        if dup_values:
            v = rng.choice(np.array([0.25, 0.5, 1.0], dtype=np.float32), size=k)
        else:
            v = np.abs(rng.standard_normal(k)).astype(np.float32) + np.float32(1e-3)
        cols.extend(c.tolist())
        vals.extend(v.tolist())
        row_ptr.append(len(cols))
    label = rng.choice(np.array([-1, 1], dtype=np.int8), size=n_rows)
    return (np.asarray(row_ptr, dtype=np.int64), np.asarray(cols, dtype=np.int32),
            np.asarray(vals, dtype=np.float32), label.astype(np.int8))


@pytest.fixture
def rng():
    return np.random.default_rng(1234)
