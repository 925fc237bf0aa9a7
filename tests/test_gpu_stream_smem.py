"""The streaming pass's shared-memory bound belongs to the kernel, not to a context: plain contexts of two dims in one process,
the smaller one set up after the larger one has streamed, both keep streaming (each pass over 4 096 rows takes k_stream_rows)
and give the counts of the fp64 row kernel."""
import numpy as np
import pytest

from helpers import data_from_csr

pytestmark = pytest.mark.gpu


def _ctx(dim, seed, n=4096):
    from distributed_sgd_b200.native import NativeCtx
    rng = np.random.default_rng(seed)
    lens = rng.integers(1, 9, size=n)
    rp = np.concatenate([[0], np.cumsum(lens)]).astype(np.int64)
    col = np.concatenate([np.sort(rng.choice(dim, size=k, replace=False)) for k in lens]).astype(np.int32)
    val = (rng.integers(1, 257, size=rp[-1]) / 64.0).astype(np.float32)
    lab = rng.choice(np.array([-1, 1], np.int8), size=n)
    data = data_from_csr(rp, col, val, lab, dim)
    ctx = NativeCtx(0, dim, 0.0)
    ctx.load_csr(data.row_ptr, data.col, data.val, data.label)
    ctx.set_dim_sparsity(np.zeros(dim))
    ctx.set_weights(rng.integers(-64, 65, size=dim) / 512.0)
    return ctx


def test_a_smaller_dim_set_up_later_does_not_break_a_larger_ones_streaming_pass():
    big = _ctx(5001, 1)
    first = big.eval_counts(0, 4096)                  # the larger dim streams first
    small = _ctx(700, 2)
    small_counts = small.eval_counts(0, 4096)         # the smaller dim streams after it
    assert big.eval_counts(0, 4096) == first          # and the larger one streams again
    assert small.eval_counts(0, 4096) == small_counts
    for ctx, (h, c, _) in ((big, first), (small, small_counts)):   # three passes below 2 048 rows: the fp64 row kernel
        parts = [ctx.eval_counts(b, e) for b, e in ((0, 2047), (2047, 4094), (4094, 4096))]
        assert (h, c) == (sum(p[0] for p in parts), sum(p[1] for p in parts))
