"""SparseLogistic's loss sums and gradients checked exactly (tests/loss_sum_model.py states the loss sum's semantics).

a. A one-row evaluation returns exactly R(v) for the device's softplus value v: these per-row values are the ground truth
   of every pass sum below, whatever CUDA's exp / log1p give in the last ulp (checked against the oracle only loosely).
b. Passes of every size and form (range, list, reversed, shuffled, with repeats, device-drawn sample) against the exact sum
   of the per-row values, within one ulp; every form of one multiset gives the same bits.
c. Planted losses: with x = 1, y = +1 and |z| >= 800, softplus(z) is z or 0 exactly, so limb edges, carries, the largest
   summed value, the NaN rule and the 2^-160 resolution are planted exactly.
d. Passes whose limb words would pass 2^64: 2^25 repeats of one row, and 4097 values just below 2^52.
e. Step losses against an evaluation of the same ids at the same weights (one worker, and virtual workers whose sums are
   folded in fp64).
f. Dyadic rows whose sigma is 1/2, 1 or 0: gradients and whole trajectories bit for bit against LogisticOracle.
"""
import math
import os
import socket
import sys
from fractions import Fraction

import numpy as np
import pytest

from loss_sum_model import MAX_VALUE, R, describe, exact_sum, r_units, within_one_ulp

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LAM = 1e-5
N_BIG = 100_000
UNIT = 2.0 ** -160


def _sm_count():
    from distributed_sgd_b200.native import NativeCtx
    with NativeCtx(0, 16, 0.1) as c:
        return int(c.info()["sm_count"])


@pytest.fixture(scope="module")
def sm():
    return _sm_count()


def _row_values(ctx, n):
    """Per-row device losses R(v_r) of rows [0, n) at the resident weights, from one-row evaluations."""
    out = np.empty(n)
    for r in range(n):
        out[r] = ctx.eval_samples_sums(np.array([r], np.int32))[0]
    return out


@pytest.fixture(scope="module")
def big():
    """A realistic synthetic set, its oracle, two weight vectors (unit scale; scales spread over 10^-1.5 .. 10^3, whose
    losses run from below 2^-161 to above 10^3) and the per-row device losses at each."""
    from distributed_sgd_b200.native import NativeCtx
    from distributed_sgd_b200.utils import synthetic_rcv1
    from oracle.logistic import LogisticOracle
    data = synthetic_rcv1(n_rows=N_BIG, seed=31)
    ctx = NativeCtx(0, data.dim, LAM, logistic=True)
    ctx.load_csr(data.row_ptr, data.col, data.val, data.label)
    d = ctx.compute_dim_sparsity(N_BIG)
    orc = LogisticOracle(data.row_ptr, data.col, data.val, data.label, data.dim, LAM)
    orc.set_dim_sparsity(d)
    rng = np.random.default_rng(5)
    weights = {
        "wide": rng.standard_normal(data.dim) * 10.0 ** rng.uniform(-1.5, 3.0, data.dim),
        "unit": np.where(rng.random(data.dim) < 0.3, 0.5 * rng.standard_normal(data.dim), 0.0),
    }
    rows = {"wide": N_BIG, "unit": 2048}
    vals, units = {}, {}
    for name, w in weights.items():
        ctx.set_weights(w)
        vals[name] = _row_values(ctx, rows[name])
        units[name] = np.array([r_units(v) for v in vals[name]], dtype=object)
    yield dict(data=data, ctx=ctx, orc=orc, w=weights, vals=vals, units=units)
    ctx.close()


def _exact(units, ids):
    """Exact sum of the per-row values of `ids` (every occurrence), from their units of 2^-160."""
    return Fraction(int(units[np.asarray(ids)].sum()), 1 << 160)


def _rounding_scale(data, w, n):
    """Per row of [0, n): nnz * sum_j |x_j w_j|, the scale of the fp64 dot's rounding differences (rows are not empty)."""
    end = int(data.row_ptr[n])
    a = np.abs(data.val[:end].astype(np.float64) * w[data.col[:end]])
    return np.add.reduceat(a, data.row_ptr[:n]) * np.diff(data.row_ptr[:n + 1])


# ---- a. per-row device losses ---------------------------------------------------------------------------------------------

@pytest.mark.parametrize("name", ["wide", "unit"])
def test_one_row_sums_are_exact_limb_values(big, name):
    data, orc, w, v = big["data"], big["orc"], big["w"][name], big["vals"][name]
    n = len(v)
    # a single value's limbs convert back without rounding: every one-row sum is a multiple of 2^-160 and its own R
    assert all(R(x) == x for x in v.tolist())
    ref = orc.sample_losses(w, begin=0, n=n)
    # sanity only: the oracle's softplus, with the dot's rounding (slope sigma <= 1.5 softplus) and half a unit of R
    tol = ref * (1e-12 + 1.5 * 2.0 ** -53 * _rounding_scale(data, w, n)) + 2.0 ** -161
    bad = np.flatnonzero(~(np.abs(v - ref) <= tol))
    assert bad.size == 0, f"row {bad[0]}: device {v[bad[0]]!r}, oracle {ref[bad[0]]!r}"
    if name == "wide":
        # the values cover every limb: from below the resolution to above 10^3
        u = big["units"][name]
        assert (v == 0).any() and v.max() > 1e3
        for k in range(5):
            assert any((int(x) >> (40 * k)) & ((1 << 40) - 1) for x in u), f"no value has bits in limb {k}"


# ---- b. pass sums against the exact model ----------------------------------------------------------------------------------

def _sizes(sm):
    return [1, 2, 7, 8, 9, 64 * sm - 1, 64 * sm, 64 * sm + 1, 2047, 2048, N_BIG]


@pytest.mark.parametrize("name", ["wide", "unit"])
def test_pass_sums_are_exact_in_every_form(big, sm, name):
    from distributed_sgd_b200.native import host_lib
    data, ctx, orc, w = big["data"], big["ctx"], big["orc"], big["w"][name]
    units = big["units"][name]
    ctx.set_weights(w)
    rng = np.random.default_rng(17)
    for n in _sizes(sm):
        if n > len(units):
            continue
        ids = np.arange(n, dtype=np.int32)
        ex = _exact(units, ids)
        key = 0x5EED0000 + n
        drawn = np.fromiter((host_lib().dsgd_feistel_pos(p, n, key) for p in range(n)), dtype=np.int32, count=n)
        assert np.array_equal(np.sort(drawn), ids)
        forms = {
            "range": ctx.eval_sums(0, n),
            "list": ctx.eval_samples_sums(ids),
            "reversed": ctx.eval_samples_sums(ids[::-1].copy()),
            "shuffled": ctx.eval_samples_sums(rng.permutation(ids)),
            "sample": ctx.eval_sampled_sums(0, n, key, 0, n),
            "drawn list": ctx.eval_samples_sums(drawn),
        }
        s0, c0, _ = forms["range"]
        assert within_one_ulp(s0, ex), f"n={n}: " + describe(s0, ex)
        for form, (s, c, _) in forms.items():
            assert s == s0 and c == c0, f"n={n}, {form}: {s!r} / {c} against the range's {s0!r} / {c0}"
        assert c0 == round(orc.loss_acc(w, begin=0, n=n)[1] * n)
        # repeats: every occurrence counts; the same multiset in another order gives the same bits
        rep = rng.integers(0, n, size=n + 5).astype(np.int32)
        ex_rep = _exact(units, rep)
        s_rep, c_rep, _ = ctx.eval_samples_sums(rep)
        assert within_one_ulp(s_rep, ex_rep), f"n={n} with repeats: " + describe(s_rep, ex_rep)
        s_rep2, c_rep2, _ = ctx.eval_samples_sums(rng.permutation(rep))
        assert s_rep2 == s_rep and c_rep2 == c_rep
        assert c_rep == round(orc.loss_acc(w, idx=rep)[1] * len(rep))
        # part of a device-drawn sample of a larger range: the host reproduces the ids
        if n < len(units):
            m, k = len(units), min(n, 3001)
            part = np.fromiter((host_lib().dsgd_feistel_pos(p, m, key) for p in range(k)), dtype=np.int64, count=k)
            s_part = ctx.eval_sampled_sums(0, m, key, 0, k)[0]
            ex_part = _exact(units, part)
            assert within_one_ulp(s_part, ex_part), f"sample {k} of {m}: " + describe(s_part, ex_part)
            assert ctx.eval_samples_sums(part.astype(np.int32))[0] == s_part


# ---- c. planted limb edges -------------------------------------------------------------------------------------------------

NAN_ROW = "nan"   # a row with two columns at weights +inf and -inf: its dot is NaN
Z_RES_IN = math.log(0.9) - 160 * math.log(2.0)    # loss ~0.9 units of 2^-160: R = 2^-160
Z_RES_OUT = math.log(0.3) - 160 * math.log(2.0)   # loss ~0.3 units: R = 0


def _planted_ctx(zs):
    """One row per entry, x = 1 and y = +1 on the row's own column(s), weights such that z = the entry."""
    from distributed_sgd_b200.native import NativeCtx
    from oracle.logistic import LogisticOracle
    rp, col, w = [0], [], []
    for z in zs:
        if isinstance(z, str):
            col += [len(w), len(w) + 1]
            w += [math.inf, -math.inf]
        else:
            col.append(len(w))
            w.append(float(z))
        rp.append(len(col))
    dim = max(len(w), 2)
    w = np.array(w + [0.0] * (dim - len(w)))
    rp, col = np.array(rp, np.int64), np.array(col, np.int32)
    val, lab = np.ones(len(col), np.float32), np.ones(len(zs), np.int8)
    ctx = NativeCtx(0, dim, LAM, logistic=True)
    ctx.load_csr(rp, col, val, lab)
    ctx.set_dim_sparsity(np.zeros(dim))
    return ctx, LogisticOracle(rp, col, val, lab, dim, LAM), w


def _planted_value(z):
    """The exact per-row loss the device must report for a planted z."""
    if isinstance(z, str) or not z < MAX_VALUE:
        return math.nan
    if z >= 800.0:
        return z
    if z <= -800.0 or z == Z_RES_OUT or z < -112.0:
        return 0.0
    assert z == Z_RES_IN
    return UNIT


LIMB3_ONES = 1025.0 - 2.0 ** -40   # fraction bits 2^-1 .. 2^-40 all set
TOP = MAX_VALUE - 0.5              # the largest value that is summed
PLANTED = {
    "limb3 all ones": [LIMB3_ONES],
    "limb3 zero": [1024.0, 2.0 ** 40, 2.0 ** 45 + 3.0],
    "carry out of limb 3": [LIMB3_ONES] * 3 + [1024.0 + 2.0 ** -40],
    "carry across the integer split": [2.0 ** 40 - 2.0 ** -12] * 5 + [2.0 ** 41 + 0.75, 2.0 ** 40 + 2.0 ** -12],
    "largest value": [TOP],
    "largest value twice": [TOP, TOP],
    "carries the reader needs": [TOP, TOP, MAX_VALUE - 1.0],
    "carries the reader needs, below the top": [3.0 * 2.0 ** 50 - 0.5] * 2 + [MAX_VALUE - 1.0],
    "largest and smallest": [TOP, Z_RES_IN, LIMB3_ONES, -1000.0, 800.0],
    "2^52": [1024.0, MAX_VALUE],
    "+inf": [1024.0, math.inf],
    "nan row": [LIMB3_ONES, NAN_ROW, 2048.0],
    "nan rows and negative margins": [NAN_ROW, -1000.0, NAN_ROW, -900.0, 1e6],
    "below the resolution": [-200.0] * 1000,
    "resolution": [Z_RES_IN] * 1000 + [Z_RES_OUT] * 1000,
    "resolution one row": [Z_RES_IN],
    "just below the resolution": [Z_RES_OUT],
}


@pytest.mark.parametrize("case", list(PLANTED))
def test_planted_sums(case):
    zs = PLANTED[case]
    ctx, orc, w = _planted_ctx(zs)
    try:
        ctx.set_weights(w)
        n = len(zs)
        for r, z in enumerate(zs[:8]):
            got, want = ctx.eval_samples_sums([r])[0], _planted_value(z)
            assert got == want or (math.isnan(got) and math.isnan(want)), f"row {r} (z = {z!r}): {got!r}, want {want!r}"
        ex = exact_sum([_planted_value(z) for z in zs])
        ids = np.arange(n, dtype=np.int32)
        forms = [ctx.eval_sums(0, n), ctx.eval_samples_sums(ids[::-1].copy()),
                 ctx.eval_samples_sums(np.random.default_rng(n).permutation(ids))]
        correct = round(orc.loss_acc(w, begin=0, n=n)[1] * n)
        for s, c, _ in forms:
            assert within_one_ulp(s, ex), f"{case}: " + describe(s, ex)
            assert c == correct
        # a double-sized list of the same rows: every occurrence counts
        s2 = ctx.eval_samples_sums(np.concatenate([ids, ids]))[0]
        ex2 = None if ex is None else 2 * ex
        assert within_one_ulp(s2, ex2), f"{case}, twice: " + describe(s2, ex2)
    finally:
        ctx.close()


# ---- d. the wraps ----------------------------------------------------------------------------------------------------------

def test_many_repeats_of_one_row():
    """2^25 ids of one row with loss log1p(1): 2^25 * 2^40 passed 2^64 in a limb word."""
    ctx, _, _ = _planted_ctx([0.0])
    try:
        ctx.set_weights(np.zeros(2))
        v = ctx.eval_samples_sums([0])[0]
        assert abs(v - math.log(2.0)) <= 2.3e-16 * math.log(2.0)
        n = 1 << 25
        ids = np.zeros(n, dtype=np.int32)
        s, c, _ = ctx.eval_samples_sums(ids)
        del ids
        ex = exact_sum([v], repeat=n)
        assert float(ex) == ex                                   # a power-of-two multiple: the sum is a double
        assert within_one_ulp(s, ex), describe(s, ex)
        assert c == 0
    finally:
        ctx.close()


def test_values_just_below_2_52():
    """4097 values of 2^52 - 1: the sum of the integer parts passes 2^63 (and 2^64)."""
    big = MAX_VALUE - 1.0
    ctx, _, w = _planted_ctx([big] * 4097)
    try:
        ctx.set_weights(w)
        ex = exact_sum([big], repeat=4097)
        for s, _, _ in (ctx.eval_sums(0, 4097), ctx.eval_samples_sums(np.zeros(4097, np.int32)),
                        ctx.eval_samples_sums(np.arange(4096, -1, -1, dtype=np.int32))):
            assert within_one_ulp(s, ex), describe(s, ex)
        s = ctx.eval_sums(0, 4096)[0]
        assert within_one_ulp(s, exact_sum([big], repeat=4096)), describe(s, exact_sum([big], repeat=4096))
    finally:
        ctx.close()


# ---- e. step losses --------------------------------------------------------------------------------------------------------

def _ulps(a, b):
    return abs(a - b) / math.ulp(b)


@pytest.mark.parametrize("counts", [[1], [64], [2048], [40, 24], [50, 31, 7]])
def test_step_loss_matches_the_evaluation(big, counts):
    """A step reports lambda ||w||^2 + S / n for the sum S an evaluation of the same ids gives at the same weights; the
    virtual workers' sums are folded in fp64 in worker order."""
    ctx, w = big["ctx"], big["w"]["wide"]
    tot = sum(counts)
    rng = np.random.default_rng(tot)
    ctx.set_weights(w * 1e-2)
    ctx.set_workers(counts, len(counts))
    try:
        for _ in range(3):
            ids = rng.choice(N_BIG, size=tot, replace=False).astype(np.int32)
            fold, off = 0.0, 0
            for k, nk in enumerate(counts):
                s, _, n2 = ctx.eval_samples_sums(ids[off:off + nk])
                fold = s if k == 0 else fold + s
                off += nk
            want = LAM * n2 + fold / tot
            got = ctx.sync_steps(ids, tot, 1, 0.25)[0]
            assert _ulps(got, want) <= 2.0, f"{got!r} against {want!r}"
    finally:
        ctx.set_workers([], 0)


# ---- f. dyadic gradients and trajectories ----------------------------------------------------------------------------------

LAM_D = 2.0 ** -10
LR_D = 2.0 ** -6
BIAS = 2048.0
TINY_X = 2.0 ** -66   # passes the value filter; times sigma = 1/2 it falls below 1e-20


def _dyadic_data(n_rows, dim, seed, with_half):
    """Rows whose sigma is exactly 1/2 (all weights 0: z = 0), 1 (a bias column at +-BIAS: z = BIAS) or 0 (z = -BIAS, the
    row is dropped).  Every row has columns 0 and dim - 1; values are multiples of 1/2 up to 2, so every sum is exact.
    Returns (data, w, d): only the bias columns have weights, and d is 2^-3 on the column of the sigma = 0 rows with y = +1
    only, so that c = 2 lambda (w . d) = -0.5 is exact and stays constant."""
    from helpers import data_from_csr
    rng = np.random.default_rng(seed)
    b_pos, b_neg, c_pos, c_neg, tiny = dim - 5, dim - 4, dim - 3, dim - 2, 1
    rp, col, val, lab = [0], [], [], []
    for _ in range(n_rows):
        y = int(rng.choice([-1, 1]))
        cls = int(rng.integers(0 if with_half else 1, 3))        # 0: sigma 1/2, 1: sigma 1, 2: sigma 0
        cols = {0, dim - 1} | set(rng.integers(2, dim - 5, size=int(rng.integers(1, 7))).tolist())
        special = {}
        if cls == 1:
            special[b_pos if y > 0 else b_neg] = 1.0
        elif cls == 2:
            special[c_pos if y > 0 else c_neg] = 1.0
        elif rng.random() < 0.5:
            special[tiny] = TINY_X * y                          # x * y * sigma = 2^-67 for every such row
        for c in sorted(cols | set(special)):
            col.append(c)
            val.append(special.get(c, float(rng.choice([-2.0, -1.5, -1.0, -0.5, 0.5, 1.0, 1.5, 2.0]))))
        rp.append(len(col))
        lab.append(y)
    w = np.zeros(dim)
    w[b_pos], w[b_neg], w[c_pos], w[c_neg] = BIAS, -BIAS, -BIAS, BIAS
    d = np.zeros(dim)
    d[c_pos] = 2.0 ** -3
    return data_from_csr(rp, col, val, lab, dim), w, d


@pytest.fixture(scope="module")
def dyadic(sm):
    from distributed_sgd_b200.native import NativeCtx
    from oracle.logistic import LogisticOracle
    data, w, d = _dyadic_data(max(64 * sm + 600, 6000), 700, 3, with_half=True)
    ctx = NativeCtx(0, data.dim, LAM_D, logistic=True)
    ctx.load_csr(data.row_ptr, data.col, data.val, data.label)
    ctx.set_dim_sparsity(d)
    orc = LogisticOracle(data.row_ptr, data.col, data.val, data.label, data.dim, LAM_D)
    orc.set_dim_sparsity(d)
    yield data, ctx, orc, w
    ctx.close()


def test_dyadic_rows_have_the_planned_sigmas(dyadic):
    data, ctx, orc, w = dyadic
    z = data.label.astype(np.float64) * np.array([float(np.dot(data.val[a:b].astype(np.float64), w[data.col[a:b]]))
                                                 for a, b in zip(data.row_ptr[:-1], data.row_ptr[1:])])
    assert set(np.unique(z).tolist()) == {0.0, BIAS, -BIAS}
    assert (np.abs(data.val) == TINY_X).any()


def _grad_sizes(sm):
    return [1, 7, 64 * sm - 1, 64 * sm + 1, 2048, 5000]


@pytest.mark.parametrize("which", range(6))
@pytest.mark.parametrize("resident", [False, True])
def test_dyadic_gradient_bit_for_bit(dyadic, sm, which, resident):
    data, ctx, orc, w = dyadic
    n = _grad_sizes(sm)[which]
    idx = np.random.default_rng(n).choice(data.n_rows, size=n, replace=False).astype(np.int32)
    if resident:
        ctx.set_weights(w)
        g = ctx.gradient(idx)
    else:
        g = ctx.gradient(idx, w)
    g_ref, c = orc.gradient(w, idx)
    assert c == -0.5
    assert np.array_equal(g == 0, g_ref == 0), "gradient support differs"
    diff = np.flatnonzero(g != g_ref)
    assert diff.size == 0, f"column {diff[0]}: {g[diff[0]]!r} against {g_ref[diff[0]]!r}"


@pytest.fixture(scope="module")
def dyadic_run():
    """Rows of sigma 1 and 0 only: every row keeps |z| >= 800 for the whole run, so trajectories stay dyadic."""
    from distributed_sgd_b200.native import NativeCtx
    from oracle.logistic import LogisticOracle
    data, w, d = _dyadic_data(4000, 500, 4, with_half=False)
    ctx = NativeCtx(0, data.dim, LAM_D, logistic=True)
    ctx.load_csr(data.row_ptr, data.col, data.val, data.label)
    ctx.set_dim_sparsity(d)
    orc = LogisticOracle(data.row_ptr, data.col, data.val, data.label, data.dim, LAM_D)
    orc.set_dim_sparsity(d)
    yield data, ctx, orc, w
    ctx.close()


@pytest.mark.parametrize("counts", [[64], [1], [32, 32], [16, 8, 24, 16]])
def test_dyadic_trajectory_bit_for_bit(dyadic_run, counts):
    data, ctx, orc, w0 = dyadic_run
    steps, tot = 20, sum(counts)
    rng = np.random.default_rng(tot + len(counts))
    idx = np.concatenate([rng.choice(data.n_rows, size=tot, replace=False) for _ in range(steps)]).astype(np.int32)
    ctx.set_weights(w0)
    ctx.set_workers(counts, len(counts))
    try:
        losses = ctx.sync_steps(idx, tot, steps, LR_D)
    finally:
        ctx.set_workers([], 0)
    w_ref, losses_ref = orc.sync_steps(w0, idx, counts, LR_D, n_steps=steps)
    w = ctx.get_weights()
    z = data.label * np.array([float(np.dot(data.val[a:b].astype(np.float64), w_ref[data.col[a:b]]))
                               for a, b in zip(data.row_ptr[:-1], data.row_ptr[1:])])
    assert (np.abs(z) >= 800.0).all()                           # the run stayed where sigma is 0 or 1
    assert np.array_equal(losses, losses_ref), np.flatnonzero(losses != losses_ref)
    diff = np.flatnonzero(w != w_ref)
    assert diff.size == 0, f"column {diff[0]}: {w[diff[0]]!r} against {w_ref[diff[0]]!r}"


def _free_port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def _dyadic_worker(rank, world, port, q):
    sys.path.insert(0, ROOT)
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    import torch
    import torch.distributed as dist
    from distributed_sgd_b200.core import Group
    from distributed_sgd_b200.native import NativeCtx
    from oracle.logistic import LogisticOracle

    torch.cuda.set_device(rank)
    dist.init_process_group("gloo", init_method=f"tcp://127.0.0.1:{port}", rank=rank, world_size=world)
    group = Group()
    data, w0, d = _dyadic_data(4000, 500, 4, with_half=False)
    batch, steps = 48, 20
    ctx = NativeCtx(rank, data.dim, LAM_D, rank=rank, world=world, logistic=True)
    ctx.load_csr(data.row_ptr, data.col, data.val, data.label)
    ctx.set_dim_sparsity(d)
    uid = NativeCtx.comm_unique_id() if rank == 0 else b""
    ctx.comm_init(group.broadcast_bytes(uid, 0))
    rng = np.random.default_rng(9)
    per = data.n_rows // world
    idx = np.stack([np.concatenate([k * per + rng.choice(per, size=batch, replace=False) for k in range(world)])
                    for _ in range(steps)]).astype(np.int32)
    mine = idx.reshape(steps, world, batch)[:, rank, :]
    ctx.set_weights(w0)
    losses = ctx.sync_steps(mine.reshape(-1), batch, steps, LR_D)
    w = ctx.get_weights()
    orc = LogisticOracle(data.row_ptr, data.col, data.val, data.label, data.dim, LAM_D)
    orc.set_dim_sparsity(d)
    w_ref, losses_ref = orc.sync_steps(w0, idx.reshape(-1), [batch] * world, LR_D, n_steps=steps)
    q.put((rank, bool(np.array_equal(losses, losses_ref)), bool(np.array_equal(w, w_ref))))
    ctx.close()
    dist.destroy_process_group()


def test_two_gpu_nccl_dyadic_trajectory_bit_for_bit():
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    import torch.multiprocessing as mp
    ctxmp = mp.get_context("spawn")
    q = ctxmp.Queue()
    port = _free_port()
    procs = [ctxmp.Process(target=_dyadic_worker, args=(r, 2, port, q)) for r in range(2)]
    for p in procs:
        p.start()
    res = [q.get(timeout=300) for _ in procs]
    for p in procs:
        p.join(timeout=60)
    for rank, same_losses, same_w in res:
        assert same_losses, f"rank {rank}: step losses differ from the oracle"
        assert same_w, f"rank {rank}: weights differ from the oracle"
