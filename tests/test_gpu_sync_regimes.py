"""The persistent sync step (k_sync_persistent, csrc/dsgd_persistent.cuh) in the regimes random RCV1-shaped rows never
reach, against the fp64 oracle.

A. Grid sweep on one GPU: 1, 2, 7, S/2 + 1 and S CTAs (S = SM count; S both as a plain and as a cooperative launch), batches
   on both sides of G and 32 G (32 G + 1 runs k_rows + k_update<true>), dims around the update threads' register columns
   (U = 192 G: U - 1, 2 U, 2 U + 1) and the RCV1 dim, 20 steps split over two calls without set_weights in between; and one
   run that alternates persistent and fallback batches and grid sizes, against one oracle trajectory.
B. Stage layout: rows of 0 to 2000 non-zeros placed so that a CTA's rows fill the 2560-pair stage exactly, spill from it,
   fill the 128-entry chunk list exactly, or miss it (whole rows from global memory, FetchLocal/FetchLL::get1); empty steps
   and steps in which every row fails the gate.  A Python mirror of the producer's layout checks each case reaches its
   branch.  One GPU at G = 1 and 2, and fused K = 2 on one GPU; dyadic values bit for bit, random fp32 values at tolerance.
C. The 1e-20 filter of the reference's Sparse at every place the step applies it, and D1. the fixed-point accumulator of
   {W.d, ||W||^2} (zero, negative and > 2^40 partials from different CTAs): hand-built dyadic cases through the persistent
   kernel, the fallback, fused K = 2 and two virtual workers (k_finish_acc), weights bit for bit.
D2. Losses of steps whose gradient is empty (loss = lambda ||W||^2) at weight scales down to 1e-16, through every path.
E. Ranks wired with the peer exchange only refuse steps the fused kernel cannot take.

Tolerances (README): losses rtol 1e-12, supports exact, weights rtol 1e-11 / atol 1e-15; bit for bit where the values are
dyadic and every sum is exact.
"""
import numpy as np
import pytest

from helpers import data_from_csr, fused_ranks, make_pair

pytestmark = pytest.mark.gpu

UPD_THREADS = 6 * 32            # update threads per CTA (kPUpd warps); U = UPD_THREADS * G
MAX_ROWS = 32                   # kMaxRowsPerCta: larger batches run k_rows + k_update<true>
CHUNK_PAIRS, MAX_CHUNKS, STAGE_PAIRS = 128, 128, 2560   # kChunkPairs, kPMaxChunks, kPStagePairs
SLICE_MAX = 14 * 32             # K GPUs: columns of one CTA's slice, dim + 1 counter column included
EPS = 1e-20


@pytest.fixture(scope="module")
def S():
    from distributed_sgd_b200.native import NativeCtx
    ctx = NativeCtx(0, 8, 0.0)
    s = int(ctx.info()["sm_count"])
    ctx.close()
    return s


def _csr(rows, labels, dim):
    """rows: list of (cols, vals) in storage order."""
    rp = np.zeros(len(rows) + 1, np.int64)
    rp[1:] = np.cumsum([len(c) for c, _ in rows])
    col = np.concatenate([np.asarray(c, np.int32) for c, _ in rows] + [np.zeros(0, np.int32)])
    val = np.concatenate([np.asarray(v, np.float32) for _, v in rows] + [np.zeros(0, np.float32)])
    return data_from_csr(rp, col, val, np.asarray(labels, np.int8), dim)


def _pair(data, lam, d=None, **kw):
    ctx, orc = make_pair(data, lam, **kw)
    if d is not None:
        ctx.set_dim_sparsity(d)
        orc.set_dim_sparsity(d)
    return ctx, orc


def _check(losses, w, losses_ref, w_ref, what, exact=False):
    if exact:
        np.testing.assert_array_equal(w, w_ref, err_msg=what)
    np.testing.assert_allclose(losses, losses_ref, rtol=1e-12, atol=0, err_msg=what)
    assert np.array_equal(w != 0, w_ref != 0), f"{what}: supports differ"
    np.testing.assert_allclose(w, w_ref, rtol=1e-11, atol=1e-15, err_msg=what)


def _fits_fused(dim, G):
    return ((dim + 1 + G - 1) // G + 31) // 32 * 32 <= SLICE_MAX


# ---- two ranks of the fused exchange on one GPU (helpers.fused_ranks) --------------------------------------------------

def _fused_run(data, lam, d, G, w0, per_rank, lr):
    """per_rank[r]: int32 [steps, batch_r] of rank r.  Runs both ranks in one launch (fused_ranks checks the replicas are
    identical), returns rank 0's (losses, weights)."""
    res = fused_ranks(data, lam, d, [G, G], w0, [(per_rank, None)], lr)
    return res["losses"][0], res["w"][0]


def _fused_oracle(orc, w0, per_rank, lr):
    steps = per_rank[0].shape[0]
    idx = np.concatenate([per_rank[0], per_rank[1]], axis=1)
    return orc.sync_steps(w0, idx.reshape(-1), [per_rank[0].shape[1], per_rank[1].shape[1]], lr, n_steps=steps)


# ---- A. grid sweep --------------------------------------------------------------------------------------------------

def _synth(dim, n_rows, seed):
    from distributed_sgd_b200.utils import synthetic_rcv1
    return synthetic_rcv1(n_rows=n_rows, dim=dim, seed=seed, mean_nnz=min(94.5, dim / 8.0), max_nnz=min(2000, dim // 2))


def _grid(S, name):
    """(grid limit passed to set_grid_limit, CTAs of the launch)."""
    limit = {"G1": 1, "G2": 2, "G7": 7, "half": S // 2 + 1, "S_plain": S, "S_coop": 0}[name]
    return limit, (limit or S)


def _dim(kind, G):
    U = UPD_THREADS * G
    return {"U-1": U - 1, "2U": 2 * U, "2U+1": 2 * U + 1, "rcv1": 47237}[kind]


ALL_DIMS = ["U-1", "2U", "2U+1", "rcv1"]
GRID_CASES = ([("G1", k) for k in ALL_DIMS] + [("G2", "U-1"), ("G2", "2U+1")] + [("G7", k) for k in ALL_DIMS]
              + [("half", "2U+1"), ("S_plain", "2U"), ("S_coop", "2U+1")])
SWEEP_STEPS = (17, 3)           # first call: every one of the 8 stage slots is used at least twice


def _sweep_lr(batch):
    return 0.5 / batch          # the gradient is a sum over the batch: keep lr * batch bounded


@pytest.mark.parametrize("grid,dim_kind", GRID_CASES)
def test_grid_sweep(S, grid, dim_kind):
    limit, G = _grid(S, grid)
    dim = _dim(dim_kind, G)
    batches = sorted({b for b in (1, G - 1, G, G + 1, 32 * G - 1, 32 * G, 32 * G + 1) if b > 0})
    n_rows = 32 * G + 64
    data = _synth(dim, n_rows, seed=1000 * G + dim)
    ctx, orc = make_pair(data, lam=1e-2)
    ctx.set_grid_limit(limit)
    rng = np.random.default_rng(dim + G)
    steps = sum(SWEEP_STEPS)
    try:
        for b in batches:
            lr = _sweep_lr(b)
            idx = np.stack([rng.choice(n_rows, size=b, replace=False) for _ in range(steps)]).astype(np.int32)
            w0 = rng.standard_normal(dim) * (rng.random(dim) < 0.3) * 0.1
            ctx.set_weights(w0)
            a = SWEEP_STEPS[0]
            losses = np.concatenate([ctx.sync_steps(idx[:a].reshape(-1), b, a, lr),
                                     ctx.sync_steps(idx[a:].reshape(-1), b, steps - a, lr)])
            w_ref, losses_ref = orc.sync_steps(w0, idx.reshape(-1), [b], lr, n_steps=steps)
            _check(losses, ctx.get_weights(), losses_ref, w_ref, f"G {G} ({grid}), dim {dim}, batch {b}")
    finally:
        ctx.close()


def test_mixed_sequence(S):
    """Persistent and fallback batches and grid sizes alternate from call to call; the weights stay resident throughout."""
    half = S // 2 + 1
    calls = [(7, 20, 17), (7, 32 * 7 + 1, 3), (2, 64, 17), (0, 100, 5), (1, 33, 2), (half, 32 * half, 17), (0, 32 * S + 1, 2),
             (1, 1, 17)]
    dim, n_rows = 47237, 32 * S + 64
    data = _synth(dim, n_rows, seed=3)
    ctx, orc = make_pair(data, lam=1e-2)
    rng = np.random.default_rng(4)
    w_ref = rng.standard_normal(dim) * (rng.random(dim) < 0.3) * 0.1
    ctx.set_weights(w_ref)
    try:
        for limit, b, n in calls:
            ctx.set_grid_limit(limit)
            lr = _sweep_lr(b)
            idx = np.stack([rng.choice(n_rows, size=b, replace=False) for _ in range(n)]).astype(np.int32).reshape(-1)
            losses = ctx.sync_steps(idx, b, n, lr)
            w_ref, losses_ref = orc.sync_steps(w_ref, idx, [b], lr, n_steps=n)
            np.testing.assert_allclose(losses, losses_ref, rtol=1e-12, atol=0, err_msg=f"limit {limit}, batch {b}")
        w = ctx.get_weights()
        assert np.array_equal(w != 0, w_ref != 0)
        np.testing.assert_allclose(w, w_ref, rtol=1e-11, atol=1e-15)
    finally:
        ctx.close()


# ---- B. stage layout ------------------------------------------------------------------------------------------------

def stage_layout(nnzs):
    """Mirror of the producer's layout of one CTA's rows in a stage (k_sync_persistent, producer warp): pairs (padded to
    even), chunks of 128 pairs, listed while the inclusive chunk prefix fits the 128-entry chunk list, in the shared-memory
    ring while listed and the inclusive pair prefix fits the 2560-pair stage."""
    nnz = np.asarray(nnzs, np.int64)
    pairs = 2 * ((nnz + 1) // 2)
    chunks = (pairs + CHUNK_PAIRS - 1) // CHUNK_PAIRS
    listed = np.cumsum(chunks) <= MAX_CHUNKS
    in_ring = listed & (np.cumsum(pairs) <= STAGE_PAIRS)
    return pairs, chunks, listed, in_ring


STAGE_CASES = {   # non-zeros of one CTA's rows, in row order
    "lengths": [0, 1, 2, 127, 128, 129, 255, 256, 257, 2000],
    "lengths_reversed": [2000, 257, 256, 255, 129, 128, 127, 2, 1, 0],
    "ring_2560": [2000, 558, 2],
    "ring_2562": [2000, 558, 2, 2],
    "chunks_128": [1024] * 16,
    "chunks_129": [1024] * 16 + [1],
    "unlisted": [1024] * 16 + [300, 0, 5, 129],
    "all_empty": [0] * 9,
    "gate_fails": [40] * 12,
}
STAGE_BRANCH = {   # what each case is built to reach, on the mirror
    "lengths": lambda p, c, l, r: l.all() and (r & (c > 1)).any() and (l & ~r & (c > 0)).any(),
    "lengths_reversed": lambda p, c, l, r: l.all() and (r & (c > 1)).any() and (l & ~r & (c > 0)).sum() >= 3,
    "ring_2560": lambda p, c, l, r: p.sum() == STAGE_PAIRS and r.all(),
    "ring_2562": lambda p, c, l, r: p.sum() == STAGE_PAIRS + 2 and r[:-1].all() and l[-1] and not r[-1],
    "chunks_128": lambda p, c, l, r: c.sum() == MAX_CHUNKS and l.all(),
    "chunks_129": lambda p, c, l, r: c.sum() == MAX_CHUNKS + 1 and l[:-1].all() and not l[-1],
    "unlisted": lambda p, c, l, r: (~l).sum() >= 3 and (~l & (p == 0)).any() and (~l & (c > 1)).any(),
    "all_empty": lambda p, c, l, r: (c == 0).all(),
    "gate_fails": lambda p, c, l, r: l.all() and r.all(),
}
STAGE_DIM = 2047                # fused K = 2 at 5 CTAs per rank: slices of 416 columns fit the 448 column threads
STAGE_STEPS = 3
STAGE_PATHS = {"one_gpu_G1": (1, 1), "one_gpu_G2": (2, 1), "fused_K2_G5": (5, 2)}   # (CTAs per rank, ranks)
STAGE_INSTANCES = 5 * 2 * STAGE_STEPS


def test_stage_cases_reach_their_branch():
    for name, nnzs in STAGE_CASES.items():
        assert STAGE_BRANCH[name](*stage_layout(nnzs)), name


@pytest.fixture(scope="module", params=["dyadic", "fp32"])
def stage_data(request):
    """Every case of STAGE_CASES STAGE_INSTANCES times over (fresh columns and values each time).  Weights are positive on
    every column and values positive, so a row's dot is positive: y = +1 rows pass the gate, y = -1 rows (all of
    "gate_fails") fail it."""
    dyadic = request.param == "dyadic"
    rng = np.random.default_rng(17 if dyadic else 18)
    rows, labels, inst = [], [], {}
    for name, nnzs in STAGE_CASES.items():
        inst[name] = []
        for _ in range(STAGE_INSTANCES):
            ids = []
            for n in nnzs:
                cols = rng.choice(STAGE_DIM, size=n, replace=False)
                vals = rng.integers(1, 1025, size=n) / 256.0 if dyadic else rng.random(n) * 2.0 + 1e-3
                ids.append(len(rows))
                rows.append((cols, vals))
                labels.append(-1 if name == "gate_fails" else int(rng.choice([-1, 1])))
            inst[name].append(ids)
    w0 = (rng.integers(1, 257, size=STAGE_DIM) / 64.0) if dyadic else (rng.random(STAGE_DIM) + 0.05)
    return _csr(rows, labels, STAGE_DIM), inst, w0, dyadic


def _stage_steps(inst, G, rank):
    """[steps, G * n] sample ids: CTA b of the launch owns step positions b + m * G, and gets instance m-th row of its own
    instance of the case."""
    out = []
    for s in range(STAGE_STEPS):
        ctas = [inst[(s * 2 + rank) * 5 + b] for b in range(G)]
        out.append([ctas[i % G][i // G] for i in range(G * len(ctas[0]))])
    return np.asarray(out, np.int32)


@pytest.mark.parametrize("path", list(STAGE_PATHS))
def test_stage_layout(stage_data, path):
    data, inst, w0, dyadic = stage_data
    G, K = STAGE_PATHS[path]
    lam, lr = (0.0, 2.0 ** -6) if dyadic else (1e-3, 2.0 ** -6)
    failures = []
    ctx = orc = None
    if K == 1:
        ctx, orc = make_pair(data, lam)
        ctx.set_grid_limit(G)
    else:
        _, orc = make_pair(data, lam)
    try:
        for name, nnzs in STAGE_CASES.items():
            assert STAGE_BRANCH[name](*stage_layout(nnzs)), name
            what = f"{path}, {'dyadic' if dyadic else 'fp32'} values, case {name}"
            if K == 1:
                idx = _stage_steps(inst[name], G, 0)
                ctx.set_weights(w0)
                losses = ctx.sync_steps(idx.reshape(-1), idx.shape[1], STAGE_STEPS, lr)
                w = ctx.get_weights()
                w_ref, losses_ref = orc.sync_steps(w0, idx.reshape(-1), [idx.shape[1]], lr, n_steps=STAGE_STEPS)
            else:
                per_rank = [_stage_steps(inst[name], G, r) for r in range(K)]
                losses, w = _fused_run(data, lam, None, G, w0, per_rank, lr)
                w_ref, losses_ref = _fused_oracle(orc, w0, per_rank, lr)
            try:
                if name in ("all_empty", "gate_fails"):
                    np.testing.assert_array_equal(w_ref, w0)      # nothing to scatter: the weights do not move
                    hinge = 1.0 if name == "all_empty" else 0.0
                    np.testing.assert_allclose(losses_ref, lam * np.sum(w0 * w0) + hinge, rtol=1e-13)
                else:
                    assert np.count_nonzero(w_ref != w0) > 0, "the case moved no weight"
                _check(losses, w, losses_ref, w_ref, what, exact=dyadic)
                if dyadic:
                    np.testing.assert_array_equal(losses, losses_ref, err_msg=what)
            except AssertionError as e:
                failures.append(f"{name}: {e}")
    finally:
        if ctx is not None:
            ctx.close()
    assert not failures, "\n".join(failures)


# ---- C / D1. the 1e-20 filter and the fixed-point accumulator, hand-built --------------------------------------------

def _hand_case(name):
    """dict(rows=[(cols, vals, y)], workers=(ids of worker 0, ids of worker 1), single=ids of the one-worker batch, dim, d,
    lam, lr, w0, expect={col: w after one step} with one worker, expect2=... with two workers)."""
    c = dict(dim=64, lam=0.0, lr=1.0, expect2=None)
    dim = 400 if name.startswith("wd_") else 64
    c["dim"] = dim
    w0, d = np.zeros(dim), np.zeros(dim)
    c["w0"], c["d"] = w0, d
    one = dict(workers=([0], [0]), single=[0])
    if name == "residual":              # w - step = 2^-72 ~ 2.1e-22 must become 0
        w0[3] = 2.0 ** -20 + 2.0 ** -72
        c.update(rows=[([3], [2.0 ** -20], 1)], expect={3: 0.0}, **one)
    elif name == "tiny_step":           # mean * lr = 2^-70 <= 1e-20 on column 1: no update there
        w0[1] = 1.0
        c.update(rows=[([1, 2], [2.0 ** -40, 1.0], 1)], lr=2.0 ** -30, expect={1: 1.0, 2: -(2.0 ** -30)}, **one)
    elif name == "tiny_mean":           # two workers: s = 2^-66 on column 4, s / 2 = 2^-67 <= 1e-20: no update there
        w0[4], w0[5] = 2.0 ** -40, 1.0
        c.update(rows=[([4], [2.0 ** -66], 1), ([5], [0.5], 1)], workers=([0], [1]), single=[0, 1],
                 expect={4: 2.0 ** -40 - 2.0 ** -66, 5: 0.5}, expect2={4: 2.0 ** -40, 5: 0.75})
    elif name in ("c_at_eps", "c_above_eps"):   # W.d = 1, lambda = 1e-20 / 2: c = 1e-20 exactly (not added), or one ulp above
        w0[0], d[0] = 1.0, 1.0
        lam = EPS / 2 if name == "c_at_eps" else np.nextafter(EPS / 2, 1.0)
        c.update(rows=[([4], [2.0 ** -66], 1)], lam=lam, **one,
                 expect={4: -(2.0 ** -66)} if name == "c_at_eps" else {4: -(2.0 ** -66 + np.nextafter(EPS, 1.0))})
    elif name == "g_plus_c":            # c = -(2^-40 - 2^-80): g + c = 2^-80 <= 1e-20 on column 1, the key is absent
        w0[0], d[0] = -(1.0 - 2.0 ** -40), 1.0
        cc = -(2.0 ** -40 - 2.0 ** -80)
        c.update(rows=[([1, 6], [2.0 ** -40, 0.5], 1)], lam=2.0 ** -41, lr=2.0 ** 20, **one,   # unfiltered: w1 = -2^-60
                 expect={1: 0.0, 6: -((0.5 + cc) * 2.0 ** 20)})
    elif name == "tiny_products":       # w.d = 2^-80 dropped from c (lambda 2^40 would make c = 2^-39); x.w = 2^-80 dropped
        w0[0], d[0], w0[2] = 2.0 ** -40, 2.0 ** -40, 2.0 ** -40      # from the dot: dot 0, the y = -1 row passes the gate
        c.update(rows=[([2, 5], [2.0 ** -40, 0.5], -1)], lam=2.0 ** 40, expect={2: 2.0 ** -39, 5: 0.5}, **one)
    elif name == "tiny_value":          # x = 2^-70 <= 1e-20 is absent: dot 0 (not 2^-46), the y = -1 row passes the gate
        w0[1] = 2.0 ** 24
        c.update(rows=[([1, 5], [2.0 ** -70, 0.5], -1)], expect={1: 2.0 ** 24, 5: 0.5}, **one)
    elif name == "cancel_rows":         # KA5: column 3 cancels exactly inside the batch, so it gets no + c
        w0[0], d[0] = 1.0, 1.0
        c.update(rows=[([3, 5], [0.5, 0.25], 1), ([3, 9], [0.5, 0.75], -1)], lam=0.25, lr=0.5,
                 workers=([0, 1], [0, 1]), single=[0, 1], expect={3: 0.0, 5: -0.375, 9: 0.125})
    elif name == "wd_zero":             # partials +0.5 (CTA of column 0) and -0.5 (CTA of column 192): W.d = 0, c = 0
        w0[0], d[0], w0[192], d[192] = 1.0, 0.5, -1.0, 0.5
        c.update(rows=[([5], [0.5], 1)], lam=0.25, lr=0.5, expect={5: -0.25}, **one)
    elif name == "wd_negative":         # W.d = -1.5 + 0.25: c = -0.625
        w0[0], d[0], w0[192], d[192] = -3.0, 0.5, 0.5, 0.5
        c.update(rows=[([5], [0.5], 1)], lam=0.25, lr=0.5, expect={5: 0.0625}, **one)
    elif name == "wd_big":              # partials 2^41 + 2^15 and -(2^41 - 2^25), ||W||^2 < 2^52 per CTA: c = 2^-4 + 2^-14
        w0[0], d[0], w0[192], d[192] = 2.0 ** 25 + 0.5, 2.0 ** 16, -(2.0 ** 25), 2.0 ** 16 - 1
        c.update(rows=[([5], [0.5], 1)], lam=2.0 ** -30, lr=0.5, expect={5: -(0.25 + 2.0 ** -5 + 2.0 ** -15)}, **one)
    else:
        raise KeyError(name)
    if c["expect2"] is None:
        c["expect2"] = c["expect"]
    return c


HAND_CASES = ["residual", "tiny_step", "tiny_mean", "c_at_eps", "c_above_eps", "g_plus_c", "tiny_products", "tiny_value",
              "cancel_rows", "wd_zero", "wd_negative", "wd_big"]
HAND_PATHS = ["persistent_G2", "fallback_G1", "fused_K2_G5", "two_workers"]
HAND_STEPS = 3                  # fused K = 2 takes c from the accumulator from its third step on


def _hand_data(c):
    rows = [(cols, vals) for cols, vals, _ in c["rows"]] + [([], [])]   # the last row is empty: padding for batch 33
    labels = [y for _, _, y in c["rows"]] + [1]
    return _csr(rows, labels, c["dim"]), len(rows) - 1


@pytest.mark.parametrize("path", HAND_PATHS)
@pytest.mark.parametrize("name", HAND_CASES)
def test_filter_and_accumulator_edges(name, path):
    c = _hand_case(name)
    data, empty = _hand_data(c)
    w0, lam, lr, d = c["w0"], c["lam"], c["lr"], c["d"]
    two = path in ("fused_K2_G5", "two_workers")
    if path == "fused_K2_G5":
        assert _fits_fused(c["dim"], 5)
        per_rank = [np.tile(np.asarray(c["workers"][r], np.int32), (HAND_STEPS, 1)) for r in range(2)]
        losses, w = _fused_run(data, lam, d, 5, w0, per_rank, lr)
        _, orc = _pair(data, lam, d)
        w_ref, losses_ref = _fused_oracle(orc, w0, per_rank, lr)
        w1_ref, _ = _fused_oracle(orc, w0, [p[:1] for p in per_rank], lr)
    else:
        ctx, orc = _pair(data, lam, d)
        if path == "two_workers":
            ids = list(c["workers"][0]) + list(c["workers"][1])
            ctx.set_workers([len(c["workers"][0]), len(c["workers"][1])], k_total=2)
            counts = [len(c["workers"][0]), len(c["workers"][1])]
        else:
            ids = list(c["single"]) + ([empty] * (33 - len(c["single"])) if path == "fallback_G1" else [])
            ctx.set_grid_limit(1 if path == "fallback_G1" else 2)
            counts = [len(ids)]
        idx = np.tile(np.asarray(ids, np.int32), HAND_STEPS)
        ctx.set_weights(w0)
        losses = ctx.sync_steps(idx, len(ids), HAND_STEPS, lr)
        w = ctx.get_weights()
        ctx.close()
        w_ref, losses_ref = orc.sync_steps(w0, idx, counts, lr, n_steps=HAND_STEPS)
        w1_ref, _ = orc.sync_steps(w0, idx[:len(ids)], counts, lr, n_steps=1)
    for j, v in (c["expect2"] if two else c["expect"]).items():
        assert w1_ref[j] == v, (j, w1_ref[j], v)               # the case is what it says on the oracle
    _check(losses, w, losses_ref, w_ref, f"{name} via {path}", exact=True)


# ---- D2. losses of empty-gradient steps at small weight scales -------------------------------------------------------

SMALL_DIM = 20000               # a multiple of 32: in the fused exchange a warp's first column is the counter column


@pytest.fixture(scope="module")
def small_weight_data(S):
    """Weights on 2 % of the columns, |w| in [1, 2) (times the scale), random signs; every row holds 8 columns of ONE sign
    with values in [0.5, 1.5) and y = -sign: y (x.w) < 0 in every row, so the hinge is 0 and the gradient empty."""
    rng = np.random.default_rng(23)
    sup = np.flatnonzero(rng.random(SMALL_DIM) < 0.02)
    base = np.zeros(SMALL_DIM)
    base[sup] = (1.0 + rng.random(sup.size)) * rng.choice([-1.0, 1.0], size=sup.size)
    pos, neg = sup[base[sup] > 0], sup[base[sup] < 0]
    n_rows = 32 * S + 64
    rows, labels = [], []
    for i in range(n_rows):
        s = 1 if i % 2 == 0 else -1
        rows.append((rng.choice(pos if s > 0 else neg, size=8, replace=False), 0.5 + rng.random(8)))
        labels.append(-s)
    return _csr(rows, labels, SMALL_DIM), base


@pytest.mark.parametrize("path", ["persistent_32S", "fallback_32S+1", "fused_K2"])
@pytest.mark.parametrize("scale", [1e-6, 1e-9, 1e-12, 1e-16])
def test_small_weight_losses(S, small_weight_data, scale, path):
    """loss = lambda ||W||^2 exactly as the oracle sums it, whichever kernel sums ||W||^2: the persistent kernel through its
    fixed-point accumulator, k_update<true> in fp64, the fused exchange through the accumulator from its second step on."""
    data, base = small_weight_data
    w0 = base * scale
    lam, lr, steps = 1e-3, 0.5, 3
    rng = np.random.default_rng(int(-np.log10(scale)))
    _, orc = make_pair(data, lam)
    if path == "fused_K2":
        G = S // 2
        assert _fits_fused(SMALL_DIM, G)
        per_rank = [np.stack([rng.choice(data.n_rows, size=32 * G, replace=False) for _ in range(steps)]).astype(np.int32)
                    for _ in range(2)]
        losses, w = _fused_run(data, lam, None, G, w0, per_rank, lr)
        w_ref, losses_ref = _fused_oracle(orc, w0, per_rank, lr)
    else:
        b = 32 * S + (1 if path == "fallback_32S+1" else 0)
        idx = np.stack([rng.choice(data.n_rows, size=b, replace=False) for _ in range(steps)]).astype(np.int32).reshape(-1)
        ctx, _ = make_pair(data, lam)
        ctx.set_weights(w0)
        losses = ctx.sync_steps(idx, b, steps, lr)
        w = ctx.get_weights()
        ctx.close()
        w_ref, losses_ref = orc.sync_steps(w0, idx, [b], lr, n_steps=steps)
    np.testing.assert_array_equal(w_ref, w0)                  # the gradient is empty: nothing moves
    np.testing.assert_allclose(losses_ref, lam * np.sum(w0 * w0), rtol=1e-13)   # hinge 0: the loss is lambda ||W||^2
    np.testing.assert_array_equal(w, w0)
    np.testing.assert_allclose(losses, losses_ref, rtol=1e-12, atol=0, err_msg=f"scale {scale}, {path}")


# ---- E. exchange-only ranks -----------------------------------------------------------------------------------------

@pytest.mark.parametrize("what", ["batch_above_32G", "dim_above_448G"])
def test_exchange_only_ranks_refuse_what_the_fused_kernel_cannot_take(S, what):
    """Ranks wired with dsgd_xchg_attach and no communicator have no step-by-step path: a batch above 32 G per rank or
    dim + 1 above 448 G must raise DsgdState before anything is launched."""
    from distributed_sgd_b200.native import DsgdState
    G = S // 2 if what == "batch_above_32G" else 2
    dim = 2000 if what == "batch_above_32G" else SLICE_MAX * G
    batch = 32 * G + 1 if what == "batch_above_32G" else 4
    assert (batch > 32 * G) or not _fits_fused(dim, G)
    data = _synth(dim, batch + 8, seed=5)
    ctxs = []
    try:
        for r in range(2):
            ctx, _ = make_pair(data, 1e-3, rank=r, world=2)
            ctx.set_grid_limit(G)
            ctx.reserve(batch, 1)
            ctxs.append(ctx)
        ctxs[0].xchg_attach(1, ctxs[1])
        ctxs[1].xchg_attach(0, ctxs[0])
        for ctx in ctxs:
            ctx.set_weights(np.zeros(dim))
            before = ctx.launch_count()
            with pytest.raises(DsgdState, match="fused peer-exchange kernel cannot take this step"):
                ctx.sync_steps(np.arange(batch, dtype=np.int32), batch, 1, 0.5)
            assert ctx.launch_count() == before
    finally:
        for c in ctxs:
            c.close()
