"""The fused K-rank sync step (k_sync_persistent<..., kMulti = true>, csrc/dsgd_persistent.cuh) bit for bit against the
oracle's K-worker master step (one_sync_step in oracle/dsgd_oracle.c; core/Master.scala:184-197).  K contexts share one GPU
through dsgd_set_grid_limit + dsgd_xchg_attach (helpers.fused_ranks), one host thread per rank.

A. The fold over the replies, K = 3: each reply is regularized on its own support, then the replies are folded left to right
   in rank order with the 1e-20 filter after every +.  Columns whose result depends on the order (a large reply on rank 0, 1
   or 2 next to two 2^-53 replies), on where the filter sits (r0 + r1 lands within 1e-20 of zero before r2 is added), on
   absent replies (only rank 2; ranks 0 and 2); lambda = 0 and a lambda whose c is one exact term.
B. Unequal per-rank batches: the loss of a step is decoded from the sum of the ranks' packed counters (hinge + 2^32 B):
   (48, 7), (34, 34, 32), 32 G mispredicted rows next to one row, and an epoch shaped like MasterSync.fit's calls.
C. Slice and bitmap edges, K = 2: dim + 1 = 0, 1, 31 (mod 32), a 448-column slice, CTAs that own no column, ranks whose grids
   differ; rows on column 0, column dim - 1 and the first and last column of every CTA's slice.  A Python mirror of the
   kernel's slice / j_col / warp_act checks that each case reaches the layout it names.
D. Launch sequences: eleven launches of 1 to 5 steps with and without set_weights in between (lambda > 0, so that a stale c
   would show), then the streaming dsgd_eval (>= 2048 rows, reads the fp32 copy of the weights), eval_counts and gradient on
   the resident weights against a one-rank context holding the same weights.
E. Every run of A-D checks dsgd_xchg_stats of every rank against its exact model (helpers.xchg_model), including a reply
   entry that sums to 2^-80 inside one rank and so must not be sent.

Exactness: the REDs inside one rank add in any order, so every rank's batch sum must be exact: rows hold dyadic fp32 values.
c = 2 lambda W.d is one exact term: d is non-zero on one column j0 that no row touches.  With K = 2 and a dyadic learning
rate the weights stay dyadic and ||W||^2 is exact, so losses are compared bit for bit too; with K = 3 the mean s / 3 is
inexact, so where lambda > 0 the losses are compared at the suite's tolerance (rtol 1e-12) and the weights bit for bit.

K stops at 3, as in test_gpu_fused_one_gpu.py: four spinning kernels sharing one GPU are not promised to be co-scheduled.
"""
import numpy as np
import pytest

from helpers import data_from_csr, fused_ranks, xchg_model
from oracle.oracle import Oracle

pytestmark = pytest.mark.gpu

EPS = 1e-20
SLICE_MAX = 14 * 32             # barrier-synchronised threads per CTA: one column of the CTA's slice each
E53 = 2.0 ** -53


@pytest.fixture(scope="module")
def S():
    from distributed_sgd_b200.native import NativeCtx
    ctx = NativeCtx(0, 8, 0.0)
    s = int(ctx.info()["sm_count"])
    ctx.close()
    return s


def _csr(rows, dim):
    """rows: list of (cols, vals, y)."""
    rp = np.zeros(len(rows) + 1, np.int64)
    rp[1:] = np.cumsum([len(c) for c, _, _ in rows])
    col = np.concatenate([np.asarray(c, np.int32) for c, _, _ in rows] + [np.zeros(0, np.int32)])
    val = np.concatenate([np.asarray(v, np.float32) for _, v, _ in rows] + [np.zeros(0, np.float32)])
    assert np.array_equal(val.astype(np.float64), np.concatenate([np.asarray(v, np.float64) for _, v, _ in rows] + [[]]))
    return data_from_csr(rp, col, val, np.asarray([y for _, _, y in rows], np.int8), dim)


def _d_one(dim, j0):
    d = np.zeros(dim)
    d[j0] = 1.0
    return d


def _oracle(data, lam, d):
    orc = Oracle(data.row_ptr, data.col, data.val, data.label, data.dim, lam)
    orc.set_dim_sparsity(d)
    return orc


def _oracle_run(orc, w0, calls, lr):
    w, losses = np.asarray(w0, np.float64), []
    for ids, w_new in calls:
        if w_new is not None:
            w = np.asarray(w_new, np.float64)
        idx = np.concatenate([np.asarray(a, np.int32) for a in ids], axis=1)
        w, ls = orc.sync_steps(w, idx.reshape(-1), [a.shape[1] for a in ids], lr, n_steps=idx.shape[0])
        losses.append(ls)
    return w, np.concatenate(losses)


def _run_and_check(data, lam, d, grids, w0, calls, lr, exact_losses=True, after=None, what=""):
    """Runs the ranks, checks weights bit for bit, losses bit for bit (or at rtol 1e-12) and every rank's exchange counters
    against the exact model.  Returns (fused_ranks' result, oracle, final oracle weights)."""
    res = fused_ranks(data, lam, d, grids, w0, calls, lr, after=after)
    orc = _oracle(data, lam, d)
    w_ref, losses_ref = _oracle_run(orc, w0, calls, lr)
    np.testing.assert_array_equal(res["w"][0], w_ref, err_msg=f"{what}: weights")
    if exact_losses:
        np.testing.assert_array_equal(res["losses"][0], losses_ref, err_msg=f"{what}: losses")
    else:
        np.testing.assert_allclose(res["losses"][0], losses_ref, rtol=1e-12, atol=0, err_msg=f"{what}: losses")
    model = xchg_model(orc, w0, calls, lr)
    for r in range(len(grids)):
        assert tuple(res["xstats"][r]) == model[r], f"{what}: rank {r} xchg_stats {res['xstats'][r]}, model {model[r]}"
    return res, orc, w_ref


def _random_rows(rng, n, cols, nnz, y=None, k_max=32):
    """n rows of `nnz` distinct columns drawn from `cols`, values k / 16 (k in 1..k_max), labels y or random."""
    cols = np.asarray(cols)
    return [(np.sort(rng.choice(cols, size=nnz, replace=False)), rng.integers(1, k_max + 1, size=nnz) / 16.0,
             int(y if y is not None else rng.choice([-1, 1]))) for _ in range(n)]


def _dyadic_w0(rng, dim, j0, frac=0.3):
    w0 = rng.integers(-32, 33, size=dim) / 8.0 * (rng.random(dim) < frac)
    w0[j0] = 1.0
    return w0


# ---- A. the fold over the replies, K = 3 ------------------------------------------------------------------------------

def _filt(v):
    return v if abs(v) > EPS else 0.0


def _fold(replies, c, order, filter_each=True):
    """Mirror of the column threads' fold: each reply filtered and, where non-zero, + c (filtered); replies folded in `order`
    with the filter after every + (or, filter_each=False, only at the end)."""
    s, first = 0.0, True
    for k in order:
        v = _filt(replies[k])
        if v != 0.0 and c != 0.0 and abs(c) > EPS:
            v = _filt(v + c)
        s = v if first else (_filt(s + v) if filter_each else s + v)
        first = False
    return _filt(s)


def _update(w, s, K, lr):
    return w if s == 0.0 else _filt(w - _filt(_filt(s / K) * lr))


FOLD_J0, FOLD_DIM = 0, 64
TINY_A, TINY_B = 2.0 ** -60 * (1 + 2.0 ** -20), 2.0 ** -60
FOLD_COLS = {   # column: raw reply of ranks 0, 1, 2 (their batch sums of y x) and the sum a left fold gives at lambda = 0
    3: ((1.0, E53, E53), 1.0),                    # large reply on rank 0: right fold 1 + 2^-52
    4: ((E53, 1.0, E53), 1.0),                    # large reply on rank 1: rank 2's own-first fold 1 + 2^-52
    5: ((E53, E53, 1.0), 1.0 + 2.0 ** -52),       # large reply on rank 2: right fold and rank 2's own-first fold 1
    6: ((TINY_A, -TINY_B, TINY_B), TINY_B),       # r0 + r1 = 2^-80 is filtered before r2: 2^-60, not 2^-60 + 2^-80
    7: ((0.0, 0.0, 0.75), 0.75),                  # only rank 2 sends
    8: ((0.5, 0.0, 0.25), 0.75),                  # the middle reply is absent
    9: ((2.0 ** -80, 0.0, 0.0), 0.0),             # 2^-60 (1 + 2^-20) - 2^-60 inside rank 0: filtered, never sent
    10: ((1.0, 0.0, 0.0), 1.0),                   # anchors: w0 = 8 keeps every row's dot positive for the three steps
    11: ((0.0, 1.0, 0.0), 1.0),
    12: ((0.0, 0.0, 1.0), 1.0),
    13: ((-1.0, 0.0, 0.0), -1.0),                 # rank 0's y = -1 row: w0 = -8 keeps its dot negative
}
FOLD_STEPS, FOLD_LR = 3, 1.0
# rank 1's own-first order (1, 0, 2) only swaps the operands of the first +, which never changes a sum
FOLD_ORDERS = {"descending": [2, 1, 0], "own first (rank 2)": [2, 0, 1]}


def _fold_case():
    """Rank 0: rows 0 (y = +1) and 1 (y = -1); rank 1: row 2; rank 2: row 3.  Within a rank no two entries of one column
    except column 9, whose two entries sum to 2^-80 exactly."""
    per_rank = [dict(), dict(), dict()]
    for j, (rep, _) in FOLD_COLS.items():
        for r in range(3):
            if rep[r] != 0.0 and j not in (9, 13):
                per_rank[r][j] = rep[r]
    per_rank[0][9] = TINY_A
    rows = [(sorted(p), [p[j] for j in sorted(p)], 1) for p in per_rank]
    rows.insert(1, ([9, 13], [TINY_B, 1.0], -1))
    w0 = np.zeros(FOLD_DIM)
    w0[FOLD_J0] = 1.0
    w0[[10, 11, 12]] = 8.0
    w0[13] = -8.0
    ids = [np.array([[0, 1]] * FOLD_STEPS, np.int32), np.array([[2]] * FOLD_STEPS, np.int32),
           np.array([[3]] * FOLD_STEPS, np.int32)]
    return _csr(rows, FOLD_DIM), w0, ids


@pytest.mark.parametrize("grids", ["small", "widest"])
@pytest.mark.parametrize("lam", [0.0, 2.0 ** -31])
def test_rank_order_fold(S, lam, grids):
    data, w0, ids = _fold_case()
    d = _d_one(FOLD_DIM, FOLD_J0)
    c = lam * 2.0 * 1.0                           # W.d = w0[j0] * 1: one exact term, and column j0 never moves
    G = [2, 3, 1] if grids == "small" else [S // 3 - 4] * 3
    # the case is what it says: the oracle's first step is the left fold of the table, and every other order gives
    # different weights on at least one column
    orc = _oracle(data, lam, d)
    w1, _ = orc.sync_steps(w0, np.concatenate([a[0] for a in ids]), [2, 1, 1], FOLD_LR)
    for j, (rep, s_left) in FOLD_COLS.items():
        if lam == 0.0:
            assert _fold(rep, c, [0, 1, 2]) == s_left, j
        assert w1[j] == _update(w0[j], _fold(rep, c, [0, 1, 2]), 3, FOLD_LR), (j, w1[j])
    for name, order in FOLD_ORDERS.items():
        assert any(_fold(rep, c, order) != _fold(rep, c, [0, 1, 2]) for rep, _ in FOLD_COLS.values()), name
    if lam == 0.0:
        assert _fold(FOLD_COLS[6][0], c, [0, 1, 2], filter_each=False) != FOLD_COLS[6][1]
        assert w1[5] == -((1.0 + 2.0 ** -52) / 3) and w1[3] == w1[4] == -(1.0 / 3)
    _run_and_check(data, lam, d, G, w0, [(ids, None)], FOLD_LR, exact_losses=(lam == 0.0), what=f"fold, lambda {lam}")


# ---- B. unequal per-rank batches --------------------------------------------------------------------------------------

UNEQUAL_DIM, UNEQUAL_J0 = 3000, 0


def _unequal_data(n_rows, seed):
    rng = np.random.default_rng(seed)
    rows = _random_rows(rng, n_rows, np.arange(1, UNEQUAL_DIM), 12)
    return _csr(rows, UNEQUAL_DIM), _dyadic_w0(rng, UNEQUAL_DIM, UNEQUAL_J0), rng


@pytest.mark.parametrize("batches", [(48, 7), (34, 34, 32)])
def test_unequal_rank_batches(batches):
    K = len(batches)
    steps = 5
    data, w0, rng = _unequal_data(sum(batches) * steps, seed=31 + K)
    perm = rng.permutation(data.n_rows).astype(np.int32).reshape(steps, -1)
    cuts = np.cumsum((0,) + batches)
    ids = [np.ascontiguousarray(perm[:, cuts[r]:cuts[r + 1]]) for r in range(K)]
    res, _, _ = _run_and_check(data, 0.0, _d_one(UNEQUAL_DIM, UNEQUAL_J0), [8] * K, w0, [(ids, None)], 2.0 ** -3,
                               what=f"batches {batches}")
    assert len(set(res["losses"][0].tolist())) > 1, "the hinge counts do not change: a weak case"


@pytest.mark.parametrize("grid", ["G5", "widest"])
def test_full_grid_batch_next_to_one_row(S, grid):
    """Rank 0 takes 32 G rows, every one mispredicted (y = +1, dot > 0: hinge 2 each), rank 1 one row: the loss is
    (64 G + h1) / (32 G + 1), which neither rank's own counter gives."""
    G = 5 if grid == "G5" else S // 2
    dim, j0 = 2048, 0                              # dim + 1 <= 448 * 5: the G5 slices fit
    rng = np.random.default_rng(G)
    P = np.arange(1, 257)                          # rank 0's columns: w0 = 64 keeps every dot positive for the three steps
    rows = _random_rows(rng, 32 * G, P, 8, y=1, k_max=16)
    rows.append(([300, 301, 302], [0.5, 0.25, 1.0], -1))    # rank 1: w = 0 there, dot 0: passes the gate, hinge 1
    data = _csr(rows, dim)
    w0 = np.zeros(dim)
    w0[P] = 64.0
    w0[j0] = 1.0
    steps = 3
    ids = [np.tile(np.arange(32 * G, dtype=np.int32), (steps, 1)), np.full((steps, 1), 32 * G, np.int32)]
    res, _, _ = _run_and_check(data, 0.0, _d_one(dim, j0), [G, G], w0, [(ids, None)], 2.0 ** -6, what=f"32 G + 1, G {G}")
    assert res["losses"][0][0] == (64 * G + 1) / (32 * G + 1)


def test_epoch_shaped_like_master_sync_fit(S):
    """SplitStrategy.vanilla over n_train = 1000 rows, K = 3, batch 100: groups of 334, 334 and 332 rows; every epoch is
    three steps of 100 rows per rank and a last step of 34, 34 and 32 rows -- two launches per epoch, two epochs."""
    K, n_train, batch = 3, 1000, 100
    data, w0, rng = _unequal_data(n_train, seed=7)
    size = -(-n_train // K)
    groups = [np.arange(a, min(a + size, n_train)) for a in range(0, n_train, size)]
    calls = []
    for _ in range(2):
        steps = [[rng.choice(g, size=min(batch, len(g) - b), replace=False).astype(np.int32) for g in groups]
                 for b in range(0, size, batch)]
        assert [len(a) for a in steps[-1]] == [34, 34, 32] and all(len(a) == batch for s in steps[:-1] for a in s)
        calls.append(([np.stack([s[r] for s in steps[:-1]]) for r in range(K)], None))
        calls.append(([steps[-1][r][None, :] for r in range(K)], None))
    _run_and_check(data, 0.0, _d_one(UNEQUAL_DIM, UNEQUAL_J0), [S // 3 - 4] * K, w0, calls, 2.0 ** -3, what="epoch")


# ---- C. slice and bitmap edges, K = 2 ---------------------------------------------------------------------------------

def slice_layout(dim, G):
    """Mirror of the kMulti column threads: slice = roundup32(ceil((dim + 1) / G)); thread x of CTA b owns column
    j_col = b * slice + x if x < slice and j_col <= dim (column dim is the counter); a warp takes part in the exchange
    (warp_act) if its first column exists.  Returns (slice, [(first, last) column of each CTA, or None], active warps)."""
    sl = ((dim + 1 + G - 1) // G + 31) // 32 * 32
    owned = [(b * sl, min((b + 1) * sl, dim + 1) - 1) if b * sl <= dim else None for b in range(G)]
    warps = sum(1 for b in range(G) for w in range(sl // 32) if b * sl + 32 * w <= dim)
    return sl, owned, warps


EDGE_CASES = {   # name: (dim, CTAs of rank 0, CTAs of rank 1)
    "dim+1=0_mod32": (1023, 3, 3),
    "dim+1=1_mod32": (1024, 3, 3),
    "dim+1=31_mod32": (1022, 3, 3),
    "slice_448": (448 * 3 - 1, 3, 3),
    "empty_last_cta": (100, 5, 5),
    "empty_ctas_grids_differ": (100, 5, 7),
    "grids_differ": (1023, 3, 5),
    "grids_differ_448": (448 * 3 - 1, 3, 4),
}


def _edge_reaches(name, dim, G0, G1):
    lay = [slice_layout(dim, G) for G in (G0, G1)]
    for sl, owned, warps in lay:
        assert sl <= SLICE_MAX and warps == (dim + 1 + 31) // 32
        assert [o for o in owned if o is not None][-1][1] == dim      # the counter column has an owner
    if name == "dim+1=0_mod32":
        return (dim + 1) % 32 == 0
    if name == "dim+1=1_mod32":
        return (dim + 1) % 32 == 1                                   # the counter column is alone in its bitmap word
    if name == "dim+1=31_mod32":
        return (dim + 1) % 32 == 31
    if name == "slice_448":
        return lay[0][0] == lay[1][0] == SLICE_MAX
    if name == "empty_last_cta":
        return lay[0][1][-1] is None and lay[1][1][-1] is None
    if name == "empty_ctas_grids_differ":
        return lay[0][1].count(None) >= 1 and lay[1][1].count(None) >= 3 and G0 != G1
    if name == "grids_differ":
        return lay[0][0] != lay[1][0]
    if name == "grids_differ_448":
        return lay[0][0] == SLICE_MAX and lay[1][0] < SLICE_MAX
    raise KeyError(name)


def test_edge_cases_reach_their_layout():
    for name, (dim, G0, G1) in EDGE_CASES.items():
        assert _edge_reaches(name, dim, G0, G1), name


def _edge_cols(dim, grids):
    cols = {0, dim - 1}
    for G in grids:
        for o in slice_layout(dim, G)[1]:
            if o is not None:
                cols.update(c for c in o if c < dim)
    return sorted(cols)


@pytest.mark.parametrize("name", list(EDGE_CASES))
def test_slice_and_bitmap_edges(name):
    dim, G0, G1 = EDGE_CASES[name]
    assert _edge_reaches(name, dim, G0, G1), name
    edges = _edge_cols(dim, (G0, G1))
    j0 = dim // 2 + 1
    assert j0 not in edges
    rng = np.random.default_rng(dim + 100 * G0 + G1)
    rows = []
    for r in range(2):   # both ranks: every edge column, four per row, y = +1 at w = 0 (dot 0: the gate passes)
        for a in range(0, len(edges), 4):
            cs = edges[a:a + 4]
            rows.append((cs, rng.integers(1, 33, size=len(cs)) / 16.0, 1))
    n_edge = len(rows) // 2
    inner = sorted(set(range(dim)) - set(edges) - {j0})
    rows += _random_rows(rng, 64, inner, 12)      # the rest of the batch: other columns, random labels and weights
    data = _csr(rows, dim)
    w0 = np.zeros(dim)
    w0[inner] = rng.integers(-16, 17, size=len(inner)) / 8.0
    w0[j0] = 1.0
    lam, lr, steps = 2.0 ** -6, 2.0 ** -2, 3
    rand = np.arange(2 * n_edge, len(rows), dtype=np.int32)
    step_ids = [[np.concatenate([np.arange(r * n_edge, (r + 1) * n_edge), rand[r * 32:r * 32 + 5 + s]]).astype(np.int32)
                 for r in range(2)] for s in range(steps)]
    # one launch per step: a launch takes one batch shape, and each step adds one random row to every rank
    calls = [([step_ids[s][r][None, :] for r in range(2)], None) for s in range(steps)]
    res, orc, _ = _run_and_check(data, lam, _d_one(dim, j0), [G0, G1], w0, calls, lr, what=name)
    w1, _ = orc.sync_steps(w0, np.concatenate(step_ids[0]), [len(a) for a in step_ids[0]], lr)
    assert np.all(w1[edges] != w0[edges]), "the first step does not move every edge column"


# ---- D. launch sequences ----------------------------------------------------------------------------------------------

SEQ_DIM, SEQ_J0, SEQ_ROWS = 2000, 0, 2304
SEQ_LENGTHS = [1, 1, 2, 3, 1, 5, 2, 1, 4, 1, 3]
SEQ_BATCHES = [(24, 17), (9, 30), (24, 17), (1, 1), (32, 5), (24, 17), (7, 7), (40, 3), (24, 17), (2, 33), (24, 17)]
SEQ_SET_AT = {3: 0.5, 7: 2.0}   # launch index: w[j0] (so c) of the weights installed before it


@pytest.mark.parametrize("reset", ["carry_over", "set_weights"])
def test_launch_sequence_then_resident_requests(reset):
    from distributed_sgd_b200.native import NativeCtx
    rng = np.random.default_rng(41 if reset == "set_weights" else 42)
    rows = _random_rows(rng, SEQ_ROWS, np.arange(1, SEQ_DIM), 10)
    data = _csr(rows, SEQ_DIM)
    d = _d_one(SEQ_DIM, SEQ_J0)
    lam, lr = 2.0 ** -6, 2.0 ** -4
    w0 = _dyadic_w0(rng, SEQ_DIM, SEQ_J0)
    calls, last_set = [], w0
    for i, (n, (b0, b1)) in enumerate(zip(SEQ_LENGTHS, SEQ_BATCHES)):
        ids = [rng.choice(SEQ_ROWS, size=(n, b), replace=False if n * b <= SEQ_ROWS else True).astype(np.int32)
               for b in (b0, b1)]
        w = None
        if reset == "set_weights" and i in SEQ_SET_AT:
            w = _dyadic_w0(rng, SEQ_DIM, SEQ_J0)
            w[SEQ_J0] = SEQ_SET_AT[i]
            last_set = w
        calls.append((ids, w))
    big = rng.choice(SEQ_ROWS, size=2048 + 37, replace=True).astype(np.int32)    # the streaming pass (>= 2048 rows)
    small = rng.choice(SEQ_ROWS, size=45, replace=False).astype(np.int32)

    def requests(ctx, w=None):
        return (ctx.eval(0, SEQ_ROWS, w), ctx.eval_counts(0, SEQ_ROWS, w), ctx.eval(100, 2200, w),
                ctx.gradient(big, w), ctx.gradient(small, w))

    res, _, w_ref = _run_and_check(data, lam, d, [6, 8], w0, calls, lr, after=lambda r, ctx: requests(ctx),
                                   what=f"launch sequence, {reset}")
    one = NativeCtx(0, SEQ_DIM, lam)
    try:
        one.load_csr(data.row_ptr, data.col, data.val, data.label)
        one.set_dim_sparsity(d)
        one.set_weights(w_ref)
        want = requests(one)
        before = requests(one, last_set)
    finally:
        one.close()
    for r in range(2):
        got = res["after"][r]
        for k, what in enumerate(["eval", "eval_counts", "eval of rows [100, 2200)", "gradient (streaming)", "gradient"]):
            np.testing.assert_array_equal(np.asarray(got[k]), np.asarray(want[k]), err_msg=f"rank {r}: {what}")
    # the launches move the predictions: a stale fp32 copy of the weights would give other evaluations
    assert before[1][:2] != want[1][:2]
