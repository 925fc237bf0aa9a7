"""Rows of several 128-pair chunks in the persistent sync step (consume_stage, csrc/dsgd_persistent.cuh), bit for bit.

A stage whose rows are all in the chunk list and take at most kCons = 8 chunks finishes each row of several chunks in the
warps that hold its chunks, after a named barrier of the row's own; any other stage takes the second pass after a barrier of
all consumer warps.  Each case below is one CTA's rows of a step.  A Python mirror of the producer's layout checks which path
each case takes.  The same steps run at 5 CTAs (one instance of the case per CTA: the path the case is built for) and at
1 CTA (five instances in one CTA: always more than 8 chunks, the second pass), on every weighting (none, class, sample)
with and without the L1 penalty, and on fused K = 2 ranks on one GPU.  Values, weights and rates are dyadic and lambda is 0,
so every sum is exact: the weights must equal the checker's bit for bit, and the two paths must agree bit for bit on the
weights and the losses.  Values and weights are positive, so rows of label -1 fail the gate and rows of label +1 pass it.
"""
import numpy as np
import pytest

from helpers import csr, fused_ranks, make_pair
from oracle import sw as SW

pytestmark = pytest.mark.gpu

CHUNK_PAIRS, MAX_CHUNKS, CONS = 128, 128, 8     # kChunkPairs, kPMaxChunks, kPCons
DIM = 2047                                     # fused K = 2 at 5 CTAs per rank: slices of 416 columns fit its column threads
G_CASE = 5                                     # CTAs that hold one instance of a case each
STEPS = 3
INSTANCES = G_CASE * 2 * STEPS                 # one instance per CTA, step and rank

CASES = {   # non-zeros of one CTA's rows, in row order -> (chunks, path)
    "multi_beside_single": [300, 40, 100, 7],  # 3 + 1 + 1 + 1
    "two_chunks": [200, 60],                   # 2 + 1
    "eight_chunks": [1024],                    # one row of exactly kCons chunks
    "four_two_chunk_rows": [256, 250, 129, 200],   # 2 + 2 + 2 + 2 = kCons: four row barriers
    "three_multi_and_empty": [300, 129, 0, 257],   # 3 + 2 + 0 + 3 = kCons
    "kcons_plus_one": [1024, 5],               # 8 + 1: the second pass
    "one_row_nine_chunks": [1025],             # 1026 pairs: 9 chunks, the second pass
}
PATH = {"multi_beside_single": "per_row", "two_chunks": "per_row", "eight_chunks": "per_row",
        "four_two_chunk_rows": "per_row", "three_multi_and_empty": "per_row", "kcons_plus_one": "two_pass",
        "one_row_nine_chunks": "two_pass"}
FORMS = {   # (class weights or None, sample weights, lambda1)
    "unweighted": (None, False, 0.0), "class": ((0.5, 2.0), False, 0.0), "sample": ((0.5, 2.0), True, 0.0),
    "unweighted_l1": (None, False, 2.0 ** -7), "class_l1": ((0.5, 2.0), False, 2.0 ** -7),
    "sample_l1": ((0.5, 2.0), True, 2.0 ** -7),
}
LR = 2.0 ** -6


def stage_path(nnzs):
    """Mirror of the producer's choice (k_sync_persistent, producer warp): (chunks, rows of several chunks, path)."""
    nnz = np.asarray(nnzs, np.int64)
    chunks = (2 * ((nnz + 1) // 2) + CHUNK_PAIRS - 1) // CHUNK_PAIRS
    listed = np.cumsum(chunks) <= MAX_CHUNKS
    multi = int(np.sum(listed & (chunks > 1)))
    per_row = bool(listed.all()) and int(chunks[listed].sum()) <= CONS
    return int(chunks.sum()), multi, ("per_row" if per_row or multi == 0 else "two_pass")


def test_cases_take_their_path():
    for name, nnzs in CASES.items():
        chunks, multi, path = stage_path(nnzs)
        assert multi > 0 and path == PATH[name], (name, chunks, multi, path)
        # five instances in one CTA: always the second pass
        assert stage_path(nnzs * G_CASE)[2] == "two_pass" and len(nnzs) * G_CASE <= 32, name
    assert stage_path(CASES["eight_chunks"])[0] == CONS and stage_path(CASES["kcons_plus_one"])[0] == CONS + 1
    assert stage_path(CASES["four_two_chunk_rows"])[1] == 4


@pytest.fixture(scope="module")
def case_data():
    """INSTANCES fresh instances of every case: dyadic values in [2^-8, 4] on distinct columns, random labels."""
    rng = np.random.default_rng(29)
    rows, labels, inst = [], [], {}
    for name, nnzs in CASES.items():
        inst[name] = []
        for _ in range(INSTANCES):
            ids = []
            for n in nnzs:
                ids.append(len(rows))
                rows.append((rng.choice(DIM, size=n, replace=False), rng.integers(1, 1025, size=n) / 256.0))
                labels.append(int(rng.choice([-1, 1])))
            inst[name].append(ids)
    w0 = rng.integers(1, 257, size=DIM) / 64.0
    sw = rng.integers(1, 17, size=len(rows)) / 4.0
    return csr(rows, np.asarray(labels, np.int8), DIM), inst, w0, sw


def steps_of(inst, rank=0):
    """[STEPS, G_CASE * rows] sample ids: position b + m * G_CASE is row m of the instance CTA b holds at G_CASE CTAs."""
    out = []
    for s in range(STEPS):
        ctas = [inst[(s * 2 + rank) * G_CASE + b] for b in range(G_CASE)]
        out.append([ctas[i % G_CASE][i // G_CASE] for i in range(G_CASE * len(ctas[0]))])
    return np.asarray(out, np.int32)


def run_one_gpu(data, form, sw, grid, idx, w0):
    cw, weighted, lam1 = FORMS[form]
    ctx, _ = make_pair(data, 0.0)
    try:
        ctx.set_grid_limit(grid)
        if cw is not None:
            ctx.set_class_weights(*cw)
        if weighted:
            ctx.set_sample_weights(sw)
        if lam1:
            ctx.set_l1(lam1)
        ctx.set_weights(w0)
        losses = ctx.sync_steps(idx.reshape(-1), idx.shape[1], STEPS, LR)
        return losses, ctx.get_weights()
    finally:
        ctx.close()


@pytest.mark.parametrize("form", list(FORMS))
def test_one_gpu_both_paths_and_checker(case_data, form):
    data, inst, w0, sw = case_data
    cw, weighted, lam1 = FORMS[form]
    _, orc = make_pair(data, 0.0)
    failures = []
    for name in CASES:
        idx = steps_of(inst[name])
        per_row = run_one_gpu(data, form, sw, G_CASE, idx, w0)
        two_pass = run_one_gpu(data, form, sw, 1, idx, w0)
        w_ref, l_ref = SW.sync_steps(orc, w0, idx.reshape(-1), [idx.shape[1]], [LR] * STEPS, sw if weighted else None,
                                     *(cw or (1.0, 1.0)), lambda1=lam1)
        try:
            assert np.count_nonzero(w_ref != w0) > 0, "the case moved no weight"
            np.testing.assert_array_equal(per_row[1], two_pass[1], err_msg="weights: 5 CTAs against 1 CTA")
            np.testing.assert_array_equal(per_row[0], two_pass[0], err_msg="losses: 5 CTAs against 1 CTA")
            np.testing.assert_array_equal(per_row[1], w_ref, err_msg="weights against the checker")
            np.testing.assert_allclose(per_row[0], l_ref, rtol=1e-13, atol=0, err_msg="losses against the checker")
        except AssertionError as e:
            failures.append(f"{form}, case {name}: {e}")
    assert not failures, "\n".join(failures)


def test_fused_two_ranks_on_one_gpu(case_data):
    data, inst, w0, _ = case_data
    _, orc = make_pair(data, 0.0)
    failures = []
    for name in CASES:
        per_rank = [steps_of(inst[name], r) for r in range(2)]
        res = fused_ranks(data, 0.0, None, [G_CASE, G_CASE], w0, [(per_rank, None)], LR)
        idx = np.concatenate(per_rank, axis=1)
        w_ref, l_ref = orc.sync_steps(w0, idx.reshape(-1), [per_rank[0].shape[1], per_rank[1].shape[1]], LR, n_steps=STEPS)
        try:
            assert np.count_nonzero(w_ref != w0) > 0, "the case moved no weight"
            np.testing.assert_array_equal(res["w"][0], w_ref, err_msg="weights against the oracle")
            np.testing.assert_array_equal(res["losses"][0], l_ref, err_msg="losses against the oracle")
        except AssertionError as e:
            failures.append(f"case {name}: {e}")
    assert not failures, "\n".join(failures)
