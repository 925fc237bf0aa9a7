"""The numpy model of the row fold (tests/row_fold_model.py) and the adversarial rows the GPU test feeds the device
(tests/test_gpu_row_fold.py): the model is the fold the kernels document, it is exact where the sum is, and every class
of adversarial row really tells the row fold from the folds some kernels used before (U, W)."""
from fractions import Fraction

import numpy as np
import pytest

import row_fold_model as M


def literal_row_fold(p):
    """The row fold of one window of products, written out one lane and one chunk at a time."""
    dot = 0.0
    for c0 in range(0, len(p), 128):
        lanes = [0.0] * 32
        for l in range(32):
            for u in range(4):
                k = c0 + l + 32 * u
                if k < len(p):
                    lanes[l] = lanes[l] + p[k]
        for o in (16, 8, 4, 2, 1):
            lanes = [lanes[l] + lanes[l ^ o] for l in range(32)]
        dot = dot + lanes[0]
    return dot


def literal_fold_w(p):
    lanes = [0.0] * 32
    for k, v in enumerate(p):
        lanes[k % 32] = lanes[k % 32] + v
    for o in (16, 8, 4, 2, 1):
        lanes = [lanes[l] + lanes[l ^ o] for l in range(32)]
    return lanes[0]


def literal_fold_u(p):
    lanes = [0.0] * 32
    for u in range(0, len(p) // 2):
        lanes[u % 32] = lanes[u % 32] + p[2 * u]
        lanes[u % 32] = lanes[u % 32] + p[2 * u + 1]
    for o in (16, 8, 4, 2, 1):
        lanes = [lanes[l] + lanes[l ^ o] for l in range(32)]
    return lanes[0]


def _padded(rows):
    L = max(128, -(-max(len(r) for r in rows) // 128) * 128)
    P = np.zeros((len(rows), L))
    for i, r in enumerate(rows):
        P[i, :len(r)] = r
    return P


@pytest.mark.parametrize("n", [1, 2, 31, 32, 33, 127, 128, 129, 255, 256, 257, 640, 1000])
def test_vectorised_folds_equal_the_literal_folds(n):
    """Non-dyadic products of mixed sign and scale: every rounding shows, so the vectorised model must take the order."""
    rng = np.random.default_rng(n)
    rows = [rng.standard_normal(n) * np.exp2(rng.integers(-40, 40, size=n)) for _ in range(6)]
    rows = [np.concatenate([r, [0.0]]) if n % 2 else r for r in rows]   # a window is a whole number of 16-byte units
    P = _padded(rows)
    for i, r in enumerate(rows):
        assert M.fold_row(P)[i] == literal_row_fold(list(r))
        assert M.fold_w(P)[i] == literal_fold_w(list(r))
        assert M.fold_u(P)[i] == literal_fold_u(list(r))
        left = 0.0
        for v in r:
            left = left + v
        assert M.fold_l(P)[i] == left


def test_window_products_follow_storage_order_and_filter():
    rp = np.array([0, 3, 3, 5], np.int64)
    col = np.array([2, 0, 1, 1, 2], np.int32)
    val = np.array([1.0, 2.0 ** -70, 0.5, 0.25, -1.0], np.float32)
    w = np.array([1.0, 2.0 ** -60, 3.0])
    P = M.window_products(rp, col, val, w, [0, 1, 2])
    assert P.shape == (3, 128)
    # x = 2^-70 is absent (filt), 0.5 * 2^-60 survives, 0.25 * 2^-60 = 2^-62 survives; the empty row is all zeros
    assert P[0, :3].tolist() == [3.0, 0.0, 2.0 ** -61]
    assert not P[1].any()
    assert P[2, :2].tolist() == [2.0 ** -62, -3.0]


@pytest.mark.parametrize("n", [3, 64, 128, 129, 500, 1000])
def test_every_fold_is_the_exact_sum_where_the_sum_is_exact(n):
    """Integer products times one power of two: every partial sum is exact, so every fold is the Fraction sum."""
    rng = np.random.default_rng(n + 7)
    rows = [rng.integers(-1000, 1001, size=n) * 2.0 ** -30 for _ in range(8)]
    rows = [np.concatenate([r, [0.0]]) if n % 2 else r for r in rows]
    P = _padded(rows)
    for f in (M.fold_row, M.fold_w, M.fold_u, M.fold_l):
        got = f(P)
        for i, r in enumerate(rows):
            assert Fraction(got[i]) == sum(Fraction(v) for v in r), f.__name__


def _dots(x):
    P = _padded([np.concatenate([x, [0.0]]) if len(x) % 2 else x])
    return M.fold_row(P)[0], M.fold_w(P)[0], M.fold_u(P)[0], M.fold_l(P)[0]


def test_row_a():
    c, w, u, l = _dots(np.array(M.ROW_A))
    assert (c, w, u, l) == (2.0 ** -59, 2.0 ** -59, 0.0, 2.0 ** -60)
    assert M.pred(c) == -1 and M.pred(u) == 0 and np.sign(l) == np.sign(c)


def test_short_rows_separate_the_row_fold_from_u_and_keep_the_oracles_sign():
    rows = M.short_rows(5, 48)
    assert len(rows) == 48 and all(3 <= len(x) <= 32 for x in rows)
    opposite = 0
    for x in rows:
        c, w, u, l = _dots(x)
        assert c == w                                    # one chunk: the row fold is W
        assert np.sign(c) != np.sign(u)
        assert np.sign(l) == np.sign(c)
        opposite += int(c * u < 0)
    assert opposite > 0                                  # some rows have opposite non-zero signs, not only zero vs non-zero


@pytest.mark.parametrize("n", [256, 320, 640, 960])
@pytest.mark.parametrize("sign", [1.0, -1.0])
def test_long_rows_separate_the_row_fold_from_w(n, sign):
    x = M.long_row(n, sign)
    c, w, u, l = _dots(x)
    assert c == 0.0 and w == sign * 2.0 ** -59
    assert np.sign(l) != np.sign(c)      # the oracle's fold differs here too: the GPU test checks this class on the model
    assert (np.abs(x) > M.EPS).all()


def test_data_set_columns_sum_exactly():
    """Every column holds one magnitude class (a pool) of x values, so any subset's sum of +-x is exact at lambda = 0."""
    d = M.build_rows(3)
    rp, col, val = M.to_csr(d["rows"])
    assert (np.abs(val[val != 0]) > M.EPS).all()
    base = M.N_POOLS * M.POOL_COLS
    for j in np.unique(col):
        v = np.abs(val[col == j].astype(np.float64))
        q = v / (M.POOL_UNIT[j // M.POOL_COLS] if j < base else 2.0 ** -8)
        assert (q == np.round(q)).all() and q.sum() < 2.0 ** 50, j
    kinds = set(d["kind"].tolist())
    assert kinds == {"row_a", "short", "long", "ordinary", "empty"}
    lab = d["labels"]
    assert (lab == 1).any() and (lab == -1).any()
    # the initial weights are 1 on every pool column and non-dyadic on the ordinary ones
    w = d["w"]
    assert (w[:base] == 1.0).all() and np.mean(w[base:] * 2.0 ** 20 != np.round(w[base:] * 2.0 ** 20)) > 0.9


def test_model_margins_of_the_data_set_separate_the_folds():
    d = M.build_rows(3)
    rp, col, val = M.to_csr(d["rows"])
    ids = np.arange(len(d["rows"]))
    P = M.window_products(rp, col, val, d["w"], ids)
    c, w, u = M.fold_row(P), M.fold_w(P), M.fold_u(P)
    adv = np.isin(d["kind"], ["row_a", "short", "long"])
    assert ((np.sign(c) != np.sign(u)) | (np.sign(c) != np.sign(w)))[adv].all()
    assert (c[d["kind"] == "empty"] == 0).all()
