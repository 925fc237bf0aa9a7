"""The streaming pass (k_stream_rows, csrc/dsgd_stream.cuh) at the ends of the fp32 range: rows whose fp32 dot overflows,
rows on subnormal weights, weights beyond fp32, through every streamed form, on request and on resident weights.

Each family is one weight vector and one data set of N rows.  Pass positions that are multiples of 32 hold the family's
planted rows, so that they start at lane 0 of their block in every block size (32, 16 or 8 rows); copies sit at other
positions, between ordinary and empty rows.  tests/stream_band_model.py gives every row's decision at each start lane, and
the start of every row of a pass follows from the work split (stream_launch), so each pass's count of recomputed rows
(dsgd_stream_exact_rows) is known exactly.  Every decision must be the filtered fp64 one (Oracle.forward, and the exact
sign of the row's products), wherever the row sits; gradients are compared bit for bit: every column holds one value
(times the labels and class weights), so every column sum is exact in any order.
"""
import numpy as np
import pytest

import stream_band_model as M
from helpers import data_from_csr, make_pair
from test_gpu_streaming import split_bounds

pytestmark = pytest.mark.gpu

MIN_STREAM_ROWS = 2048          # kStreamMinRows (csrc/dsgd_api.cu)
N_ROWS = 32 * 100 + 17          # rows of a family's data set: a ragged last block
N_KROWS = 1500                  # k_rows takes passes below 2048 rows
N_ORD_COLS = 1024               # ordinary columns; the planted rows' columns follow
CW = (2.0, 0.5)                 # class weights of the per-class forms
KEY = 0x5EED


class Family:
    """Planted rows (name -> (cols, vals)) on their own columns, and the weights; ordinary rows on the first columns."""

    def __init__(self, ord_w, ord_scale):
        self.w = list(ord_w)
        self.ord_scale = ord_scale
        self.kinds = {}

    def col(self, wv):
        self.w.append(wv)
        return len(self.w) - 1

    def plant(self, name, pairs):
        """pairs: [(x, w)], one fresh column per pair."""
        self.kinds[name] = ([self.col(wv) for _, wv in pairs], [x for x, _ in pairs])


def _units(name, fam, units):
    """A row of units [((x0, w0), (x1, w1))]."""
    fam.plant(name, [p for u in units for p in u])


def _filler(k):
    """k units of small products: (1 on w 1, 1 on w -1) cancel exactly in both fp32 and fp64."""
    return [((1.0, 1.0), (1.0, -1.0))] * k


def overflow_family(rng):
    fam = Family(rng.uniform(0.5, 1.5, N_ORD_COLS) * np.where(rng.random(N_ORD_COLS) < 0.5, -1, 1), 1.0)
    Z = (1.0, 0.0)
    big, neg, small = (2e36, 100.0), (-3.3e36, 100.0), (-1e36, 100.0)
    for tag, other in (("other", neg), ("same", small)):
        # a single product: 4e36 * 100 = 4e38 is +inf in fp32
        _units(f"product_{tag}", fam, [((4e36, 100.0), Z), (other, Z), (other, Z)])
        # a unit's fma: 2e38 + 2e38 (the first row of the issue's table, and its same-sign twin)
        _units(f"fma_{tag}", fam, [(big, big), (other, Z), (other, Z)])
        # a lane's running sum: units 0 and 32 share a lane at every start
        _units(f"lane_{tag}", fam, [(big, Z), (other, Z), (other, Z)] + _filler(29) + [(big, Z)])
        # the butterfly: units 0 and 16 meet in its first step at start 0
        _units(f"butterfly_{tag}", fam, [(big, Z), (other, Z), (other, Z)] + _filler(13) + [(big, Z)])
    # +inf and -inf in two units: NaN; the fp64 dot is negative
    _units("nan", fam, [(big, big), ((-2e36, 100.0), (-2.5e36, 100.0))])
    # sum|x| = 6e38 rounds up to inf: the band is inf
    fam.plant("yabs_inf", [(3e38, 1e-10), (-3e38, 2e-10)])
    return fam


def subnormal_family(rng, wmax_col=None):
    """Every weight below 2^-126 (max|w| < 7.8e-39: the fp32 band was 0).  wmax_col: one more column of that weight, read by
    no row (max|w| in [1e-38, 1e-31]: the fp32 band was subnormal), and ordinary rows on weights near 2^-119, which that
    band decides."""
    s = 2.0 ** -149
    ord_unit = s if wmax_col is None else 2.0 ** -130
    fam = Family(rng.integers(1000, 4000, N_ORD_COLS) * ord_unit * np.where(rng.random(N_ORD_COLS) < 0.5, -1, 1), 2.0 ** 100)
    a = 2.0 ** 100
    for i, (x0, x1, w0, w1) in enumerate([(a, -2 * a, 21.375, 10.625),        # the second row of the issue's table
                                          (-a, 2 * a, 21.375, 10.625),        # mirrored values
                                          (a, -2 * a, -21.375, -10.625),      # mirrored weights
                                          (-2 * a, a, 10.625, 21.375),        # swapped pairs
                                          (a, -2 * a, 41.375, 20.625),
                                          (2.0 ** 110, -2.0 ** 111, 1001.375, 500.625)]):
        fam.plant(f"pair_{i}", [(x0, w0 * s), (x1, w1 * s)])
    fam.plant("pair_exact", [(a, 21.0 * s), (-2 * a, 10.5 * s)])              # rounds 10.5 to 10: fp32 +2^-49, fp64 0
    fam.plant("many", [(a * (1 + (k % 3) / 4), (37.375 + 3 * k) * s * (-1) ** k) for k in range(70)])
    if wmax_col is not None:
        fam.w.append(wmax_col)
    return fam


def beyond_family(rng):
    """Weights beyond fp32 (+-inf shadows) and NaN: max|w32| is inf, the band is inf, every non-empty row is recomputed."""
    fam = Family(rng.uniform(0.5, 1.5, N_ORD_COLS) * np.where(rng.random(N_ORD_COLS) < 0.5, -1, 1), 1.0)
    pinf, ninf, nan = fam.col(1e39), fam.col(-3.5e38), fam.col(np.nan)
    c = [fam.col(1.0) for _ in range(8)]
    fam.kinds["touch_pinf"] = ([c[0], pinf, c[1]], [1.0, 0.5, -4.0])
    fam.kinds["touch_ninf"] = ([ninf, c[2]], [0.25, 1.0])
    fam.kinds["touch_both"] = ([pinf, ninf, c[3]], [1.0, 1.0, 1.0])                 # fp32 +inf - inf: NaN
    fam.kinds["touch_nan"] = ([nan, c[4], c[5]], [1.0, 1.0, -0.5])
    fam.kinds["pad_inf"] = ([c[6], pinf], [2.0, 1e-21])                             # the inf column holds a filtered 0
    fam.kinds["all_filtered"] = ([c[7], pinf, ninf], [1e-21, 5e-21, -1e-25])        # yabs 0: the band is inf * 0
    return fam


def nan_family(rng):
    """A NaN weight with a finite max|w32|: only the rows that read it are recomputed."""
    fam = Family(rng.uniform(0.5, 1.5, N_ORD_COLS) * np.where(rng.random(N_ORD_COLS) < 0.5, -1, 1), 1.0)
    nan = fam.col(np.nan)
    c = [fam.col(1.0) for _ in range(3)]
    fam.kinds["touch_nan"] = ([nan, c[0], c[1]], [1.0, 1.0, -0.5])
    fam.kinds["nan_padding"] = ([c[2], nan], [-2.0, 1e-22])
    return fam


FAMILIES = {
    "overflow": overflow_family,
    "subnormal": subnormal_family,
    "band_subnormal": lambda rng: subnormal_family(rng, wmax_col=1e-35),
    "beyond": beyond_family,
    "nan": nan_family,
}


def ordinary_rows(rng, fam, n):
    """Rows of 1..70 pairs of dyadic values on the ordinary columns that the band decides at every start lane."""
    w = np.asarray(fam.w, np.float64)
    out = []
    for _ in range(4):
        if len(out) >= n:
            break
        cand = []
        for _ in range(2 * n):
            L = int(rng.choice([1, 2, 3, 5, 8, 13, 31, 64, 65, 70]))
            cols = np.sort(rng.choice(N_ORD_COLS, size=L, replace=False))
            cand.append((cols, (rng.choice([0.25, 0.5, 1.0], size=L) * fam.ord_scale).astype(np.float32)))
        if np.isinf(M.shadow_max(M.shadow(w))):
            out += cand                                          # an infinite band: nothing is decided
        else:
            ok = np.all(M.decide_starts(cand, w) != M.RECOMPUTE, axis=1)
            out += [r for r, k in zip(cand, ok) if k]
    assert len(out) >= n, "too few ordinary rows outside the band"
    return out[:n]


def build(name):
    """(data, w, kind of every row ('' ordinary, 'empty', or the planted kind), decisions (N, 32), exact signs (N,))"""
    rng = np.random.default_rng(list(FAMILIES).index(name) + 101)
    fam = FAMILIES[name](rng)
    names = list(fam.kinds)
    ords = iter(ordinary_rows(rng, fam, N_ROWS))
    rows, kind = [], []
    for i in range(N_ROWS):
        r = i % 32
        if r == 0:
            k = names[(i // 32) % len(names)]                     # lane 0 in every block size
        elif r in (7, 19):
            k = names[(i // 32 + r) % len(names)]                 # copies elsewhere
        elif r in (3, 4, 25):
            k = "empty"
        else:
            k = ""
        kind.append(k)
        rows.append(([], []) if k == "empty" else (fam.kinds[k] if k else next(ords)))
    w = np.asarray(fam.w, np.float64)
    dim = w.size
    rp = np.concatenate([[0], np.cumsum([len(c) for c, _ in rows])]).astype(np.int64)
    col = np.concatenate([np.asarray(c, np.int32) for c, _ in rows])
    val = np.concatenate([np.asarray(v, np.float32) for _, v in rows])
    lab = np.where(rng.random(N_ROWS) < 0.5, -1, 1).astype(np.int8)
    data = data_from_csr(rp, col, val, lab, dim)
    dec = M.decide_starts(rows, w)
    exact = np.array([M.exact_sign(c, v, w) for c, v in rows])
    return data, w, np.array(kind), dec, exact


@pytest.fixture(scope="module", params=list(FAMILIES))
def family(request):
    data, w, kind, dec, exact = build(request.param)
    # the model's decisions are right wherever a row starts, and every planted row at lane 0 goes to the row fold
    assert np.all((dec == M.RECOMPUTE) | (dec == exact[:, None]))
    planted = (kind != "") & (kind != "empty")
    assert np.all(dec[planted, 0] == M.RECOMPUTE)
    if request.param != "beyond":
        assert np.all(dec[kind == ""] != M.RECOMPUTE)                # ordinary rows stay on the fast path
    ctx, orc = make_pair(data, lam=0.0)
    # the fp64 sums of the oracle have the exact signs: the designs leave no room for a summation order
    np.testing.assert_array_equal(orc.forward(w, np.arange(N_ROWS, dtype=np.int32)), -exact.astype(np.float64))
    S = ctx.info()["sm_count"]
    print(f"{request.param}: {int(planted.sum())} planted rows, lane-0 decisions "
          f"{dict(zip(*np.unique(dec[planted, 0], return_counts=True)))}; device {ctx.info()['name']}, {S} SMs")
    yield request.param, data, w, kind, dec, exact, ctx, orc, S
    ctx.close()


def n_units(data):
    return (np.diff(data.row_ptr) + 1) // 2


def expected_recomputes(data, dec, ids, S):
    """Rows of the pass [data rows ids, in order] that the band sends to the row fold."""
    u = n_units(data)[ids]
    if ids.size < MIN_STREAM_ROWS:
        return 0
    start = M.pass_starts(u, S) % 32
    return int(np.sum((u > 0) & (dec[ids, start] == M.RECOMPUTE)))


def host_ids(row_begin, row_end, key, lo, hi):
    from distributed_sgd_b200.native import host_lib
    h, n = host_lib(), row_end - row_begin
    return (row_begin + np.fromiter((h.dsgd_feistel_pos(p, n, key) for p in range(lo, hi)), dtype=np.int64,
                                    count=hi - lo)).astype(np.int32)


def hinge_correct(preds, labels):
    return int(np.sum(1 - labels * preds)), int(np.sum(preds == labels))


class Recomputes:
    """The rows each call sent to the row fold, against the model's count; checked after the call's results, so that a
    wrong decision shows as such."""

    def __init__(self, ctx):
        self.ctx, self.seen = ctx, []

    def __call__(self, expect, fn, *args):
        before = self.ctx.stream_exact_rows()
        out = fn(*args)
        self.seen.append((fn.__name__, self.ctx.stream_exact_rows() - before, expect))
        return out

    def check(self):
        assert all(got == want for _, got, want in self.seen), self.seen


@pytest.mark.parametrize("resident", [False, True])
def test_every_streamed_form(family, resident):
    from oracle import cw as CWO
    name, data, w, kind, dec, exact, ctx, orc, S = family
    lab = data.label.astype(np.int64)
    counted = Recomputes(ctx)
    wa = None if resident else w
    if resident:
        ctx.set_weights(w)
    ids = np.arange(N_ROWS, dtype=np.int32)
    want = expected_recomputes(data, dec, ids, S)
    p_ref = orc.forward(w, ids)
    # forward on a list
    ctx.set_class_weights(1.0, 1.0)
    preds = counted(want, ctx.forward, ids, wa)
    np.testing.assert_array_equal(preds, p_ref)
    np.testing.assert_array_equal(ctx.forward(ids[:N_KROWS], wa), preds[:N_KROWS])            # k_rows
    # the contiguous form
    h_ref, c_ref = hinge_correct(p_ref, lab)
    h, c, _ = counted(want, ctx.eval_counts, 0, N_ROWS, wa)
    assert (h, c) == (h_ref, c_ref)
    loss_sum, c2, _ = counted(want, ctx.eval_sums, 0, N_ROWS, wa)
    assert (loss_sum, c2) == (float(h_ref), c_ref)
    assert ctx.eval_counts(0, N_KROWS, wa)[:2] == hinge_correct(p_ref[:N_KROWS], lab[:N_KROWS])
    # a device-drawn sample (a list pass in the draw's order)
    k = N_ROWS - 600
    sid = host_ids(0, N_ROWS, KEY, 0, k)
    want_s = expected_recomputes(data, dec, sid, S)
    hs, cs = hinge_correct(p_ref[sid], lab[sid])
    assert counted(want_s, ctx.eval_sampled_counts, 0, N_ROWS, KEY, 0, k, wa)[:2] == (hs, cs)
    assert counted(want_s, ctx.eval_sampled_sums, 0, N_ROWS, KEY, 0, k, wa)[:2] == (float(hs), cs)
    # the unweighted gradient (scatter form)
    g_ref, _ = orc.gradient(w, ids)
    np.testing.assert_array_equal(counted(want, ctx.gradient, ids, wa), g_ref)
    np.testing.assert_array_equal(ctx.gradient(ids[:N_KROWS], wa), orc.gradient(w, ids[:N_KROWS])[0])
    # the per-class form: the evaluation and the gradient under class weights
    ctx.set_class_weights(*CW)
    try:
        ce = counted(want, ctx.eval_class, 0, N_ROWS, wa)
        sums_ref, counts_ref = CWO.eval_class(orc, w, ids)
        assert [ce.loss_pos, ce.loss_neg] == list(sums_ref)
        assert [ce.correct_pos, ce.correct_neg, ce.n_pos, ce.n_neg] == list(counts_ref)
        g_cw = counted(want, ctx.gradient, ids, wa)
        np.testing.assert_array_equal(g_cw, CWO.gradient(orc, w, ids, *CW)[0])
        np.testing.assert_array_equal(ctx.gradient(ids[:N_KROWS], wa), CWO.gradient(orc, w, ids[:N_KROWS], *CW)[0])
    finally:
        ctx.set_class_weights(1.0, 1.0)
    counted.check()
    # the count is the planted rows', and in the families with finite weights no ordinary row is among them
    if name != "beyond":
        start = M.pass_starts(n_units(data)[ids], S) % 32
        assert np.all(dec[ids[kind == ""], start[kind == ""]] != M.RECOMPUTE)
    else:
        assert want == int(np.sum(n_units(data) > 0))


def test_a_pass_of_32_row_blocks(family):
    """The data set repeated past the first pass with 32-row blocks: dynamically claimed blocks, the half-size tail."""
    name, data, w, kind, dec, exact, ctx, orc, S = family
    counted = Recomputes(ctx)
    b32 = split_bounds(S)[2]
    base = np.arange(N_ROWS // 32 * 32, dtype=np.int32)
    reps = -(-b32 // base.size) + 1
    ids = np.tile(base, reps)
    assert ids.size > b32 and np.all(ids[::32] % 32 == 0)                # every 32nd position holds a planted row
    want = expected_recomputes(data, dec, ids, S)
    p_ref = np.tile(orc.forward(w, base), reps)
    np.testing.assert_array_equal(counted(want, ctx.forward, ids, w), p_ref)
    g_ref, _ = orc.gradient(w, ids)
    np.testing.assert_array_equal(counted(want, ctx.gradient, ids, w), g_ref)
    counted.check()
