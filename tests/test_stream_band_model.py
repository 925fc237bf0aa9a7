"""The CPU model of the streaming pass's row decision (tests/stream_band_model.py) over the whole fp32 range: whenever the
rule decides a row from its fp32 dot, the sign is the exact sign of the filtered fp64 products.  The earlier rule (an fp32
band, infinite dots decided) is restated beside it, and the sweep must catch it deciding wrongly, so that the sweep reaches
the rows the rule exists for.  No GPU."""
from fractions import Fraction

import numpy as np
import pytest

import stream_band_model as M

F32_MAX = M.FLT_MAX
DIM = 600


def _rand_f32_log(rng, lo, hi, n):
    """fp32 magnitudes log-uniform in [lo, hi] with random signs."""
    v = np.exp(rng.uniform(np.log(lo), np.log(hi), size=n)).astype(np.float32)
    return np.where(rng.random(n) < 0.5, -v, v).astype(np.float32)


def _weights(rng, kind):
    """One weight vector of DIM columns per sweep batch."""
    if kind == "span":                                   # 2^-149 .. FLT_MAX, then beyond fp32, inf and NaN
        w = np.where(rng.random(DIM) < 0.5, -1.0, 1.0) * 2.0 ** rng.uniform(-149, 128, size=DIM)
        w[rng.choice(DIM, 6, replace=False)] = [3.5e38, -1e39, 1e100, np.inf, -np.inf, np.nan]
        return w
    if kind == "span_finite":                             # the same without the columns beyond fp32 (max|w32| finite)
        return np.where(rng.random(DIM) < 0.5, -1.0, 1.0) * 2.0 ** rng.uniform(-149, 128, size=DIM)
    if kind == "near_max":                               # products near FLT_MAX: every overflow site
        return np.where(rng.random(DIM) < 0.5, -1.0, 1.0) * rng.uniform(1.0, 100.0, size=DIM)
    if kind == "subnormal":                              # every |w| below 2^-126: fp32 keeps 1 to 23 bits of each
        return np.where(rng.random(DIM) < 0.5, -1.0, 1.0) * rng.uniform(1.0, 2.0 ** 23, size=DIM) * 2.0 ** -149
    if kind == "tiny":                                   # max|w| below 7.8e-39: the fp32 band was 0
        return np.where(rng.random(DIM) < 0.5, -1.0, 1.0) * rng.uniform(1.0, 4.0e3, size=DIM) * 2.0 ** -149
    if kind == "band_subnormal":                         # max|w| in [1e-38, 1e-31]: the fp32 band was subnormal
        w = np.where(rng.random(DIM) < 0.5, -1.0, 1.0) * rng.uniform(1.0, 2.0 ** 23, size=DIM) * 2.0 ** -149
        w[0] = 10.0 ** rng.uniform(-38, -31)
        return w
    raise KeyError(kind)


def _row_random(rng, w, lo, hi):
    """A row of 1..140 pairs (up to 70 units: one lane adds across three slots) with values log-uniform in [lo, hi]."""
    L = int(rng.choice([1, 2, 3, 4, 7, 16, 63, 64, 65, 66, 67, 130, 140]))
    cols = rng.choice(DIM, size=L, replace=False)
    return cols, _rand_f32_log(rng, lo, hi, L)


def _row_cancel(rng, w, w32max, scale_x, k):
    """A near-cancelling row like those of test_stream_margin_sweep_and_recompute_counter: units (x, x) on columns
    (2j, 2j + 1) with w[2j + 1] = -w[2j], and a last column whose product is k times the row's band.  The weights of the
    pairs are set here (columns 0 .. 2 * 150 - 1 are reserved for them), the target on a column from 300 on."""
    m = int(rng.integers(1, 70))
    js = np.sort(rng.choice(150, size=m, replace=False))
    x = (rng.random(m) + 0.05).astype(np.float32) * np.float32(scale_x)
    xt = np.float32(scale_x * (rng.random() + 0.5))
    cols = np.concatenate([np.stack([2 * js, 2 * js + 1], axis=1).reshape(-1), [300 + int(rng.integers(0, DIM - 300))]])
    vals = np.concatenate([np.repeat(x, 2), [xt]]).astype(np.float32)
    ya = float(np.float32(2 * np.sum(np.abs(x).astype(np.float64)) + abs(float(xt))))
    band = 1.5 * 2.0 ** -24 * max(w32max, 2.0 ** -126) * ya * (((cols.size + 1) // 2 >> 5) + 10)
    w[cols[-1]] = k * band / float(xt) * (1 if rng.random() < 0.5 else -1)
    return cols, vals


def _row_overflow(rng, w):
    """Products near FLT_MAX of both signs, 2..70 units: the fp32 chain overflows in a product, a unit's fma, a lane's sum
    or the butterfly, and the fp64 dot is finite with either sign."""
    L = int(rng.choice([2, 4, 6, 8, 34, 66, 70, 130]))
    cols = rng.choice(DIM, size=L, replace=False)
    mag = np.abs(w[cols])
    x = (rng.uniform(0.3, 1.2, size=L) * F32_MAX / mag).astype(np.float32)
    x = np.where(rng.random(L) < 0.5, -x, x).astype(np.float32)
    x[rng.random(L) < 0.2] = np.float32(1.0)             # small products in between
    return cols, x


def _row_subnormal(rng, w):
    """Two to four pairs of large x on subnormal weights: fp32 rounds each weight by up to 2^-150, not 2^-24 |w|."""
    L = int(rng.integers(2, 5))
    cols = rng.choice(DIM, size=L, replace=False)
    x = (2.0 ** rng.integers(70, 128, size=L) * rng.choice([1.0, -1.0, 1.5, -1.5, 1.25], size=L)).astype(np.float32)
    return cols, x


def _row_subnormal_pair(rng, w):
    """x = (2^a, -2^(a+1)) on weights (m0 2^-149, m1 2^-149) with m0 = 2 m1 + 1/8: the fp64 dot is 2^(a-152), and fp32's
    rounding of the two weights to integers m can give the other sign (the second row of the issue's table, scaled)."""
    a = int(rng.integers(60, 126))
    c0, c1 = rng.choice(DIM, size=2, replace=False)
    m1 = int(rng.integers(1, 2000)) + float(rng.choice([0.5 + 1 / 8, 0.5 - 1 / 8, 0.625, 0.375]))
    s = 1.0 if rng.random() < 0.5 else -1.0
    w[c0], w[c1] = s * (2 * m1 + 0.125) * 2.0 ** -149, s * m1 * 2.0 ** -149
    sx = 1.0 if rng.random() < 0.5 else -1.0
    return np.array([c0, c1]), np.array([sx * 2.0 ** a, -sx * 2.0 ** (a + 1)], np.float32)


def sweep_batches(seed=2024):
    """[(rows, w)]: about 13 000 rows over the fp32 range, each batch with its own weight vector."""
    rng = np.random.default_rng(seed)
    batches = []
    for kind, n, gen in (
            ("span", 1500, lambda w: _row_random(rng, w, 1e-21, F32_MAX)),
            ("span_finite", 1500, lambda w: _row_random(rng, w, 1e-21, F32_MAX)),
            ("near_max", 2500, lambda w: _row_overflow(rng, w)),
            ("subnormal", 1500, lambda w: _row_subnormal(rng, w)),
            ("tiny", 1500, lambda w: _row_subnormal(rng, w)),
            ("tiny", 1000, lambda w: _row_subnormal_pair(rng, w)),
            ("band_subnormal", 1000, lambda w: _row_subnormal(rng, w))):
        w = _weights(rng, kind)
        batches.append((kind, [gen(w) for _ in range(n)], w))
    # near-cancelling rows at k x their band, k from 1e-3 to 1e3, at x and w scales across the range
    for sx, sw in ((1.0, 1.0), (2.0 ** 100, 2.0 ** -140), (2.0 ** -60, 2.0 ** 60), (2.0 ** 60, 2.0 ** 60),
                   (2.0 ** 120, 2.0 ** -135), (2.0 ** -40, 2.0 ** 10)):
        w = np.zeros(DIM)
        w[0:300:2] = (rng.standard_normal(150) + np.sign(rng.standard_normal(150)) * 0.1) * sw
        w[1:300:2] = -w[0:300:2]
        w32max = float(M.shadow_max(M.shadow(w)))
        ks = np.geomspace(1e-3, 1e3, 400)
        batches.append((f"cancel_{sx:g}_{sw:g}", [_row_cancel(rng, w, w32max, sx, k) for k in ks], w))
    return batches


@pytest.fixture(scope="module")
def swept():
    """Per batch: (kind, rows, w, exact signs, decisions at start 0, decisions at a random start, decisions of the earlier rule)."""
    rng = np.random.default_rng(7)
    out = []
    for kind, rows, w in sweep_batches():
        exact = np.array([M.exact_sign(c, v, w) for c, v in rows])
        d0 = M.decide(rows, w)[0]
        ds = M.decide(rows, w, start=rng.integers(0, 32, size=len(rows)))[0]
        dp = M.decide(rows, w, fp32_band=True)[0]
        out.append((kind, rows, w, exact, d0, ds, dp))
    return out


def test_the_two_rows_of_the_issue_and_their_mirrors():
    """An infinite fp32 dot whose fp64 dot has the other sign, and subnormal weights whose fp32 rounding flips the sign:
    the earlier rule decides both wrongly, the rule recomputes both."""
    w = np.zeros(8)
    w[[0, 1, 2, 4]] = 100.0
    x = [2e36, 2e36, -3.3e36, 1.0, -3.3e36, 1.0]
    w2 = np.zeros(8)
    w2[0], w2[1] = 21.375 * 2.0 ** -149, 10.625 * 2.0 ** -149
    for rows, ww, sign in ((([0, 1, 2, 3, 4, 5], x),), w, -1), ((([0, 1], [2.0 ** 100, -2.0 ** 101]),), w2, 1):
        for mirror in (1.0, -1.0):
            r = [(c, list(np.float32(mirror) * np.asarray(v, np.float32))) for c, v in rows]
            assert M.exact_sign(*r[0], ww) == sign * mirror
            dec, d32, t = M.decide(r, ww)
            assert dec[0] == M.RECOMPUTE, (d32, t)
            pdec, pd32, pt = M.decide(r, ww, fp32_band=True)
            assert pdec[0] == -sign * mirror, (pd32, pt)
    # the table's numbers: dot32 = +inf against 9.5e32; dot32 = -2^-49 against 2e-20 with a band scale of 0
    assert np.isposinf(M.decide([([0, 1, 2, 3, 4, 5], x)], w, fp32_band=True)[1][0])
    assert M.decide([([0, 1], [2.0 ** 100, -2.0 ** 101])], w2, fp32_band=True)[1][0] == -2.0 ** -49
    assert np.float32(1.5) * np.float32(2.0 ** -24) * M.shadow_max(M.shadow(w2)) == 0.0


def test_sweep_decides_only_exact_signs(swept):
    n = sum(len(b[1]) for b in swept)
    assert n > 10_000
    for kind, rows, w, exact, d0, ds, dp in swept:
        for d in (d0, ds):
            bad = np.flatnonzero((d != M.RECOMPUTE) & (d != exact))
            assert bad.size == 0, f"{kind}: rows {bad[:5]} decided {d[bad[:5]]}, exact {exact[bad[:5]]}: {rows[bad[0]]}"


def test_sweep_reaches_both_outcomes_and_the_fp32_band_failures(swept):
    """The sweep is not vacuous: in every batch the rule decides rows and recomputes rows, and over the sweep the earlier
    rule decides wrong signs in the overflow and tiny-weight batches.  The batch whose weights go beyond fp32
    has an infinite max|w32|, hence an infinite band: every row is recomputed."""
    wrong = {}
    for kind, rows, w, exact, d0, ds, dp in swept:
        if kind == "span":
            assert np.all(d0 == M.RECOMPUTE) and np.all(ds == M.RECOMPUTE)
        else:
            assert np.any(d0 != M.RECOMPUTE) and np.any(d0 == M.RECOMPUTE), kind
        wrong[kind] = wrong.get(kind, 0) + int(np.sum((dp != M.RECOMPUTE) & (dp != exact)))
    assert wrong["near_max"] > 0 and wrong["tiny"] > 0, wrong
    # where the earlier rule holds, nothing is wrong: near-1 scales and max|w| well above 2^-126
    assert wrong["cancel_1_1"] == 0 and wrong["cancel_1.15292e+18_1.15292e+18"] == 0, wrong


def test_ordinary_rows_are_decided():
    """Rows of values near 1 on weights near 1 are far outside the band, at every start: the fast path stays fast."""
    rng = np.random.default_rng(3)
    w = rng.uniform(0.5, 1.5, size=DIM) * np.where(rng.random(DIM) < 0.5, -1, 1)
    w[:4] = [1.0, 1.0, 1.0, 1.0]
    rows = []
    for _ in range(2000):
        L = int(rng.integers(1, 140))
        rows.append((rng.choice(DIM, size=L, replace=False), rng.uniform(0.25, 2.0, size=L).astype(np.float32)))
    exact = np.array([M.exact_sign(c, v, w) for c, v in rows])
    # the fp64 dots of random rows are rarely within 1e-4 of 0; keep the ones that are not, and assert all are decided
    far = np.array([abs(float(np.dot(v.astype(np.float64), w[c]))) > 1e-3 * np.sum(np.abs(v)) for c, v in rows])
    for start in (None, rng.integers(0, 32, size=len(rows))):
        dec = M.decide(rows, w, start=start)[0]
        assert np.all(dec[far] == exact[far])


def test_fma32_rounds_once():
    """The model's fp32 fma against exact rationals rounded to nearest-even fp32, on products of every scale."""
    rng = np.random.default_rng(5)
    n = 20000
    a = _rand_f32_log(rng, 1e-20, 1e19, n)
    b = _rand_f32_log(rng, 2.0 ** -149, 1e19, n)
    c = (-(a.astype(np.float64) * b) * (1 + rng.uniform(-2.0 ** -20, 2.0 ** -20, size=n))).astype(np.float32)
    c[::3] = _rand_f32_log(rng, 2.0 ** -149, 1e38, n)[::3]
    got = M._fma32(a, b, c)
    for i in range(0, n, 7):
        ex = Fraction(float(a[i])) * Fraction(float(b[i])) + Fraction(float(c[i]))
        lo = np.float32(float(ex))                            # within one fp32 ulp of ex; pick the nearest, ties to even
        cands = [np.nextafter(lo, np.float32(-np.inf)), lo, np.nextafter(lo, np.float32(np.inf))]
        dist = [abs(Fraction(float(v)) - ex) for v in cands]
        best = min(dist)
        near = [v for v, d in zip(cands, dist) if d == best]
        want = near[0] if len(near) == 1 else [v for v in near if (v.view(np.int32) & 1) == 0][0]
        assert got[i] == want, (a[i], b[i], c[i], got[i], want)


def test_yabs_rounds_up_and_overflows_to_inf():
    rows = [([0, 1], [3e38, 3e38]), ([0, 1, 2], [1e-21, 1e-25, -1e-20]), ([0], [np.float32(0.1)]), ([], [])]
    ya = M.yabs(rows)
    assert np.isposinf(ya[0]) and ya[1] == 0.0 and ya[3] == 0.0
    assert float(ya[2]) >= float(np.float32(0.1)) and ya[2] == np.float32(0.1)   # exact: one fp32 value


def test_block_starts_follow_the_work_split():
    """Blocks of 8 rows below 48 * W blocks' worth, halves in the last fifth; every multiple of 32 starts a block."""
    for S in (1, 4, 132):
        for n in (2048, 2049, 5000, 33 * 1000 + 7):
            first = M.block_starts(n, S)
            assert first[0] == 0 and np.all(first <= np.arange(n)) and np.all(np.diff(first) >= 0)
            assert np.all(first[::32] == np.arange(0, n, 32))
            starts = np.unique(first)
            size = np.diff(np.append(starts, n))
            assert set(size[:-1].tolist()) <= {8, 16, 32} and size[-1] <= 32
