"""The planted layouts of tests/topic_edges_data.py reach what they claim, on the host: their margins are the intended
values, the numpy models and the C checkers agree on every layout, and each tuning status, each threshold branch, each
tile-edge candidate and each kind of ranking tie occurs.  tests/test_gpu_topic_edges.py runs the same layouts on the
device, so its coverage can be checked here without a GPU."""
import numpy as np
import pytest

import topic_edges_data as E
from oracle import topic_rank as rank_oracle
from oracle import topic_thresh as thresh_oracle
from oracle import topics as topics_oracle
from oracle.oracle import Oracle
from topic_ranking_model import order, topic_ranking
from topic_thresholds_model import BELOW_FBR, NO_MARGIN, NO_POSITIVE, TUNED, midpoint, thresholded_words, tune
from topics_model import topic_words


def _orc(lay):
    d = lay.data
    return Oracle(d.row_ptr, d.col, d.val, d.label, d.dim, 2.0 ** -6)


def _checker_tune(lay, m):
    d = lay.data
    return thresh_oracle.topic_thresh(_orc(lay), d.topics.ptr, d.topics.ids, lay.T, lay.fbr, idx=lay.ids, margins=m)


def _same(a, b):
    return np.array_equal(a[0].view(np.int64), b[0].view(np.int64)) and np.array_equal(a[1], b[1])


def _sorted_candidates(m):
    return sorted({float(v) + 0.0 for v in m[~np.isnan(m)]})


def _intended(lay):
    """the margin each single-column row is planted to have: filt(W[t, c]) (+ filt of the intercept), exactly"""
    d = lay.data
    dim = d.dim
    Wf = np.where(np.abs(lay.W) > 1e-20, lay.W, 0.0)
    out = {}
    for r in range(d.n_rows):
        cols = d.col[d.row_ptr[r]:d.row_ptr[r + 1]]
        if len(cols) == 1:
            v = Wf[:, cols[0]] + 0.0
        elif len(cols) == 0:
            v = np.zeros(lay.T)
        else:
            continue
        with np.errstate(invalid="ignore"):
            out[r] = v + Wf[:, dim] if lay.intercept else v
    return out


def _all_layouts():
    yield "tiles", E.tune_tiles()
    for icpt in (False, True):
        yield f"values{int(icpt)}", E.tune_values(icpt)
    for T in E.RANK_TS[:7]:
        for icpt in (False, True):
            yield f"rank{T}_{int(icpt)}", E.rank_layout(T, icpt)


@pytest.mark.parametrize("name,lay", list(_all_layouts()), ids=lambda x: x if isinstance(x, str) else "")
def test_host_margins_are_the_planted_values(name, lay):
    with np.errstate(invalid="ignore"):
        m = lay.row_margins()
    for r, v in _intended(lay).items():
        assert E.same_bits(m[:, r], v), (name, r)
    d = lay.data
    nan_rows = [r for r in range(d.n_rows) if d.row_ptr[r + 1] - d.row_ptr[r] == 2]
    for r in nan_rows:                                              # NaN exactly where both +inf and -inf are planted
        na, nb = d.col[d.row_ptr[r]:d.row_ptr[r] + 2]
        planted = (lay.W[:, na] == np.inf) & (lay.W[:, nb] == -np.inf)
        if lay.intercept:                                           # or an infinite sum against an opposite intercept
            with np.errstate(invalid="ignore"):
                s, b = lay.W[:, na] + lay.W[:, nb], lay.W[:, d.dim]
            planted |= np.isinf(s) & np.isinf(b) & (np.sign(s) != np.sign(b))
        assert np.array_equal(np.isnan(m[:, r]), planted), (name, r)


def test_tile_layout_reaches_every_thread_and_tile_edge():
    lay = E.tune_tiles()
    m, has = lay.margins(), lay.has()
    got = tune(m, has)
    assert _same(got, _checker_tune(lay, m))
    thr, words = got
    ends = {}
    for t in range(lay.T):
        rows, P, nan, D, tp, pp, status, j = (int(x) for x in words[8 * t:8 * t + 8])
        assert status == TUNED and nan == lay.marks["nan_positions"] and rows == len(lay.ids)
        c = _sorted_candidates(m[t])
        ends[t] = int(np.sum(m[t] <= c[j])) - 1                     # the chosen group's last sorted position
    for t, e in lay.marks["end_at"].items():
        assert ends[t] == e, (t, ends[t], e)
    assert 2047 in ends.values() and 2048 in ends.values() and 4095 in ends.values()
    # every planted run end is a group end of the ascending topics, and the long run spans tile 3 with mixed bytes
    srt = np.sort(m[0][~np.isnan(m[0])])
    group_ends = set(np.flatnonzero(np.diff(srt) != 0).tolist()) | {srt.size - 1}
    assert set(E.TILE_ENDS) <= group_ends
    lo, hi = lay.marks["long_run"]
    assert lo <= 3 * E.TILE and 4 * E.TILE - 1 <= hi and not any(lo <= e < hi for e in group_ends)
    order_ = np.argsort(m[0], kind="stable")
    assert 0 < has[order_[lo:hi + 1], 13].sum() < hi + 1 - lo
    last = lay.marks["last_candidate"]
    assert words[8 * last + 7] == words[8 * last + 3] - 1 and thr[last] == np.inf


@pytest.mark.parametrize("intercept", [False, True])
def test_value_layout_reaches_every_branch(intercept):
    lay = E.tune_values(intercept)
    m, has = lay.margins(), lay.has()
    got = tune(m, has, lay.fbr)
    assert _same(got, _checker_tune(lay, m))
    thr, words = got
    w = {name: [int(x) for x in words[8 * t:8 * t + 8]] for t, name in enumerate(E.VALUE_TOPICS)}
    tau = dict(zip(E.VALUE_TOPICS, thr))
    cand = {name: _sorted_candidates(m[t]) for t, name in enumerate(E.VALUE_TOPICS)}
    n = lay.marks["n"]
    # -inf chosen: the midpoint of -inf and c_1 is -inf, so tau is c_1
    c = cand["neg_inf_chosen"]
    assert w["neg_inf_chosen"][6:] == [TUNED, 0] and c[0] == -np.inf and c[0] / 2 + c[1] / 2 == -np.inf
    assert tau["neg_inf_chosen"] == c[1] and w["neg_inf_chosen"][4:6] == [4, 4]
    # adjacent doubles: the midpoint rounds to c_j, tau is c_(j+1)
    c, j = cand["adjacent_doubles"], w["adjacent_doubles"][7]
    assert c[j] == 1.0 and c[j + 1] == E.NEXT_UP and c[j] / 2 + c[j + 1] / 2 == 1.0 and tau["adjacent_doubles"] == E.NEXT_UP
    assert E.NEXT_DOWN in c and w["adjacent_doubles"][4:6] == [9, 9]
    # 1e308 and DBL_MAX: the halves' sum is finite (the plain sum is not), and it is tau
    c, j = cand["huge_neighbours"], w["huge_neighbours"][7]
    with np.errstate(over="ignore"):
        assert c[j] == 1e308 and c[j + 1] == E.DBL_MAX and np.isinf(np.float64(c[j]) + np.float64(c[j + 1]))
    assert tau["huge_neighbours"] == midpoint(c[j], c[j + 1]) and c[j] < tau["huge_neighbours"] < c[j + 1]
    # +inf as the chosen last group: tau = +inf predicts only the rows below it
    r = w["inf_last_group"]
    assert r[6:] == [TUNED, r[3] - 1] and tau["inf_last_group"] == np.inf and cand["inf_last_group"][-1] == np.inf
    assert r[4] == r[5] == n - lay.marks["inf_rows"] and r[1] == n
    # +inf as the only non-NaN margin: one candidate, nothing predicted at tau = +inf
    r = w["inf_only"]
    assert r[2] == 3 and r[3] == 1 and r[6:] == [TUNED, 0] and r[4:6] == [0, 0] and tau["inf_only"] == np.inf
    assert w["no_positive"][1] == 0 and w["no_positive"][6] == NO_POSITIVE and tau["no_positive"] == 0.0
    assert w["no_positive"][5] == int(np.sum(m[5] < 0.0)) > 0
    r = w["below_fbr"]
    assert r[6:] == [BELOW_FBR, 0] and r[4:6] == [0, 3] and tau["below_fbr"] == midpoint(*cand["below_fbr"][:2])
    r = w["fbr_equal"]
    assert r[6:] == [TUNED, 2] and (2 * r[4]) / (r[1] + r[5]) == lay.fbr and r[4:6] == [2, 6]
    r = w["all_nan"]
    if intercept:
        assert r[2] == n and r[3] == 0 and r[6:] == [NO_MARGIN, -1] and r[4:6] == [0, 0] and tau["all_nan"] == 0.0
    else:
        assert r[3] == 1 and r[6:] == [TUNED, 0] and r[4:6] == [n, n] and tau["all_nan"] == np.inf
    assert {int(s) for s in words[6::8]} == ({TUNED, NO_POSITIVE, BELOW_FBR, NO_MARGIN} if intercept else
                                             {TUNED, NO_POSITIVE, BELOW_FBR})


def test_group_sizes():
    assert E.tune_group(131_100, 1024) == 1023 and 1024 % 1023 == 1
    assert E.tune_group(1025 * 65_473, 3) == 1 and 1025 * 65_473 > 1 << 26
    assert E.tune_group(1025, 3) == 3


def test_group_layout_agrees_with_the_checker_own_dots():
    lay = E.tune_groups(3, 1025)
    d = lay.data
    m = lay.margins()
    got = tune(m, lay.has())
    assert _same(got, _checker_tune(lay, m))
    own = thresh_oracle.topic_thresh(_orc(lay), d.topics.ptr, d.topics.ids, lay.T, 0.0, W=lay.W, idx=lay.ids)
    assert _same(got, own) and (got[1][6::8] == TUNED).all()


@pytest.mark.parametrize("T", E.RANK_TS)
def test_rank_layout_models_and_checkers_agree_and_ties_are_planted(T):
    for intercept in (False, True) if T < 1000 else (False,):
        lay = E.rank_layout(T, intercept)
        d = lay.data
        m, has = lay.margins(), lay.has()
        orc = _orc(lay)
        K = min(T, 32)
        ref = topic_ranking(m, has, K)
        for k in E.rank_ks(T):
            cw, cs = rank_oracle.topic_rank(orc, d.topics.ptr, d.topics.ids, T, k, idx=lay.ids, margins=m)
            rw, rs = E.slice_k(*ref, K, k)
            assert np.array_equal(cw, rw) and np.array_equal(cs, rs), (T, intercept, k)
        tw = topic_words(m, has)
        assert np.array_equal(topics_oracle.topics(orc, d.topics.ptr, d.topics.ids, T, idx=lay.ids, margins=m), tw)
        for thr in E.rank_thresholds(lay):
            assert not np.isnan(thr).any() and (m == thr[:, None]).any(axis=1).all()
            stand = np.where(m < thr[:, None], -1.0, np.where(m > thr[:, None], 1.0, np.where(np.isnan(m), np.nan, 0.0)))
            got = thresholded_words(m, has, thr)
            chk = topics_oracle.topics(orc, d.topics.ptr, d.topics.ids, T, idx=lay.ids, margins=stand)
            assert np.array_equal(np.delete(got, 8 * T + 2), np.delete(chk, 8 * T + 2)) and got[8 * T + 2] == tw[8 * T + 2]
        w = ref[0]
        assert w[4] > 0 and w[2] > 0 and w[3] > 0                      # rows with every topic, NaN rows, rows without
        # the NaN row scores NaN at topic T - 1 alone; the tie rule decides orders among equal margins
        rm = lay.row_margins()
        nan_cols = np.isnan(rm).any(axis=0)
        assert all(np.flatnonzero(np.isnan(rm[:, r])).tolist() == [T - 1] for r in np.flatnonzero(nan_cols))
        same_lane = across = 0
        for r in range(d.n_rows):
            o = order(rm[:, r])[:K]
            for a, b in zip(o, o[1:]):
                if rm[a, r] == rm[b, r]:
                    assert a < b
                    same_lane += (a & 31) == (b & 31)
                    across += (a & 31) != (b & 31)
        assert across > 0 and (same_lane > 0) == (T > 32)
        if T >= 4:                                                      # several topics tied at +inf, several at -inf
            assert (rm == np.inf).sum(axis=0).max() >= 2 and (rm == -np.inf).sum(axis=0).max() >= 2
