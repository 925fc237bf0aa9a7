"""Planted-margin layouts for the edge tests of the topic kernels (tests/test_host_topic_edges.py checks what each layout
reaches on the host; tests/test_gpu_topic_edges.py runs them on the device).

* Rows.  A row holds x = 1.0 (exact in fp32) on one column c, so topic t's margin on it is filt(W[t, c]), and with an
  intercept fl(filt(W[t, c]) + filt(W[t, dim])).  A NaN row holds 1.0 on the two columns `na` < `nb`; the topics that are
  to score NaN there carry +inf and -inf on them.  A row with no non-zero scores 0 (its intercept with one).
* Margins from the host only.  `host_margins` folds the CSR with tests/row_fold_model.py, the device's one summation
  order; no reference here reads a margin the device computed.
* Runs.  A request's positions are a list of row ids with repeats, so runs of equal margins sit at exact places of each
  topic's sorted segment; rows sharing a weight value make one run with mixed has-topic bytes.
* Topics.  Each topic's rows are chosen so that its best F1 candidate, status and threshold branch are the planted ones.
"""
from dataclasses import dataclass, field

import numpy as np

from row_fold_model import filt, fold_row, window_products

INF = float("inf")
DBL_MAX = float(np.finfo(np.float64).max)
TUNE_KEYS = 1 << 27          # keys per topic group of dsgd_tune_topic_thresholds: G = max(1, min(T, 2^27 // n))
TILE = 256 * 8               # positions per tile of the tuning scan: 256 threads of 8 consecutive positions


def tune_group(n: int, T: int) -> int:
    """topics per group of a tuning request over n positions"""
    return max(1, min(T, TUNE_KEYS // n))


def host_margins(data, W, rows, intercept: bool) -> np.ndarray:
    """[T, len(rows)] margins of the listed rows by the row fold model (and the intercept's fl add)"""
    rows = np.asarray(rows, dtype=np.int64)
    W = np.asarray(W, dtype=np.float64)
    out = np.empty((W.shape[0], rows.size))
    with np.errstate(invalid="ignore", over="ignore"):
        for t, w in enumerate(W):
            m = fold_row(window_products(data.row_ptr, data.col, data.val, w, rows))
            out[t] = m + filt(w[data.dim]) if intercept else m
    return out


def same_bits(a, b) -> bool:
    """equal fp64 arrays bit for bit, NaN matching NaN (the device's NaN has another sign bit than numpy's)"""
    a, b = np.asarray(a, dtype=np.float64), np.asarray(b, dtype=np.float64)
    na, nb = np.isnan(a), np.isnan(b)
    return a.shape == b.shape and np.array_equal(na, nb) and np.array_equal(a[~na].view(np.int64), b[~nb].view(np.int64))


@dataclass
class Layout:
    data: object                 # Data with its topic CSR
    W: np.ndarray                # [T, wdim]
    ids: np.ndarray              # int32 positions (row ids, repeats allowed)
    intercept: bool
    fbr: float = 0.0
    marks: dict = field(default_factory=dict)   # what the planted topics are meant to reach

    @property
    def T(self) -> int:
        return self.W.shape[0]

    def row_margins(self) -> np.ndarray:
        """[T, n_rows] host margins of every row"""
        return host_margins(self.data, self.W, np.arange(self.data.n_rows), self.intercept)

    def margins(self) -> np.ndarray:
        """[T, positions] host margins of the request"""
        return self.row_margins()[:, self.ids]

    def has(self) -> np.ndarray:
        """bool [positions, T]"""
        return self.data.topics.indicator()[self.ids]


def _data(cols, dim, has_rows):
    """Data of rows holding 1.0 on the listed columns, with the topics of the bool [rows, T] array has_rows"""
    from distributed_sgd_b200.utils.dataset import Data, Topics
    rp = np.zeros(len(cols) + 1, dtype=np.int64)
    rp[1:] = np.cumsum([len(c) for c in cols])
    col = np.array([c for cs in cols for c in cs], dtype=np.int32)
    label = np.where(np.arange(len(cols)) % 3 == 0, 1, -1).astype(np.int8)
    topics = Topics.from_indicator(has_rows, [f"T{t}" for t in range(has_rows.shape[1])])
    return Data(rp, col, np.ones(col.size, dtype=np.float32), label, dim, topics=topics)


def _positions(counts, seed):
    """row r repeated counts[r] times, shuffled (the sort places the runs, not the list order)"""
    ids = np.repeat(np.arange(len(counts)), counts).astype(np.int32)
    return np.random.default_rng(seed).permutation(ids).astype(np.int32)


# ---- the tuning scan's thread and tile edges ------------------------------------------------------------------------------

# run ends: thread edges 8q - 1 and 8q, tile edges 2048q - 1 .. 2048q + 1
TILE_ENDS = (7, 8, 15, 2046, 2047, 2048, 2049, 4095, 4096)


def tune_tiles() -> Layout:
    """Runs of equal margins ending at the sorted positions TILE_ENDS, then one run of 4203 positions (4097 .. 8299, with
    tile 3 wholly inside it) made of twelve rows of one level with mixed has-topic bytes, three short runs and a NaN run
    of 37 positions at the end.  Levels (k - 6) / 2 of run k, so the signs and a run at 0 are in it.
      topics 0 .. 8: the rows up to TILE_ENDS[t] (best candidate: the run ending there, F1 = 1)
      topic 9: the rows up to 4096 and every other row of the long run (best: the long run's end)
      topic 10: descending levels, random rows; topic 11: ascending levels, random rows
      topic 12: every row, NaN rows included (best: the last candidate, tau = +inf)
      topic 13: every other row of the long run alone (best: the long run's end)"""
    lengths = [TILE_ENDS[0] + 1] + list(np.diff(TILE_ENDS))
    runs = [[n] for n in lengths]                                   # a run: its rows' repeat counts
    runs[3] = [677, 677, 677]                                       # 2031 positions in three rows
    runs.append([350] * 11 + [353])                                 # the long run
    runs += [[1], [2], [3]]
    long_run = 9
    level_rows = [(k, c) for k, run in enumerate(runs) for c in run]   # (run, count) per row
    n_level = len(level_rows)
    nan_counts = [20, 17]
    na, nb = n_level, n_level + 1
    dim = n_level + 2
    cols = [(r,) for r in range(n_level)] + [(na, nb)] * len(nan_counts)
    run_of = np.array([k for k, _ in level_rows])
    level = (run_of - 6) * 0.5
    ends = np.cumsum([sum(r) for r in runs]) - 1
    assert tuple(ends[:len(TILE_ENDS)]) == TILE_ENDS and ends[long_run] == 8299
    T = 14
    W = np.zeros((T, dim))
    W[:, :n_level] = level
    W[10, :n_level] = -level
    W[:, na], W[:, nb] = INF, -INF
    n_rows = n_level + len(nan_counts)
    has = np.zeros((n_rows, T), dtype=bool)
    for t in range(len(TILE_ENDS)):
        has[:n_level, t] = run_of <= t
    in_long = np.flatnonzero(run_of == long_run)
    has[:n_level, 9] = run_of <= 8
    has[in_long[::2], 9] = True
    rng = np.random.default_rng(11)
    has[:, 10] = rng.random(n_rows) < 0.4
    has[:, 11] = rng.random(n_rows) < 0.3
    has[:, 12] = True
    has[in_long[1::2], 13] = True
    counts = [c for _, c in level_rows] + nan_counts
    marks = {"end_at": {**{t: e for t, e in enumerate(TILE_ENDS)}, 9: 8299, 13: 8299},
             "long_run": (4097, 8299), "nan_positions": sum(nan_counts), "last_candidate": 12}
    return Layout(_data(cols, dim, has), W, _positions(counts, 1), False, 0.0, marks)


# ---- the tuning's value edges ---------------------------------------------------------------------------------------------

NEXT_UP, NEXT_DOWN = float(np.nextafter(1.0, INF)), float(np.nextafter(1.0, -INF))
VALUE_COUNTS = [3, 1, 2, 2, 4, 1, 3, 2, 5, 1, 2, 3]   # positions of the twelve level rows; then two NaN rows, 2 and 1
VALUE_FBR = 0.5
VALUE_TOPICS = ("neg_inf_chosen", "adjacent_doubles", "huge_neighbours", "inf_last_group", "inf_only", "no_positive",
                "below_fbr", "fbr_equal", "all_nan")


def tune_values(intercept: bool) -> Layout:
    """One topic per threshold branch, at fbr = 0.5 (its weights over the twelve level rows, then na, nb):
      neg_inf_chosen: the rows at -inf; the midpoint of -inf and c_1 is -inf, so tau falls back to c_1
      adjacent_doubles: the rows at or below 1.0, next margin nextafter(1.0): the midpoint rounds to 1.0, tau = c_1
      huge_neighbours: the rows at or below 1e308, next margin DBL_MAX: the halves' sum is finite, the plain sum is not
      inf_last_group: every row, two rows at +inf: best is the +inf group, tau = +inf counts only the rows below it
      inf_only: +inf on every level row, NaN on the NaN rows: one candidate, at +inf; the level rows are positive
      no_positive: no row (status 1); below_fbr: best F1 0.4 (status 2); fbr_equal: best F1 exactly 0.5 (status 0)
      all_nan: -inf everywhere; with the intercept's +inf every margin is NaN (status 3), without it one -inf group"""
    T = len(VALUE_TOPICS)
    n_level = len(VALUE_COUNTS)
    na, nb = n_level, n_level + 1
    dim = n_level + 2
    W = np.zeros((T, dim + intercept))
    W[0, :dim] = [-INF, 0.5, 1.0, 1.5, 2.0, -INF, 2.5, 3.0, 3.5, 4.0, 4.5, 5.0, 0.25, 0.25]
    W[1, :dim] = [NEXT_DOWN, 1.0, -3.0, 2.0, 5.0, 7.0, 1.0, 9.0, 11.0, NEXT_UP, 13.0, 15.0, 8.0, 8.0]
    W[2, :dim] = [-1e308, 1e308, DBL_MAX, INF, -5.0, 1.0, 2.0, 3.0, 4.0, 1e308, DBL_MAX, -1e308, 0.0, 0.0]
    W[3, :dim] = [1.0, 2.0, 3.0, 4.0, INF, -1.0, -2.0, 0.5, INF, 6.0, 7.0, 8.0, 0.125, 0.125]
    W[4, :dim] = [INF] * n_level + [INF, -INF]
    W[5, :dim] = [-2.0, -1.0, 0.0, 1.0, 2.0, -0.0, -0.5, 0.5, 3.0, -3.0, 0.0, 1.0, -0.25, 0.0]
    W[6, :dim] = [-4.0, -3.0, -2.0, -1.0, 1.0, 2.0, 3.0, 4.0, 5.0, 6.0, 7.0, 8.0, 4.5, 4.5]
    W[7, :dim] = [5.0, 6.0, -3.0, -2.0, 7.0, 8.0, 9.0, -1.0, 10.0, 11.0, 12.0, 13.0, 7.0, 7.0]
    W[8, :dim] = -INF
    if intercept:
        W[8, dim] = INF
    cols = [(r,) for r in range(n_level)] + [(na, nb)] * 2
    n_rows = n_level + 2
    has = np.zeros((n_rows, T), dtype=bool)
    has[[0, 5], 0] = True
    has[[0, 1, 2, 6], 1] = True
    has[[0, 1, 4, 5, 6, 7, 8, 9, 11, 12, 13], 2] = True        # every row whose margin is at most 1e308
    has[:, 3] = True
    has[:n_level, 4] = True
    has[3, 6] = True                                            # after 6 positions, 2 of its own: F1 = 4 / 10
    has[7, 7] = True                                            # after 4 positions, 2 of its own: F1 = 4 / 8
    has[:, 8] = True
    counts = VALUE_COUNTS + [2, 1]
    marks = {"n": sum(counts), "inf_rows": VALUE_COUNTS[4] + VALUE_COUNTS[8]}
    return Layout(_data(cols, dim, has), W, _positions(counts, 2), intercept, VALUE_FBR, marks)


# ---- the topic groups of a tuning request ---------------------------------------------------------------------------------

def tune_groups(T: int, n_pos: int, n_rows: int = 400, seed: int = 5) -> Layout:
    """T topics over n_pos positions drawn from n_rows single-column rows.  The weights take a few values (runs of ties),
    topic t's rows are random at a share that varies with t, and the last topic is planted apart (its own weights and
    rows), so a last group of one topic has a result of its own."""
    rng = np.random.default_rng(seed)
    dim = n_rows
    W = rng.integers(-6, 7, size=(T, dim)) * 0.25
    W[-1] = rng.permutation(dim) * 0.5 - dim / 4
    share = 0.05 + 0.4 * (np.arange(T) % 7) / 7
    has = rng.random((n_rows, T)) < share
    has[:, -1] = W[-1] < 10.0                                   # the lowest rows: a tuned prefix
    has[0, -1] = False
    ids = rng.integers(0, n_rows, size=n_pos).astype(np.int32)
    return Layout(_data([(r,) for r in range(n_rows)], dim, has), W, ids, False)


# ---- ranking at every warp shape ------------------------------------------------------------------------------------------

RANK_TS = (2, 31, 32, 33, 63, 64, 65, 1023, 1024)
RANK_PATTERNS = ("all_tied", "same_lane", "adjacent_even", "adjacent_odd", "infs", "few_values", "distinct")


def rank_ks(T: int):
    return sorted({1, min(T, 5), min(T, 32)})


def slice_k(words, sums, K: int, k: int):
    """the ranking words and sums of k <= K from those of K: the row words, hits 1..k and the limbs of A, B, C_1..C_k"""
    return np.concatenate([words[:8 + k], words[8 + K:8 + K + 7 * (2 + k)]]), sums[:2 + k]


def rank_layout(T: int, intercept: bool, seed: int = 0) -> Layout:
    """One column per pattern of RANK_PATTERNS (its margins over the topics):
      all_tied: every topic 0.75; same_lane: (t mod 32) / 2 - 4, so t ties with t + 32; adjacent_even: t ties with t + 1
      for even t; adjacent_odd: for odd t (31 with 32, 63 with 64); infs: +inf at t = 0 mod 3, -inf at 1 mod 3;
      few_values: five values, ties everywhere; distinct: no tie.
    A NaN row scores NaN at topic T - 1 only (the last lane's highest mask bit); a row with no non-zero scores 0.
    On each pattern column: a row with every topic, a row with exactly a tied set, a random row and a row without topics.
    The intercept (0.5, 0.75 at t = 3 mod 4) keeps the same-lane ties.  Positions: every row once, shuffled, and a few
    again."""
    rng = np.random.default_rng(1000 * T + seed)
    t = np.arange(T)
    P = len(RANK_PATTERNS)
    na, nb = P, P + 1
    dim = P + 2
    W = np.zeros((T, dim + intercept))
    W[:, 0] = 0.75
    W[:, 1] = (t % 32) * 0.5 - 4.0
    W[:, 2] = (t // 2) * 0.25 - 2.0
    W[:, 3] = ((t + 1) // 2) * 0.25 - 2.0
    W[:, 4] = np.where(t % 3 == 0, INF, np.where(t % 3 == 1, -INF, rng.integers(-4, 5, size=T) * 0.5))
    W[:, 5] = rng.integers(-2, 3, size=T) * 0.5
    W[:, 6] = rng.permutation(T) * 0.125 - T / 16
    W[:, na] = rng.integers(-4, 5, size=T) * 0.5
    W[:, nb] = rng.integers(-4, 5, size=T) * 0.5
    W[T - 1, na], W[T - 1, nb] = INF, -INF
    if intercept:
        W[:, dim] = np.where(t % 4 == 3, 0.75, 0.5)
    tied = [t,                                                          # all_tied
            t[t % 32 == 3 % T],                                        # same_lane: lane 3 (lane 1 at T = 2)
            t[t // 2 == min(2, (T - 1) // 2)],                          # adjacent_even: {4, 5}
            t[(t + 1) // 2 == min(16, T // 2)],                        # adjacent_odd: {31, 32}
            t[t % 3 == 0],                                             # infs: the +inf topics
            t[W[:, 5] == W[:, 5].min()],                               # few_values: the top tie
            t[W[:, 6].argsort()[:3]]]                                  # distinct: the top three
    cols, sets = [], []
    for p in range(P):
        for s in (t, tied[p], t[rng.random(T) < 0.3], t[:0]):
            cols.append((p,))
            sets.append(s)
    cols.append((4,))                                                   # infs again: exactly the -inf topics
    sets.append(t[t % 3 == 1])
    for s in (t, t[rng.random(T) < 0.3]):                               # NaN rows
        cols.append((na, nb))
        sets.append(s)
    for s in (t, t[:1], t[-1:]):                                        # rows with no non-zero
        cols.append(())
        sets.append(s)
    has = np.zeros((len(cols), T), dtype=bool)
    for r, s in enumerate(sets):
        has[r, s] = True
    n_rows = len(cols)
    ids = np.concatenate([rng.permutation(n_rows), rng.integers(0, n_rows, size=6)]).astype(np.int32)
    marks = {"tied": {name: tied[p] for p, name in enumerate(RANK_PATTERNS)}, "row_of": {name: 4 * p for p, name in
                                                                                         enumerate(RANK_PATTERNS)}}
    return Layout(_data(cols, dim, has), W, ids, intercept, marks=marks)


def rank_thresholds(lay: Layout):
    """thresholds equal to planted margins: the same_lane row's (finite) and the infs row's (+-inf and finite)"""
    m = lay.row_margins()
    return [m[:, lay.marks["row_of"][name]].copy() for name in ("same_lane", "infs")]
