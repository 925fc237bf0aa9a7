"""Row data for the hot path: the counterpart of utils/Dataset.scala.

`Data` is the array form of the reference's `Array[(Vec, Int)]` (utils/Dataset.scala:11): CSR with
0-based int32 columns (reference feature key - 1), fp32 values and +/-1 int8 labels.

  * `rcv1(folder, full)` reads the text files the reference reads (utils/Dataset.scala:13-58).
  * `synthetic_rcv1(...)` generates RCV1-shaped rows deterministically from one seed (there is no RCV1
    copy and no network here); the generator is C (csrc/dsgd_host.c) so the full 700 k x 47 236 set takes
    seconds.
  * `Topics` are the rows' topic sets of a multi-label collection: `rcv1(..., topics=True)` reads every qrels line, and
    `synthetic_topics(data, n_topics)` plants topics on existing rows.
"""
from __future__ import annotations

import ctypes as C
import os
from dataclasses import dataclass
from typing import Optional, Tuple

import numpy as np

from .. import native

RCV1_FEATURES = 47236  # utils/Dataset.scala:16


@dataclass(frozen=True)
class Topics:
    """The topics of each row, as a CSR: row r has the topic ids ids[ptr[r]:ptr[r + 1]], strictly ascending, each an index
    into `names`."""
    ptr: np.ndarray   # int64[n_rows + 1]
    ids: np.ndarray   # int32[nnz]
    names: tuple      # str per topic; a topic's index is its position

    def __post_init__(self):
        ptr = np.ascontiguousarray(self.ptr, dtype=np.int64).reshape(-1)
        ids = np.ascontiguousarray(self.ids, dtype=np.int32).reshape(-1)
        names = tuple(self.names)
        object.__setattr__(self, "ptr", ptr)
        object.__setattr__(self, "ids", ids)
        object.__setattr__(self, "names", names)
        if ptr.size < 1 or ptr[0] != 0 or (np.diff(ptr) < 0).any() or int(ptr[-1]) != ids.size:
            raise ValueError("Topics: ptr must start at 0, be monotone and end at the id count")
        if not names or not all(isinstance(n, str) for n in names) or len(set(names)) != len(names):
            raise ValueError("Topics: names must be distinct strings, at least one")
        if ids.size and (ids.min() < 0 or ids.max() >= len(names)):
            raise ValueError(f"Topics: an id outside [0, {len(names)})")
        # strictly ascending within a row: every step inside a row goes up
        inner = np.ones(ids.size, dtype=bool)
        inner[ptr[:-1][np.diff(ptr) > 0]] = False
        if ids.size > 1 and (np.diff(ids)[inner[1:]] <= 0).any():
            raise ValueError("Topics: the ids of a row must be strictly ascending")

    @property
    def n_rows(self) -> int:
        return self.ptr.size - 1

    @property
    def n_topics(self) -> int:
        return len(self.names)

    def rows(self, begin: int, end: int) -> "Topics":
        """The topics of rows [begin, end)."""
        a, b = int(self.ptr[begin]), int(self.ptr[end])
        return Topics(self.ptr[begin:end + 1] - a, self.ids[a:b], self.names)

    def indicator(self) -> np.ndarray:
        """bool[n_rows, n_topics]: row r has topic t."""
        out = np.zeros((self.n_rows, self.n_topics), dtype=bool)
        out[np.repeat(np.arange(self.n_rows), np.diff(self.ptr)), self.ids] = True
        return out

    def labels(self, t: int) -> np.ndarray:
        """int8[n_rows]: +1 when the row has topic t, else -1."""
        has = np.zeros(self.n_rows, dtype=bool)
        has[np.repeat(np.arange(self.n_rows), np.diff(self.ptr))[self.ids == t]] = True
        return np.where(has, 1, -1).astype(np.int8)

    def select(self, names) -> "Topics":
        """Only the named topics, in the given order (a KeyError names one that is missing)."""
        missing = [x for x in names if x not in self.names]
        if missing:
            raise KeyError(f"topics: {missing[0]!r} is not a topic of the data")
        return Topics.from_indicator(self.indicator()[:, [self.names.index(x) for x in names]], names)

    @staticmethod
    def from_indicator(has: np.ndarray, names) -> "Topics":
        has = np.asarray(has, dtype=bool)
        ptr = np.zeros(has.shape[0] + 1, dtype=np.int64)
        np.cumsum(has.sum(axis=1), out=ptr[1:])
        return Topics(ptr, np.nonzero(has)[1].astype(np.int32), tuple(names))


@dataclass
class Data:
    row_ptr: np.ndarray  # int64[n_rows + 1]
    col: np.ndarray      # int32[nnz], 0-based, ascending within a row
    val: np.ndarray      # float32[nnz]
    label: np.ndarray    # int8[n_rows], +1 / -1
    dim: int
    weight: Optional[np.ndarray] = None   # float64[n_rows]: per-row sample weights (finite, >= 0), None: every row weighs 1
    topics: Optional[Topics] = None       # each row's topics (a multi-label set), None: the binary label only

    @property
    def n_rows(self) -> int:
        return len(self.row_ptr) - 1

    @property
    def nnz(self) -> int:
        return int(self.row_ptr[-1])

    def __len__(self) -> int:
        return self.n_rows

    def split_at(self, n: int) -> Tuple["Data", "Data"]:
        """`data.splitAt(n)` (Main.scala:52)."""
        n = max(0, min(int(n), self.n_rows))
        cut = int(self.row_ptr[n])
        wa, wb = (None, None) if self.weight is None else (self.weight[:n], self.weight[n:])
        ta, tb = (None, None) if self.topics is None else (self.topics.rows(0, n), self.topics.rows(n, self.n_rows))
        a = Data(self.row_ptr[:n + 1].copy(), self.col[:cut], self.val[:cut], self.label[:n], self.dim, wa, ta)
        b = Data(self.row_ptr[n:] - cut, self.col[cut:], self.val[cut:], self.label[n:], self.dim, wb, tb)
        return a, b

    def head(self, n: int) -> "Data":
        return self.split_at(n)[0]

    def algorithmic_bytes(self, rows: Optional[np.ndarray] = None) -> int:
        """SURVEY.md 8(d): 8*nnz_i + 16 bytes per sample (col id + fp32 value per non-zero; two row
        pointers, the sample index and the label)."""
        lens = np.diff(self.row_ptr)
        if rows is not None:
            lens = lens[np.asarray(rows, dtype=np.int64)]
        return int(8 * lens.sum() + 16 * lens.size)


def has_sample_weights(*parts: Optional["Data"]) -> bool:
    """Whether any of the given row sets carries per-row sample weights."""
    return any(p is not None and p.weight is not None for p in parts)


def sample_weights_of(*parts: Optional["Data"]) -> np.ndarray:
    """The sample weights of the given row sets end to end, ones for a set without weights (float64)."""
    return np.concatenate([np.ones(p.n_rows, dtype=np.float64) if p.weight is None
                           else np.asarray(p.weight, dtype=np.float64).reshape(-1) for p in parts if p is not None])


def load_sample_weights(path: str, n_rows: int) -> np.ndarray:
    """The sample weights of a `.npy` file: one finite weight >= 0 per row of a set of n_rows rows, as float64."""
    w = np.load(path, allow_pickle=False)
    if w.ndim != 1 or w.size != n_rows:
        raise ValueError(f"sample-weight: {path} holds an array of shape {w.shape}, expected ({n_rows},): one weight per row")
    if not np.issubdtype(w.dtype, np.number) or np.iscomplexobj(w):
        raise ValueError(f"sample-weight: {path} holds {w.dtype} values, expected real numbers")
    w = w.astype(np.float64)
    bad = np.flatnonzero(~(np.isfinite(w) & (w >= 0.0)))
    if bad.size:
        raise ValueError(f"sample-weight: weight {w[bad[0]]!r} of row {int(bad[0])} is not finite and >= 0")
    return w


SAMPLE_WEIGHT_ASYNC = "sample-weight: sample weights belong to sync training; asynchronous (Hogwild) training has none"


def synthetic_rcv1(n_rows: int = 700_000, dim: int = RCV1_FEATURES, seed: int = 0, mean_nnz: float = 94.5,
                   sigma: float = 0.7, max_nnz: int = 2000, zipf_s: float = 1.1, zipf_q: float = 20.0,
                   label_noise: float = 0.1, return_w_star: bool = False):
    """RCV1-shaped synthetic rows (SURVEY.md 8d): density ~0.2 % (mean 94.5 nnz/row, lognormal row
    lengths clipped to [1, 2000]); columns drawn without replacement per row from a Zipf-Mandelbrot
    popularity 1/(rank + q + 1)^s scattered over the id space by a fixed shuffle, sorted ascending;
    values |N(0,1)| row-L2-normalised fp32; labels sign(x.w* + noise) from a planted dense w*."""
    h = native.host_lib()
    p = native.SynthParams(seed, n_rows, dim, mean_nnz, sigma, max_nnz, zipf_s, zipf_q, label_noise)
    row_ptr = np.zeros(n_rows + 1, dtype=np.int64)
    nnz = h.dsgd_synth_row_ptr(C.byref(p), row_ptr.ctypes.data_as(C.c_void_p))
    if nnz < 0:
        raise ValueError("synthetic_rcv1: bad parameters")
    col = np.empty(nnz, dtype=np.int32)
    val = np.empty(nnz, dtype=np.float32)
    label = np.empty(n_rows, dtype=np.int8)
    w_star = np.empty(dim, dtype=np.float64)
    rc = h.dsgd_synth_fill(C.byref(p), row_ptr.ctypes.data_as(C.c_void_p), col.ctypes.data_as(C.c_void_p),
                           val.ctypes.data_as(C.c_void_p), label.ctypes.data_as(C.c_void_p),
                           w_star.ctypes.data_as(C.c_void_p))
    if rc != 0:
        raise MemoryError("synthetic_rcv1: generator failed")
    data = Data(row_ptr, col, val, label, dim)
    return (data, w_star) if return_w_star else data


def synthetic_topics(data: Data, n_topics: int, seed: int = 0) -> Topics:
    """Topics planted on the rows of `data`, named "T0", "T1", ...: one planted vector w*_t per topic, and row r has topic t
    when x_r . w*_t plus noise is above the quantile that leaves a share p_t of the rows above it.  The shares are skewed as
    in RCV1: p_t = max(0.35 / (t + 1)^0.9, 0.004), a few popular topics and many rare ones.  The vectors are random
    combinations of 32 shared directions, so that topics correlate.  Every topic has a positive among the first 80 % of the
    rows (the train share of a 0.8 split): where the threshold leaves none, that share's top-scored row gets it.  numpy only,
    deterministic from the seed."""
    n, T = data.n_rows, int(n_topics)
    if T < 1 or n < 2:
        raise ValueError("synthetic_topics: needs at least one topic and two rows")
    rng = np.random.default_rng(seed)
    K = 32
    B = rng.standard_normal((data.dim, K)).astype(np.float32)
    A = rng.standard_normal((K, T))
    Z = np.zeros((n, K), dtype=np.float64)   # X B, row by row in chunks of about 2^20 non-zeros
    lens = np.diff(data.row_ptr)
    r0 = 0
    while r0 < n:
        r1 = int(np.searchsorted(data.row_ptr, data.row_ptr[r0] + (1 << 20), side="right"))
        r1 = min(max(r1 - 1, r0 + 1), n)
        a, b = int(data.row_ptr[r0]), int(data.row_ptr[r1])
        if b > a:
            prod = B[data.col[a:b]] * data.val[a:b, None]
            rows = np.repeat(np.arange(r1 - r0), lens[r0:r1])
            Z[r0:r1] = np.stack([np.bincount(rows, weights=prod[:, k], minlength=r1 - r0) for k in range(K)], axis=1)
        r0 = r1
    S = Z @ A
    S += 0.5 * S.std(axis=0, keepdims=True) * rng.standard_normal(S.shape)
    p = np.maximum(0.35 / np.arange(1, T + 1) ** 0.9, 0.004)
    thr = np.array([np.quantile(S[:, t], 1.0 - p[t]) for t in range(T)])
    has = S > thr
    n_train = max(1, int(0.8 * n))
    for t in np.flatnonzero(~has[:n_train].any(axis=0)):
        has[int(np.argmax(S[:n_train, t])), t] = True
    return Topics.from_indicator(has, [f"T{t}" for t in range(T)])


def _read_topics(qrels: str, ids: np.ndarray) -> Topics:
    """Every qrels line of the documents ids (row r is document ids[r]): names sorted, a repeated (topic, doc) line once,
    lines of other documents left out."""
    h = native.host_lib()
    n_lines, n_names, n_bytes = C.c_int64(), C.c_int32(), C.c_int64()
    if h.dsgd_rcv1_topics_count(qrels.encode(), C.byref(n_lines), C.byref(n_names), C.byref(n_bytes)) != 0:
        raise FileNotFoundError(qrels)
    buf = C.create_string_buffer(max(n_bytes.value, 1))
    line_topic = np.empty(n_lines.value, dtype=np.int32)
    line_doc = np.empty(n_lines.value, dtype=np.int64)
    if h.dsgd_rcv1_topics_parse(qrels.encode(), n_lines.value, n_names.value, n_bytes.value, buf,
                                line_topic.ctypes.data_as(C.c_void_p), line_doc.ctypes.data_as(C.c_void_p)) != 0:
        raise ValueError(f"{qrels}: the file changed while it was read")
    seen = buf.raw[:n_bytes.value].split(b"\0")[:n_names.value]
    names = sorted(x.decode() for x in seen)
    rank = np.empty(len(seen), dtype=np.int64)
    rank[np.argsort([x.decode() for x in seen], kind="stable")] = np.arange(len(seen))
    row_of = np.full(max(int(ids.max(initial=0)), int(line_doc.max(initial=0))) + 1, -1, dtype=np.int64)
    row_of[ids] = np.arange(ids.size)
    keep = line_doc >= 0
    rows = np.where(keep, row_of[np.where(keep, line_doc, 0)], -1)
    keep &= rows >= 0
    key = np.unique(rows[keep] * len(names) + rank[line_topic[keep]])
    ptr = np.zeros(ids.size + 1, dtype=np.int64)
    np.cumsum(np.bincount(key // len(names), minlength=ids.size), out=ptr[1:])
    return Topics(ptr, (key % len(names)).astype(np.int32), tuple(names))


def _read_vectors(path: str, dim: int):
    h = native.host_lib()
    n, nnz = C.c_int64(), C.c_int64()
    if h.dsgd_rcv1_count(path.encode(), C.byref(n), C.byref(nnz)) != 0:
        raise FileNotFoundError(path)
    row_ptr = np.zeros(n.value + 1, dtype=np.int64)
    col = np.empty(nnz.value, dtype=np.int32)
    val = np.empty(nnz.value, dtype=np.float32)
    ids = np.empty(n.value, dtype=np.int64)
    rc = h.dsgd_rcv1_parse(path.encode(), dim, n.value, nnz.value, row_ptr.ctypes.data_as(C.c_void_p),
                           col.ctypes.data_as(C.c_void_p), val.ctypes.data_as(C.c_void_p),
                           ids.ctypes.data_as(C.c_void_p))
    if rc != 0:
        raise ValueError(f"{path}: malformed RCV1 vectors file (code {rc})")
    # the count is an upper bound: a key repeated within a line is stored once
    nnz = int(row_ptr[-1])
    return row_ptr, col[:nnz], val[:nnz], ids


def rcv1(folder: str, full: bool = True, features_count: int = RCV1_FEATURES, topics: bool = False) -> Data:
    """utils/Dataset.scala:13-58: train file (+ the four test parts when `full`), labels from the qrels
    file (+1 iff CCAT; the last line of a document wins, quirk Q10).  topics=True: Data.topics holds every qrels line of
    each document as well (names sorted, a repeated line once); the binary label stays the CCAT label."""
    files = [os.path.join(folder, "lyrl2004_vectors_train.dat")]
    if full:
        files += [os.path.join(folder, f"lyrl2004_vectors_test_pt{d}.dat") for d in range(4)]
    parts = [_read_vectors(f, features_count) for f in files]
    row_ptr = [np.zeros(1, dtype=np.int64)]
    off = 0
    for rp, _, _, _ in parts:
        row_ptr.append(rp[1:] + off)
        off += int(rp[-1])
    row_ptr = np.concatenate(row_ptr)
    col = np.concatenate([p[1] for p in parts])
    val = np.concatenate([p[2] for p in parts])
    ids = np.concatenate([p[3] for p in parts])
    label = np.zeros(len(ids), dtype=np.int8)
    h = native.host_lib()
    qrels = os.path.join(folder, "rcv1-v2.topics.qrels")
    if h.dsgd_rcv1_labels(qrels.encode(), ids.ctypes.data_as(C.c_void_p), len(ids), label.ctypes.data_as(C.c_void_p)) != 0:
        raise FileNotFoundError(qrels)
    if (label == 0).any():
        raise KeyError("rcv1: a document has no qrels line (labels(id) throws in the reference, Dataset.scala:58)")
    return Data(row_ptr, col, val, label, features_count, None, _read_topics(qrels, ids) if topics else None)


def write_rcv1(data: Data, folder: str, first_id: int = 1, name: str = "lyrl2004_vectors_train.dat") -> None:
    """Export rows in the reference's text format so a JVM run of the reference can read the same data."""
    os.makedirs(folder, exist_ok=True)
    h = native.host_lib()
    rc = h.dsgd_rcv1_write(os.path.join(folder, name).encode(), os.path.join(folder, "rcv1-v2.topics.qrels").encode(),
                           data.n_rows, data.row_ptr.ctypes.data_as(C.c_void_p), data.col.ctypes.data_as(C.c_void_p),
                           data.val.ctypes.data_as(C.c_void_p), data.label.ctypes.data_as(C.c_void_p), first_id)
    if rc != 0:
        raise OSError("write_rcv1 failed")
