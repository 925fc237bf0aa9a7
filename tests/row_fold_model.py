"""numpy model of the row fold (dsgd_kernels.cuh, row_fold): the one fp64 summation order of x . w on the device, and of the
two folds some kernels used before it (W: lane-strided over the whole window; U: 16-byte units of two pairs lane-strided),
plus the oracle's index-order fold L.  Every fold works on a (rows, window pairs) matrix of the filtered products; a row is
padded with +0.0 products to a multiple of 128 pairs, which adds nothing to any lane sum (no lane sum is -0).  numpy adds
and multiplies float64 with one rounding each and no contraction, like the library (built with --fmad=false), so the model
gives the device's bits.

Also here: the adversarial rows that tell the folds apart, and a small CSR data set built from them for the GPU test.
Each row carries its design in x; its columns have weight 1 and are taken from pools of one magnitude each, so
that every column's gradient sum is exact in any order at lambda = 0."""
import numpy as np

EPS = 1e-20
LANES, CHUNK = 32, 128


def filt(v):
    v = np.asarray(v, np.float64)
    return np.where(np.abs(v) > EPS, v, 0.0)


def window_products(row_ptr, col, val, w, rows):
    """(len(rows), L) filtered products filt(filt(x) * w) in window (storage) order, L a multiple of 128."""
    rows = np.asarray(rows, np.int64)
    lens = (row_ptr[rows + 1] - row_ptr[rows]).astype(np.int64)
    L = max(CHUNK, int(-(-max(int(lens.max(initial=0)), 1) // CHUNK)) * CHUNK)
    P = np.zeros((rows.size, L))
    if rows.size == 0:
        return P
    pos = np.arange(L)[None, :]
    mask = pos < lens[:, None]
    src = (row_ptr[rows][:, None] + pos)[mask]
    x = filt(val[src].astype(np.float64))
    P[mask] = filt(x * np.asarray(w, np.float64)[col[src]])
    return P


def butterfly(v):
    """The xor butterfly 16, 8, 4, 2, 1 over the last axis (32 lanes); every lane ends with the same value: lane 0's."""
    lanes = np.arange(LANES)
    for o in (16, 8, 4, 2, 1):
        v = v + v[..., lanes ^ o]
    return v[..., 0]


def fold_row(P):
    """The row fold: per 128-pair chunk lane l sums pairs l + 32 u, u = 0..3, from +0.0; butterfly; 0.0 + partials in order."""
    n, L = P.shape
    Q = P.reshape(n, L // CHUNK, 4, LANES)
    acc = np.zeros((n, L // CHUNK, LANES))
    for u in range(4):
        acc = acc + Q[:, :, u, :]
    part = butterfly(acc)
    dot = np.zeros(n)
    for c in range(part.shape[1]):
        dot = dot + part[:, c]
    return dot


def fold_w(P):
    """W: lane l sums pairs l + 32 k over the whole window, in order, from +0.0; then the butterfly."""
    n, L = P.shape
    Q = P.reshape(n, L // LANES, LANES)
    acc = np.zeros((n, LANES))
    for k in range(Q.shape[1]):
        acc = acc + Q[:, k, :]
    return butterfly(acc)


def fold_u(P):
    """U: units of two pairs; lane l sums units l + 32 k in order (the unit's two pairs in order), from +0.0; butterfly."""
    n, L = P.shape
    Q = P.reshape(n, L // (2 * LANES), LANES, 2)
    acc = np.zeros((n, LANES))
    for k in range(Q.shape[1]):
        acc = acc + Q[:, k, :, 0]
        acc = acc + Q[:, k, :, 1]
    return butterfly(acc)


def fold_l(P):
    """L: the oracle's left fold in index order from 0.0."""
    dot = np.zeros(P.shape[0])
    for k in range(P.shape[1]):
        dot = dot + P[:, k]
    return dot


def pred(dot):
    """-signum(x . w)"""
    return -np.sign(dot)


# ---- adversarial rows: x values only (the columns carry weight 1) ------------------------------------------------------

ROW_A = [1.0, 2.0 ** -60, -1.0, 2.0 ** -60]    # W = C = 2^-59, U = 0, L = 2^-60
SHORT_SET = np.array([0.5, 1.0, 2.0 ** -53, 3 * 2.0 ** -54])
A_FILL = 2.0 ** -20


def short_rows(seed, n_rows):
    """Rows of 3 to 32 values from +-SHORT_SET whose row fold and U fold differ in sign (or zero against non-zero), and
    whose L has the row fold's sign; found by a seeded random search."""
    rng = np.random.default_rng(seed)
    out = []
    while len(out) < n_rows:
        m = int(rng.integers(3, 33))
        X = rng.choice(SHORT_SET, size=(4096, m)) * rng.choice([-1.0, 1.0], size=(4096, m))
        P = np.zeros((4096, CHUNK))
        P[:, :m] = X
        c, u, l = fold_row(P), fold_u(P), fold_l(P)
        ok = (np.sign(c) != np.sign(u)) & (np.sign(l) == np.sign(c))
        for i in np.flatnonzero(ok)[: n_rows - len(out)]:
            out.append(X[i].copy())
    return out


def long_row(n, sign=1.0):
    """n pairs, n a multiple of 64 in [256, 1024]: lane 0 holds +-1/2 twice in chunk 0 and twice in chunk 1 (partials 1 and
    -1), lane 1 holds 2^-61 twice in both, every other slot +-2^-20 in pairs that cancel within a lane and a chunk.  The row
    fold gives 1 + 2^-60 -> 1, then 1 - 1 = 0; W gives lane 1's 2^-59."""
    assert n % 64 == 0 and 256 <= n <= 1024
    x = np.empty(n)
    k = np.arange(n)
    visit = k // LANES
    x[:] = np.where(visit % 2 == 0, A_FILL, -A_FILL)
    for v, val in ((0, 0.5), (3, 0.5), (4, -0.5), (7, -0.5)):
        x[v * LANES] = val
    for v in (0, 3, 4, 7):
        x[v * LANES + 1] = 2.0 ** -61
    # keep every other lane's chunk sums cancelling: lane 0 / 1 visits 1, 2 and 5, 6 are +-2^-20 pairs already
    return sign * x


def pool_of(v):
    """Which column pool a value's magnitude belongs to (one magnitude class per pool keeps column sums exact)."""
    a = abs(v)
    if a >= 0.5:
        return 0
    if a == A_FILL:
        return 1
    if a >= 2.0 ** -54:
        return 2
    return 3


N_POOLS = 4
POOL_UNIT = [0.5, A_FILL, 2.0 ** -54, 2.0 ** -61]   # every value of pool p is an integer multiple of POOL_UNIT[p]
POOL_COLS = 1024            # columns per pool (a row uses at most 1024 of one pool)


def build_rows(seed, n_short=48, long_lengths=(256, 320, 640, 960), n_long_each=8, n_ordinary=160, ord_dim=4096,
               ord_nnz=(1, 200), n_empty=8):
    """Adversarial, ordinary and empty rows, interleaved.  Returns dict(rows=[(cols, vals)], labels, kind=[str], dim,
    w=initial weights: 1 on the pool columns, non-dyadic on the ordinary ones)."""
    rng = np.random.default_rng(seed)
    adv = [("row_a", np.array(ROW_A))] * 8 + [("short", x) for x in short_rows(seed, n_short)]
    for n in long_lengths:
        adv += [("long", long_row(n, s)) for s in [1.0, -1.0] * (n_long_each // 2)]
    base = N_POOLS * POOL_COLS
    dim = base + ord_dim
    rows, kind = [], []

    def adv_row(x):
        cols = np.empty(len(x), np.int64)
        for p in range(N_POOLS):
            sel = np.flatnonzero([pool_of(v) == p for v in x])
            cols[sel] = p * POOL_COLS + rng.choice(POOL_COLS, size=sel.size, replace=False)
        return cols, x

    items = [("adv", a) for a in adv] + [("ordinary", None)] * n_ordinary + [("empty", None)] * n_empty
    for i in rng.permutation(len(items)):
        what, a = items[i]
        if what == "adv":
            rows.append(adv_row(a[1]))
            kind.append(a[0])
        elif what == "ordinary":
            m = int(rng.integers(ord_nnz[0], ord_nnz[1] + 1))
            rows.append((base + rng.choice(ord_dim, size=m, replace=False), rng.integers(1, 1025, size=m) / 256.0))
            kind.append("ordinary")
        else:
            rows.append((np.zeros(0, np.int64), np.zeros(0)))
            kind.append("empty")
    w = np.ones(dim)
    w[base:] = rng.standard_normal(ord_dim) * 0.37
    labels = rng.choice(np.array([-1, 1], np.int8), size=len(rows))
    return dict(rows=rows, labels=labels, kind=np.array(kind), dim=dim, w=w)


def to_csr(rows):
    rp = np.zeros(len(rows) + 1, np.int64)
    rp[1:] = np.cumsum([len(c) for c, _ in rows])
    col = np.concatenate([np.asarray(c, np.int32) for c, _ in rows])
    val = np.concatenate([np.asarray(v, np.float32) for _, v in rows])
    return rp, col, val


# ---- what the device computes, decided by the row fold -------------------------------------------------------------------

class Model:
    """Margins, predictions, counters, gradients and sync / async updates at lambda = 0 whose every decision is the row
    fold's.  The gradient sums are exact on the data of build_rows (dyadic x, one magnitude class per column), so their
    order does not matter."""

    def __init__(self, row_ptr, col, val, label, dim):
        self.rp, self.col, self.val = np.asarray(row_ptr, np.int64), np.asarray(col), np.asarray(val, np.float32)
        self.y = np.asarray(label, np.float64)
        self.dim = dim

    def margins(self, w, ids):
        return fold_row(window_products(self.rp, self.col, self.val, w, ids))

    def counts(self, w, ids):
        """(hinge sum, correct count) of SparseSVM over the rows ids."""
        ids = np.asarray(ids, np.int64)
        p, y = pred(self.margins(w, ids)), self.y[ids]
        return int(np.sum(1 - y * p)), int(np.sum(p == y))

    def raw_gradient(self, w, ids):
        """(sum of y x over the rows that pass the gate, hinge sum)."""
        ids = np.asarray(ids, np.int64)
        dot = self.margins(w, ids)
        y = self.y[ids]
        g = np.zeros(self.dim)
        for r, yy in zip(ids[~(y * dot < 0.0)], y[~(y * dot < 0.0)]):
            b, e = self.rp[r], self.rp[r + 1]
            np.add.at(g, self.col[b:e], filt(filt(self.val[b:e].astype(np.float64)) * yy))
        return filt(g), int(np.sum(1 - y * pred(dot)))

    def sync_steps(self, w, ids, counts, lr, n_steps):
        """Master.scala:194,197 at lambda = 0 with len(counts) workers: (weights, per-step losses)."""
        w = np.array(w, np.float64)
        ids = np.asarray(ids, np.int64).reshape(n_steps, -1)
        losses = []
        K = len(counts)
        for s in range(n_steps):
            g, h, off = np.zeros(self.dim), 0, 0
            for k in range(K):
                gk, hk = self.raw_gradient(w, ids[s, off:off + counts[k]])
                g, h, off = filt(g + gk), h + hk, off + counts[k]
            losses.append(h / float(ids.shape[1]))
            nz = g != 0.0
            step = filt(filt(g / float(K)) * lr)
            w[nz] = filt(w[nz] - step[nz])
        return w, np.array(losses)

    def async_run(self, w, ids, batch, lr):
        """One Hogwild lane replaying batches at lambda = 0: w <- filt(w - filt(filt(sum / B) * lr))."""
        w = np.array(w, np.float64)
        ids = np.asarray(ids, np.int64).reshape(-1, batch)
        for b in ids:
            g, _ = self.raw_gradient(w, b)
            nz = g != 0.0
            delta = filt(filt(g / float(batch)) * lr)
            w[nz] = filt(w[nz] - delta[nz])
        return w
