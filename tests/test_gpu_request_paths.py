"""Every request entry point of the C ABI: forward, gradient, the nine evaluations, margins, probabilities and the three
metrics calls.

* The kernels one call launches (the dsgd_launch_count delta), on an SVM and a logistic context, over fewer and more ids than
  kStreamMinRows (2048, csrc/dsgd_api.cu) where the SVM's streaming pass takes over; with the resident weights and with the
  same weights passed in, which must give the same bits.  The logistic gradient adds to g with fp64 atomics in the order the
  rows arrive, so its gradient agrees to rounding and its loss (a fixed-point sum) to the bit.
* The error each bad argument gets on its own, and a message that names the entry point that was called.
* A list of more ids than rows is refused while an async loop is started, even after the loop ended by itself: growing a
  buffer then would wait for every kernel on the device, and a loop that runs until stopped never ends."""
import os
import subprocess
import sys

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LAM = 1e-4
N_ROWS = 6000
KEY = 0x9E3779B97F4A7C15
SIZES = {"small": 300, "large": 4000}          # ids (or rows) of one call: below and above kStreamMinRows

# entry point -> one call over the rows that `ids` stands for, with weights w (None: the resident ones)
REQUESTS = {
    "forward": lambda c, ids, w: c.forward(ids, w),
    "gradient": lambda c, ids, w: c.gradient(ids, w, want_loss=True),
    "eval": lambda c, ids, w: c.eval(7, 7 + ids.size, w),
    "eval_counts": lambda c, ids, w: c.eval_counts(7, 7 + ids.size, w),
    "eval_sums": lambda c, ids, w: c.eval_sums(7, 7 + ids.size, w),
    "eval_sampled_counts": lambda c, ids, w: c.eval_sampled_counts(7, N_ROWS, KEY, 5, 5 + ids.size, w),
    "eval_sampled_sums": lambda c, ids, w: c.eval_sampled_sums(7, N_ROWS, KEY, 5, 5 + ids.size, w),
    "eval_samples_counts": lambda c, ids, w: c.eval_samples_counts(ids, w),
    "eval_samples_sums": lambda c, ids, w: c.eval_samples_sums(ids, w),
    "margins": lambda c, ids, w: c.margins(ids, w),
    "probabilities": lambda c, ids, w: c.probabilities(ids, w),
    "eval_metrics": lambda c, ids, w: c.eval_metrics(7, 7 + ids.size, w),
    "eval_sampled_metrics": lambda c, ids, w: c.eval_sampled_metrics(7, N_ROWS, KEY, 5, 5 + ids.size, w),
    "eval_samples_metrics": lambda c, ids, w: c.eval_samples_metrics(ids, w),
}
SVM_ONLY = {"eval_counts", "eval_sampled_counts", "eval_samples_counts"}
LOGISTIC_ONLY = {"probabilities"}

# (model, size, entry point) -> launch_count() delta of one call (resident weights, weights passed in)
LAUNCHES = {
    ('svm', 'large', 'forward'): (1, 3),
    ('svm', 'large', 'gradient'): (3, 5),
    ('svm', 'large', 'eval'): (2, 4),
    ('svm', 'large', 'eval_counts'): (2, 4),
    ('svm', 'large', 'eval_sums'): (2, 4),
    ('svm', 'large', 'eval_sampled_counts'): (3, 5),
    ('svm', 'large', 'eval_sampled_sums'): (3, 5),
    ('svm', 'large', 'eval_samples_counts'): (2, 4),
    ('svm', 'large', 'eval_samples_sums'): (2, 4),
    ('svm', 'large', 'margins'): (1, 3),
    ('svm', 'large', 'eval_metrics'): (2, 4),
    ('svm', 'large', 'eval_sampled_metrics'): (3, 5),
    ('svm', 'large', 'eval_samples_metrics'): (2, 4),
    ('svm', 'small', 'forward'): (1, 3),
    ('svm', 'small', 'gradient'): (3, 5),
    ('svm', 'small', 'eval'): (2, 4),
    ('svm', 'small', 'eval_counts'): (2, 4),
    ('svm', 'small', 'eval_sums'): (2, 4),
    ('svm', 'small', 'eval_sampled_counts'): (3, 5),
    ('svm', 'small', 'eval_sampled_sums'): (3, 5),
    ('svm', 'small', 'eval_samples_counts'): (2, 4),
    ('svm', 'small', 'eval_samples_sums'): (2, 4),
    ('svm', 'small', 'margins'): (1, 3),
    ('svm', 'small', 'eval_metrics'): (2, 4),
    ('svm', 'small', 'eval_sampled_metrics'): (3, 5),
    ('svm', 'small', 'eval_samples_metrics'): (2, 4),
    ('logistic', 'large', 'forward'): (1, 3),
    ('logistic', 'large', 'gradient'): (3, 5),
    ('logistic', 'large', 'eval'): (2, 4),
    ('logistic', 'large', 'eval_sums'): (2, 4),
    ('logistic', 'large', 'eval_sampled_sums'): (3, 5),
    ('logistic', 'large', 'eval_samples_sums'): (2, 4),
    ('logistic', 'large', 'margins'): (1, 3),
    ('logistic', 'large', 'probabilities'): (1, 3),
    ('logistic', 'large', 'eval_metrics'): (2, 4),
    ('logistic', 'large', 'eval_sampled_metrics'): (3, 5),
    ('logistic', 'large', 'eval_samples_metrics'): (2, 4),
    ('logistic', 'small', 'forward'): (1, 3),
    ('logistic', 'small', 'gradient'): (3, 5),
    ('logistic', 'small', 'eval'): (2, 4),
    ('logistic', 'small', 'eval_sums'): (2, 4),
    ('logistic', 'small', 'eval_sampled_sums'): (3, 5),
    ('logistic', 'small', 'eval_samples_sums'): (2, 4),
    ('logistic', 'small', 'margins'): (1, 3),
    ('logistic', 'small', 'probabilities'): (1, 3),
    ('logistic', 'small', 'eval_metrics'): (2, 4),
    ('logistic', 'small', 'eval_sampled_metrics'): (3, 5),
    ('logistic', 'small', 'eval_samples_metrics'): (2, 4),
}

FORM = {"forward": "list", "gradient": "list", "eval": "range", "eval_counts": "range", "eval_sums": "range",
        "eval_sampled_counts": "drawn", "eval_sampled_sums": "drawn", "eval_samples_counts": "list",
        "eval_samples_sums": "list", "margins": "list", "probabilities": "list", "eval_metrics": "range",
        "eval_sampled_metrics": "drawn", "eval_samples_metrics": "list"}
GOOD_ROWS = {"list": [1, 2, 3], "range": (10, 20), "drawn": (10, 20, 1, 0, 5)}
BAD_ROWS = {
    "list": [[0, N_ROWS], [-1, 3], [], "NULL"],
    "range": [(0, N_ROWS + 1), (-1, 5), (9, 8), (4, 4)],
    "drawn": [(0, N_ROWS + 1, 1, 0, 5), (-1, 10, 1, 0, 5), (5, 5, 1, 0, 0), (10, 20, 1, -1, 3), (10, 20, 1, 0, 11),
              (10, 20, 1, 4, 12), (10, 20, 1, 3, 3), (10, 20, 1, 5, 4)],
}
# entry points whose first output pointer must not be NULL
NEEDS_OUT = {"forward", "gradient", "margins", "probabilities", "eval_metrics", "eval_sampled_metrics",
             "eval_samples_metrics"}

# (entry point, context, rows (None: GOOD_ROWS of its form), NULL output, expected exception class name or None)
ERRORS = [
    ('forward', 'svm', [0, 6000], False, 'DsgdRange'),
    ('forward', 'svm', [-1, 3], False, 'DsgdRange'),
    ('forward', 'svm', [], False, None),
    ('forward', 'svm', 'NULL', False, 'DsgdInvalid'),
    ('forward', 'empty_svm', None, False, 'DsgdState'),
    ('forward', 'svm', None, True, 'DsgdInvalid'),
    ('gradient', 'svm', [0, 6000], False, 'DsgdRange'),
    ('gradient', 'svm', [-1, 3], False, 'DsgdRange'),
    ('gradient', 'svm', [], False, 'DsgdEmpty'),
    ('gradient', 'svm', 'NULL', False, 'DsgdInvalid'),
    ('gradient', 'empty_svm', None, False, 'DsgdState'),
    ('gradient', 'svm', None, True, 'DsgdInvalid'),
    ('eval', 'svm', (0, 6001), False, 'DsgdRange'),
    ('eval', 'svm', (-1, 5), False, 'DsgdRange'),
    ('eval', 'svm', (9, 8), False, 'DsgdRange'),
    ('eval', 'svm', (4, 4), False, 'DsgdEmpty'),
    ('eval', 'empty_svm', None, False, 'DsgdState'),
    ('eval_counts', 'svm', (0, 6001), False, 'DsgdRange'),
    ('eval_counts', 'svm', (-1, 5), False, 'DsgdRange'),
    ('eval_counts', 'svm', (9, 8), False, 'DsgdRange'),
    ('eval_counts', 'svm', (4, 4), False, 'DsgdEmpty'),
    ('eval_counts', 'empty_svm', None, False, 'DsgdState'),
    ('eval_counts', 'logistic', None, False, 'DsgdState'),
    ('eval_sums', 'svm', (0, 6001), False, 'DsgdRange'),
    ('eval_sums', 'svm', (-1, 5), False, 'DsgdRange'),
    ('eval_sums', 'svm', (9, 8), False, 'DsgdRange'),
    ('eval_sums', 'svm', (4, 4), False, 'DsgdEmpty'),
    ('eval_sums', 'empty_svm', None, False, 'DsgdState'),
    ('eval_sampled_counts', 'svm', (0, 6001, 1, 0, 5), False, 'DsgdRange'),
    ('eval_sampled_counts', 'svm', (-1, 10, 1, 0, 5), False, 'DsgdRange'),
    ('eval_sampled_counts', 'svm', (5, 5, 1, 0, 0), False, 'DsgdEmpty'),
    ('eval_sampled_counts', 'svm', (10, 20, 1, -1, 3), False, 'DsgdInvalid'),
    ('eval_sampled_counts', 'svm', (10, 20, 1, 0, 11), False, 'DsgdInvalid'),
    ('eval_sampled_counts', 'svm', (10, 20, 1, 4, 12), False, 'DsgdInvalid'),
    ('eval_sampled_counts', 'svm', (10, 20, 1, 3, 3), False, 'DsgdEmpty'),
    ('eval_sampled_counts', 'svm', (10, 20, 1, 5, 4), False, 'DsgdEmpty'),
    ('eval_sampled_counts', 'empty_svm', None, False, 'DsgdState'),
    ('eval_sampled_counts', 'logistic', None, False, 'DsgdState'),
    ('eval_sampled_sums', 'svm', (0, 6001, 1, 0, 5), False, 'DsgdRange'),
    ('eval_sampled_sums', 'svm', (-1, 10, 1, 0, 5), False, 'DsgdRange'),
    ('eval_sampled_sums', 'svm', (5, 5, 1, 0, 0), False, 'DsgdEmpty'),
    ('eval_sampled_sums', 'svm', (10, 20, 1, -1, 3), False, 'DsgdInvalid'),
    ('eval_sampled_sums', 'svm', (10, 20, 1, 0, 11), False, 'DsgdInvalid'),
    ('eval_sampled_sums', 'svm', (10, 20, 1, 4, 12), False, 'DsgdInvalid'),
    ('eval_sampled_sums', 'svm', (10, 20, 1, 3, 3), False, 'DsgdEmpty'),
    ('eval_sampled_sums', 'svm', (10, 20, 1, 5, 4), False, 'DsgdEmpty'),
    ('eval_sampled_sums', 'empty_svm', None, False, 'DsgdState'),
    ('eval_samples_counts', 'svm', [0, 6000], False, 'DsgdRange'),
    ('eval_samples_counts', 'svm', [-1, 3], False, 'DsgdRange'),
    ('eval_samples_counts', 'svm', [], False, 'DsgdEmpty'),
    ('eval_samples_counts', 'svm', 'NULL', False, 'DsgdInvalid'),
    ('eval_samples_counts', 'empty_svm', None, False, 'DsgdState'),
    ('eval_samples_counts', 'logistic', None, False, 'DsgdState'),
    ('eval_samples_sums', 'svm', [0, 6000], False, 'DsgdRange'),
    ('eval_samples_sums', 'svm', [-1, 3], False, 'DsgdRange'),
    ('eval_samples_sums', 'svm', [], False, 'DsgdEmpty'),
    ('eval_samples_sums', 'svm', 'NULL', False, 'DsgdInvalid'),
    ('eval_samples_sums', 'empty_svm', None, False, 'DsgdState'),
    ('margins', 'svm', [0, 6000], False, 'DsgdRange'),
    ('margins', 'svm', [-1, 3], False, 'DsgdRange'),
    ('margins', 'svm', [], False, 'DsgdEmpty'),
    ('margins', 'svm', 'NULL', False, 'DsgdInvalid'),
    ('margins', 'empty_svm', None, False, 'DsgdState'),
    ('margins', 'svm', None, True, 'DsgdInvalid'),
    ('probabilities', 'logistic', [0, 6000], False, 'DsgdRange'),
    ('probabilities', 'logistic', [-1, 3], False, 'DsgdRange'),
    ('probabilities', 'logistic', [], False, 'DsgdEmpty'),
    ('probabilities', 'logistic', 'NULL', False, 'DsgdInvalid'),
    ('probabilities', 'empty_logistic', None, False, 'DsgdState'),
    ('probabilities', 'logistic', None, True, 'DsgdInvalid'),
    ('probabilities', 'svm', None, False, 'DsgdState'),
    ('eval_metrics', 'svm', (0, 6001), False, 'DsgdRange'),
    ('eval_metrics', 'svm', (-1, 5), False, 'DsgdRange'),
    ('eval_metrics', 'svm', (9, 8), False, 'DsgdRange'),
    ('eval_metrics', 'svm', (4, 4), False, 'DsgdEmpty'),
    ('eval_metrics', 'empty_svm', None, False, 'DsgdState'),
    ('eval_metrics', 'svm', None, True, 'DsgdInvalid'),
    ('eval_sampled_metrics', 'svm', (0, 6001, 1, 0, 5), False, 'DsgdRange'),
    ('eval_sampled_metrics', 'svm', (-1, 10, 1, 0, 5), False, 'DsgdRange'),
    ('eval_sampled_metrics', 'svm', (5, 5, 1, 0, 0), False, 'DsgdEmpty'),
    ('eval_sampled_metrics', 'svm', (10, 20, 1, -1, 3), False, 'DsgdInvalid'),
    ('eval_sampled_metrics', 'svm', (10, 20, 1, 0, 11), False, 'DsgdInvalid'),
    ('eval_sampled_metrics', 'svm', (10, 20, 1, 4, 12), False, 'DsgdInvalid'),
    ('eval_sampled_metrics', 'svm', (10, 20, 1, 3, 3), False, 'DsgdEmpty'),
    ('eval_sampled_metrics', 'svm', (10, 20, 1, 5, 4), False, 'DsgdEmpty'),
    ('eval_sampled_metrics', 'empty_svm', None, False, 'DsgdState'),
    ('eval_sampled_metrics', 'svm', None, True, 'DsgdInvalid'),
    ('eval_samples_metrics', 'svm', [0, 6000], False, 'DsgdRange'),
    ('eval_samples_metrics', 'svm', [-1, 3], False, 'DsgdRange'),
    ('eval_samples_metrics', 'svm', [], False, 'DsgdEmpty'),
    ('eval_samples_metrics', 'svm', 'NULL', False, 'DsgdInvalid'),
    ('eval_samples_metrics', 'empty_svm', None, False, 'DsgdState'),
    ('eval_samples_metrics', 'svm', None, True, 'DsgdInvalid'),
    ('gradient', 'no_d', None, False, 'DsgdState'),
]


def request_ids(n):
    return np.random.default_rng(n).integers(0, N_ROWS, size=n).astype(np.int32)


def bits(x):
    if isinstance(x, tuple):
        return tuple(bits(v) for v in x)
    if isinstance(x, np.ndarray):
        return x.dtype.str, x.tobytes()
    return float(x).hex() if isinstance(x, float) else x


def entry_points(model):
    return [n for n in REQUESTS if n not in (LOGISTIC_ONLY if model == "svm" else SVM_ONLY)]


def make_contexts():
    """model -> (ctx with N_ROWS rows, dimSparsity and resident weights w, w); plus the contexts of the error table:
    `empty_*` without rows, `no_d` with rows and no dimSparsity."""
    from distributed_sgd_b200.native import NativeCtx
    from distributed_sgd_b200.utils import synthetic_rcv1
    data = synthetic_rcv1(n_rows=N_ROWS, seed=31)
    rng = np.random.default_rng(31)
    w = np.where(rng.random(data.dim) < 0.6, rng.standard_normal(data.dim) * 0.1, 0.0)
    out = {}
    for model in ("svm", "logistic"):
        ctx = NativeCtx(0, data.dim, LAM, logistic=model == "logistic")
        ctx.load_csr(data.row_ptr, data.col, data.val, data.label)
        ctx.compute_dim_sparsity(N_ROWS)
        ctx.set_weights(w)
        out[model] = ctx
        out["empty_" + model] = NativeCtx(0, data.dim, LAM, logistic=model == "logistic")
    out["no_d"] = NativeCtx(0, data.dim, LAM)
    out["no_d"].load_csr(data.row_ptr, data.col, data.val, data.label)
    return out, w


def observe_launches(ctxs, w, model, size):
    """entry point -> ((delta, delta), (result, result)): one call with the resident weights and one with w passed in."""
    ctx, ids, out = ctxs[model], request_ids(SIZES[size]), {}
    for name in entry_points(model):
        deltas, results = [], []
        for wa in (None, w):
            before = ctx.launch_count()
            results.append(REQUESTS[name](ctx, ids, wa))
            deltas.append(ctx.launch_count() - before)
        out[name] = (tuple(deltas), tuple(results))
    return out


def raw_call(ctx, name, rows, null_out):
    """dsgd_<name> through ctypes with `rows` in its form and no weights: (exception class name or None, message)."""
    from distributed_sgd_b200.native import _EXC
    if FORM[name] == "list":
        ids = None if rows == "NULL" else np.asarray(rows, np.int32)
        args = (None if ids is None else ids.ctypes.data, 3 if ids is None else ids.size)
    else:
        args = tuple(rows)
    preds, grad, m8 = np.zeros(N_ROWS + 8), np.zeros(ctx.dim), np.zeros(8, np.int64)
    outs = {"forward": (preds.ctypes.data,), "gradient": (grad.ctypes.data, None), "eval": (None, None),
            "margins": (preds.ctypes.data,), "probabilities": (preds.ctypes.data,)}.get(name)
    if outs is None:
        outs = (m8.ctypes.data,) if "metrics" in name else (None, None, None)
    if null_out:
        outs = (None,) + outs[1:]
    rc = getattr(ctx._l, "dsgd_" + name)(ctx._h, None, *args, *outs)
    return (None if rc == 0 else _EXC[rc].__name__), (ctx._l.dsgd_last_error(ctx._h) or b"").decode()


def error_cases():
    """(entry point, context, rows, NULL output): each bad argument on its own."""
    cases = []
    for name in REQUESTS:
        own = "logistic" if name in LOGISTIC_ONLY else "svm"
        cases += [(name, own, rows, False) for rows in BAD_ROWS[FORM[name]]]
        cases.append((name, "empty_" + own, None, False))
        if name in NEEDS_OUT:
            cases.append((name, own, None, True))
        if name in SVM_ONLY:
            cases.append((name, "logistic", None, False))
        if name in LOGISTIC_ONLY:
            cases.append((name, "svm", None, False))
    cases.append(("gradient", "no_d", None, False))
    return cases


@pytest.fixture(scope="module")
def ctxs():
    out, w = make_contexts()
    yield out, w
    for c in out.values():
        c.close()


@pytest.mark.parametrize("size", sorted(SIZES))
@pytest.mark.parametrize("model", ["svm", "logistic"])
def test_launches_and_resident_weights(ctxs, model, size):
    got = observe_launches(*ctxs, model, size)
    assert {name: d for name, (d, _) in got.items()} == {k[2]: v for k, v in LAUNCHES.items() if k[:2] == (model, size)}
    (g0, loss0), (g1, loss1) = got.pop("gradient")[1] if model == "logistic" else ((0.0, 0.0), (0.0, 0.0))
    np.testing.assert_allclose(g0, g1, rtol=1e-12, atol=1e-18)
    assert bits(loss0) == bits(loss1)
    assert [name for name, (_, (a, b)) in got.items() if bits(a) != bits(b)] == []


def test_errors(ctxs):
    assert len(ERRORS) == len(error_cases())
    for name, kind, rows, null_out, expected in ERRORS:
        ctx = ctxs[0][kind]
        got, msg = raw_call(ctx, name, GOOD_ROWS[FORM[name]] if rows is None else rows, null_out)
        assert got == expected, (name, kind, rows, null_out, msg)
        if expected is not None:
            assert msg.startswith(f"dsgd_{name}: "), (name, kind, rows, null_out, msg)
    w = ctxs[1]                                       # the contexts still answer after the refusals
    assert bits(ctxs[0]["svm"].eval_sums(0, N_ROWS)) == bits(ctxs[0]["svm"].eval_sums(0, N_ROWS, w))


_LOOP = r"""
import sys, time
sys.path.insert(0, {root!r})
import numpy as np
from distributed_sgd_b200.native import DsgdState, NativeCtx
from distributed_sgd_b200.utils import synthetic_rcv1
data = synthetic_rcv1(n_rows=3000, seed=8)
ctx = NativeCtx(0, data.dim, 1e-4, is_async=True)
ctx.load_csr(data.row_ptr, data.col, data.val, data.label)
ctx.compute_dim_sparsity(3000)
ctx.start_async(np.zeros(data.dim), np.arange(3000, dtype=np.int32), 8, 0.1, concurrency=1, max_updates=64, seed=1)
try:
    t0 = time.time()
    while ctx.async_running():
        if time.time() - t0 > 60:
            raise SystemExit("the loop did not end by itself")
        time.sleep(0.01)
    ids = np.zeros(3001, np.int32)
    refused = []
    for name in ("forward", "gradient", "eval_samples_counts", "eval_samples_sums", "margins", "eval_samples_metrics"):
        try:
            getattr(ctx, name)(ids)
        except DsgdState as e:
            refused.append(name if str(e).split("] ", 1)[1].startswith("dsgd_" + name + ": ") else name + "?")
    print("REFUSED", " ".join(refused))
finally:
    ctx.stop_async()
print("AFTER", len(ctx.forward(ids)))
ctx.close()
"""


def test_longer_list_than_rows_is_refused_while_a_loop_is_started():
    """The loop ends by itself on max_updates; the context still counts as running until stop_async, so the list requests
    refuse a list their buffers cannot hold, and take it once the loop is stopped.  The subprocess has a timeout."""
    r = subprocess.run([sys.executable, "-s", "-c", _LOOP.format(root=ROOT)], cwd=ROOT, capture_output=True, text=True,
                       timeout=180)
    assert r.returncode == 0, r.stdout + r.stderr
    assert ("REFUSED forward gradient eval_samples_counts eval_samples_sums margins eval_samples_metrics\nAFTER 3001"
            in r.stdout), r.stdout + r.stderr
