"""ctypes binding of libdsgd.so (the C ABI in include/dsgd.h) and libdsgd_host.so (data preparation).

This is the only place the Python host touches native code.  There is no fallback: if libdsgd.so is
missing or no H100 is usable, the call raises (NativeLibraryMissing / DsgdError) -- nothing in this
package computes the hot path on the CPU.
"""
from __future__ import annotations

import ctypes as C
import json
import math
import os
import subprocess
from typing import NamedTuple, Optional, Tuple

import numpy as np

_PKG = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_PKG, "libdsgd.so")
HOST_LIB_PATH = os.path.join(_PKG, "libdsgd_host.so")
HEADER_PATH = os.path.join(os.path.dirname(_PKG), "include", "dsgd.h")

UNIQUE_ID_BYTES = 128
IPC_HANDLE_BYTES = 64
FLAG_ASYNC = 1
FLAG_LOGISTIC = 2
FLAG_SQUARED_HINGE = 4
FLAG_MODIFIED_HUBER = 8
FLAG_INTERCEPT = 16   # an unregularised intercept: weight vectors are dim + 1 long, the intercept last
# NativeCtx(model=...) -> the model flag of dsgd_create
MODEL_FLAGS = {"svm": 0, "logistic": FLAG_LOGISTIC, "squared_hinge": FLAG_SQUARED_HINGE, "modified_huber": FLAG_MODIFIED_HUBER}
REPLICA_SELF, REPLICA_MASTER = 0, 1

OK, ERR_INVALID, ERR_STATE, ERR_EMPTY, ERR_RANGE, ERR_CUDA, ERR_NCCL, ERR_NOMEM, ERR_TIMEOUT = 0, -1, -2, -3, -4, -5, -6, -7, -8
# words of the dsgd_eval_*metrics calls: TP, FN, positives without a +-1 prediction, FP, TN, negatives without one, U2, NaN rows
METRICS_WORDS = 8
CALIBRATION_INFO_WORDS = 5   # DSGD_CALIBRATION_INFO_WORDS
CALIBRATION_MAX_BINS = 64    # DSGD_CALIBRATION_MAX_BINS
CALIBRATION_WSUMS = 3        # DSGD_CALIBRATION_WSUMS: W+, W-, the NaN rows' weight
WCALIBRATION_SUMS = 4        # DSGD_WCALIBRATION_SUMS: weighted Brier and log-loss sums, weight used, infinite-term weight
ISOTONIC_INFO_WORDS = 5      # DSGD_ISOTONIC_INFO_WORDS: blocks, points, rows used, NaN rows, distinct scores
ISOTONIC_EVAL_WORDS = 3      # DSGD_ISOTONIC_EVAL_WORDS: rows used, rows left out, rows with an infinite log-loss term
BOOTSTRAP_WORDS = 9          # DSGD_BOOTSTRAP_WORDS: the METRICS_WORDS of a replicate, then its size (sum of m_i)
BOOTSTRAP_MAX_ROWS = 1 << 26  # the rows of one bootstrap request
MAX_TOPICS = 1024             # DSGD_MAX_TOPICS


def topic_words(n_topics: int) -> int:
    """DSGD_TOPIC_WORDS(T): eight words per topic, then eight row words"""
    return 8 * int(n_topics) + 8


TOPIC_RANK_MAX_K = 32         # DSGD_TOPIC_RANK_MAX_K


def topic_rank_words(k: int) -> int:
    """DSGD_TOPIC_RANK_WORDS(k): eight row words, k hit words, then 2 + k fixed-point sums of seven words each"""
    return 8 + int(k) + 7 * (2 + int(k))


def topic_tune_words(n_topics: int) -> int:
    """DSGD_TOPIC_TUNE_WORDS(T): eight words per topic (rows, P, NaN rows, D, tp, predicted, status, j)"""
    return 8 * int(n_topics)


class NativeLibraryMissing(ImportError):
    pass


class DsgdError(RuntimeError):
    """A failing C-ABI call.  `.code` is the DSGD_ERR_* value."""

    def __init__(self, code: int, msg: str):
        super().__init__(f"[dsgd {code}] {msg}")
        self.code = code


class DsgdInvalid(DsgdError, ValueError):  # the reference's require(...) -> IllegalArgumentException
    pass


class DsgdState(DsgdError):  # "slave is in synchronous mode", "already running"
    pass


class DsgdEmpty(DsgdError, ValueError):  # Vec.sum on an empty list (math/Vec.scala:129)
    pass


class DsgdRange(DsgdError, IndexError):  # ArrayIndexOutOfBoundsException on data(idx)
    pass


_EXC = {ERR_INVALID: DsgdInvalid, ERR_STATE: DsgdState, ERR_EMPTY: DsgdEmpty, ERR_RANGE: DsgdRange}


def build(verbose: bool = False) -> None:
    """Compile libdsgd.so (nvcc, sm_90a) and libdsgd_host.so (gcc) in-tree."""
    r = subprocess.run(["make", "-C", os.path.join(_PKG, "csrc"), "all"], capture_output=True, text=True)
    if verbose or r.returncode != 0:
        print(r.stdout)
        print(r.stderr)
    if r.returncode != 0:
        raise RuntimeError("building libdsgd.so failed")


_lib = None
_host = None

_vp, _i32, _i64, _f64, _u32, _u64 = C.c_void_p, C.c_int32, C.c_int64, C.c_double, C.c_uint32, C.c_uint64

# name -> argtypes; every function returns int unless listed in _RESTYPE
ABI = {
    "dsgd_create": [C.POINTER(_vp), C.c_int, _i32, _f64, C.c_int, C.c_int, _u32],
    "dsgd_destroy": [_vp],
    "dsgd_last_error": [_vp],
    "dsgd_info": [_vp],
    "dsgd_set_stream": [_vp, _vp],
    "dsgd_synchronize": [_vp],
    "dsgd_timer_start": [_vp],
    "dsgd_timer_stop": [_vp, C.POINTER(C.c_float)],
    "dsgd_launch_count": [_vp, C.POINTER(_i64)],
    "dsgd_profile_begin": [_vp, _i32],
    "dsgd_profile_end": [_vp, C.POINTER(C.c_float), C.POINTER(_i64)],
    "dsgd_load_csr": [_vp, _i64, _i64, _vp, _vp, _vp, _vp],
    "dsgd_set_dim_sparsity": [_vp, _vp],
    "dsgd_compute_dim_sparsity": [_vp, _i64, _vp],
    "dsgd_set_weights": [_vp, _vp],
    "dsgd_get_weights": [_vp, _vp],
    "dsgd_forward": [_vp, _vp, _vp, _i64, _vp],
    "dsgd_gradient": [_vp, _vp, _vp, _i64, _vp, C.POINTER(_f64)],
    "dsgd_eval": [_vp, _vp, _i64, _i64, C.POINTER(_f64), C.POINTER(_f64)],
    "dsgd_margins": [_vp, _vp, _vp, _i64, _vp],
    "dsgd_probabilities": [_vp, _vp, _vp, _i64, _vp],
    "dsgd_calibrated_probabilities": [_vp, _vp, _vp, _i64, _f64, _f64, _vp],
    "dsgd_isotonic_probabilities": [_vp, _vp, _vp, _i64, _vp, _vp, _i64, _vp],
    "dsgd_comm_unique_id": [_vp],
    "dsgd_comm_init": [_vp, _vp],
    "dsgd_xchg_export": [_vp, _vp],
    "dsgd_xchg_import": [_vp, C.c_int, _vp],
    "dsgd_xchg_attach": [_vp, C.c_int, _vp],
    "dsgd_xchg_stats": [_vp, C.POINTER(_i64), C.POINTER(_i64), C.POINTER(_i64)],
    "dsgd_debug_timeline": [_vp, _vp],
    "dsgd_stream_exact_rows": [_vp, C.POINTER(_i64)],
    "dsgd_set_grid_limit": [_vp, _i32],
    "dsgd_reserve": [_vp, _i64, _i64],
    "dsgd_set_workers": [_vp, _i32, _vp, _i32],
    "dsgd_sync_step": [_vp, _vp, _i64, _f64, C.POINTER(_f64)],
    "dsgd_sync_steps": [_vp, _vp, _i64, _i64, _f64, _vp],
    "dsgd_sync_steps_lr": [_vp, _vp, _i64, _i64, _vp, _vp],
    "dsgd_stage_samples": [_vp, _vp, _i64],
    "dsgd_sync_steps_staged": [_vp, _i64, _i64, _i64, _f64, C.c_int],
    "dsgd_read_losses": [_vp, _vp, _i64],
    "dsgd_average_begin": [_vp],
    "dsgd_average_end": [_vp],
    "dsgd_average_weights": [_vp, _vp, C.POINTER(_i64)],
    "dsgd_set_l1": [_vp, _f64],
    "dsgd_dim": [_vp, C.POINTER(_i32)],
    "dsgd_weights_l1": [_vp, _vp, C.POINTER(_f64), C.POINTER(_i64)],
    "dsgd_set_class_weights": [_vp, _f64, _f64],
    "dsgd_get_class_weights": [_vp, C.POINTER(_f64), C.POINTER(_f64)],
    "dsgd_set_sample_weights": [_vp, _vp, _i64],
    "dsgd_async_host_master": [_vp, _vp],
    "dsgd_ipc_export": [_vp, C.c_int, _vp],
    "dsgd_ipc_import": [_vp, C.c_int, _vp],
    "dsgd_peer_attach": [_vp, C.c_int, _vp, C.c_int],
    "dsgd_async_replay": [_vp, _vp, _vp, _i32, _i64, _f64],
    "dsgd_async_running": [_vp, C.POINTER(C.c_int)],
    "dsgd_async_master_weights": [_vp, _vp],
    "dsgd_async_outbox_enable": [_vp],
    "dsgd_async_outbox_read": [_vp, _vp],
    "dsgd_async_elapsed_ms": [_vp, C.POINTER(C.c_float)],
    "dsgd_start_async": [_vp, _vp, _vp, _i64, _i32, _f64, _i32, _i64, _u64],
    "dsgd_stop_async": [_vp],
    "dsgd_update_grad": [_vp, _vp, _vp, _i64],
    "dsgd_async_updates": [_vp, C.POINTER(_i64)],
    "dsgd_load_topics": [_vp, _i32, _vp, _vp],
    "dsgd_select_topic": [_vp, _i32],
}
_RESTYPE = {"dsgd_last_error": C.c_char_p, "dsgd_info": C.c_char_p}

# The evaluation families: each has a range, a drawn-sample and an id-list entry point, (ctx, w) and the rows of that form
# (_ROW_PREFIX), then the family's own arguments (below)
_ROW_PREFIX = {"range": [_vp, _vp, _i64, _i64], "drawn": [_vp, _vp, _i64, _i64, _u64, _i64, _i64], "list": [_vp, _vp, _vp, _i64]}
_PI64, _PF64 = C.POINTER(_i64), C.POINTER(_f64)
_QUALITY = [_f64, _f64, _i32, _vp, _vp, _vp, _vp, _vp]                  # (a, b), n_bins, the quality outputs
_ISO_QUALITY = [_vp, _vp, _i64, _i32, _vp, _vp, _vp, _vp, _vp]          # the map (x, y, k), n_bins, the quality outputs
_BOOTSTRAP = [_u64, _i64, _i64, _vp, _vp, _vp]                          # bkey, [b_begin, b_end), the replicate outputs
_ROW_FAMILIES = {
    "eval_counts": [_PI64, _PI64, _PF64], "eval_sums": [_PF64, _PI64, _PF64], "eval_class": [_PF64, _vp, _vp],
    "eval_weighted": [_PF64, _vp, _vp], "eval_metrics": [_vp], "eval_curve": [_vp, _PF64, _PI64, _vp, _vp, _vp],
    "eval_weighted_curve": [_vp, _vp, _PI64, _vp, _vp, _vp], "eval_bootstrap": _BOOTSTRAP,
    "eval_weighted_bootstrap": _BOOTSTRAP, "calibrate": [_vp, _vp, _vp], "calibrate_weighted": [_vp, _vp, _vp, _vp],
    "eval_calibration": _QUALITY, "eval_weighted_calibration": _QUALITY, "calibrate_isotonic": [_PI64] + [_vp] * 5,
    "calibrate_isotonic_weighted": [_PI64] + [_vp] * 6, "eval_isotonic_calibration": _ISO_QUALITY,
    "eval_weighted_isotonic_calibration": _ISO_QUALITY,
}


def row_methods(family: str) -> dict:
    """{form: NativeCtx method} of an evaluation family, each bound to the entry point dsgd_<method>: eval_<rest>,
    eval_sampled_<rest> and eval_samples_<rest> for an evaluation; <fit>, <fit>_sampled and <fit>_samples for the others
    (the fits and the tuning)."""
    if not family.startswith("eval_"):
        return {"range": family, "drawn": f"{family}_sampled", "list": f"{family}_samples"}
    rest = family[len("eval_"):]
    return {"range": f"eval_{rest}", "drawn": f"eval_sampled_{rest}", "list": f"eval_samples_{rest}"}


ABI.update({"dsgd_" + name: _ROW_PREFIX[form] + tail for family, tail in _ROW_FAMILIES.items()
            for form, name in row_methods(family).items()})
# the topic family takes T weight vectors and their count between (ctx, W) and the rows, then the words; the topic ranking
# family takes k after the count, then words and sums
ABI.update({"dsgd_" + name: _ROW_PREFIX[form][:2] + [_i32] + _ROW_PREFIX[form][2:] + [_vp]
            for form, name in row_methods("eval_topics").items()})
ABI.update({"dsgd_" + name: _ROW_PREFIX[form][:2] + [_i32, _i32] + _ROW_PREFIX[form][2:] + [_vp, _vp]
            for form, name in row_methods("eval_topic_ranking").items()})
ABI["dsgd_topics_topk"] = [_vp, _vp, _i32, _i32, _vp, _i64, _vp, _vp]
# the threshold tuning takes the count and fbr before the rows, then thresholds and words; the thresholded topic family takes
# the count and the thresholds before the rows, then the words
ABI.update({"dsgd_" + name: _ROW_PREFIX[form][:2] + [_i32, _f64] + _ROW_PREFIX[form][2:] + [_vp, _vp]
            for form, name in row_methods("tune_topic_thresholds").items()})
ABI.update({"dsgd_" + name: _ROW_PREFIX[form][:2] + [_i32, _vp] + _ROW_PREFIX[form][2:] + [_vp]
            for form, name in row_methods("eval_thresholded_topics").items()})


def lib():
    """Load libdsgd.so; raises NativeLibraryMissing if it has not been built."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise NativeLibraryMissing(
                f"{LIB_PATH} not found: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
                "(nvcc, sm_90a).  There is no CPU fallback for the hot path.")
        l = C.CDLL(LIB_PATH)
        for name, args in ABI.items():
            fn = getattr(l, name)  # AttributeError here == header and library disagree
            fn.argtypes = args
            fn.restype = _RESTYPE.get(name, C.c_int)
        _lib = l
    return _lib


class SynthParams(C.Structure):
    _fields_ = [("seed", C.c_uint64), ("n_rows", C.c_int64), ("dim", C.c_int32), ("mean_nnz", C.c_double),
                ("sigma", C.c_double), ("max_nnz", C.c_int32), ("zipf_s", C.c_double), ("zipf_q", C.c_double),
                ("label_noise", C.c_double)]


def host_lib():
    global _host
    if _host is None:
        if not os.path.exists(HOST_LIB_PATH):
            raise NativeLibraryMissing(f"{HOST_LIB_PATH} not found: run __graft_entry__.build()")
        h = C.CDLL(HOST_LIB_PATH)
        h.dsgd_synth_row_ptr.restype = C.c_int64
        h.dsgd_synth_row_ptr.argtypes = [C.POINTER(SynthParams), _vp]
        h.dsgd_synth_fill.argtypes = [C.POINTER(SynthParams), _vp, _vp, _vp, _vp, _vp]
        h.dsgd_rcv1_count.argtypes = [C.c_char_p, C.POINTER(_i64), C.POINTER(_i64)]
        h.dsgd_rcv1_parse.argtypes = [C.c_char_p, _i32, _i64, _i64, _vp, _vp, _vp, _vp]
        h.dsgd_rcv1_labels.argtypes = [C.c_char_p, _vp, _i64, _vp]
        h.dsgd_rcv1_topics_count.argtypes = [C.c_char_p, C.POINTER(_i64), C.POINTER(_i32), C.POINTER(_i64)]
        h.dsgd_rcv1_topics_parse.argtypes = [C.c_char_p, _i64, _i32, _i64, C.c_char_p, _vp, _vp]
        h.dsgd_rcv1_write.argtypes = [C.c_char_p, C.c_char_p, _i64, _vp, _vp, _vp, _vp, _i64]
        h.dsgd_draw_epoch.restype = C.c_int64
        h.dsgd_draw_epoch.argtypes = [C.c_uint64, _i64, _i32, _vp, _vp, _i32, _vp, _vp, _i64]
        h.dsgd_feistel_pos.restype = C.c_uint32
        h.dsgd_feistel_pos.argtypes = [C.c_uint32, C.c_uint64, C.c_uint64]
        h.dsgd_bootstrap_draw.restype = C.c_int
        h.dsgd_bootstrap_draw.argtypes = [C.c_uint64, C.c_uint64, C.c_uint64]
        _host = h
    return _host


class _Rows(NamedTuple):
    """The rows of one request: the C arguments of its form, the number of rows, and the id array those arguments point
    into (held here so that it outlives the call)."""
    args: tuple
    n: int
    ids: Optional[np.ndarray] = None


def _range(row_begin: int, row_end: int) -> _Rows:
    return _Rows((row_begin, row_end), row_end - row_begin)


def _drawn(row_begin: int, row_end: int, key: int, pos_begin: int, pos_end: int) -> _Rows:
    """Positions [pos_begin, pos_end) of a sample drawn on the device from rows [row_begin, row_end): the key goes in as
    64 bits."""
    return _Rows((row_begin, row_end, int(key) & 0xFFFFFFFFFFFFFFFF, pos_begin, pos_end), pos_end - pos_begin)


def _list(samples) -> _Rows:
    ids = _arr(samples, np.int32)
    return _Rows((_ptr(ids), ids.size), ids.size, ids)


# out-parameters of the dsgd_eval_*counts and dsgd_eval_*sums calls: (hinge sum | loss sum, correct count, ||w||^2)
_COUNTS = (_i64, _i64, _f64)


class ClassEval(NamedTuple):
    """One per-class evaluation (dsgd_eval*_class): ||w||^2, the unweighted loss sums and the correct and row counts of the
    y = +1 and y = -1 rows."""
    norm_squared: float
    loss_pos: float
    loss_neg: float
    correct_pos: int
    correct_neg: int
    n_pos: int
    n_neg: int

    def weighted_loss_sum(self, w_pos: float, w_neg: float) -> float:
        return w_pos * self.loss_pos + w_neg * self.loss_neg


class WeightedEval(NamedTuple):
    """One weighted evaluation (dsgd_eval*_weighted): ||w||^2, the fixed-point sums over the rows of c_i L_i, of c_i over the
    correctly predicted rows and of c_i (c_i = class weight x sample weight), and the row and correct counts."""
    norm_squared: float
    loss_sum: float
    correct_weight: float
    weight_sum: float
    n: int
    correct: int

_SUMS = (_f64, _i64, _f64)

WCURVE_WORDS = 13   # DSGD_WCURVE_WORDS


class WeightedCurve(NamedTuple):
    """One weighted curve (dsgd_eval*_weighted_curve): the metrics words (counts), the DSGD_WCURVE_WORDS weighted words
    (include/dsgd.h), the number of points m, the points (thresholds, W+(>= t) and W-(>= t); empty arrays for a words-only
    pass), and the weighted ROC AUC and average precision derived from the words."""
    words: np.ndarray
    wsums: np.ndarray
    n_points: int
    thr: np.ndarray
    tpw: np.ndarray
    fpw: np.ndarray
    auc: float
    ap: float


def weighted_auc_ap(words, wsums) -> tuple:
    """(AUC, AP) of a weighted curve: U2w / (2 W+ W-), NaN when a score is NaN or W+ or W- is 0; S_ap / W+, NaN when a score
    is NaN or W+ is 0, and 1 when W- is 0."""
    nan, wp, wn = int(words[7]) > 0, float(wsums[11]), float(wsums[12])
    auc = math.nan if nan or wp == 0.0 or wn == 0.0 else float(wsums[6]) / (2.0 * wp * wn)
    ap = math.nan if nan or wp == 0.0 else 1.0 if wn == 0.0 else float(wsums[8]) / wp
    return auc, ap


def _ptr(a: Optional[np.ndarray]):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


def _arr(a, dtype, n: Optional[int] = None, what: str = "array") -> np.ndarray:
    a = np.ascontiguousarray(a, dtype=dtype).reshape(-1)
    if n is not None and a.size != n:
        raise DsgdInvalid(ERR_INVALID, f"{what}: expected {n} elements, got {a.size}")
    return a


class NativeCtx:
    """One dsgd_ctx == one GPU worker (a reference Slave with its SparseSVM, or with the model named by `model`: "svm",
    "logistic", "squared_hinge" or "modified_huber"; `logistic=True` is model="logistic").  intercept=True: the model fits an
    unregularised intercept (DSGD_FLAG_INTERCEPT), and every weight vector in or out is wdim = dim + 1 long, the intercept
    last; d stays dim long."""

    def __init__(self, device: int, dim: int, lam: float, rank: int = 0, world: int = 1, is_async: bool = False,
                 logistic: bool = False, model: Optional[str] = None, intercept: bool = False):
        if model is None:
            model = "logistic" if logistic else "svm"
        elif model not in MODEL_FLAGS or (logistic and model != "logistic"):
            raise ValueError(f"NativeCtx: model must be one of {', '.join(MODEL_FLAGS)} (got {model!r}, logistic={logistic})")
        self._l = lib()
        self._h = C.c_void_p()
        self.dim, self.lam, self.rank, self.world, self.device = int(dim), float(lam), int(rank), int(world), int(device)
        self.model = model
        self.logistic = model == "logistic"
        self.intercept = bool(intercept)
        self.wdim = self.dim + (1 if self.intercept else 0)
        flags = (FLAG_ASYNC if is_async else 0) | MODEL_FLAGS[model] | (FLAG_INTERCEPT if self.intercept else 0)
        rc = self._l.dsgd_create(C.byref(self._h), device, dim, lam, rank, world, flags)
        if rc != OK:
            msg = (self._l.dsgd_last_error(None) or b"").decode()
            self._h = C.c_void_p()
            raise _EXC.get(rc, DsgdError)(rc, msg)
        self.n_rows = 0
        self.n_topics = 0

    # -- plumbing --
    def _ck(self, rc: int):
        if rc != OK:
            raise _EXC.get(rc, DsgdError)(rc, (self._l.dsgd_last_error(self._h) or b"").decode())

    def close(self):
        if getattr(self, "_h", None) and self._h.value:
            self._l.dsgd_destroy(self._h)
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def __enter__(self):
        return self

    def __exit__(self, *a):
        self.close()

    def info(self) -> dict:
        return json.loads(self._l.dsgd_info(self._h).decode())

    def set_stream(self, cuda_stream: Optional[int]):
        self._ck(self._l.dsgd_set_stream(self._h, C.c_void_p(cuda_stream) if cuda_stream else None))

    def synchronize(self):
        self._ck(self._l.dsgd_synchronize(self._h))

    def timer_start(self):
        self._ck(self._l.dsgd_timer_start(self._h))

    def timer_stop(self) -> float:
        ms = C.c_float()
        self._ck(self._l.dsgd_timer_stop(self._h, C.byref(ms)))
        return ms.value

    def launch_count(self) -> int:
        n = C.c_int64()
        self._ck(self._l.dsgd_launch_count(self._h, C.byref(n)))
        return n.value

    def profile_begin(self, sample_every: int = 1):
        self._ck(self._l.dsgd_profile_begin(self._h, sample_every))

    def profile_end(self) -> Tuple[float, int]:
        """(mean duration in ms of the sampled gradient-kernel launches, number sampled)."""
        ms, n = C.c_float(), C.c_int64()
        self._ck(self._l.dsgd_profile_end(self._h, C.byref(ms), C.byref(n)))
        return ms.value, n.value

    # -- data / model --
    def load_csr(self, row_ptr, col, val, label):
        row_ptr = _arr(row_ptr, np.int64)
        n_rows = row_ptr.size - 1
        nnz = int(row_ptr[-1]) if row_ptr.size else 0
        col, val, label = _arr(col, np.int32), _arr(val, np.float32), _arr(label, np.int8, n_rows, "label")
        if col.size != val.size or col.size < nnz:
            raise DsgdInvalid(ERR_INVALID, "load_csr: col/val shorter than row_ptr[-1]")
        self._ck(self._l.dsgd_load_csr(self._h, n_rows, nnz, _ptr(row_ptr), _ptr(col), _ptr(val), _ptr(label)))
        self.n_rows = n_rows
        self.n_topics = 0

    def set_dim_sparsity(self, d):
        d = _arr(d, np.float64, self.dim, "dim_sparsity")
        self._ck(self._l.dsgd_set_dim_sparsity(self._h, _ptr(d)))

    def compute_dim_sparsity(self, n_train: int) -> np.ndarray:
        out = np.zeros(self.dim, dtype=np.float64)
        self._ck(self._l.dsgd_compute_dim_sparsity(self._h, n_train, _ptr(out)))
        return out

    def set_weights(self, w):
        w = _arr(w, np.float64, self.wdim, "weights")
        self._ck(self._l.dsgd_set_weights(self._h, _ptr(w)))

    def get_weights(self) -> np.ndarray:
        out = np.zeros(self.wdim, dtype=np.float64)
        self._ck(self._l.dsgd_get_weights(self._h, _ptr(out)))
        return out

    # -- requests --
    def _w(self, w):
        return None if w is None else _arr(w, np.float64, self.wdim, "weights")

    def _call(self, fn: str, w, rows: _Rows, *args):
        """dsgd_<fn>(ctx, w, *rows, *args), checked; w None: the resident weights."""
        w = self._w(w)
        self._ck(getattr(self._l, "dsgd_" + fn)(self._h, _ptr(w), *rows.args, *args))

    def forward(self, samples, w=None) -> np.ndarray:
        rows = _list(samples)
        return self._request("forward", w, rows, np.zeros(rows.n, dtype=np.float64))

    def gradient(self, samples, w=None, want_loss: bool = False):
        out = np.zeros(self.wdim, dtype=np.float64)
        loss = C.c_double()
        self._call("gradient", w, _list(samples), _ptr(out), C.byref(loss) if want_loss else None)
        return (out, loss.value) if want_loss else out

    def _request(self, fn: str, w, rows: _Rows, out):
        """dsgd_<fn>(ctx, w, *rows, out...).  out: an array, filled and returned, or ctypes scalar types, passed by reference
        and returned as a tuple of values."""
        if isinstance(out, np.ndarray):
            self._call(fn, w, rows, _ptr(out))
            return out
        vals = [t() for t in out]
        self._call(fn, w, rows, *[C.byref(v) for v in vals])
        return tuple([v.value for v in vals])

    def eval(self, row_begin: int, row_end: int, w=None) -> Tuple[float, float]:
        return self._request("eval", w, _range(row_begin, row_end), (_f64, _f64))

    def eval_counts(self, row_begin: int, row_end: int, w=None) -> Tuple[int, int, float]:
        """(hinge sum, correct count, ||w||^2) over rows [row_begin, row_end) -- exact shardable form."""
        return self._request("eval_counts", w, _range(row_begin, row_end), _COUNTS)

    def eval_sampled_counts(self, row_begin: int, row_end: int, key: int, pos_begin: int, pos_end: int,
                            w=None) -> Tuple[int, int, float]:
        """(hinge sum, correct count, ||w||^2) over positions [pos_begin, pos_end) of the sample drawn on the device from rows
        [row_begin, row_end) with `key` (dsgd_eval_sampled_counts)."""
        return self._request("eval_sampled_counts", w, _drawn(row_begin, row_end, key, pos_begin, pos_end), _COUNTS)

    def eval_samples_counts(self, samples, w=None) -> Tuple[int, int, float]:
        """The same counters over a list of row ids; repeats count every time (dsgd_eval_samples_counts)."""
        return self._request("eval_samples_counts", w, _list(samples), _COUNTS)

    def eval_sums(self, row_begin: int, row_end: int, w=None) -> Tuple[float, int, float]:
        """(loss sum, correct count, ||w||^2) over rows [row_begin, row_end), for either model (dsgd_eval_sums)."""
        return self._request("eval_sums", w, _range(row_begin, row_end), _SUMS)

    def eval_sampled_sums(self, row_begin: int, row_end: int, key: int, pos_begin: int, pos_end: int,
                          w=None) -> Tuple[float, int, float]:
        """(loss sum, correct count, ||w||^2) over positions [pos_begin, pos_end) of the device-drawn sample
        (dsgd_eval_sampled_sums)."""
        return self._request("eval_sampled_sums", w, _drawn(row_begin, row_end, key, pos_begin, pos_end), _SUMS)

    def eval_samples_sums(self, samples, w=None) -> Tuple[float, int, float]:
        """(loss sum, correct count, ||w||^2) over a list of row ids; repeats count every time (dsgd_eval_samples_sums)."""
        return self._request("eval_samples_sums", w, _list(samples), _SUMS)

    # -- scores and ranking metrics --
    def margins(self, samples, w=None) -> np.ndarray:
        """x . w in fp64 for each listed row (dsgd_margins)."""
        rows = _list(samples)
        return self._request("margins", w, rows, np.zeros(rows.n, dtype=np.float64))

    def probabilities(self, samples, w=None) -> np.ndarray:
        """P(y = +1 | x) for each listed row (dsgd_probabilities): sigmoid(-x . w) on a SparseLogistic context,
        (clip(-x . w, -1, 1) + 1) / 2 on a SparseModifiedHuber one; other models raise DsgdState."""
        rows = _list(samples)
        return self._request("probabilities", w, rows, np.zeros(rows.n, dtype=np.float64))

    def eval_metrics(self, row_begin: int, row_end: int, w=None) -> np.ndarray:
        """The METRICS_WORDS exact counts over rows [row_begin, row_end) (dsgd_eval_metrics)."""
        return self._request("eval_metrics", w, _range(row_begin, row_end), np.zeros(METRICS_WORDS, dtype=np.int64))

    def eval_sampled_metrics(self, row_begin: int, row_end: int, key: int, pos_begin: int, pos_end: int,
                             w=None) -> np.ndarray:
        """The same counts over positions [pos_begin, pos_end) of the device-drawn sample (dsgd_eval_sampled_metrics)."""
        return self._request("eval_sampled_metrics", w, _drawn(row_begin, row_end, key, pos_begin, pos_end),
                             np.zeros(METRICS_WORDS, dtype=np.int64))

    def eval_samples_metrics(self, samples, w=None) -> np.ndarray:
        """The same counts over a list of row ids; repeats count every time (dsgd_eval_samples_metrics)."""
        return self._request("eval_samples_metrics", w, _list(samples), np.zeros(METRICS_WORDS, dtype=np.int64))

    # -- calibration --
    def _calibrate(self, fn: str, w, rows: _Rows):
        """dsgd_<fn>: (A, B, objective, info) of one Platt fit; info = the CALIBRATION_INFO_WORDS words {iterations, status,
        rows used, NaN rows, points evaluated}."""
        ab = np.zeros(2, dtype=np.float64)
        info = np.zeros(CALIBRATION_INFO_WORDS, dtype=np.int64)
        obj = C.c_double()
        self._call(fn, w, rows, _ptr(ab), C.byref(obj), _ptr(info))
        return float(ab[0]), float(ab[1]), obj.value, info

    def calibrate(self, row_begin: int, row_end: int, w=None):
        """Platt scaling of x . w over rows [row_begin, row_end) (dsgd_calibrate): (A, B, objective, info) with
        P(y = +1 | x) = 1 / (1 + exp(A x . w + B))."""
        return self._calibrate("calibrate", w, _range(row_begin, row_end))

    def calibrate_sampled(self, row_begin: int, row_end: int, key: int, pos_begin: int, pos_end: int, w=None):
        """The same over positions [pos_begin, pos_end) of the device-drawn sample (dsgd_calibrate_sampled)."""
        return self._calibrate("calibrate_sampled", w, _drawn(row_begin, row_end, key, pos_begin, pos_end))

    def calibrate_samples(self, samples, w=None):
        """The same over a list of row ids; repeats count every time (dsgd_calibrate_samples)."""
        return self._calibrate("calibrate_samples", w, _list(samples))

    def calibrated_probabilities(self, samples, a: float, b: float, w=None) -> np.ndarray:
        """sigmoid(-(a x . w + b)) for each listed row, either model (dsgd_calibrated_probabilities)."""
        rows = _list(samples)
        out = np.zeros(rows.n, dtype=np.float64)
        self._call("calibrated_probabilities", w, rows, float(a), float(b), _ptr(out))
        return out

    def _eval_calibration(self, fn: str, w, rows: _Rows, a: float, b: float, n_bins: int):
        """dsgd_<fn>: (sums, bin_rows, bin_pos, bin_psum, words): sums = {Brier, log loss} sums, words = {rows used, rows
        left out}."""
        m = max(int(n_bins), 1)
        sums, words = np.zeros(2, dtype=np.float64), np.zeros(2, dtype=np.int64)
        rows_b, pos_b, psum = np.zeros(m, dtype=np.int64), np.zeros(m, dtype=np.int64), np.zeros(m, dtype=np.float64)
        self._call(fn, w, rows, float(a), float(b), int(n_bins), _ptr(sums), _ptr(rows_b), _ptr(pos_b), _ptr(psum),
                   _ptr(words))
        return sums, rows_b, pos_b, psum, words

    def eval_calibration(self, row_begin: int, row_end: int, a: float, b: float, n_bins: int = 10, w=None):
        """Brier and log-loss sums and n_bins reliability bins at (a, b) over rows [row_begin, row_end)
        (dsgd_eval_calibration)."""
        return self._eval_calibration("eval_calibration", w, _range(row_begin, row_end), a, b, n_bins)

    def eval_sampled_calibration(self, row_begin: int, row_end: int, key: int, pos_begin: int, pos_end: int, a: float,
                                 b: float, n_bins: int = 10, w=None):
        """The same over positions [pos_begin, pos_end) of the device-drawn sample (dsgd_eval_sampled_calibration)."""
        return self._eval_calibration("eval_sampled_calibration", w, _drawn(row_begin, row_end, key, pos_begin, pos_end), a, b,
                                      n_bins)

    def eval_samples_calibration(self, samples, a: float, b: float, n_bins: int = 10, w=None):
        """The same over a list of row ids; repeats count every time (dsgd_eval_samples_calibration)."""
        return self._eval_calibration("eval_samples_calibration", w, _list(samples), a, b, n_bins)

    # -- weighted calibration --
    def _calibrate_weighted(self, fn: str, w, rows: _Rows):
        """dsgd_<fn>: (A, B, objective, info, wsums) of one weighted Platt fit; info as _calibrate's, wsums = the
        CALIBRATION_WSUMS doubles {W+, W-, NaN rows' weight}."""
        ab = np.zeros(2, dtype=np.float64)
        info = np.zeros(CALIBRATION_INFO_WORDS, dtype=np.int64)
        wsums = np.zeros(CALIBRATION_WSUMS, dtype=np.float64)
        obj = C.c_double()
        self._call(fn, w, rows, _ptr(ab), C.byref(obj), _ptr(info), _ptr(wsums))
        return float(ab[0]), float(ab[1]), obj.value, info, wsums

    def calibrate_weighted(self, row_begin: int, row_end: int, w=None):
        """Platt scaling with every row counted by its weight c_i over rows [row_begin, row_end) (dsgd_calibrate_weighted)."""
        return self._calibrate_weighted("calibrate_weighted", w, _range(row_begin, row_end))

    def calibrate_weighted_sampled(self, row_begin: int, row_end: int, key: int, pos_begin: int, pos_end: int, w=None):
        """The same over positions [pos_begin, pos_end) of the device-drawn sample (dsgd_calibrate_weighted_sampled)."""
        return self._calibrate_weighted("calibrate_weighted_sampled", w, _drawn(row_begin, row_end, key, pos_begin, pos_end))

    def calibrate_weighted_samples(self, samples, w=None):
        """The same over a list of row ids; repeats count every time (dsgd_calibrate_weighted_samples)."""
        return self._calibrate_weighted("calibrate_weighted_samples", w, _list(samples))

    def _eval_weighted_calibration(self, fn: str, w, rows: _Rows, a: float, b: float, n_bins: int):
        """dsgd_<fn>: (sums, bin_weight, bin_pos_weight, bin_psum, words): sums = the WCALIBRATION_SUMS doubles {Brier sum,
        log-loss sum, weight used, infinite-term weight}, words = {rows used, rows left out}."""
        m = max(int(n_bins), 1)
        sums, words = np.zeros(WCALIBRATION_SUMS, dtype=np.float64), np.zeros(2, dtype=np.int64)
        wb, pwb, psum = np.zeros(m), np.zeros(m), np.zeros(m)
        self._call(fn, w, rows, float(a), float(b), int(n_bins), _ptr(sums), _ptr(wb), _ptr(pwb), _ptr(psum), _ptr(words))
        return sums, wb, pwb, psum, words

    def eval_weighted_calibration(self, row_begin: int, row_end: int, a: float, b: float, n_bins: int = 10, w=None):
        """Weighted Brier and log-loss sums and n_bins weighted reliability bins at (a, b) over rows [row_begin, row_end)
        (dsgd_eval_weighted_calibration)."""
        return self._eval_weighted_calibration("eval_weighted_calibration", w, _range(row_begin, row_end), a, b, n_bins)

    def eval_sampled_weighted_calibration(self, row_begin: int, row_end: int, key: int, pos_begin: int, pos_end: int,
                                          a: float, b: float, n_bins: int = 10, w=None):
        """The same over positions [pos_begin, pos_end) of the device-drawn sample (dsgd_eval_sampled_weighted_calibration)."""
        return self._eval_weighted_calibration("eval_sampled_weighted_calibration", w,
                                               _drawn(row_begin, row_end, key, pos_begin, pos_end), a, b, n_bins)

    def eval_samples_weighted_calibration(self, samples, a: float, b: float, n_bins: int = 10, w=None):
        """The same over a list of row ids; repeats count every time (dsgd_eval_samples_weighted_calibration)."""
        return self._eval_weighted_calibration("eval_samples_weighted_calibration", w, _list(samples), a, b, n_bins)

    # -- isotonic calibration --
    def _calibrate_isotonic(self, fn: str, w, rows: _Rows):
        """dsgd_<fn>: (x, y, block_rows, block_pos, info) of one isotonic fit over the rows; info = the ISOTONIC_INFO_WORDS
        words {blocks, points, rows used, NaN rows, distinct scores}."""
        size = max(int(rows.n), 1)
        x, y = np.zeros(size, dtype=np.float64), np.zeros(size, dtype=np.float64)
        br, bp = np.zeros(size, dtype=np.int64), np.zeros(size, dtype=np.int64)
        info, k = np.zeros(ISOTONIC_INFO_WORDS, dtype=np.int64), C.c_int64()
        self._call(fn, w, rows, C.byref(k), _ptr(x), _ptr(y), _ptr(br), _ptr(bp), _ptr(info))
        nb = int(info[0])
        return x[:k.value].copy(), y[:k.value].copy(), br[:nb].copy(), bp[:nb].copy(), info

    def calibrate_isotonic(self, row_begin: int, row_end: int, w=None):
        """Isotonic regression of the labels on s = -x . w over rows [row_begin, row_end) (dsgd_calibrate_isotonic):
        (x, y, block_rows, block_pos, info), x ascending, P(y = +1 | x) = numpy.interp(s, x, y)."""
        return self._calibrate_isotonic("calibrate_isotonic", w, _range(row_begin, row_end))

    def calibrate_isotonic_sampled(self, row_begin: int, row_end: int, key: int, pos_begin: int, pos_end: int, w=None):
        """The same over positions [pos_begin, pos_end) of the device-drawn sample (dsgd_calibrate_isotonic_sampled)."""
        return self._calibrate_isotonic("calibrate_isotonic_sampled", w, _drawn(row_begin, row_end, key, pos_begin, pos_end))

    def calibrate_isotonic_samples(self, samples, w=None):
        """The same over a list of row ids; repeats count every time (dsgd_calibrate_isotonic_samples)."""
        return self._calibrate_isotonic("calibrate_isotonic_samples", w, _list(samples))

    def isotonic_probabilities(self, samples, x, y, w=None) -> np.ndarray:
        """numpy.interp(-x_i . w, x, y) for each listed row, any model (dsgd_isotonic_probabilities)."""
        rows = _list(samples)
        x, y = _arr(x, np.float64), _arr(y, np.float64)
        out = np.zeros(rows.n, dtype=np.float64)
        self._call("isotonic_probabilities", w, rows, _ptr(x), _ptr(y), x.size if x.size == y.size else -1, _ptr(out))
        return out

    def _eval_isotonic_calibration(self, fn: str, w, rows: _Rows, x, y, n_bins: int):
        """dsgd_<fn>: (sums, bin_rows, bin_pos, bin_psum, words): sums = {Brier sum, log-loss sum over the finite terms},
        words = {rows used, rows left out, rows with an infinite term}."""
        x, y = _arr(x, np.float64), _arr(y, np.float64)
        m = max(int(n_bins), 1)
        sums, words = np.zeros(2, dtype=np.float64), np.zeros(ISOTONIC_EVAL_WORDS, dtype=np.int64)
        rows_b, pos_b, psum = np.zeros(m, dtype=np.int64), np.zeros(m, dtype=np.int64), np.zeros(m, dtype=np.float64)
        self._call(fn, w, rows, _ptr(x), _ptr(y), x.size if x.size == y.size else -1, int(n_bins), _ptr(sums), _ptr(rows_b),
                   _ptr(pos_b), _ptr(psum), _ptr(words))
        return sums, rows_b, pos_b, psum, words

    def _calibrate_isotonic_weighted(self, fn: str, w, rows: _Rows):
        """dsgd_<fn>: (x, y, block_weight, block_pos_weight, info, wsums) of one weighted isotonic fit over the rows; info as
        _calibrate_isotonic's (rows and scores of positive weight), wsums = {W+, W-}."""
        size = max(int(rows.n), 1)
        x, y, bw, bp = (np.zeros(size, dtype=np.float64) for _ in range(4))
        info, k, ws = np.zeros(ISOTONIC_INFO_WORDS, dtype=np.int64), C.c_int64(), np.zeros(2)
        self._call(fn, w, rows, C.byref(k), _ptr(x), _ptr(y), _ptr(bw), _ptr(bp), _ptr(info), _ptr(ws))
        nb = int(info[0])
        return x[:k.value].copy(), y[:k.value].copy(), bw[:nb].copy(), bp[:nb].copy(), info, ws

    def calibrate_isotonic_weighted(self, row_begin: int, row_end: int, w=None):
        """Isotonic regression with every row counted by its weight c_i over rows [row_begin, row_end)
        (dsgd_calibrate_isotonic_weighted)."""
        return self._calibrate_isotonic_weighted("calibrate_isotonic_weighted", w, _range(row_begin, row_end))

    def calibrate_isotonic_weighted_sampled(self, row_begin: int, row_end: int, key: int, pos_begin: int, pos_end: int,
                                            w=None):
        """The same over positions [pos_begin, pos_end) of the device-drawn sample."""
        return self._calibrate_isotonic_weighted("calibrate_isotonic_weighted_sampled", w,
                                                 _drawn(row_begin, row_end, key, pos_begin, pos_end))

    def calibrate_isotonic_weighted_samples(self, samples, w=None):
        """The same over a list of row ids; repeats count every time."""
        return self._calibrate_isotonic_weighted("calibrate_isotonic_weighted_samples", w, _list(samples))

    def _eval_weighted_isotonic_calibration(self, fn: str, w, rows: _Rows, x, y, n_bins: int):
        """dsgd_<fn>: (sums, bin_weight, bin_pos_weight, bin_psum, words): sums = {Brier sum, log-loss sum over the finite
        terms, weight used, weight of the infinite terms}, words = {rows used, rows left out, rows with an infinite term}."""
        x, y = _arr(x, np.float64), _arr(y, np.float64)
        m = max(int(n_bins), 1)
        sums, words = np.zeros(WCALIBRATION_SUMS), np.zeros(ISOTONIC_EVAL_WORDS, dtype=np.int64)
        wb, pwb, psum = np.zeros(m), np.zeros(m), np.zeros(m)
        self._call(fn, w, rows, _ptr(x), _ptr(y), x.size if x.size == y.size else -1, int(n_bins), _ptr(sums), _ptr(wb),
                   _ptr(pwb), _ptr(psum), _ptr(words))
        return sums, wb, pwb, psum, words

    def eval_weighted_isotonic_calibration(self, row_begin: int, row_end: int, x, y, n_bins: int = 10, w=None):
        """Weighted quality at the isotonic map (x, y) over rows [row_begin, row_end)."""
        return self._eval_weighted_isotonic_calibration("eval_weighted_isotonic_calibration", w, _range(row_begin, row_end),
                                                        x, y, n_bins)

    def eval_sampled_weighted_isotonic_calibration(self, row_begin: int, row_end: int, key: int, pos_begin: int,
                                                   pos_end: int, x, y, n_bins: int = 10, w=None):
        """The same over positions [pos_begin, pos_end) of the device-drawn sample."""
        return self._eval_weighted_isotonic_calibration("eval_sampled_weighted_isotonic_calibration", w,
                                                        _drawn(row_begin, row_end, key, pos_begin, pos_end), x, y, n_bins)

    def eval_samples_weighted_isotonic_calibration(self, samples, x, y, n_bins: int = 10, w=None):
        """The same over a list of row ids; repeats count every time."""
        return self._eval_weighted_isotonic_calibration("eval_samples_weighted_isotonic_calibration", w, _list(samples), x, y,
                                                        n_bins)

    def eval_isotonic_calibration(self, row_begin: int, row_end: int, x, y, n_bins: int = 10, w=None):
        """Brier and log-loss sums and n_bins reliability bins at the map (x, y) over rows [row_begin, row_end)
        (dsgd_eval_isotonic_calibration)."""
        return self._eval_isotonic_calibration("eval_isotonic_calibration", w, _range(row_begin, row_end), x, y, n_bins)

    def eval_sampled_isotonic_calibration(self, row_begin: int, row_end: int, key: int, pos_begin: int, pos_end: int, x, y,
                                          n_bins: int = 10, w=None):
        """The same over positions [pos_begin, pos_end) of the device-drawn sample (dsgd_eval_sampled_isotonic_calibration)."""
        return self._eval_isotonic_calibration("eval_sampled_isotonic_calibration", w,
                                               _drawn(row_begin, row_end, key, pos_begin, pos_end), x, y, n_bins)

    def eval_samples_isotonic_calibration(self, samples, x, y, n_bins: int = 10, w=None):
        """The same over a list of row ids; repeats count every time (dsgd_eval_samples_isotonic_calibration)."""
        return self._eval_isotonic_calibration("eval_samples_isotonic_calibration", w, _list(samples), x, y, n_bins)

    def _curve(self, fn: str, w, rows: _Rows, curve: bool):
        """dsgd_<fn>: (words, ap, thr, tp, fp) with the m points of a curve pass over the rows, or (words, ap, m) when not
        `curve` (the average-precision-only pass)."""
        n = max(rows.n, 0)
        words = np.zeros(METRICS_WORDS, dtype=np.int64)
        ap, m = C.c_double(), C.c_int64()
        thr = np.zeros(n, dtype=np.float64) if curve else None
        tp = np.zeros(n, dtype=np.int64) if curve else None
        fp = np.zeros(n, dtype=np.int64) if curve else None
        self._call(fn, w, rows, _ptr(words), C.byref(ap), C.byref(m), _ptr(thr), _ptr(tp), _ptr(fp))
        if not curve:
            return words, ap.value, m.value
        k = m.value
        return words, ap.value, thr[:k].copy(), tp[:k].copy(), fp[:k].copy()

    def eval_curve(self, row_begin: int, row_end: int, w=None, curve: bool = True):
        """ROC / precision-recall points and average precision over rows [row_begin, row_end) (dsgd_eval_curve): (words,
        ap, thr, tp, fp), one point per distinct score, highest first; curve=False: (words, ap, number of points)."""
        return self._curve("eval_curve", w, _range(row_begin, row_end), curve)

    def eval_sampled_curve(self, row_begin: int, row_end: int, key: int, pos_begin: int, pos_end: int, w=None,
                           curve: bool = True):
        """The same over positions [pos_begin, pos_end) of the device-drawn sample (dsgd_eval_sampled_curve)."""
        return self._curve("eval_sampled_curve", w, _drawn(row_begin, row_end, key, pos_begin, pos_end), curve)

    def eval_samples_curve(self, samples, w=None, curve: bool = True):
        """The same over a list of row ids; repeats count every time (dsgd_eval_samples_curve)."""
        return self._curve("eval_samples_curve", w, _list(samples), curve)

    # -- bootstrap --
    def _bootstrap(self, fn: str, w, rows: _Rows, bkey: int, b_begin: int, b_end: int):
        """dsgd_<fn>: (words[b_end - b_begin, BOOTSTRAP_WORDS], ap[...], loss_sum[...]) of replicates [b_begin, b_end)."""
        k = max(int(b_end) - int(b_begin), 0)
        words = np.zeros((max(k, 1), BOOTSTRAP_WORDS), dtype=np.int64)
        ap = np.zeros(max(k, 1), dtype=np.float64)
        loss = np.zeros(max(k, 1), dtype=np.float64)
        self._call(fn, w, rows, int(bkey) & 0xFFFFFFFFFFFFFFFF, int(b_begin), int(b_end), _ptr(words), _ptr(ap), _ptr(loss))
        return words[:k], ap[:k], loss[:k]

    def eval_bootstrap(self, row_begin: int, row_end: int, bkey: int, b_begin: int, b_end: int, w=None):
        """Poisson-bootstrap replicates [b_begin, b_end) of rows [row_begin, row_end) with key bkey (dsgd_eval_bootstrap):
        (words, ap, loss_sum), one row per replicate -- the metrics words and size, the average precision and the loss sum of
        the replicate's expanded list."""
        return self._bootstrap("eval_bootstrap", w, _range(row_begin, row_end), bkey, b_begin, b_end)

    def eval_sampled_bootstrap(self, row_begin: int, row_end: int, key: int, pos_begin: int, pos_end: int, bkey: int,
                               b_begin: int, b_end: int, w=None):
        """The same over positions [pos_begin, pos_end) of the device-drawn sample (dsgd_eval_sampled_bootstrap)."""
        return self._bootstrap("eval_sampled_bootstrap", w, _drawn(row_begin, row_end, key, pos_begin, pos_end), bkey,
                               b_begin, b_end)

    def eval_samples_bootstrap(self, samples, bkey: int, b_begin: int, b_end: int, w=None):
        """The same over a list of row ids, position i being list index i (dsgd_eval_samples_bootstrap)."""
        return self._bootstrap("eval_samples_bootstrap", w, _list(samples), bkey, b_begin, b_end)

    # -- sync --
    def set_workers(self, counts, k_total: int = 0):
        """Logical workers on this ctx: counts[v] samples each per step; k_total = Vec.mean divisor."""
        counts = _arr(counts, np.int32)
        self._ck(self._l.dsgd_set_workers(self._h, counts.size, _ptr(counts) if counts.size else None, k_total))

    @staticmethod
    def comm_unique_id() -> bytes:
        buf = (C.c_uint8 * UNIQUE_ID_BYTES)()
        rc = lib().dsgd_comm_unique_id(C.cast(buf, C.c_void_p))
        if rc != OK:
            raise DsgdError(rc, (lib().dsgd_last_error(None) or b"").decode())
        return bytes(buf)

    def comm_init(self, uid: bytes):
        assert len(uid) == UNIQUE_ID_BYTES
        buf = (C.c_uint8 * UNIQUE_ID_BYTES).from_buffer_copy(uid)
        self._ck(self._l.dsgd_comm_init(self._h, C.cast(buf, C.c_void_p)))

    def xchg_export(self) -> bytes:
        buf = (C.c_uint8 * IPC_HANDLE_BYTES)()
        self._ck(self._l.dsgd_xchg_export(self._h, C.cast(buf, C.c_void_p)))
        return bytes(buf)

    def xchg_import(self, peer_rank: int, handle: bytes):
        buf = (C.c_uint8 * IPC_HANDLE_BYTES).from_buffer_copy(handle)
        self._ck(self._l.dsgd_xchg_import(self._h, peer_rank, C.cast(buf, C.c_void_p)))

    def xchg_attach(self, peer_rank: int, peer: "NativeCtx"):
        self._ck(self._l.dsgd_xchg_attach(self._h, peer_rank, peer._h))

    def setup_peer_exchange(self, group) -> None:
        """One process per GPU: swap exchange-block handles through the process group and map every peer's block
        (the fused multi-GPU sync step then needs no NCCL)."""
        handles = group.all_gather_bytes(self.xchg_export())
        for r, h in enumerate(handles):
            if r != self.rank:
                self.xchg_import(r, h)
        group.barrier()

    def xchg_stats(self) -> Tuple[int, int, int]:
        """(value words, bitmap words) this rank stored into EACH peer so far, and the SGD steps of those launches."""
        v, b, n = C.c_int64(), C.c_int64(), C.c_int64()
        self._ck(self._l.dsgd_xchg_stats(self._h, C.byref(v), C.byref(b), C.byref(n)))
        return v.value, b.value, n.value

    def reserve(self, n_samples: int, n_steps: int):
        """Allocate the sync path's device buffers now (see dsgd_reserve: needed when several ctxs share one GPU)."""
        self._ck(self._l.dsgd_reserve(self._h, n_samples, n_steps))

    def set_grid_limit(self, n_ctas: int):
        """CTAs of the persistent sync kernel (0: one per SM) -- lets several ranks share one GPU in tests."""
        self._ck(self._l.dsgd_set_grid_limit(self._h, n_ctas))

    TIMELINE_WORDS = 256 * 16 + 4 * 160 * 4

    def debug_timeline(self) -> np.ndarray:
        """Phase stamps of the last persistent launch (needs DSGD_PERSIST_TIMELINE in the environment)."""
        out = np.zeros(self.TIMELINE_WORDS, dtype=np.int64)
        self._ck(self._l.dsgd_debug_timeline(self._h, _ptr(out)))
        return out

    def stream_exact_rows(self) -> int:
        """Rows the streaming pass recomputed in fp64 (rounding band) since this ctx was created."""
        n = C.c_int64()
        self._ck(self._l.dsgd_stream_exact_rows(self._h, C.byref(n)))
        return n.value

    def sync_step(self, samples, lr: float, want_loss: bool = True):
        samples = _arr(samples, np.int32)
        loss = C.c_double()
        self._ck(self._l.dsgd_sync_step(self._h, _ptr(samples), samples.size, lr, C.byref(loss) if want_loss else None))
        return loss.value if want_loss else None

    def sync_steps(self, samples, n_per_step: int, n_steps: int, lr: float, want_losses: bool = True):
        samples = _arr(samples, np.int32, n_per_step * n_steps, "samples")
        losses = np.zeros(n_steps, dtype=np.float64) if want_losses else None
        self._ck(self._l.dsgd_sync_steps(self._h, _ptr(samples), n_per_step, n_steps, lr, _ptr(losses)))
        return losses

    def sync_steps_lr(self, samples, n_per_step: int, lrs, want_losses: bool = True):
        """len(lrs) steps; step s uses the learning rate lrs[s] (exactly len(lrs) one-step sync_steps calls)."""
        lrs = _arr(lrs, np.float64)
        n_steps = lrs.size
        samples = _arr(samples, np.int32, n_per_step * n_steps, "samples")
        losses = np.zeros(n_steps, dtype=np.float64) if want_losses else None
        self._ck(self._l.dsgd_sync_steps_lr(self._h, _ptr(samples), n_per_step, n_steps, _ptr(lrs), _ptr(losses)))
        return losses

    def stage_samples(self, samples):
        samples = _arr(samples, np.int32)
        self._ck(self._l.dsgd_stage_samples(self._h, _ptr(samples), samples.size))

    def sync_steps_staged(self, first: int, n_per_step: int, n_steps: int, lr: float, want_losses: bool = False):
        self._ck(self._l.dsgd_sync_steps_staged(self._h, first, n_per_step, n_steps, lr, 1 if want_losses else 0))

    def read_losses(self, n_steps: int) -> np.ndarray:
        out = np.zeros(n_steps, dtype=np.float64)
        self._ck(self._l.dsgd_read_losses(self._h, _ptr(out), n_steps))
        return out

    # -- averaged SGD (sync mode) --
    def average_begin(self):
        """Zero the running sum of the weights and its step count; every following sync step adds its new weights."""
        self._ck(self._l.dsgd_average_begin(self._h))

    def average_end(self):
        """Stop adding to the sum; the sum and the count stay readable."""
        self._ck(self._l.dsgd_average_end(self._h))

    def average_weights(self) -> Tuple[np.ndarray, int]:
        """(mean of the weights after every step averaged since average_begin, number of those steps)."""
        out = np.zeros(self.wdim, dtype=np.float64)
        n = C.c_int64()
        self._ck(self._l.dsgd_average_weights(self._h, _ptr(out), C.byref(n)))
        return out, n.value

    # -- L1 penalty (sync mode) --
    def set_l1(self, lambda1: float):
        """Every following sync step soft-thresholds every weight at lr * lambda1 after its update (0: off)."""
        self._ck(self._l.dsgd_set_l1(self._h, float(lambda1)))

    def weights_l1(self, w=None) -> Tuple[float, int]:
        """(||w||_1, number of non-zero weights) of w, or of the resident weights when w is None."""
        w = self._w(w)
        l1, nnz = C.c_double(), C.c_int64()
        self._ck(self._l.dsgd_weights_l1(self._h, _ptr(w), C.byref(l1), C.byref(nnz)))
        return l1.value, nnz.value

    # -- class weights (sync mode) and the per-class evaluations --
    def set_class_weights(self, w_pos: float, w_neg: float):
        """Every following sync step and gradient request scales the gradient and the loss of a row by the weight of its label."""
        self._ck(self._l.dsgd_set_class_weights(self._h, float(w_pos), float(w_neg)))

    def get_class_weights(self) -> Tuple[float, float]:
        wp, wn = C.c_double(), C.c_double()
        self._ck(self._l.dsgd_get_class_weights(self._h, C.byref(wp), C.byref(wn)))
        return wp.value, wn.value

    def _class(self, fn: str, w, rows: _Rows) -> "ClassEval":
        nrm = C.c_double()
        sums, counts = np.zeros(2, dtype=np.float64), np.zeros(4, dtype=np.int64)
        self._call(fn, w, rows, C.byref(nrm), _ptr(sums), _ptr(counts))
        return ClassEval(nrm.value, float(sums[0]), float(sums[1]), *[int(c) for c in counts])

    def eval_class(self, row_begin: int, row_end: int, w=None) -> "ClassEval":
        """Per-class loss sums (unweighted), correct counts and row counts over rows [row_begin, row_end) (dsgd_eval_class)."""
        return self._class("eval_class", w, _range(row_begin, row_end))

    def eval_sampled_class(self, row_begin: int, row_end: int, key: int, pos_begin: int, pos_end: int, w=None) -> "ClassEval":
        """The same over positions [pos_begin, pos_end) of the device-drawn sample (dsgd_eval_sampled_class)."""
        return self._class("eval_sampled_class", w, _drawn(row_begin, row_end, key, pos_begin, pos_end))

    def eval_samples_class(self, samples, w=None) -> "ClassEval":
        """The same over a list of row ids; repeats count every time (dsgd_eval_samples_class)."""
        return self._class("eval_samples_class", w, _list(samples))

    # -- topics (sync mode): one-vs-rest labels and the one-pass multi-label evaluation --
    def load_topics(self, topic_ptr, topic_id, n_topics: int):
        """Each loaded row's topic ids (CSR: topic_ptr int64[n_rows + 1], ids strictly ascending within a row, each in
        [0, n_topics)); the ctx keeps the loaded labels beside them (dsgd_load_topics)."""
        topic_ptr = _arr(topic_ptr, np.int64, self.n_rows + 1, "topic_ptr")
        topic_id = _arr(topic_id, np.int32)
        if topic_id.size != int(topic_ptr[-1]):
            raise DsgdInvalid(ERR_INVALID, f"load_topics: {topic_id.size} ids, topic_ptr ends at {int(topic_ptr[-1])}")
        self._ck(self._l.dsgd_load_topics(self._h, int(n_topics), _ptr(topic_ptr), _ptr(topic_id)))
        self.n_topics = int(n_topics)

    def select_topic(self, topic: int):
        """Labels "has topic t" (+1 / -1) for every following call; -1: the labels load_csr loaded (dsgd_select_topic)."""
        self._ck(self._l.dsgd_select_topic(self._h, int(topic)))

    def _topics(self, fn: str, W, rows: _Rows) -> np.ndarray:
        W = self._topic_W(fn, W)
        out = np.zeros(topic_words(W.shape[0]), dtype=np.int64)
        self._ck(getattr(self._l, "dsgd_" + fn)(self._h, _ptr(W), W.shape[0], *rows.args, _ptr(out)))
        return out

    def eval_topics(self, row_begin: int, row_end: int, W) -> np.ndarray:
        """The DSGD_TOPIC_WORDS(T) words of the T weight vectors W[T, wdim] over rows [row_begin, row_end): per topic the
        metrics words for "has topic t" (U2 left 0), then the row words (dsgd_eval_topics)."""
        return self._topics("eval_topics", W, _range(row_begin, row_end))

    def eval_sampled_topics(self, row_begin: int, row_end: int, key: int, pos_begin: int, pos_end: int, W) -> np.ndarray:
        """The same over positions [pos_begin, pos_end) of the device-drawn sample (dsgd_eval_sampled_topics)."""
        return self._topics("eval_sampled_topics", W, _drawn(row_begin, row_end, key, pos_begin, pos_end))

    def eval_samples_topics(self, samples, W) -> np.ndarray:
        """The same over a list of row ids; repeats count every time (dsgd_eval_samples_topics)."""
        return self._topics("eval_samples_topics", W, _list(samples))

    def _topic_W(self, fn: str, W) -> np.ndarray:
        W = np.ascontiguousarray(W, dtype=np.float64)
        if W.ndim != 2 or W.shape[1] != self.wdim:
            raise DsgdInvalid(ERR_INVALID, f"{fn}: W must be [T, {self.wdim}], got {W.shape}")
        return W

    def _thresholded_topics(self, fn: str, W, thresholds, rows: _Rows) -> np.ndarray:
        W = self._topic_W(fn, W)
        thr = np.ascontiguousarray(thresholds, dtype=np.float64).reshape(-1)
        if thr.size != W.shape[0]:
            raise DsgdInvalid(ERR_INVALID, f"{fn}: {thr.size} thresholds for {W.shape[0]} weight vectors")
        out = np.zeros(topic_words(W.shape[0]), dtype=np.int64)
        self._ck(getattr(self._l, "dsgd_" + fn)(self._h, _ptr(W), W.shape[0], _ptr(thr), *rows.args, _ptr(out)))
        return out

    def eval_thresholded_topics(self, row_begin: int, row_end: int, W, thresholds) -> np.ndarray:
        """eval_topics with topic t predicted present when its margin is below thresholds[t], absent above it, and not
        predicted at it or for a NaN margin (dsgd_eval_thresholded_topics)."""
        return self._thresholded_topics("eval_thresholded_topics", W, thresholds, _range(row_begin, row_end))

    def eval_sampled_thresholded_topics(self, row_begin: int, row_end: int, key: int, pos_begin: int, pos_end: int, W,
                                        thresholds) -> np.ndarray:
        """The same over positions [pos_begin, pos_end) of the device-drawn sample (dsgd_eval_sampled_thresholded_topics)."""
        return self._thresholded_topics("eval_sampled_thresholded_topics", W, thresholds,
                                        _drawn(row_begin, row_end, key, pos_begin, pos_end))

    def eval_samples_thresholded_topics(self, samples, W, thresholds) -> np.ndarray:
        """The same over a list of row ids; repeats count every time (dsgd_eval_samples_thresholded_topics)."""
        return self._thresholded_topics("eval_samples_thresholded_topics", W, thresholds, _list(samples))

    def _tune(self, fn: str, W, fbr: float, rows: _Rows) -> Tuple[np.ndarray, np.ndarray]:
        W = self._topic_W(fn, W)
        thr = np.zeros(W.shape[0], dtype=np.float64)
        words = np.zeros(topic_tune_words(W.shape[0]), dtype=np.int64)
        self._ck(getattr(self._l, "dsgd_" + fn)(self._h, _ptr(W), W.shape[0], float(fbr), *rows.args, _ptr(thr),
                                                  _ptr(words)))
        return thr, words

    def tune_topic_thresholds(self, row_begin: int, row_end: int, W, fbr: float = 0.0) -> Tuple[np.ndarray, np.ndarray]:
        """(thresholds float64[T], words int64[8 T]): each topic's F1-optimal margin threshold (SCut, with the fbr fallback)
        over rows [row_begin, row_end), and per topic the words rows, P, NaN rows, D, tp and rows predicted at the
        threshold, status and candidate (dsgd_tune_topic_thresholds)."""
        return self._tune("tune_topic_thresholds", W, fbr, _range(row_begin, row_end))

    def tune_topic_thresholds_sampled(self, row_begin: int, row_end: int, key: int, pos_begin: int, pos_end: int, W,
                                      fbr: float = 0.0) -> Tuple[np.ndarray, np.ndarray]:
        """The same over positions [pos_begin, pos_end) of the device-drawn sample (dsgd_tune_topic_thresholds_sampled)."""
        return self._tune("tune_topic_thresholds_sampled", W, fbr, _drawn(row_begin, row_end, key, pos_begin, pos_end))

    def tune_topic_thresholds_samples(self, samples, W, fbr: float = 0.0) -> Tuple[np.ndarray, np.ndarray]:
        """The same over a list of row ids; repeats count every time (dsgd_tune_topic_thresholds_samples)."""
        return self._tune("tune_topic_thresholds_samples", W, fbr, _list(samples))

    def _topic_ranking(self, fn: str, W, k: int, rows: _Rows) -> Tuple[np.ndarray, np.ndarray]:
        W = self._topic_W(fn, W)
        k = int(k)
        if not 1 <= k <= TOPIC_RANK_MAX_K:
            raise DsgdInvalid(ERR_INVALID, f"{fn}: k = {k}; 1 .. min(T, {TOPIC_RANK_MAX_K})")
        words = np.zeros(topic_rank_words(k), dtype=np.int64)
        sums = np.zeros(2 + k, dtype=np.float64)
        self._ck(getattr(self._l, "dsgd_" + fn)(self._h, _ptr(W), W.shape[0], k, *rows.args, _ptr(words), _ptr(sums)))
        return words, sums

    def eval_topic_ranking(self, row_begin: int, row_end: int, W, k: int) -> Tuple[np.ndarray, np.ndarray]:
        """(words, sums) of the ranking of every row's topics by the T weight vectors W[T, wdim] over rows
        [row_begin, row_end): the DSGD_TOPIC_RANK_WORDS(k) words (row counts, coverage, mis-ordered pairs, hits in the top j,
        then the limbs of the sums A, B, C_1..C_k) and the 2 + k sums' values (dsgd_eval_topic_ranking)."""
        return self._topic_ranking("eval_topic_ranking", W, k, _range(row_begin, row_end))

    def eval_sampled_topic_ranking(self, row_begin: int, row_end: int, key: int, pos_begin: int, pos_end: int, W,
                                   k: int) -> Tuple[np.ndarray, np.ndarray]:
        """The same over positions [pos_begin, pos_end) of the device-drawn sample (dsgd_eval_sampled_topic_ranking)."""
        return self._topic_ranking("eval_sampled_topic_ranking", W, k, _drawn(row_begin, row_end, key, pos_begin, pos_end))

    def eval_samples_topic_ranking(self, samples, W, k: int) -> Tuple[np.ndarray, np.ndarray]:
        """The same over a list of row ids; repeats count every time (dsgd_eval_samples_topic_ranking)."""
        return self._topic_ranking("eval_samples_topic_ranking", W, k, _list(samples))

    def topics_topk(self, samples, W, k: int) -> Tuple[np.ndarray, np.ndarray]:
        """(ids int32[n, k], margins float64[n, k]): each listed row's first k topics by score -x . W_t (the margins
        ascending, ties to the lower t) among its non-NaN scores, and their margins; -1 and NaN past them.  Needs no loaded
        topics (dsgd_topics_topk)."""
        W = self._topic_W("topics_topk", W)
        rows = _list(samples)
        k = int(k)
        ids = np.zeros((rows.n, max(k, 0)), dtype=np.int32)
        m = np.zeros((rows.n, max(k, 0)), dtype=np.float64)
        self._ck(self._l.dsgd_topics_topk(self._h, _ptr(W), W.shape[0], k, *rows.args, _ptr(ids), _ptr(m)))
        return ids, m

    # -- sample weights (sync mode) and the weighted evaluations --
    def set_sample_weights(self, sw):
        """One weight per loaded row (finite, >= 0) for every following sync step, gradient request and weighted evaluation;
        None clears them (dsgd_set_sample_weights)."""
        if sw is None:
            self._ck(self._l.dsgd_set_sample_weights(self._h, None, 0))
            return
        sw = _arr(sw, np.float64)
        self._ck(self._l.dsgd_set_sample_weights(self._h, _ptr(sw), sw.size))

    def _weighted(self, fn: str, w, rows: _Rows) -> "WeightedEval":
        nrm = C.c_double()
        sums, counts = np.zeros(3, dtype=np.float64), np.zeros(2, dtype=np.int64)
        self._call(fn, w, rows, C.byref(nrm), _ptr(sums), _ptr(counts))
        return WeightedEval(nrm.value, float(sums[0]), float(sums[1]), float(sums[2]), int(counts[0]), int(counts[1]))

    def eval_weighted(self, row_begin: int, row_end: int, w=None) -> "WeightedEval":
        """Weighted loss, correct-weight and weight sums over rows [row_begin, row_end) (dsgd_eval_weighted)."""
        return self._weighted("eval_weighted", w, _range(row_begin, row_end))

    def eval_sampled_weighted(self, row_begin: int, row_end: int, key: int, pos_begin: int, pos_end: int,
                              w=None) -> "WeightedEval":
        """The same over positions [pos_begin, pos_end) of the device-drawn sample (dsgd_eval_sampled_weighted)."""
        return self._weighted("eval_sampled_weighted", w, _drawn(row_begin, row_end, key, pos_begin, pos_end))

    def eval_samples_weighted(self, samples, w=None) -> "WeightedEval":
        """The same over a list of row ids; repeats count every time (dsgd_eval_samples_weighted)."""
        return self._weighted("eval_samples_weighted", w, _list(samples))

    def _weighted_curve(self, fn: str, w, rows: _Rows, curve: bool) -> "WeightedCurve":
        words, wsums, m = np.zeros(METRICS_WORDS, dtype=np.int64), np.zeros(WCURVE_WORDS), C.c_int64()
        pts = [np.zeros(max(rows.n, 0)) if curve else None for _ in range(3)]
        self._call(fn, w, rows, _ptr(words), _ptr(wsums), C.byref(m), *[_ptr(a) for a in pts])
        k = m.value
        thr, tpw, fpw = [a[:k].copy() if curve else np.zeros(0) for a in pts]
        return WeightedCurve(words, wsums, k, thr, tpw, fpw, *weighted_auc_ap(words, wsums))

    def eval_weighted_curve(self, row_begin: int, row_end: int, w=None, curve: bool = True) -> "WeightedCurve":
        """ROC / precision-recall points, AUC and AP over rows [row_begin, row_end), every row counted by its weight
        c_i = class weight x sample weight (dsgd_eval_weighted_curve); curve=False: the words only."""
        return self._weighted_curve("eval_weighted_curve", w, _range(row_begin, row_end), curve)

    def eval_sampled_weighted_curve(self, row_begin: int, row_end: int, key: int, pos_begin: int, pos_end: int, w=None,
                                    curve: bool = True) -> "WeightedCurve":
        """The same over positions [pos_begin, pos_end) of the device-drawn sample (dsgd_eval_sampled_weighted_curve)."""
        return self._weighted_curve("eval_sampled_weighted_curve", w, _drawn(row_begin, row_end, key, pos_begin, pos_end),
                                    curve)

    def eval_samples_weighted_curve(self, samples, w=None, curve: bool = True) -> "WeightedCurve":
        """The same over a list of row ids; repeats count every time (dsgd_eval_samples_weighted_curve)."""
        return self._weighted_curve("eval_samples_weighted_curve", w, _list(samples), curve)

    # -- weighted bootstrap --
    def _weighted_bootstrap(self, fn: str, w, rows: _Rows, bkey: int, b_begin: int, b_end: int):
        """dsgd_<fn>: (words[b_end - b_begin, 2], wsums[..., WCURVE_WORDS], loss_sum[...]) of replicates [b_begin, b_end)."""
        k = max(int(b_end) - int(b_begin), 0)
        words = np.zeros((max(k, 1), 2), dtype=np.int64)
        wsums = np.zeros((max(k, 1), WCURVE_WORDS), dtype=np.float64)
        loss = np.zeros(max(k, 1), dtype=np.float64)
        self._call(fn, w, rows, int(bkey) & 0xFFFFFFFFFFFFFFFF, int(b_begin), int(b_end), _ptr(words), _ptr(wsums), _ptr(loss))
        return words[:k], wsums[:k], loss[:k]

    def eval_weighted_bootstrap(self, row_begin: int, row_end: int, bkey: int, b_begin: int, b_end: int, w=None):
        """Weighted Poisson-bootstrap replicates [b_begin, b_end) of rows [row_begin, row_end) with key bkey, every row
        counted by c_i = class weight x sample weight (dsgd_eval_weighted_bootstrap): (words, wsums, loss_sum), one row per
        replicate -- its size and NaN-score rows, the weighted curve words and the weighted loss sum of its expanded list."""
        return self._weighted_bootstrap("eval_weighted_bootstrap", w, _range(row_begin, row_end), bkey, b_begin, b_end)

    def eval_sampled_weighted_bootstrap(self, row_begin: int, row_end: int, key: int, pos_begin: int, pos_end: int,
                                        bkey: int, b_begin: int, b_end: int, w=None):
        """The same over positions [pos_begin, pos_end) of the device-drawn sample (dsgd_eval_sampled_weighted_bootstrap)."""
        return self._weighted_bootstrap("eval_sampled_weighted_bootstrap", w,
                                        _drawn(row_begin, row_end, key, pos_begin, pos_end), bkey, b_begin, b_end)

    def eval_samples_weighted_bootstrap(self, samples, bkey: int, b_begin: int, b_end: int, w=None):
        """The same over a list of row ids, position i being list index i (dsgd_eval_samples_weighted_bootstrap)."""
        return self._weighted_bootstrap("eval_samples_weighted_bootstrap", w, _list(samples), bkey, b_begin, b_end)

    # -- async --
    def async_host_master(self, w0):
        """Host the master's replica (GradState.grad + update counter) on this GPU."""
        w0 = _arr(w0, np.float64, self.dim, "weights")
        self._ck(self._l.dsgd_async_host_master(self._h, _ptr(w0)))

    def ipc_export(self, which: int = REPLICA_SELF) -> bytes:
        buf = (C.c_uint8 * IPC_HANDLE_BYTES)()
        self._ck(self._l.dsgd_ipc_export(self._h, which, C.cast(buf, C.c_void_p)))
        return bytes(buf)

    def peer_attach(self, peer_rank: int, peer: "NativeCtx", which: int = REPLICA_SELF):
        """Same-process peer (several ctxs driven by one host process)."""
        self._ck(self._l.dsgd_peer_attach(self._h, peer_rank, peer._h, which))

    def async_replay(self, w0, samples, batch: int, lr: float):
        """Replays recorded batches on one lane; w0 None starts from the replica as it is (peers' pushes included)."""
        w0 = None if w0 is None else _arr(w0, np.float64, self.dim, "weights")
        samples = _arr(samples, np.int32)
        if samples.size % batch:
            raise DsgdInvalid(ERR_INVALID, "async_replay: len(samples) is not a multiple of batch")
        self._ck(self._l.dsgd_async_replay(self._h, _ptr(w0), _ptr(samples), batch, samples.size // batch, lr))

    def async_running(self) -> bool:
        r = C.c_int()
        self._ck(self._l.dsgd_async_running(self._h, C.byref(r)))
        return bool(r.value)

    def async_elapsed_ms(self) -> float:
        ms = C.c_float()
        self._ck(self._l.dsgd_async_elapsed_ms(self._h, C.byref(ms)))
        return ms.value

    def async_master_weights(self) -> np.ndarray:
        out = np.zeros(self.dim, dtype=np.float64)
        self._ck(self._l.dsgd_async_master_weights(self._h, _ptr(out)))
        return out

    def async_outbox_enable(self):
        """One more target of every delta of this worker: the accumulator a host relay forwards to colleagues that are not GPU
        peers (core/Slave.scala:104-105).  Call before start_async."""
        self._ck(self._l.dsgd_async_outbox_enable(self._h))

    def async_outbox_read(self) -> np.ndarray:
        """Sum of -delta since async_outbox_enable (safe while the loop runs)."""
        out = np.zeros(self.dim, dtype=np.float64)
        self._ck(self._l.dsgd_async_outbox_read(self._h, _ptr(out)))
        return out

    def ipc_import(self, peer_rank: int, handle: bytes):
        buf = (C.c_uint8 * IPC_HANDLE_BYTES).from_buffer_copy(handle)
        self._ck(self._l.dsgd_ipc_import(self._h, peer_rank, C.cast(buf, C.c_void_p)))

    def start_async(self, w0, assigned, batch: int, lr: float, concurrency: int = 1, max_updates: int = 0, seed: int = 0):
        w0 = None if w0 is None else _arr(w0, np.float64, self.dim, "weights")
        assigned = _arr(assigned, np.int32)
        self._ck(self._l.dsgd_start_async(self._h, _ptr(w0), _ptr(assigned), assigned.size, batch, lr, concurrency,
                                          max_updates, seed))

    def stop_async(self):
        self._ck(self._l.dsgd_stop_async(self._h))

    def update_grad(self, idx, val):
        idx, val = _arr(idx, np.int32), _arr(val, np.float64)
        if idx.size != val.size:
            raise DsgdInvalid(ERR_INVALID, "update_grad: idx and val differ in length")
        self._ck(self._l.dsgd_update_grad(self._h, _ptr(idx), _ptr(val), idx.size))

    def async_updates(self) -> int:
        n = C.c_int64()
        self._ck(self._l.dsgd_async_updates(self._h, C.byref(n)))
        return n.value
