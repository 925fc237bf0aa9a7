"""Every public evaluation method of Master against a recording device context, on CPU.  For the whole split, a
device-drawn sample and a jvm_exact id list; at world 1, at rank 1 of world 2 and at rank 0 of world 2 with a one-row
sample (an empty share); for the SVM, the logistic model and an L1 penalty; without weights, with class weights and with
sample weights; over the train and the test rows: the exact context calls (names, positional arguments and keywords, in
order), the collectives with their payloads, the sample draws and the returned value."""
import math
from types import SimpleNamespace

import numpy as np
import pytest

from distributed_sgd_b200.core.master import (BOOTSTRAP_METRICS, MasterSync, bootstrap_key, bootstrap_pack,
                                               bootstrap_summary, bootstrap_unpack, bootstrap_values, calibration_dict,
                                               curve_dict, isotonic_calibration_dict, metrics_dict, sampled_key,
                                               weighted_bootstrap_values, weighted_calibration_dict, weighted_curve_dict)
from distributed_sgd_b200.ml import Calibration, IsotonicCalibration, SparseLogistic, SparseSVM
from distributed_sgd_b200.ml import split_strategy
from distributed_sgd_b200.ml.one_vs_rest import topic_ranking_report, topic_report
from distributed_sgd_b200.native import ClassEval, DsgdEmpty, WeightedCurve, WeightedEval, topic_rank_words, topic_words
from distributed_sgd_b200.utils.dataset import Data
from distributed_sgd_b200.utils.jvm_random import JvmRandom

N_TRAIN, N_TEST, DIM, SEED, LAM, L1, COUNT = 13, 7, 3, 5, 0.25, 0.5, 4
CLASS_WEIGHT = (2.0, 0.5)
WTS = "w"                                    # the weights: passed through to the context untouched
TOPIC_W = np.arange(2.0 * DIM).reshape(2, DIM)
TOPICS = SimpleNamespace(names=("a", "b"), n_topics=2)
RANK_K, N_BOOT, LEVEL, N_BINS = 2, 3, 0.9, 4

# ---- canned device results, one per family --------------------------------------------------------------------------
METRICS = np.array([3, 1, 0, 1, 2, 0, 10, 0], dtype=np.int64)
WSUMS = np.arange(1.0, 14.0)
ISO = (np.array([-1.0, 2.0]), np.array([0.25, 0.75]), np.array([4, 4]), np.array([1, 3]), np.array([2, 2, 8, 0, 5]))
CAL = (0.5, -0.25, 1.0, np.array([3, 0, 8, 0]))
L1_NORM = (3.0, 4)


def canned(family, args, kw):
    if family == "eval_counts":
        return 7, 3, 2.0
    if family == "eval_sums":
        return 1.5, 3, 2.0
    if family == "eval_class":
        return ClassEval(2.0, 1.5, 2.5, 2, 1, 3, 2)
    if family == "eval_weighted":
        return WeightedEval(2.0, 4.5, 1.25, 3.5, 5, 3)
    if family == "eval_metrics":
        return METRICS
    if family == "eval_curve":
        if kw["curve"]:
            return METRICS, 0.75, np.array([0.5, -0.5]), np.array([2, 3]), np.array([0, 1])
        return METRICS, 0.75, 2
    if family == "eval_weighted_curve":
        pts = [np.array([0.5, -0.5]), np.array([1.5, 2.0]), np.array([0.0, 1.0])] if kw["curve"] else [np.zeros(0)] * 3
        return WeightedCurve(METRICS, WSUMS, 2, *pts, 0.25, 0.5)
    if family in ("eval_bootstrap", "eval_weighted_bootstrap"):
        k = args[-2] - args[-3]
        loss = np.arange(k) + 1.5
        if family == "eval_bootstrap":
            return np.tile(np.arange(9), (k, 1)) + np.arange(k)[:, None], np.full(k, 0.5), loss
        return np.tile([6, 0], (k, 1)), np.tile(WSUMS, (k, 1)) + np.arange(k)[:, None], loss
    if family == "calibrate":
        return CAL
    if family == "calibrate_weighted":
        return (*CAL, np.array([1.0, 2.0, 3.0]))
    if family == "calibrate_isotonic":
        return ISO
    if family == "calibrate_isotonic_weighted":
        return (*ISO[:2], np.array([4.0, 4.5]), np.array([1.0, 3.5]), ISO[4], np.array([1.5, 2.5]))
    if family.endswith("calibration"):
        n_bins, weighted = args[-2], "weighted" in family
        sums = np.array([2.0, 4.0, 8.0, 0.0]) if weighted else np.array([2.0, 4.0])
        rows = np.eye(n_bins)[0] * 8.0 if weighted else np.eye(n_bins, dtype=np.int64)[0] * 8
        words = np.array([8, 1, 2]) if "isotonic" in family else np.array([8, 1])
        return sums, rows, rows * 0, np.eye(n_bins)[0] * 2.0, words
    if family == "eval_topics":
        return np.arange(topic_words(len(args[-1])), dtype=np.int64)
    if family == "eval_topic_ranking":
        return np.arange(topic_rank_words(args[-1]), dtype=np.int64) % 5, np.zeros(2 + args[-1])
    if family == "weights_l1":
        return L1_NORM
    raise AssertionError(f"unexpected call {family}")


def family_of(name):
    """The family of a NativeCtx method: eval_sampled_X and eval_samples_X are eval_X, calibrate*_sampled and
    calibrate*_samples are calibrate*."""
    for form in ("sampled_", "samples_"):
        if name.startswith("eval_" + form):
            return "eval_" + name[len("eval_" + form):]
    for form in ("_sampled", "_samples"):
        if name.startswith("calibrate") and name.endswith(form):
            return name[:-len(form)]
    return name


def plain(v):
    """A value with its arrays as lists, so that call logs compare with ==."""
    if isinstance(v, np.ndarray):
        return ("array", v.tolist())
    if isinstance(v, (tuple, list)):
        return tuple(plain(x) for x in v)
    return v


class RecordingCtx:
    def __init__(self):
        self.calls = []

    def __getattr__(self, name):
        if name.startswith("__"):
            raise AttributeError(name)

        def call(*args, **kw):
            self.calls.append((name, plain(args), kw))
            return canned(family_of(name), args, kw)
        return call


class RecordingGroup:
    """A Group stand-in for rank `rank` of `world`: every other rank is taken to contribute 1 to each summed value and to
    hold the same bytes as this one."""

    def __init__(self, world, rank):
        self.world, self.rank, self.log = world, rank, []

    def all_reduce_sum(self, values):
        self.log.append(("sum", [float(v) for v in values]))
        return [float(v) + 1.0 for v in values]

    def all_reduce_max(self, value):
        self.log.append(("max", float(value)))
        return float(value) + 1.0

    def all_gather_bytes(self, payload):
        self.log.append(("gather", np.frombuffer(payload, dtype=np.float64).tolist()))
        return [payload] * self.world


def stub(n):
    return Data(np.arange(n + 1, dtype=np.int64), np.zeros(n, np.int32), np.ones(n, np.float32), np.ones(n, np.int8), DIM)


def make_master(c):
    cw = (1.0, 1.0) if c.weighting == "none" else CLASS_WEIGHT
    slave = SimpleNamespace(ctx=RecordingCtx(), world=c.world, is_async=False, n_train=N_TRAIN, n_test=N_TEST,
                            class_weight=cw, sample_weighted=c.weighting == "sample", topics=TOPICS, intercept=False)
    model = {"svm": SparseSVM(LAM), "logistic": SparseLogistic(LAM), "l1": SparseSVM(LAM, l1=L1)}[c.model]
    return MasterSync(0, stub(N_TRAIN), stub(N_TEST), model, c.world, slave=slave, group=RecordingGroup(c.world, c.rank),
                      seed=SEED, jvm_exact=c.form == "list", attach=False)


# ---- what each method must ask for ------------------------------------------------------------------------------------
class Case:
    def __init__(self, form, world, rank, count, model, weighting, test):
        self.form, self.world, self.rank, self.model, self.weighting, self.test = form, world, rank, model, weighting, test
        self.b, self.e = (N_TRAIN, N_TRAIN + N_TEST) if test else (0, N_TRAIN)
        self.count = count
        self.n = self.e - self.b if form == "whole" else min(count, self.e - self.b)
        self.ids = JvmRandom(SEED).shuffle(np.arange(self.e - self.b, dtype=np.int32))[:self.n] + np.int32(self.b)
        self.cw = (1.0, 1.0) if weighting == "none" else CLASS_WEIGHT

    def rows(self, lo=None, hi=None):
        """The row arguments of positions [lo, hi) of this case's rows (default: all of them)."""
        lo, hi = (0, self.n) if lo is None else (lo, hi)
        if self.form == "whole":
            return self.b + lo, self.b + hi
        if self.form == "drawn":
            return self.b, self.e, sampled_key(SEED, 0), lo, hi
        return (plain(self.ids[lo:hi]),)

    def share(self):
        lo, hi = (self.n * self.rank) // self.world, (self.n * (self.rank + 1)) // self.world
        return (lo, hi) if hi > lo else None

    def method(self, family):
        """The NativeCtx method of `family` for this case's form."""
        if self.form == "whole":
            return family
        if family.startswith("calibrate"):
            return family + ("_sampled" if self.form == "drawn" else "_samples")
        rest = family[len("eval_"):]
        return ("eval_sampled_" if self.form == "drawn" else "eval_samples_") + rest

    def call(self, family, *args, **kw):
        return self.method(family), self.rows() + plain(args), kw

    def penalty(self, n2, want_loss=True):
        """(lambda ||w||^2 [+ l1 ||w||_1], the calls it makes)."""
        if self.model != "l1":
            return LAM * n2, []
        if not want_loss:
            return float("nan"), []
        return LAM * n2 + L1 * L1_NORM[0], [("weights_l1", (WTS,), {})]


def loss_accuracy(c, want_loss, share, extra_count=None):
    """(calls, collectives, (loss, accuracy)) of a row-sharded loss/accuracy pass over `share` (positions, None: empty)."""
    sample, weighted = c.weighting == "sample", c.weighting == "class"
    exact = not (c.model == "logistic" or sample)
    family = ("eval_weighted" if sample else "eval_class" if weighted else
              "eval_counts" if c.model != "logistic" else "eval_sums")
    calls = []
    if share is None:
        h, cc, n2, *h_neg = (0, 0, 0.0, 0) if weighted else (0, 0, 0.0)
    else:
        rows = c.rows(*share) if extra_count is None else share
        calls.append((c.method(family) if extra_count is None else family, rows + (WTS,), {}))
        r = canned(family, (), {})
        if sample:
            h, cc, n2, h_neg = r.loss_sum, r.correct, r.norm_squared, []
        elif weighted:
            as_sum = int if exact else float
            h, cc, n2, h_neg = as_sum(r.loss_pos), r.correct_pos + r.correct_neg, r.norm_squared, [as_sum(r.loss_neg)]
        else:
            h, cc, n2, h_neg = *r, []
    counted = [] if extra_count is None else [extra_count]
    if exact:
        coll = [("sum", [float(v) for v in (h, cc, *counted, *h_neg)]), ("max", float(n2))]
        hs, cs, *rest = [float(v) + 1.0 for v in (h, cc, *counted, *h_neg)]
        n2 = float(n2) + 1.0
    else:
        mine = [float(v) for v in (h, cc, *counted, *h_neg, n2)]
        coll = [("gather", mine)]
        hs, cs, *rest = [c.world * v for v in mine[:-1]]
        n2 = mine[-1]
    n = c.n
    if extra_count is not None:
        n, *rest = rest
    pen, pen_calls = c.penalty(n2, want_loss)
    loss = pen + ((c.cw[0] * hs + c.cw[1] * rest[0]) if rest else hs) / n
    return calls + pen_calls, coll, (loss, cs / n)


def topic_words_of(c, family, *args):
    share = c.share()
    if share is None:
        words = np.zeros(topic_words(2) if family == "eval_topics" else topic_rank_words(RANK_K), dtype=np.int64)
        calls = []
    else:
        words = canned(family, (TOPIC_W, *args), {})
        words = words[0] if isinstance(words, tuple) else words
        calls = [(c.method(family), c.rows(*share) + plain((TOPIC_W, *args)), {})]
    coll = [("sum", [float(x) for x in words])]
    return calls, coll, (np.asarray(words, np.float64) + 1.0).astype(np.int64)


def class_report(c):
    pen, pen_calls = c.penalty(2.0)
    ce = canned("eval_class", (), {})
    rec_pos, rec_neg = 2 / 3, 1 / 2
    out = {"n_pos": 3, "n_neg": 2, "correct_pos": 2, "correct_neg": 1, "recall_pos": rec_pos, "recall_neg": rec_neg,
           "balanced_accuracy": (rec_pos + rec_neg) / 2.0, "accuracy": 3 / 5, "class_weight": c.cw,
           "loss": pen + (1.5 + 2.5) / 5, "weighted_loss": pen + ce.weighted_loss_sum(*c.cw) / 5}
    return [c.call("eval_class", WTS)] + pen_calls, [], out


def weighted_report_value(c, pen):
    return {"n": 5, "weight_sum": 3.5, "weighted_loss": pen + 4.5 / 5, "weighted_accuracy": 1.25 / 3.5}


def weighted_report(c):
    pen, pen_calls = c.penalty(2.0)
    return [c.call("eval_weighted", WTS)] + pen_calls, [], weighted_report_value(c, pen)


def bootstrap_side(c, weights, weighted):
    """(calls, collectives, estimates, replicate values) of one bootstrap over this case's rows."""
    bkey = bootstrap_key(SEED)
    if weighted:
        calls = [c.call("eval_weighted_curve", weights, curve=False), c.call("eval_weighted", weights)]
        pen, pen_calls = c.penalty(2.0)
        calls += [(n, (weights,), kw) for n, _, kw in pen_calls] * 2   # the report's penalty, then the bootstrap's
        curve = weighted_curve_dict(canned("eval_weighted_curve", (), {"curve": False}), curve=False)
        report = weighted_report_value(c, pen)
        est = {"accuracy": curve["accuracy"], "loss": report["weighted_loss"], "auc": curve["auc"],
               "ap": curve["average_precision"], "precision": curve["precision"], "recall": curve["recall"],
               "f1": curve["f1"]}
        family, values = "eval_weighted_bootstrap", weighted_bootstrap_values
    else:
        calls = [c.call("eval_curve", weights, curve=False), c.call("eval_sums", weights)]
        pen, pen_calls = c.penalty(2.0)
        calls += [(n, (weights,), kw) for n, _, kw in pen_calls]
        n = int(METRICS[:6].sum())
        est = {k: float(v[0]) for k, v in bootstrap_values(np.concatenate([METRICS, [n]]), [0.75], [1.5], pen).items()}
        family, values = "eval_bootstrap", bootstrap_values
    lo, hi = (N_BOOT * c.rank) // c.world, (N_BOOT * (c.rank + 1)) // c.world
    if hi > lo:
        calls.append(c.call(family, bkey, lo, hi, weights))
        mine = bootstrap_pack(*canned(family, (bkey, lo, hi, weights), {}))
    else:
        mine = np.zeros(0)
    coll = [("gather", mine.tolist())]
    reps = values(*bootstrap_unpack([mine] * c.world, weighted), pen)
    return calls, coll, est, reps


def bootstrap(c, weighted):
    calls, coll, est, reps = bootstrap_side(c, WTS, weighted)
    return calls, coll, {m: bootstrap_summary(est[m], reps[m], LEVEL) for m in BOOTSTRAP_METRICS}


def compare_bootstrap(c, weighted):
    calls, coll, sides = [], [], []
    for w in ("wa", "wb"):
        ca, co, est, reps = bootstrap_side(c, w, weighted)
        calls += ca
        coll += co
        sides.append((est, reps))
    (ea, ra), (eb, rb) = sides
    out = {}
    for m, higher in BOOTSTRAP_METRICS.items():
        d = rb[m] - ra[m]
        s = bootstrap_summary(eb[m] - ea[m], d, LEVEL)
        ok = d[~np.isnan(d)]
        s["p_better"] = float(np.mean(ok > 0 if higher else ok < 0)) if ok.size else float("nan")
        out[m] = s
    return calls, coll, out


def calibrate(c, isotonic, weighted):
    family = "calibrate" + ("_isotonic" if isotonic else "") + ("_weighted" if weighted else "")
    r = canned(family, (), {})
    if isotonic:
        info = r[4]
        extra = (True, float(r[5][0]), float(r[5][1])) if weighted else ()
        out = IsotonicCalibration(r[0], r[1], r[2], r[3], int(info[0]), int(info[2]), int(info[3]), int(info[4]), *extra)
    else:
        info = r[3]
        extra = (True, float(r[4][0]), float(r[4][1]), float(r[4][2])) if weighted else ()
        out = Calibration(r[0], r[1], r[2], int(info[0]), int(info[1]), int(info[2]), int(info[3]), *extra)
    return [c.call(family, WTS)], [], out


ISO_MAP = IsotonicCalibration(ISO[0], ISO[1], ISO[2], ISO[3], 2, 8, 0, 5)
SIGMOID = Calibration(0.5, -0.25)


def calibration_quality(c, isotonic, weighted):
    family = "eval_" + ("weighted_" if weighted else "") + ("isotonic_" if isotonic else "") + "calibration"
    params = (ISO_MAP.x, ISO_MAP.y) if isotonic else (SIGMOID.a, SIGMOID.b)
    r = canned(family, (N_BINS, WTS), {})
    convert = weighted_calibration_dict if weighted else isotonic_calibration_dict if isotonic else calibration_dict
    return [c.call(family, *params, N_BINS, WTS)], [], convert(r)


# name -> (run(master, case): the method of the whole split or its sampled form, as the case's form asks, and
# expect(case): (context calls, collectives, returned value))
METHODS = {
    "loss": (lambda m, c: m.local_loss(WTS, test_data=c.test) if c.form == "whole"
             else m.local_sampled_loss(WTS, c.count, test_data=c.test),
             lambda c: (lambda r: (r[0], r[1], r[2][0]))(loss_accuracy(c, True, c.share()))),
    "accuracy": (lambda m, c: m.local_accuracy(WTS, test_data=c.test) if c.form == "whole"
                 else m.local_sampled_accuracy(WTS, c.count, test_data=c.test),
                 lambda c: (lambda r: (r[0], r[1], r[2][1]))(loss_accuracy(c, False, c.share()))),
    "loss_accuracy": (lambda m, c: m.local_loss_accuracy(WTS, test_data=c.test) if c.form == "whole"
                      else m.local_sampled_loss_accuracy(WTS, c.count, test_data=c.test),
                      lambda c: loss_accuracy(c, True, c.share())),
    "class_report": (lambda m, c: m.local_class_report(WTS, test_data=c.test) if c.form == "whole"
                     else m.local_sampled_class_report(WTS, c.count, test_data=c.test), class_report),
    "weighted_report": (lambda m, c: m.local_weighted_report(WTS, test_data=c.test) if c.form == "whole"
                        else m.local_sampled_weighted_report(WTS, c.count, test_data=c.test), weighted_report),
    "topic_report": (lambda m, c: m.local_topic_report(TOPIC_W, test_data=c.test) if c.form == "whole"
                     else m.local_sampled_topic_report(TOPIC_W, c.count, test_data=c.test),
                     lambda c: (lambda r: (r[0], r[1], topic_report(r[2], TOPICS.names)))(
                         topic_words_of(c, "eval_topics"))),
    "topic_ranking_report": (lambda m, c: m.local_topic_ranking_report(TOPIC_W, RANK_K, test_data=c.test)
                             if c.form == "whole"
                             else m.local_sampled_topic_ranking_report(TOPIC_W, RANK_K, c.count, test_data=c.test),
                             lambda c: (lambda r: (r[0], r[1], topic_ranking_report(r[2], RANK_K)))(
                                 topic_words_of(c, "eval_topic_ranking", RANK_K))),
    "metrics": (lambda m, c: m.local_metrics(WTS, test_data=c.test) if c.form == "whole"
                else m.local_sampled_metrics(WTS, c.count, test_data=c.test),
                lambda c: ([c.call("eval_metrics", WTS)], [], metrics_dict(METRICS))),
}
for curve in (True, False):
    METHODS[f"curve[{curve}]"] = (
        lambda m, c, curve=curve: m.local_curve(WTS, test_data=c.test, curve=curve) if c.form == "whole"
        else m.local_sampled_curve(WTS, c.count, test_data=c.test, curve=curve),
        lambda c, curve=curve: ([c.call("eval_curve", WTS, curve=curve)], [],
                                curve_dict(canned("eval_curve", (), {"curve": curve}))))
    METHODS[f"weighted_curve[{curve}]"] = (
        lambda m, c, curve=curve: m.local_weighted_curve(WTS, test_data=c.test, curve=curve) if c.form == "whole"
        else m.local_sampled_weighted_curve(WTS, c.count, test_data=c.test, curve=curve),
        lambda c, curve=curve: ([c.call("eval_weighted_curve", WTS, curve=curve)], [],
                                weighted_curve_dict(canned("eval_weighted_curve", (), {"curve": curve}), curve)))
for weighted in (False, True):
    METHODS[f"bootstrap[{weighted}]"] = (
        lambda m, c, weighted=weighted: m.local_bootstrap(WTS, test_data=c.test, n_boot=N_BOOT, level=LEVEL,
                                                          weighted=weighted) if c.form == "whole"
        else m.local_sampled_bootstrap(WTS, c.count, test_data=c.test, n_boot=N_BOOT, level=LEVEL, weighted=weighted),
        lambda c, weighted=weighted: bootstrap(c, weighted))
    METHODS[f"compare_bootstrap[{weighted}]"] = (
        lambda m, c, weighted=weighted: m.compare_bootstrap("wa", "wb", test_data=c.test, n_boot=N_BOOT, level=LEVEL,
                                                            weighted=weighted),
        lambda c, weighted=weighted: compare_bootstrap(c, weighted))
    for iso in (False, True):
        method = "isotonic" if iso else "sigmoid"
        METHODS[f"calibrate[{method},{weighted}]"] = (
            lambda m, c, method=method, weighted=weighted: m.calibrate(WTS, test_data=c.test, method=method,
                                                                       weighted=weighted) if c.form == "whole"
            else m.sampled_calibrate(WTS, c.count, test_data=c.test, method=method, weighted=weighted),
            lambda c, iso=iso, weighted=weighted: calibrate(c, iso, weighted))
        METHODS[f"calibration[{method},{weighted}]"] = (
            lambda m, c, iso=iso, weighted=weighted: m.local_calibration(
                ISO_MAP if iso else SIGMOID, WTS, test_data=c.test, n_bins=N_BINS, weighted=weighted)
            if c.form == "whole" else m.local_sampled_calibration(ISO_MAP if iso else SIGMOID, WTS, c.count,
                                                                  test_data=c.test, n_bins=N_BINS, weighted=weighted),
            lambda c, iso=iso, weighted=weighted: calibration_quality(c, iso, weighted))
for name in ("distributed_loss", "distributed_accuracy"):
    METHODS[name] = (lambda m, c, name=name: getattr(m, name)(WTS), None)

WHOLE_ONLY = {"compare_bootstrap[False]", "compare_bootstrap[True]", "distributed_loss", "distributed_accuracy"}
# (world, rank, samples_count): rank 0 of 2 with a one-row sample has an empty share
PLACES = [(1, 0, COUNT), (2, 1, COUNT), (2, 0, 1)]


def same(a, b):
    """Equal values, nan equal to nan, arrays by value, dataclasses by their fields."""
    if hasattr(a, "__dataclass_fields__"):
        return type(a) is type(b) and same(vars(a), vars(b))
    if isinstance(a, dict):
        return isinstance(b, dict) and a.keys() == b.keys() and all(same(a[k], b[k]) for k in a)
    if isinstance(a, (tuple, list)):
        return isinstance(b, (tuple, list)) and len(a) == len(b) and all(same(x, y) for x, y in zip(a, b))
    if isinstance(a, np.ndarray) or isinstance(b, np.ndarray):
        a, b = np.asarray(a), np.asarray(b)
        return a.shape == b.shape and np.array_equal(a, b, equal_nan=a.dtype.kind == "f")
    if isinstance(a, float) and isinstance(b, float) and math.isnan(a) and math.isnan(b):
        return True
    return type(a) is type(b) and a == b


def expect_distributed(c, want_loss):
    groups = split_strategy.vanilla(N_TRAIN, c.world)
    mine = groups[c.rank] if c.rank < len(groups) else range(0)
    calls, coll, (loss, acc) = loss_accuracy(c, want_loss, (mine.start, mine.stop) if len(mine) else None, len(mine))
    return calls, coll, loss if want_loss else acc


@pytest.mark.parametrize("place", PLACES, ids=lambda p: f"world{p[0]}-rank{p[1]}-count{p[2]}")
@pytest.mark.parametrize("name,form", [(name, form) for name in sorted(METHODS) for form in ("whole", "drawn", "list")
                                       if form == "whole" or name not in WHOLE_ONLY])
def test_each_method_asks_for_its_rows(name, form, place):
    run, expect = METHODS[name]
    world, rank, count = place
    for model in ("svm", "logistic", "l1"):
        for weighting in ("none", "class", "sample"):
            for test in (False, True):
                c = Case(form, world, rank, count, model, weighting, test)
                if name.startswith("distributed_"):
                    c = Case("whole", world, rank, count, model, weighting, False)
                    want = expect_distributed(c, name == "distributed_loss")
                else:
                    want = expect(c)
                m = make_master(c)
                jvm_ref = JvmRandom(SEED)
                got = run(m, c)
                what = f"{name} {form} world {world} rank {rank} {model} {weighting} test={test}"
                assert m.ctx.calls == want[0], what
                assert m.group.log == want[1], what
                assert m._sampled_draws == (1 if form == "drawn" else 0), what
                if form == "list":                           # one shuffle of the split, whatever the sample size
                    jvm_ref.shuffle(np.arange(c.e - c.b, dtype=np.int32))
                    assert m.jvm.next_int() == jvm_ref.next_int(), what
                assert same(got, want[2]), what


# the message of an empty sample, per sampled method (None: the method returns nan instead)
EMPTY = {
    "local_sampled_loss": "sampled evaluation of {} rows: reduce on an empty collection",
    "local_sampled_loss_accuracy": "sampled evaluation of {} rows: reduce on an empty collection",
    "local_sampled_accuracy": None,
    "local_sampled_class_report": "sampled evaluation of {} rows: reduce on an empty collection",
    "local_sampled_weighted_report": "sampled evaluation of {} rows: reduce on an empty collection",
    "local_sampled_topic_report": "sampled topic report of {} rows: the sample is empty",
    "local_sampled_topic_ranking_report": "sampled topic ranking report of {} rows: the sample is empty",
    "local_sampled_metrics": "sampled metrics of {} rows: the sample is empty",
    "local_sampled_curve": "sampled curve of {} rows: the sample is empty",
    "local_sampled_weighted_curve": "sampled weighted curve of {} rows: the sample is empty",
    "local_sampled_bootstrap": "sampled bootstrap of {} rows: the sample is empty",
    "sampled_calibrate": "sampled calibration of {} rows: the sample is empty",
    "local_sampled_calibration": "sampled calibration quality of {} rows: the sample is empty",
}


def _call_sampled(m, name, count, test, weighted=False):
    if name == "local_sampled_topic_report":
        return m.local_sampled_topic_report(TOPIC_W, count, test_data=test)
    if name == "local_sampled_topic_ranking_report":
        return m.local_sampled_topic_ranking_report(TOPIC_W, RANK_K, count, test_data=test)
    if name == "local_sampled_calibration":
        return m.local_sampled_calibration(SIGMOID, WTS, count, test_data=test, weighted=weighted)
    if name in ("local_sampled_bootstrap", "sampled_calibrate"):
        return getattr(m, name)(WTS, count, test_data=test, weighted=weighted)
    return getattr(m, name)(WTS, count, test_data=test)


@pytest.mark.parametrize("form", ["drawn", "list"])
@pytest.mark.parametrize("name", sorted(EMPTY))
def test_an_empty_sample_asks_the_device_nothing(name, form):
    for count in (0, -2):
        for weighted in (False, True):
            c = Case(form, 2, 1, count, "l1", "class", False)
            m = make_master(c)
            jvm_ref = JvmRandom(SEED)
            if EMPTY[name] is None:
                assert math.isnan(_call_sampled(m, name, count, False, weighted))
            else:
                with pytest.raises(DsgdEmpty) as err:
                    _call_sampled(m, name, count, False, weighted)
                assert EMPTY[name].format(count) in str(err.value)
            assert m.ctx.calls == [] and m.group.log == [] and m._sampled_draws == 0
            if form == "list":                               # the reference shuffles before `take`
                jvm_ref.shuffle(np.arange(N_TRAIN, dtype=np.int32))
                assert m.jvm.next_int() == jvm_ref.next_int()


@pytest.mark.parametrize("form", ["drawn", "list"])
def test_arguments_are_checked_before_the_draw(form):
    c = Case(form, 1, 0, COUNT, "svm", "none", False)
    m = make_master(c)
    with pytest.raises(ValueError):
        m.sampled_calibrate(WTS, COUNT, method="beta")
    with pytest.raises(ValueError):
        m.local_sampled_topic_report(TOPIC_W[:1], COUNT)
    with pytest.raises(ValueError):
        m.local_sampled_topic_ranking_report(TOPIC_W[:, :1], RANK_K, COUNT)
    assert m.ctx.calls == [] and m._sampled_draws == 0
    if form == "list":                                       # no shuffle either
        assert m.jvm.next_int() == JvmRandom(SEED).next_int()
