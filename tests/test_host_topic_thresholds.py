"""Per-topic thresholds on the host, without a GPU: threshold_report's formulas, OneVsRest.predict at thresholds, the
`topic-thresholds` and `topic-threshold-fbr` keys and their refusals, row_methods for the two new families, Master's tuning
and thresholded reports against a stand-in context (not sharded, and the calls of today without thresholds), and a
two-process all-reduce of the thresholded report."""
import os
import socket
import sys
from types import SimpleNamespace

import numpy as np
import pytest

from distributed_sgd_b200.utils.dataset import Data, Topics
from topic_thresholds_model import thresholded_words, tune
from topics_model import topic_words

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DIM, T = 8, 5
NAMES = tuple(f"t{i}" for i in range(T))


def _planted(n, seed=0):
    """[T, n] tie-heavy margins with NaN and +-inf, and a [n, T] indicator with a topic no row has"""
    rng = np.random.default_rng(seed)
    m = rng.integers(-3, 4, size=(T, n)).astype(np.float64) / 2.0
    m[rng.random((T, n)) < 0.05] = np.nan
    m[rng.random((T, n)) < 0.05] = np.inf
    has = rng.random((n, T)) < 0.4
    has[:, 2] = False
    return m, has


def test_row_methods_of_the_new_families():
    from distributed_sgd_b200.native import ABI, NativeCtx, row_methods
    assert row_methods("tune_topic_thresholds") == {"range": "tune_topic_thresholds",
                                                    "drawn": "tune_topic_thresholds_sampled",
                                                    "list": "tune_topic_thresholds_samples"}
    assert row_methods("eval_thresholded_topics") == {"range": "eval_thresholded_topics",
                                                      "drawn": "eval_sampled_thresholded_topics",
                                                      "list": "eval_samples_thresholded_topics"}
    assert row_methods("calibrate_isotonic")["drawn"] == "calibrate_isotonic_sampled"
    for fam in ("tune_topic_thresholds", "eval_thresholded_topics"):
        for name in row_methods(fam).values():
            assert "dsgd_" + name in ABI and callable(getattr(NativeCtx, name))


def test_threshold_report_formulas():
    from distributed_sgd_b200.ml.one_vs_rest import threshold_report
    m, has = _planted(60)
    thr, words = tune(m, has, 0.0)
    rep = threshold_report(words, thr, NAMES)
    assert rep["rows"] == 60 and sum(rep["status_counts"].values()) == T
    assert rep["topics"]["t2"]["status"] == "no positive row" and rep["topics"]["t2"]["threshold"] == 0.0
    for t, name in enumerate(NAMES):
        r, w = rep["topics"][name], words[8 * t:8 * t + 8]
        assert r["threshold"] == thr[t] and r["positives"] == w[1] and r["tp"] == w[4] and r["predicted"] == w[5]
        assert r["distinct_margins"] == w[3] and r["candidate"] == w[7] and r["nan_margins"] == w[2]
        if r["positives"] + r["predicted"]:
            assert r["f1"] == 2 * w[4] / (w[1] + w[5])
    z = np.zeros(8 * T, dtype=np.int64)
    z[6::8] = 3
    assert all(v["f1"] != v["f1"] for v in threshold_report(z, np.zeros(T), NAMES)["topics"].values())
    with pytest.raises(ValueError, match="threshold_report"):
        threshold_report(words[:-1], thr, NAMES)


class _MarginSlave:
    def __init__(self, margins):
        self.m = margins

    def margins(self, idx, w):
        return self.m[int(w[0])][np.asarray(idx)]


def test_predict_applies_the_thresholds():
    from distributed_sgd_b200.ml.one_vs_rest import OneVsRest
    m, has = _planted(40, seed=3)
    W = np.zeros((T, DIM))
    W[:, 0] = np.arange(T)                                          # the stand-in slave reads topic t's margins
    idx = np.array([0, 5, 5, 39, 17], dtype=np.int32)
    plain = OneVsRest(W, NAMES, [{}] * T)
    assert np.array_equal(plain.predict(_MarginSlave(m), idx), (m[:, idx] < 0.0).T)
    thr = np.array([0.5, -1.0, 0.0, np.inf, -np.inf])
    tuned = OneVsRest(W, NAMES, [{}] * T, thr)
    assert np.array_equal(tuned.predict(_MarginSlave(m), idx), (m[:, idx] < thr[:, None]).T)
    assert not tuned.predict(_MarginSlave(m), idx)[:, 4].any()


def test_topic_threshold_keys_and_their_refusals():
    from distributed_sgd_b200.main import scenario
    from distributed_sgd_b200.utils.config import Config, load_config
    cfg = load_config(env={})
    assert cfg.topic_thresholds == "none" and cfg.topic_threshold_fbr == 0.0
    cfg = load_config(env={"DSGD_TOPICS": "all", "DSGD_TOPIC_THRESHOLDS": "scut", "DSGD_TOPIC_THRESHOLD_FBR": "0.1"})
    assert cfg.topic_thresholds == "scut" and cfg.topic_threshold_fbr == 0.1
    assert load_config(env={"DSGD_TOPICS": "all", "DSGD_TOPIC_THRESHOLDS": "none"}).topic_thresholds == "none"
    with pytest.raises(ValueError, match="topic-thresholds.*topics"):
        load_config(env={"DSGD_TOPIC_THRESHOLDS": "scut"})          # tuning without one-vs-rest topics
    with pytest.raises(ValueError, match="topic-thresholds: expected"):
        load_config(env={"DSGD_TOPICS": "all", "DSGD_TOPIC_THRESHOLDS": "rcut"})
    for bad in ("-0.1", "1.5", "nan"):
        with pytest.raises(ValueError, match="topic-threshold-fbr"):
            load_config(env={"DSGD_TOPICS": "all", "DSGD_TOPIC_THRESHOLDS": "scut", "DSGD_TOPIC_THRESHOLD_FBR": bad})
    with pytest.raises(ValueError, match="topic-threshold-fbr.*scut"):
        load_config(env={"DSGD_TOPICS": "all", "DSGD_TOPIC_THRESHOLD_FBR": "0.2"})
    with pytest.raises(ValueError, match="topic-thresholds"):
        scenario(Config(topic_thresholds="scut"), data=None)          # refused before any data or device is touched


# ---- Master against a stand-in context ------------------------------------------------------------------------------------

class _Ctx:
    """Stands in for NativeCtx: the models over planted margins, and a record of every call."""

    def __init__(self, m, has):
        self.m, self.has, self.calls = m, has, []

    def comm_init(self, uid):
        pass

    def eval_topics(self, lo, hi, W):
        self.calls.append(("eval_topics", lo, hi))
        return topic_words(self.m[:, lo:hi], self.has[lo:hi])

    def eval_thresholded_topics(self, lo, hi, W, thr):
        self.calls.append(("eval_thresholded_topics", lo, hi, tuple(thr)))
        return thresholded_words(self.m[:, lo:hi], self.has[lo:hi], thr)

    def tune_topic_thresholds(self, lo, hi, W, fbr):
        self.calls.append(("tune_topic_thresholds", lo, hi, fbr))
        return tune(self.m[:, lo:hi], self.has[lo:hi], fbr)

    def tune_topic_thresholds_samples(self, ids, W, fbr):
        self.calls.append(("tune_topic_thresholds_samples", tuple(ids), fbr))
        return tune(self.m[:, ids], self.has[ids], fbr)


def _master(rank, world, m, has, n_train, n_test):
    from distributed_sgd_b200.core import Group, master as master_mod
    from distributed_sgd_b200.ml import SparseSVM
    master_mod.NativeCtx.comm_unique_id = staticmethod(lambda: bytes(range(128)))
    stub = lambda n: Data(np.arange(n + 1, dtype=np.int64), np.zeros(n, np.int32), np.ones(n, np.float32),
                          np.ones(n, np.int8), DIM)
    slave = SimpleNamespace(ctx=_Ctx(m, has), world=world, is_async=False, n_train=n_train, n_test=n_test, dim=DIM,
                            topics=Topics.from_indicator(has, NAMES))
    return master_mod.MasterSync(rank, stub(n_train), stub(n_test), SparseSVM(0.5), world, slave=slave, group=Group(),
                                 seed=0), slave.ctx


def test_master_tunes_on_the_train_rows_and_reports_at_the_thresholds():
    from distributed_sgd_b200.ml.one_vs_rest import OneVsRest, threshold_report, topic_report
    m, has = _planted(70, seed=5)
    mm, ctx = _master(0, 1, m, has, 50, 20)
    ovr = OneVsRest(np.zeros((T, DIM)), NAMES, [{}] * T)
    tuned, rep = mm.tune_topic_thresholds(ovr, fbr=0.25)
    thr, words = tune(m[:, :50], has[:50], 0.25)
    assert ctx.calls == [("tune_topic_thresholds", 0, 50, 0.25)]
    assert np.array_equal(tuned.thresholds, thr) and tuned.topics == NAMES and ovr.thresholds is None
    assert rep == threshold_report(words, thr, NAMES)
    # an array model: an OneVsRest of the loaded topics comes back
    tuned_a, _ = mm.tune_topic_thresholds(np.zeros((T, DIM)), test_data=True)
    assert np.array_equal(tuned_a.thresholds, tune(m[:, 50:], has[50:])[0]) and tuned_a.topics == NAMES
    ctx.calls.clear()
    # without thresholds: exactly the calls of today
    mm.local_topic_report(ovr)
    assert ctx.calls == [("eval_topics", 50, 70)]
    ctx.calls.clear()
    r = mm.local_topic_report(tuned)
    assert ctx.calls == [("eval_thresholded_topics", 50, 70, tuple(thr))]
    assert _same(r, topic_report(thresholded_words(m[:, 50:], has[50:], thr), NAMES))
    ctx.calls.clear()
    other = np.full(T, -0.5)
    mm.local_topic_report(np.zeros((T, DIM)), thresholds=other)
    assert ctx.calls == [("eval_thresholded_topics", 50, 70, tuple(other))]
    with pytest.raises(ValueError, match="thresholds"):
        mm.local_topic_report(ovr, thresholds=[np.nan] * T)
    with pytest.raises(ValueError, match="thresholds"):
        mm.local_topic_report(ovr, thresholds=[0.0] * (T - 1))


def _free_port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def _worker(rank, world, port, q):
    sys.path.insert(0, ROOT)
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    import torch.distributed as dist
    from distributed_sgd_b200.ml.one_vs_rest import OneVsRest
    dist.init_process_group("gloo", init_method=f"tcp://127.0.0.1:{port}", rank=rank, world_size=world)
    m, has = _planted(71, seed=9)
    mm, ctx = _master(rank, world, m, has, 30, 41)
    tuned, rep = mm.tune_topic_thresholds(OneVsRest(np.zeros((T, DIM)), NAMES, [{}] * T))
    r = mm.local_topic_report(tuned, test_data=True)
    q.put({"rank": rank, "calls": ctx.calls, "report": r, "thr": tuned.thresholds, "tuning": rep})
    dist.destroy_process_group()


def test_thresholded_report_all_reduced_over_two_ranks():
    import torch.multiprocessing as mp
    from distributed_sgd_b200.ml.one_vs_rest import topic_report
    ctxmp = mp.get_context("spawn")
    q = ctxmp.Queue()
    port = _free_port()
    procs = [ctxmp.Process(target=_worker, args=(r, 2, port, q)) for r in range(2)]
    for p in procs:
        p.start()
    res = sorted([q.get(timeout=120) for _ in procs], key=lambda r: r["rank"])
    for p in procs:
        p.join(timeout=30)
    m, has = _planted(71, seed=9)
    thr = tune(m[:, :30], has[:30])[0]
    for r, share in zip(res, ((30, 50), (50, 71))):
        # every rank tunes over all the train rows, then evaluates its contiguous share of the test rows
        assert r["calls"] == [("tune_topic_thresholds", 0, 30, 0.0), ("eval_thresholded_topics", *share, tuple(thr))]
        assert np.array_equal(r["thr"], thr) and r["tuning"] == res[0]["tuning"]
    whole = topic_report(thresholded_words(m[:, 30:], has[30:], thr), NAMES)
    for r in res:
        assert _same(r["report"], whole)
    assert whole["rows"] == 41


def _same(a, b) -> bool:
    """dict equality with NaN equal to NaN"""
    if isinstance(a, dict):
        return a.keys() == b.keys() and all(_same(a[k], b[k]) for k in a)
    if isinstance(a, float) and isinstance(b, float):
        return a == b or (a != a and b != b)
    return a == b
