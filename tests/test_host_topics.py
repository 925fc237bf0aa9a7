"""One-vs-rest topics on the host, without a GPU: the qrels topic reader, Topics and their split, synthetic_topics, the
`topics` key, MasterSync.fit_one_vs_rest's call sequence against a stand-in context, the report's formulas and a
two-process all-reduce of the report's words."""
import os
import socket
import sys

import numpy as np
import pytest

from distributed_sgd_b200.utils.dataset import Data, Topics, rcv1, synthetic_rcv1, synthetic_topics, write_rcv1

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DIM = 8


# ---- the qrels topic reader ----------------------------------------------------------------------------------------------

def _rcv1_folder(tmp_path, qrels_lines, n=4):
    rp = np.arange(n + 1, dtype=np.int64)
    data = Data(rp, np.arange(n, dtype=np.int32) % 5, np.ones(n, np.float32), np.ones(n, np.int8), 10)
    write_rcv1(data, str(tmp_path), first_id=101)          # documents 101 .. 100 + n
    (tmp_path / "rcv1-v2.topics.qrels").write_text("".join(f"{t} {d} 1\n" for t, d in qrels_lines))
    return str(tmp_path)


def test_reader_keeps_every_line_sorted_names_repeats_once_and_unknown_documents_out(tmp_path):
    lines = [("GCAT", 101), ("CCAT", 101), ("E21", 101), ("CCAT", 102), ("CCAT", 102), ("M11", 103), ("CCAT", 103),
             ("GCAT", 104), ("E21", 999)]                           # 999: a document the vectors do not hold
    d = rcv1(_rcv1_folder(tmp_path, lines), full=False, features_count=10, topics=True)
    assert d.topics.names == ("CCAT", "E21", "GCAT", "M11")
    got = [[d.topics.names[i] for i in d.topics.ids[d.topics.ptr[r]:d.topics.ptr[r + 1]]] for r in range(4)]
    assert got == [["CCAT", "E21", "GCAT"], ["CCAT"], ["CCAT", "M11"], ["GCAT"]]
    # the binary label stays the last line's CCAT label (quirk Q10): 101 ends on E21, 103 on CCAT
    assert d.label.tolist() == [-1, 1, 1, -1]
    plain = rcv1(str(tmp_path), full=False, features_count=10)
    assert plain.topics is None and np.array_equal(plain.label, d.label)


def test_reader_refuses_a_document_without_a_line(tmp_path):
    with pytest.raises(KeyError):
        rcv1(_rcv1_folder(tmp_path, [("CCAT", 101), ("GCAT", 102), ("CCAT", 104)]), full=False, features_count=10,
             topics=True)


# ---- Topics and Data ----------------------------------------------------------------------------------------------------

def test_topics_validation():
    Topics(np.array([0, 2, 2, 3]), np.array([0, 2, 1]), ("a", "b", "c"))
    for ptr, ids, names in [([1, 2], [0], ("a",)), ([0, 2, 1], [0, 1], ("a", "b")), ([0, 2], [0], ("a",)),
                            ([0, 1], [3], ("a",)), ([0, 2], [1, 0], ("a", "b")), ([0, 2], [1, 1], ("a", "b")),
                            ([0, 1], [0], ("a", "a")), ([0, 0], [], ())]:
        with pytest.raises(ValueError):
            Topics(np.array(ptr), np.array(ids, dtype=np.int32), names)


def test_split_and_head_carry_topics_and_positional_construction_works():
    rp = np.arange(6, dtype=np.int64)
    d = Data(rp, np.zeros(5, np.int32), np.ones(5, np.float32), np.ones(5, np.int8), DIM)   # positional, as before
    assert d.topics is None and d.split_at(3)[1].topics is None
    top = Topics(np.array([0, 1, 1, 3, 4, 6]), np.array([2, 0, 1, 2, 0, 2]), ("x", "y", "z"))
    d = Data(rp, np.zeros(5, np.int32), np.ones(5, np.float32), np.ones(5, np.int8), DIM, None, top)
    a, b = d.split_at(3)
    assert np.array_equal(a.topics.indicator(), top.indicator()[:3]) and np.array_equal(b.topics.indicator(),
                                                                                         top.indicator()[3:])
    assert d.head(2).topics.n_rows == 2 and a.topics.names == b.topics.names == top.names
    assert top.labels(2).tolist() == [1, -1, -1, 1, 1] and top.select(["z", "x"]).names == ("z", "x")


def test_synthetic_topics_is_deterministic_and_skewed():
    data = synthetic_rcv1(n_rows=3000, dim=500, seed=3)
    a, b = synthetic_topics(data, 20, seed=5), synthetic_topics(data, 20, seed=5)
    assert np.array_equal(a.ptr, b.ptr) and np.array_equal(a.ids, b.ids) and a.names == tuple(f"T{t}" for t in range(20))
    assert not np.array_equal(synthetic_topics(data, 20, seed=6).ids, a.ids)
    has = a.indicator()
    prev = has.mean(axis=0)
    assert prev[0] > 0.25 and prev[-1] < 0.03 and prev[0] > 5 * prev[-1]      # a popular topic, rare ones
    assert has[:2400].any(axis=0).all() and (~has[:2400]).any(axis=0).all()   # both classes in the train share
    assert (has.sum(axis=1) == 0).any() and (has.sum(axis=1) > 1).any()


# ---- the `topics` key -----------------------------------------------------------------------------------------------------

def test_topics_key_and_its_async_refusal():
    from distributed_sgd_b200.main import scenario
    from distributed_sgd_b200.ml.one_vs_rest import parse_topics
    from distributed_sgd_b200.utils.config import Config, load_config
    assert load_config(env={}).topics == "" and parse_topics("") is None
    assert load_config(env={"DSGD_TOPICS": "all"}).topics == "all" and parse_topics("ALL") == "all"
    assert parse_topics(" CCAT, GCAT ") == ["CCAT", "GCAT"]
    with pytest.raises(ValueError, match="topics"):
        load_config(env={"DSGD_TOPICS": "CCAT,,GCAT"})
    with pytest.raises(ValueError, match="topics"):
        scenario(Config(is_async=True, topics="all"), data=None)     # refused before any data or device is touched


# ---- fit_one_vs_rest against a stand-in context ----------------------------------------------------------------------------

class _Ctx:
    """Stands in for NativeCtx: records the label, class-weight and step calls; the weights after a fit name its topic."""

    def __init__(self, fail_topic=None):
        self.log, self.topic, self.fail_topic, self.cw = [], -1, fail_topic, (1.0, 1.0)

    def select_topic(self, t):
        self.log.append(("select", t))
        self.topic = t

    def set_class_weights(self, a, b):
        self.log.append(("cw", a, b))
        self.cw = (a, b)

    def set_weights(self, w):
        self.log.append(("set_weights",))

    def get_weights(self):
        return np.full(DIM, float(self.topic))

    def set_workers(self, counts, k_total):
        pass

    def sync_steps(self, samples, n_per_step, n_steps, lr, want_losses=True):
        if self.topic == self.fail_topic:
            raise RuntimeError("device failure")
        self.log.append(("steps", self.topic, np.array(samples).copy()))
        return np.zeros(n_steps)

    def eval_counts(self, lo, hi, w=None):
        return hi - lo, 0, 0.0

    def eval_class(self, lo, hi, w=None):
        from distributed_sgd_b200.native import ClassEval
        return ClassEval(0.0, 1.0, 1.0, 0, 0, 1, 1)


def _topics(n):
    has = np.zeros((n, 3), dtype=bool)
    has[::2, 0] = True
    has[:3, 1] = True
    has[1::3, 2] = True
    return Topics.from_indicator(has, ("a", "b", "c"))


def _master(ctx, class_weight=None, n_train=20, n_test=5):
    from types import SimpleNamespace
    from distributed_sgd_b200.core.master import MasterSync
    from distributed_sgd_b200.ml import SparseSVM
    stub = lambda n: Data(np.arange(n + 1, dtype=np.int64), np.zeros(n, np.int32), np.ones(n, np.float32),
                          np.where(np.arange(n) % 4 == 0, 1, -1).astype(np.int8), DIM)
    cw = (2.0, 2.0 / 3.0) if class_weight == "balanced" else (1.0, 1.0)   # 5 of the 20 train labels are +1
    slave = SimpleNamespace(ctx=ctx, world=1, is_async=False, n_train=n_train, n_test=n_test, dim=DIM, class_weight=cw,
                            topics=_topics(n_train + n_test))
    return MasterSync(0, stub(n_train), stub(n_test), SparseSVM(0.1, class_weight=class_weight), 1, slave=slave, seed=0)


def _fit(m, **kw):
    return m.fit_one_vs_rest(np.zeros(DIM), 3, 4, 0.5, lambda tl: False, **kw)


def test_one_fit_per_topic_with_the_draws_of_a_fresh_master():
    ctx = _Ctx()
    m = _master(ctx)
    ovr = _fit(m)
    assert ovr.topics == ("a", "b", "c") and ovr.weights.shape == (3, DIM) and len(ovr.histories) == 3
    assert [w[0] for w in ovr.weights] == [0.0, 1.0, 2.0]
    selects = [e for e in ctx.log if e[0] == "select"]
    assert selects == [("select", 0), ("select", 1), ("select", 2), ("select", -1)]
    steps = [e for e in ctx.log if e[0] == "steps"]
    by_topic = [[s[2] for s in steps if s[1] == t] for t in range(3)]
    fresh_ctx = _Ctx()
    fresh_ctx.topic = 0
    _master(fresh_ctx).fit(np.zeros(DIM), 3, 4, 0.5, lambda tl: False)
    fresh = [e[2] for e in fresh_ctx.log if e[0] == "steps"]
    for t in range(3):                                   # every topic draws what a fresh master draws
        assert len(by_topic[t]) == len(fresh) and all(np.array_equal(a, b) for a, b in zip(by_topic[t], fresh))
    assert m._draw_cache is None and m._epochs_drawn == 0


def test_draws_are_made_once_per_epoch_for_all_topics(monkeypatch):
    from distributed_sgd_b200.core import master as master_mod
    calls = []
    real = master_mod.EpochDraw.draw.__func__
    monkeypatch.setattr(master_mod.EpochDraw, "draw", classmethod(lambda cls, *a: calls.append(a[1]) or real(cls, *a)))
    _fit(_master(_Ctx()))
    assert sorted(calls) == [0, 1, 2]


def test_balanced_weights_per_topic_and_restored():
    ctx = _Ctx()
    m = _master(ctx, class_weight="balanced")
    _fit(m, topics=["c", 0])
    cws = [e for e in ctx.log if e[0] in ("select", "cw")]
    # topic c: rows 1, 4, .., 19 of 20 -> 7 positives; topic a: 10 of 20; then the Slave's weights back
    assert cws[0] == ("select", 2) and cws[1] == ("cw", 20 / 14, 20 / 26)
    assert cws[2] == ("select", 0) and cws[3] == ("cw", 1.0, 1.0)
    assert cws[-2:] == [("select", -1), ("cw", 2.0, 2.0 / 3.0)]
    assert m.class_weight == (2.0, 2.0 / 3.0) and m.slave.class_weight == (2.0, 2.0 / 3.0)


def test_labels_and_weights_restored_when_a_fit_raises():
    ctx = _Ctx(fail_topic=1)
    m = _master(ctx, class_weight="balanced")
    with pytest.raises(RuntimeError, match="device failure"):
        _fit(m)
    assert ctx.log[-2:] == [("select", -1), ("cw", 2.0, 2.0 / 3.0)] and ctx.topic == -1
    assert m.class_weight == (2.0, 2.0 / 3.0) and m._draw_cache is None


def test_refusals_before_any_fit():
    ctx = _Ctx()
    m = _master(ctx)
    m.topics = Topics.from_indicator(np.c_[np.ones(25, bool), np.arange(25) % 2 == 0], ("all", "half"))
    with pytest.raises(ValueError, match="'all'"):
        _fit(m)
    with pytest.raises(ValueError, match="topics"):
        _fit(_master(ctx), topics=["nope"])
    m = _master(ctx)
    m.jvm = object()
    with pytest.raises(ValueError, match="jvm_exact"):
        _fit(m)
    assert not [e for e in ctx.log if e[0] in ("select", "steps")]


# ---- the report ------------------------------------------------------------------------------------------------------------

def test_report_formulas_on_planted_words():
    from distributed_sgd_b200.ml.one_vs_rest import topic_report
    words = np.zeros(8 * 3 + 8, dtype=np.int64)
    words[0:8] = [3, 1, 0, 1, 5, 0, 0, 0]        # tp fn pos_none fp tn neg_none u2 nan
    words[8:16] = [0, 0, 0, 0, 10, 0, 0, 0]      # no positive and no positive prediction: F1 undefined
    words[16:24] = [1, 0, 1, 2, 4, 2, 0, 2]
    words[24:29] = [10, 4, 6, 1, 0]
    r = topic_report(words, ("a", "b", "c"))
    assert r["topics"]["a"]["precision"] == 3 / 4 and r["topics"]["a"]["recall"] == 3 / 4 and r["topics"]["a"]["f1"] == 6 / 8
    assert np.isnan(r["topics"]["b"]["f1"]) and np.isnan(r["topics"]["b"]["precision"])
    assert r["topics"]["c"]["f1"] == 2 / 5 and r["topics"]["c"]["nan_scores"] == 2
    assert r["micro_precision"] == 4 / 7 and r["micro_recall"] == 4 / 6 and r["micro_f1"] == 8 / (8 + 3 + 1 + 1)
    assert r["macro_f1"] == (6 / 8 + 2 / 5) / 2 and r["macro_f1_topics"] == 2
    assert r["subset_accuracy"] == 0.4 and r["hamming_loss"] == (1 + 1 + 0 + 1 + 2 + 2) / 30
    assert r["top1_accuracy"] == 6 / 9 and r["rows_without_topic"] == 1 and r["rows"] == 10
    with pytest.raises(ValueError):
        topic_report(words[:-1], ("a", "b", "c"))


# ---- two ranks: the report's words are all-reduced ---------------------------------------------------------------------------

def _free_port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def _worker(rank, world, port, q):
    sys.path.insert(0, ROOT)
    import torch.distributed as dist
    from types import SimpleNamespace
    from distributed_sgd_b200.core import Group, master as master_mod
    from distributed_sgd_b200.ml import SparseSVM
    dist.init_process_group("gloo", init_method=f"tcp://127.0.0.1:{port}", rank=rank, world_size=world)
    master_mod.NativeCtx.comm_unique_id = staticmethod(lambda: bytes(range(128)))

    class Ctx:
        calls = []

        def comm_init(self, uid):
            pass

        def eval_topics(self, lo, hi, W):      # each row counts once in rows, and its index in topic 0's TP
            self.calls.append((lo, hi))
            w = np.zeros(8 * len(W) + 8, dtype=np.int64)
            w[0], w[8 * len(W)], w[8 * len(W) + 1] = sum(range(lo, hi)), hi - lo, 1
            return w

    n_train, n_test = 30, 11
    stub = lambda n: Data(np.arange(n + 1, dtype=np.int64), np.zeros(n, np.int32), np.ones(n, np.float32),
                          np.ones(n, np.int8), DIM)
    slave = SimpleNamespace(ctx=Ctx(), world=world, is_async=False, n_train=n_train, n_test=n_test, dim=DIM,
                            topics=_topics(n_train + n_test))
    m = master_mod.MasterSync(rank, stub(n_train), stub(n_test), SparseSVM(0.5), world, slave=slave, group=Group(), seed=0)
    r = m.local_topic_report(np.zeros((3, DIM)), test_data=True)
    q.put({"rank": rank, "calls": slave.ctx.calls, "tp": r["topics"]["a"]["tp"], "rows": r["rows"],
           "exact": r["subset_accuracy"]})
    dist.destroy_process_group()


def test_report_words_all_reduced_over_two_ranks():
    import torch.multiprocessing as mp
    ctxmp = mp.get_context("spawn")
    q = ctxmp.Queue()
    port = _free_port()
    procs = [ctxmp.Process(target=_worker, args=(r, 2, port, q)) for r in range(2)]
    for p in procs:
        p.start()
    res = sorted([q.get(timeout=120) for _ in procs], key=lambda r: r["rank"])
    for p in procs:
        p.join(timeout=30)
    assert res[0]["calls"] == [(30, 35)] and res[1]["calls"] == [(35, 41)]      # contiguous shares of the test rows
    for r in res:
        assert r["tp"] == sum(range(30, 41)) and r["rows"] == 11 and r["exact"] == 2 / 11
