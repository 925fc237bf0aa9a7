"""Ranking a row's topics on the host, without a GPU: the report's formulas on planted words, limbs_value against the
fixed-point model, the `topic-rank-k` key and its refusals, OneVsRest.predict_topk through Slave.topics_topk against a
stand-in context, and a two-process all-reduce whose merged limbs give the report of one pass over all rows."""
import os
import socket
import sys

import numpy as np
import pytest

from distributed_sgd_b200.utils.dataset import Data, Topics
from loss_sum_model import device_model
from topic_ranking_model import topic_ranking, topk

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DIM, T = 8, 7


def _planted(n, seed=0):
    """[T, n] tie-heavy margins with a NaN row, and a [n, T] indicator with rows without a topic and one with every topic"""
    rng = np.random.default_rng(seed)
    m = rng.integers(-3, 4, size=(T, n)).astype(np.float64)
    m[:, 1::5] = rng.standard_normal((T, len(range(1, n, 5))))
    m[2, 4] = np.nan
    has = rng.random((n, T)) < 0.35
    has[0] = False
    has[3] = True
    return m, has


# ---- the report --------------------------------------------------------------------------------------------------------------

def _block(values):
    from topic_ranking_model import limbs
    return np.array(limbs(values), dtype=np.int64)


def test_report_formulas_on_planted_words():
    from distributed_sgd_b200.ml.one_vs_rest import topic_ranking_report
    k = 2
    head = np.array([10, 4, 3, 3, 1, 9, 6, 0, 3, 5], dtype=np.int64)   # rows, N, NaN, no topic, all, coverage, pairs, 0, hits
    A, B, C1, C2 = [0.5, 0.25, 1.0], [0.125, 0.5], [1.0, 0.5, 0.5, 0.0], [1.0, 1.0, 0.5, 0.25]
    words = np.concatenate([head] + [_block(v) for v in (A, B, C1, C2)])
    r = topic_ranking_report(words, k)
    assert (r["rows"], r["ranked_rows"], r["rows_with_nan_score"], r["rows_without_topic"], r["rows_with_every_topic"]) == \
        (10, 4, 3, 3, 1)
    assert r["precision_at"] == {1: 3 / 4, 2: 5 / 8}
    assert r["recall_at"] == {1: 2.0 / 4, 2: 2.75 / 4}
    assert r["lrap"] == 1.75 / 4 and r["coverage_error"] == 9 / 4 and r["ranking_loss"] == 0.625 / 3
    with pytest.raises(ValueError):
        topic_ranking_report(words[:-1], k)
    empty = np.zeros(8 + k + 7 * (2 + k), dtype=np.int64)               # no ranked row: every ratio is NaN
    r = topic_ranking_report(empty, k)
    assert all(np.isnan(x) for x in (r["lrap"], r["coverage_error"], r["ranking_loss"], r["precision_at"][1],
                                     r["recall_at"][2]))
    every = empty.copy()
    every[[0, 1, 4, 5, 8, 9]] = [2, 2, 2, 2 * T, 2, 4]                   # two ranked rows, both with every topic
    assert np.isnan(topic_ranking_report(every, k)["ranking_loss"]) and topic_ranking_report(every, k)["precision_at"][2] == 1.0


@pytest.mark.parametrize("seed", range(5))
def test_limbs_value_is_the_device_reader(seed):
    from distributed_sgd_b200.ml.one_vs_rest import limbs_value
    rng = np.random.default_rng(seed)
    values = list(rng.integers(1, 1000, size=300) / rng.integers(1, 1000, size=300))
    values = [min(v, 1.0) for v in values] + [1.0, 0.0, 1 / 3, 2.0 ** -170]
    assert limbs_value(_block(values)) == device_model(values)
    blk = _block(values)
    raw = blk.copy()                      # limbs added over several calls, not carried: the same value
    raw[0] += 5 << 40
    raw[1] -= 5
    assert limbs_value(raw) == limbs_value(blk)
    blk[6] = 1
    assert np.isnan(limbs_value(blk))


# ---- the key -----------------------------------------------------------------------------------------------------------------

def test_topic_rank_k_key_and_its_refusals():
    from distributed_sgd_b200.main import scenario
    from distributed_sgd_b200.utils.config import Config, load_config
    assert load_config(env={}).topic_rank_k == 0
    cfg = load_config(env={"DSGD_TOPICS": "all", "DSGD_TOPIC_RANK_K": "5"})
    assert cfg.topic_rank_k == 5
    assert load_config(env={"DSGD_TOPICS": "a,b", "DSGD_TOPIC_RANK_K": "32"}).topic_rank_k == 32
    for bad in ("33", "-1"):
        with pytest.raises(ValueError, match="topic-rank-k"):
            load_config(env={"DSGD_TOPICS": "all", "DSGD_TOPIC_RANK_K": bad})
    with pytest.raises(ValueError, match="topic-rank-k.*topics"):
        load_config(env={"DSGD_TOPIC_RANK_K": "3"})                     # ranking without one-vs-rest topics
    with pytest.raises(ValueError, match="topic-rank-k"):
        scenario(Config(topic_rank_k=3), data=None)                     # refused before any data or device is touched
    with pytest.raises(ValueError, match="topics"):
        scenario(Config(is_async=True, topics="all", topic_rank_k=3), data=None)
    names = tuple(f"t{i}" for i in range(3))
    has = np.zeros((10, 3), dtype=bool)
    has[::2, 0] = True
    data = Data(np.arange(11, dtype=np.int64), np.zeros(10, np.int32), np.ones(10, np.float32), np.ones(10, np.int8), DIM,
                topics=Topics.from_indicator(has, names))
    with pytest.raises(ValueError, match="topic-rank-k: 4 exceeds the 3 topics"):
        scenario(Config(topics="all", topic_rank_k=4), data=data)


# ---- predict_topk against a stand-in context ------------------------------------------------------------------------------------

class _TopkCtx:
    """Stands in for NativeCtx: ranks planted margins of the rows with the model's tie rule."""

    def __init__(self, margins):
        self.m, self.calls = margins, []

    def topics_topk(self, samples, W, k):
        self.calls.append((np.asarray(samples).copy(), np.asarray(W).shape, k))
        return topk(self.m[:, np.asarray(samples)], k)


def test_predict_topk_goes_through_slave_topics_topk():
    from distributed_sgd_b200.core.slave import Slave
    from distributed_sgd_b200.ml.one_vs_rest import OneVsRest
    m, _ = _planted(30)
    m[1:, 29] = np.nan                                              # one non-NaN score: slots 2 and 3 are -1 and NaN
    slave = Slave.__new__(Slave)
    slave.ctx, slave.n_train = _TopkCtx(m), 30
    ovr = OneVsRest(np.zeros((T, DIM)), tuple(f"t{i}" for i in range(T)), [{}] * T)
    idx = np.array([4, 0, 17, 4, 29], dtype=np.int32)
    ids, top = ovr.predict_topk(slave, idx, 3)
    ref_ids, ref_top = topk(m[:, idx], 3)
    assert np.array_equal(ids, ref_ids) and np.array_equal(top, ref_top, equal_nan=True)
    assert slave.ctx.calls[0][1:] == ((T, DIM), 3) and np.array_equal(slave.ctx.calls[0][0], idx)
    assert ids[4].tolist() == [0, -1, -1] and top[4, 0] == m[0, 29] and np.isnan(top[4, 1:]).all()
    for i, r in enumerate(idx):                                     # ids follow the order of -margin, ties to the lower t
        order = sorted((t for t in range(T) if not np.isnan(m[t, r])), key=lambda t: (m[t, r], t))[:3]
        assert list(ids[i, :len(order)]) == order
    with pytest.raises(IndexError):
        ovr.predict_topk(slave, [30], 3)                            # a train-row wrapper, like Slave.margins


# ---- two ranks: the words and limbs are all-reduced ---------------------------------------------------------------------------

def _free_port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def _worker(rank, world, port, q):
    sys.path.insert(0, ROOT)
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    import torch.distributed as dist
    from types import SimpleNamespace
    from distributed_sgd_b200.core import Group, master as master_mod
    from distributed_sgd_b200.ml import SparseSVM
    from topic_ranking_model import topic_ranking as model
    dist.init_process_group("gloo", init_method=f"tcp://127.0.0.1:{port}", rank=rank, world_size=world)
    master_mod.NativeCtx.comm_unique_id = staticmethod(lambda: bytes(range(128)))
    n_train, n_test, k = 30, 41, 3
    m, has = _planted(n_train + n_test, seed=9)

    class Ctx:
        calls = []

        def comm_init(self, uid):
            pass

        def eval_topic_ranking(self, lo, hi, W, kk):   # the model over this rank's rows
            self.calls.append((lo, hi))
            return model(m[:, lo:hi], has[lo:hi], kk)

    stub = lambda n: Data(np.arange(n + 1, dtype=np.int64), np.zeros(n, np.int32), np.ones(n, np.float32),
                          np.ones(n, np.int8), DIM)
    slave = SimpleNamespace(ctx=Ctx(), world=world, is_async=False, n_train=n_train, n_test=n_test, dim=DIM,
                            topics=Topics.from_indicator(has, tuple(f"t{i}" for i in range(T))))
    mm = master_mod.MasterSync(rank, stub(n_train), stub(n_test), SparseSVM(0.5), world, slave=slave, group=Group(), seed=0)
    r = mm.local_topic_ranking_report(np.zeros((T, DIM)), k, test_data=True)
    q.put({"rank": rank, "calls": slave.ctx.calls, "report": r})
    dist.destroy_process_group()


def test_words_and_limbs_all_reduced_over_two_ranks():
    import torch.multiprocessing as mp
    from distributed_sgd_b200.ml.one_vs_rest import topic_ranking_report
    ctxmp = mp.get_context("spawn")
    q = ctxmp.Queue()
    port = _free_port()
    procs = [ctxmp.Process(target=_worker, args=(r, 2, port, q)) for r in range(2)]
    for p in procs:
        p.start()
    res = sorted([q.get(timeout=120) for _ in procs], key=lambda r: r["rank"])
    for p in procs:
        p.join(timeout=30)
    assert res[0]["calls"] == [(30, 50)] and res[1]["calls"] == [(50, 71)]      # contiguous shares of the test rows
    m, has = _planted(71, seed=9)
    whole = topic_ranking_report(topic_ranking(m[:, 30:], has[30:], 3)[0], 3)   # one pass over all the test rows
    for r in res:
        assert _same(r["report"], whole)
    assert whole["rows"] == 41 and whole["ranked_rows"] > 0


def _same(a, b) -> bool:
    """dict equality with NaN equal to NaN"""
    if isinstance(a, dict):
        return a.keys() == b.keys() and all(_same(a[x], b[x]) for x in a)
    return a == b or (a != a and b != b)
