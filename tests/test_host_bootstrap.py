"""Host side of the bootstrap calls (Master.local_bootstrap / local_sampled_bootstrap / compare_bootstrap, the `bootstrap`
configuration key) with a stand-in for NativeCtx: how the replicates are split over ranks and gathered, the intervals, the
undefined replicates, the pairing of compare_bootstrap by key."""
import multiprocessing as mp
import os
import socket
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LAM = 1e-5


def _reps(key, lo, hi, scale):
    """Replicate words that depend on (key, b) alone, like the device's: replicate b = 7 has no positive row."""
    words, ap, loss = [], [], []
    for b in range(lo, hi):
        r = np.random.default_rng([key & 0xFFFFFFFF, b])
        tp, fn, fp, tn = (int(x) for x in r.integers(5, 50, size=4))
        if b == 7:
            tp = fn = 0
        u2 = int(r.integers(0, 2 * max((tp + fn) * (fp + tn), 1)))
        words.append([tp, fn, 0, fp, tn, 0, u2, 0, tp + fn + fp + tn])
        ap.append(float("nan") if b == 7 else r.random() * scale)
        loss.append(float(r.integers(0, 100)) * scale)
    return np.array(words, np.int64).reshape(-1, 9), np.array(ap), np.array(loss)


class BootCtx:
    def __init__(self, dim):
        self.dim, self.calls = dim, []

    def _scale(self, w):
        return 1.0 if w is None else float(np.asarray(w)[0])

    def eval_bootstrap(self, b, e, key, lo, hi, w=None):
        self.calls.append(("eval_bootstrap", b, e, key, lo, hi))
        return _reps(key, lo, hi, self._scale(w))

    def eval_sampled_bootstrap(self, b, e, skey, plo, phi, key, lo, hi, w=None):
        self.calls.append(("eval_sampled_bootstrap", b, e, skey, plo, phi, key, lo, hi))
        return _reps(key, lo, hi, self._scale(w))

    def eval_curve(self, b, e, w=None, curve=False):
        self.calls.append(("eval_curve", b, e))
        return np.array([30, 10, 0, 5, 55, 0, 3000, 0], np.int64), 0.75 * self._scale(w), 90

    def eval_sampled_curve(self, b, e, key, lo, hi, w=None, curve=False):
        self.calls.append(("eval_sampled_curve", b, e, key, lo, hi))
        return np.array([3, 1, 0, 1, 5, 0, 30, 0], np.int64), 0.5, 9

    def eval_sums(self, b, e, w=None):
        return 50.0 * self._scale(w), 85, 4.0

    def eval_sampled_sums(self, b, e, key, lo, hi, w=None):
        return 5.0, 8, 4.0

    def comm_init(self, uid):
        pass


class BootSlave:
    def __init__(self, world, n_train, n_test, dim):
        self.ctx, self.world, self.is_async = BootCtx(dim), world, False
        self.n_train, self.n_test, self.dim = n_train, n_test, dim


def _stub(n, dim):
    from distributed_sgd_b200.utils.dataset import Data
    return Data(np.arange(n + 1, dtype=np.int64), np.zeros(n, np.int32), np.ones(n, np.float32), np.ones(n, np.int8), dim)


def _master(world=1, group=None, seed=3, n_train=101, n_test=100):
    from distributed_sgd_b200.core.master import MasterSync
    from distributed_sgd_b200.ml import SparseSVM
    slave = BootSlave(world, n_train, n_test, 16)
    m = MasterSync(0, _stub(n_train, 16), _stub(n_test, 16), SparseSVM(LAM), world, slave=slave, seed=seed, group=group,
                   attach=False)
    return m, slave.ctx


def test_replicates_split_into_contiguous_rank_ranges():
    from distributed_sgd_b200.core.master import bootstrap_share
    for n in (1, 2, 7, 1000, 1001):
        for W in (1, 2, 3, 8):
            shares = [bootstrap_share(n, W, r) for r in range(W)]
            assert shares[0][0] == 0 and shares[-1][1] == n
            assert all(a[1] == b[0] for a, b in zip(shares, shares[1:]))
            assert max(h - l for l, h in shares) - min(h - l for l, h in shares) <= 1


def test_local_bootstrap_values_and_intervals():
    from distributed_sgd_b200.core.master import BOOTSTRAP_METRICS, bootstrap_key
    m, ctx = _master()
    r = m.local_bootstrap(None, n_boot=40, level=0.9)
    assert ctx.calls[-1] == ("eval_bootstrap", 101, 201, bootstrap_key(3), 0, 40)
    assert set(r) == set(BOOTSTRAP_METRICS)
    words, ap, loss = _reps(bootstrap_key(3), 0, 40, 1.0)
    acc = (words[:, 0] + words[:, 4]) / words[:, 8]
    assert np.array_equal(r["accuracy"]["replicates"], acc)
    q = [(1 - 0.9) / 2, 1 - (1 - 0.9) / 2]                 # numpy.quantile's default method at level 0.9
    assert [r["accuracy"]["lo"], r["accuracy"]["hi"]] == list(np.quantile(acc, q))
    assert r["accuracy"]["se"] == np.std(acc, ddof=1) and r["accuracy"]["n_defined"] == 40
    assert r["accuracy"]["estimate"] == 85 / 100
    assert r["loss"]["estimate"] == LAM * 4.0 + 50.0 / 100
    assert np.array_equal(r["loss"]["replicates"], LAM * 4.0 + loss / words[:, 8])
    assert r["ap"]["estimate"] == 0.75 and r["auc"]["estimate"] == 3000 / (2 * 40 * 60)
    # replicate 7 has no positive row: its auc, ap, recall and f1 are undefined, excluded and counted out
    for k in ("auc", "ap", "recall"):
        assert np.isnan(r[k]["replicates"][7]) and r[k]["n_defined"] == 39
        ok = np.delete(r[k]["replicates"], 7)
        assert [r[k]["lo"], r[k]["hi"]] == list(np.quantile(ok, q))
    # an explicit key is used as given; n_boot must be positive
    m.local_bootstrap(None, n_boot=3, key=99)
    assert ctx.calls[-1] == ("eval_bootstrap", 101, 201, 99, 0, 3)
    with pytest.raises(ValueError):
        m.local_bootstrap(None, n_boot=0)


def test_sampled_bootstrap_draws_a_fresh_sample():
    from distributed_sgd_b200.core.master import bootstrap_key, sampled_key
    m, ctx = _master()
    r = m.local_sampled_bootstrap(None, 30, n_boot=5)
    assert ("eval_sampled_curve", 101, 201, sampled_key(3, 0), 0, 30) in ctx.calls
    assert ctx.calls[-1] == ("eval_sampled_bootstrap", 101, 201, sampled_key(3, 0), 0, 30, bootstrap_key(3), 0, 5)
    assert r["accuracy"]["estimate"] == 8 / 10
    m.local_sampled_bootstrap(None, 30, n_boot=5)
    assert ctx.calls[-1][3] == sampled_key(3, 1)


def test_compare_bootstrap_pairs_by_key():
    m, ctx = _master()
    wa, wb = np.full(16, 1.0), np.full(16, 2.0)
    r = m.compare_bootstrap(wa, wb, n_boot=20, key=5)
    boots = [c for c in ctx.calls if c[0] == "eval_bootstrap"]
    assert len(boots) == 2 and boots[0] == boots[1] == ("eval_bootstrap", 101, 201, 5, 0, 20)
    _, ap, loss = _reps(5, 0, 20, 1.0)
    d = np.delete(ap, 7)       # b's AP is twice a's in every replicate: b - a = a's AP, b better wherever defined
    assert r["ap"]["n_defined"] == 19 and np.array_equal(np.delete(r["ap"]["replicates"], 7), d)
    assert r["ap"]["estimate"] == 0.75 and r["ap"]["p_better"] == float(np.mean(d > 0))
    assert r["loss"]["p_better"] == float(np.mean(np.delete(loss, []) < 0))    # lower loss is better: b's is never lower
    same = m.compare_bootstrap(wa, wa, n_boot=20, key=5)
    for k, s in same.items():
        ok = s["replicates"][~np.isnan(s["replicates"])]
        assert s["estimate"] == 0.0 and not ok.any() and s["p_better"] == 0.0, k


def _free_port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def _worker(rank, world, port, q):
    sys.path.insert(0, ROOT)
    import torch.distributed as dist
    from distributed_sgd_b200.core import Group
    dist.init_process_group("gloo", init_method=f"tcp://127.0.0.1:{port}", rank=rank, world_size=world)
    try:
        m, ctx = _master(world=world, group=Group())
        r = m.local_bootstrap(None, n_boot=25)
        q.put({"rank": rank, "calls": [c for c in ctx.calls if c[0] == "eval_bootstrap"],
               "reps": {k: v["replicates"].tobytes() for k, v in r.items()},
               "lo": {k: v["lo"] for k, v in r.items()}})
    finally:
        dist.destroy_process_group()


def test_two_ranks_gather_the_same_bits_in_rank_order():
    from distributed_sgd_b200.core.master import bootstrap_key
    ctxmp = mp.get_context("spawn")
    q = ctxmp.Queue()
    port = _free_port()
    procs = [ctxmp.Process(target=_worker, args=(r, 2, port, q)) for r in range(2)]
    for p in procs:
        p.start()
    out = sorted((q.get(timeout=120) for _ in procs), key=lambda d: d["rank"])
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0
    key = bootstrap_key(3)
    assert out[0]["calls"] == [("eval_bootstrap", 101, 201, key, 0, 12)]
    assert out[1]["calls"] == [("eval_bootstrap", 101, 201, key, 12, 25)]
    assert out[0]["reps"] == out[1]["reps"]
    m, _ = _master()
    one = m.local_bootstrap(None, n_boot=25)
    for k, v in one.items():
        assert v["replicates"].tobytes() == out[0]["reps"][k]
        assert (np.isnan(v["lo"]) and np.isnan(out[1]["lo"][k])) or v["lo"] == out[1]["lo"][k]


def test_bootstrap_configuration_key():
    from distributed_sgd_b200.utils import load_config
    assert load_config(None, env={}).bootstrap == 0
    assert load_config(None, env={"DSGD_BOOTSTRAP": "1000"}).bootstrap == 1000
    with pytest.raises(ValueError, match="bootstrap"):
        load_config(None, env={"DSGD_BOOTSTRAP": "-1"})
    with pytest.raises(ValueError):
        load_config(None, env={"DSGD_BOOTSTRAP": "many"})
