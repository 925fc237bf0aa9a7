"""Host-side mirror of the reference's control logic (no GPU): config contract, split, early stopping, data."""
import os

import numpy as np
import pytest

from distributed_sgd_b200.ml import EarlyStopping, GradState, SplitStrategy
from distributed_sgd_b200.utils import load_config, rcv1, synthetic_rcv1, write_rcv1
from oracle import scala_semantics as S


def test_config_defaults_match_application_conf():          # resources/application.conf:15-50
    c = load_config(env={})
    assert (c.batch_size, c.learning_rate, c.lam, c.node_count, c.max_epochs) == (100, 0.5, 1e-5, 3, 10)
    assert (c.check_every, c.leaky_loss, c.patience, c.conv_delta, c.is_async, c.full) == (100, 0.9, 5, 0.01, False, False)
    assert c.port == 4000 and c.host == "127.0.0.1" and c.master_host is None


def test_config_env_overrides_and_file(tmp_path):
    c = load_config(env={"DSGD_BATCH_SIZE": "256", "DSGD_ASYNC": "true", "DSGD_LAMBDA": "0.001", "DSGD_NODE_COUNT": "8"})
    assert (c.batch_size, c.is_async, c.lam, c.node_count) == (256, True, 0.001, 8)
    conf = tmp_path / "application.conf"
    conf.write_text('dsgd {\n  batch-size = 100\n  batch-size = ${?DSGD_BATCH_SIZE}\n  lambda = 0.00001\n'
                    '  async = false\n  async = ${?DSGD_ASYNC}\n  # comment\n  host = "10.0.0.1"\n}\nkamon { metric { } }\n')
    c = load_config(str(conf), env={"DSGD_ASYNC": "yes"})
    assert (c.batch_size, c.is_async, c.host) == (100, True, "10.0.0.1")
    conf.write_text("dsgd {\n  bogus-key = 1\n}\n")
    with pytest.raises(KeyError):
        load_config(str(conf), env={})


def test_vanilla_split_is_the_references():                  # core/ml/SplitStrategy.scala:13-14
    for n, k in ((10, 4), (9, 4), (6, 2), (560000, 8), (101, 4), (5, 8)):
        assert [list(r) for r in SplitStrategy.vanilla(n, k)] == S.split_vanilla(n, k)


def test_early_stopping_mirrors_the_literal_restatement():   # core/ml/EarlyStopping.scala:13-46
    rng = np.random.default_rng(0)
    for patience, delta, min_steps in ((5, 0.01, None), (2, 0.0, None), (3, 0.1, 4), (1, 0.001, 10)):
        a = EarlyStopping.no_improvement(patience, delta, min_steps)
        b = S.early_stopping_no_improvement(patience, delta, min_steps)
        for _ in range(200):
            losses = rng.choice([0.5, 0.505, 0.6, 0.9, 0.3], size=int(rng.integers(0, 9))).tolist()
            assert a(losses) == b(losses), (patience, delta, min_steps, losses)
    assert EarlyStopping.target(0.3)([0.2, 0.9]) and not EarlyStopping.target(0.3)([0.4]) and not EarlyStopping.target(0.3)([])


def test_grad_state():                                       # core/ml/GradState.scala:6-23
    g = GradState.start_state(np.zeros(3))
    g2 = g.replace_grad(np.ones(3)).finish(0.25)
    assert g2.updates == 1 and g2.loss == 0.25 and g2.end is not None and g.end is None


def test_synthetic_generator_is_deterministic_and_rcv1_shaped():
    a, b = synthetic_rcv1(n_rows=3000, seed=4), synthetic_rcv1(n_rows=3000, seed=4)
    assert np.array_equal(a.col, b.col) and np.array_equal(a.val, b.val) and np.array_equal(a.label, b.label)
    c = synthetic_rcv1(n_rows=3000, seed=5)
    assert not np.array_equal(a.col[:100], c.col[:100])
    lens = np.diff(a.row_ptr)
    assert a.dim == 47236 and lens.min() >= 1 and lens.max() <= 2000 and 70 < lens.mean() < 120
    for r in range(0, 3000, 97):                              # sorted unique columns, L2-normalised positive rows
        cols, vals = a.col[a.row_ptr[r]:a.row_ptr[r + 1]], a.val[a.row_ptr[r]:a.row_ptr[r + 1]]
        assert np.all(np.diff(cols) > 0) and np.all(vals > 0) and abs(float(np.sum(vals.astype(np.float64) ** 2)) - 1) < 1e-5
    assert 0.35 < (a.label > 0).mean() < 0.65 and set(np.unique(a.label)) == {-1, 1}
    assert a.algorithmic_bytes() == 8 * a.nnz + 16 * a.n_rows
    head, tail = a.split_at(2400)                             # Main.scala:52
    assert head.n_rows == 2400 and tail.n_rows == 600 and head.nnz + tail.nnz == a.nnz and tail.row_ptr[0] == 0


def test_rcv1_text_round_trip(tmp_path):                      # utils/Dataset.scala:19-45 (incl. label rule)
    d = synthetic_rcv1(n_rows=300, seed=2)
    write_rcv1(d, str(tmp_path), first_id=2286)
    line = open(tmp_path / "lyrl2004_vectors_train.dat").readline()
    assert line.startswith("2286  ") and ":" in line          # "<id>  <k>:<v> ..." (two separators: parts.drop(2))
    back = rcv1(str(tmp_path), full=False)
    assert back.n_rows == 300 and np.array_equal(back.col, d.col) and np.array_equal(back.val, d.val)
    assert np.array_equal(back.label, d.label) and np.array_equal(back.row_ptr, d.row_ptr)
    with open(tmp_path / "rcv1-v2.topics.qrels", "a") as f:   # the LAST line of a document decides (quirk Q10)
        f.write("CCAT 2286 1\nGCAT 2287 1\n")
    back = rcv1(str(tmp_path), full=False)
    assert back.label[0] == 1 and back.label[1] == -1


def test_rcv1_repeated_key_keeps_the_last_value(tmp_path):   # utils/Dataset.scala:26-32: each row goes through .toMap
    """A key repeated on one line is stored once with its last value (0.25 over 0.5, in either position); a last value of
    1e-25 is stored as such and the 1e-20 filter of every consumer drops the key.  With repeats in the train file, the
    rows of the test files that follow it must still line up (the parsed arrays are shorter than the pair count)."""
    lines = {"lyrl2004_vectors_train.dat": ["10  3:0.5 7:1 3:0.25", "11  5:1 5:1e-25 9:2", "12  2:0.5 8:0.5 2:0.25 8:0.75"],
             "lyrl2004_vectors_test_pt0.dat": ["13  1:1 4:0.5"], "lyrl2004_vectors_test_pt1.dat": ["14  6:0.125"],
             "lyrl2004_vectors_test_pt2.dat": ["15  9:4 9:3"], "lyrl2004_vectors_test_pt3.dat": ["16  2:1"]}
    for name, rows in lines.items():
        (tmp_path / name).write_text("\n".join(rows) + "\n")
    (tmp_path / "rcv1-v2.topics.qrels").write_text("".join(f"CCAT {i} 1\n" for i in range(10, 17)))
    d = rcv1(str(tmp_path), full=True, features_count=10)
    assert d.n_rows == 7 and d.row_ptr.tolist() == [0, 2, 4, 6, 8, 9, 10, 11]
    assert len(d.col) == len(d.val) == 11
    rows = [dict(zip(d.col[a:b].tolist(), d.val[a:b].tolist())) for a, b in zip(d.row_ptr[:-1], d.row_ptr[1:])]
    assert rows[0] == {2: 0.25, 6: 1.0}                         # key 3 (column 2): the last value wins
    assert rows[2] == {1: 0.25, 7: 0.75}
    assert set(rows[1]) == {4, 8} and rows[1][8] == 2.0 and 0 < rows[1][4] <= 1e-20   # key 5 ends at 1e-25: filtered
    assert rows[3] == {0: 1.0, 3: 0.5} and rows[4] == {5: 0.125} and rows[5] == {8: 3.0} and rows[6] == {1: 1.0}
    assert (d.label == 1).all()


class _RecCtx:
    """Stand-in device context that records what MasterSync would send to the GPU (no arithmetic)."""

    def __init__(self, dim):
        self.dim, self.calls = dim, []

    def set_weights(self, w):
        pass

    def get_weights(self):
        return np.zeros(self.dim)

    def set_workers(self, counts, k_total):
        self.calls.append(("workers", list(map(int, counts)), int(k_total)))

    def sync_steps(self, samples, n_per_step, n_steps, lr, want_losses=True):
        self.calls.append(("steps", np.array(samples).reshape(n_steps, n_per_step).copy()))
        return np.zeros(n_steps)

    def eval_counts(self, lo, hi, w=None):
        return hi - lo, 0, 0.0


def _master(n_train, n_test=5, dim=8):
    from types import SimpleNamespace
    from distributed_sgd_b200.core.master import MasterSync
    from distributed_sgd_b200.ml import SparseSVM
    from distributed_sgd_b200.utils.dataset import Data
    stub = lambda n: Data(np.arange(n + 1, dtype=np.int64), np.zeros(n, np.int32), np.ones(n, np.float32), np.ones(n, np.int8), dim)
    slave = SimpleNamespace(ctx=_RecCtx(dim), world=1, is_async=False, n_train=n_train, n_test=n_test, dim=dim)
    return MasterSync(0, stub(n_train), stub(n_test), SparseSVM(0.1), 1, slave=slave, seed=0), slave.ctx


def test_master_sync_epoch_structure_and_reference_quirks():
    """core/Master.scala:135-138,179-188: an epoch is ceil(maxSamples / B) steps; every step takes a fresh draw of each
    worker's own range; the tail slices are shorter (Q5); vanilla(9, 4) yields 3 groups, so only 3 workers are asked and
    the mean divides by 3."""
    m, ctx = _master(n_train=9)
    m.fit(np.zeros(8), max_epochs=1, batch_size=2, learning_rate=0.5, stopping_criterion=lambda l: False, virtual_workers=4)
    workers = [c for c in ctx.calls if c[0] == "workers"]
    steps = [c[1] for c in ctx.calls if c[0] == "steps"]
    assert workers[0] == ("workers", [2, 2, 2], 3)                      # 3 groups of 3 rows -> 3 requests, divisor 3
    assert steps[0].shape == (1, 6) and steps[1].shape == (1, 3)        # steps at offsets 0 and 2: slices of 2, then of 1
    for k in range(3):                                                  # each worker samples its own contiguous range
        assert set(steps[0][0, 2 * k:2 * k + 2]) <= set(range(3 * k, 3 * k + 3))
    assert len(set(steps[0][0])) == 6                                   # without replacement inside a slice
    assert m.history["losses"] == [1.0] and m.history["test_accs"] == [0.0]


def test_master_sync_empty_slice_fails_like_the_reference():
    """Quirk Q7: groups of 3, 3, 3, 1 rows with batch 2 -> at offset 2 the short group's slice is empty, Vec.sum throws
    and the whole fit fails (math/Vec.scala:129 via core/Master.scala:187)."""
    m, ctx = _master(n_train=10)
    with pytest.raises(ValueError, match="empty list"):
        m.fit(np.zeros(8), max_epochs=1, batch_size=2, learning_rate=0.5, stopping_criterion=lambda l: False, virtual_workers=4)


def test_master_sync_stops_on_criterion_and_max_epochs():
    m, ctx = _master(n_train=8)
    seen = []
    state = m.fit(np.zeros(8), max_epochs=5, batch_size=4, learning_rate=0.5,
                  stopping_criterion=lambda losses: seen.append(list(losses)) or len(losses) >= 2)
    assert state.updates == 2 and len(m.history["test_losses"]) == 2    # stopped by the criterion after 2 epochs
    assert seen[0] == [] and len(seen[-1]) == 2                         # the criterion sees the newest-first test losses
    state = m.fit(np.zeros(8), max_epochs=3, batch_size=4, learning_rate=0.5, stopping_criterion=lambda l: False)
    assert state.updates == 3 and state.loss == m.history["losses"][-1]


def test_jvm_random_known_answers():
    """java.util.Random's well-known outputs: seed 0 -> nextInt() = -1155484576, -723955400, 1033096058, ...;
    seed 0 -> nextInt(100) = 60, 48, 29, 47, 15; seed 42 -> nextInt(10) = 0, 3, 8, 4, 0, 5, 5, 8, 9, 3."""
    from distributed_sgd_b200.utils.jvm_random import JvmRandom
    r = JvmRandom(0)
    assert [r.next_int() for _ in range(5)] == [-1155484576, -723955400, 1033096058, -1690734402, -1557280266]
    r = JvmRandom(0)
    assert [r.next_int(100) for _ in range(5)] == [60, 48, 29, 47, 15]
    r = JvmRandom(42)
    assert [r.next_int(10) for _ in range(10)] == [0, 3, 8, 4, 0, 5, 5, 8, 9, 3]
    r = JvmRandom(42)
    assert r.next_int() == -1170105035
    r = JvmRandom(7)
    assert all(0 <= r.next_int(16) < 16 for _ in range(100))           # power-of-two bound takes the multiply path


def test_scala_shuffle_and_epoch_draws():
    """scala.util.Random.shuffle (2.12): Fisher-Yates from the top with nextInt(n); the epoch helper equals shuffling a
    fresh copy of every group at every step and slicing it (core/Master.scala:184-187)."""
    from distributed_sgd_b200.utils.jvm_random import JvmRandom
    a, b = JvmRandom(0), JvmRandom(0)
    xs = list(range(10, 20))
    buf = list(xs)
    for n in range(len(buf), 1, -1):                                   # the algorithm, spelled out with next_int
        k = b.next_int(n)
        buf[n - 1], buf[k] = buf[k], buf[n - 1]
    assert a.shuffle(xs).tolist() == buf and sorted(buf) == xs
    a, b = JvmRandom(0), JvmRandom(0)
    steps = a.sync_epoch(10, 4, 2)                                     # groups 3,3,3,1 -> steps at offsets 0 and 2
    assert len(steps) == 2 and [len(g) for g in steps[0]] == [2, 2, 2, 1] and [len(g) for g in steps[1]] == [1, 1, 1, 0]
    groups = [range(0, 3), range(3, 6), range(6, 9), range(9, 10)]
    for s, batch in enumerate((0, 2)):
        for k, g in enumerate(groups):
            assert steps[s][k].tolist() == b.shuffle(list(g))[batch:batch + 2].tolist()


def test_master_sync_jvm_exact_draws():
    from types import SimpleNamespace
    from distributed_sgd_b200.core.master import MasterSync
    from distributed_sgd_b200.ml import SparseSVM
    from distributed_sgd_b200.utils.dataset import Data
    from distributed_sgd_b200.utils.jvm_random import JvmRandom
    stub = lambda n: Data(np.arange(n + 1, dtype=np.int64), np.zeros(n, np.int32), np.ones(n, np.float32), np.ones(n, np.int8), 8)
    slave = SimpleNamespace(ctx=_RecCtx(8), world=1, is_async=False, n_train=12, n_test=5, dim=8)
    m = MasterSync(0, stub(12), stub(5), SparseSVM(0.1), 1, slave=slave, seed=0, jvm_exact=True)
    m.fit(np.zeros(8), max_epochs=1, batch_size=3, learning_rate=0.5, stopping_criterion=lambda l: False, virtual_workers=2)
    steps = [c[1] for c in slave.ctx.calls if c[0] == "steps"]
    ref = JvmRandom(0).sync_epoch(12, 2, 3)
    got = np.concatenate([s.reshape(-1) for s in steps]).tolist()
    assert got == [int(i) for st in ref for g in st for i in g]


def test_jvm_async_draws():
    from distributed_sgd_b200.utils.jvm_random import JvmRandom
    assigned = np.arange(100, 200, dtype=np.int32)
    a, b = JvmRandom(0), JvmRandom(0)
    assert a.async_draws(assigned, 5).tolist() == [100 + b.next_int(100) for _ in range(5)] == [160, 148, 129, 147, 115]
    a, b = JvmRandom(3), JvmRandom(3)
    d = a.async_draws(assigned, 4, batch_size=7)                       # positions, not ids (quirk Q6)
    assert d.shape == (28,) and d.max() < 100
    assert d[:7].tolist() == b.shuffle(np.arange(100))[:7].tolist()


class _AsyncScriptCtx:
    """Stand-in device context for MasterAsync: the update counter and the test-set evaluation follow a script, so the
    host-side loop (polling, leaky loss, best weights, stop rules) can be compared with the literal restatement of
    core/MasterAsync.scala:66-177 on the SAME stream."""

    def __init__(self, dim, counter_script, eval_script, n_test):
        self.dim, self.counter, self.evals, self.n_test = dim, list(counter_script), list(eval_script), n_test
        self.poll, self.snapshots, self.stopped = -1, [], False

    def set_weights(self, w): pass
    def async_host_master(self, w): pass

    def async_updates(self):
        self.poll += 1
        return self.counter[min(self.poll, len(self.counter) - 1)]

    def async_master_weights(self):
        w = np.zeros(self.dim); w[0] = float(self.poll)       # tag the snapshot with the poll it was taken at
        self.snapshots.append(self.poll)
        return w

    def eval_counts(self, lo, hi, w=None):
        hinge, correct, n2 = self.evals[int(w[0])]
        return hinge, correct, n2

    def stop_async(self): self.stopped = True


@pytest.mark.parametrize("case", ["converges", "max_steps", "no_check_before_max_steps"])
def test_master_async_loop_matches_the_literal_restatement(case):
    """A12: MasterAsync.fit's polling loop against oracle/scala_semantics.MasterAsyncLossChecker over one recorded stream:
    which polls compute (`updates - lastStep < minStepsBetweenChecks`), the leaky averages, the best-loss rule (strict >),
    the early stop and the `updates >= n * maxEpochs` stop, and what endComputation returns."""
    from types import SimpleNamespace
    from distributed_sgd_b200.core.master import MasterAsync
    from distributed_sgd_b200.ml import SparseSVM
    from distributed_sgd_b200.utils.dataset import Data
    dim, n_train, n_test, lam, leak, every = 6, 50, 20, 0.25, 0.7, 30
    rng = np.random.default_rng(3)
    if case == "converges":
        counter = np.cumsum(rng.integers(5, 25, size=200)).tolist()
        hinge = [int(h) for h in np.r_[np.linspace(36, 8, 60), np.full(140, 8)] + rng.integers(0, 2, size=200)]
        max_epoch = 1000
    elif case == "max_steps":
        counter = np.cumsum(rng.integers(5, 25, size=200)).tolist()
        hinge = [int(h) for h in np.linspace(38, 2, 200)]                          # keeps improving: only maxSteps ends it
        max_epoch = 20                                                              # 50 * 20 = 1000 updates
    else:
        counter = [5, 12, 2000]                                                    # maxSteps is hit before any check is due
        hinge = [20, 20, 20]
        max_epoch = 20
        every = 400
    evals = [(h, n_test - h // 2, 1.5 + 0.01 * i) for i, h in enumerate(hinge)]
    stub = lambda n: Data(np.arange(n + 1, dtype=np.int64), np.zeros(n, np.int32), np.ones(n, np.float32), np.ones(n, np.int8), dim)
    ctx = _AsyncScriptCtx(dim, counter, evals, n_test)
    slave = SimpleNamespace(ctx=ctx, world=1, is_async=True, n_train=n_train, n_test=n_test, dim=dim,
                            start_async=lambda *a, **k: None, stop_async=ctx.stop_async)
    m = MasterAsync(0, stub(n_train), stub(n_test), SparseSVM(lam), 1, slave=slave)
    crit = EarlyStopping.no_improvement(patience=3, min_delta=0.01)
    state = m.fit(np.zeros(dim), max_epoch=max_epoch, batch_size=1, learning_rate=0.5, stopping_criterion=crit,
                  check_every=every, leak_loss_coef=leak, poll_seconds=0.0)
    # the same stream through the literal restatement
    polls = [(u, lam * evals[i][2] + evals[i][0] / n_test, evals[i][1] / n_test, i) for i, u in enumerate(counter)]
    ref = S.MasterAsyncLossChecker(n_train, max_epoch, S.early_stopping_no_improvement(3, 0.01), every, leak).replay(polls)
    assert m.history["ended_by"] == ref["ended_by"] == {"converges": "converged", "max_steps": "max_steps",
                                                       "no_check_before_max_steps": "max_steps"}[case]
    assert m.history["checks_at"] == ref["computed_at"]
    assert m.history["test_losses"] == ref["test_losses"] and m.history["test_accs"] == ref["test_accs"]   # bit-equal floats
    assert ctx.stopped
    if ref["computed_at"]:
        assert state.loss == ref["best_loss"] and int(state.grad[0]) == ref["best_grad"]
        assert m.history["best_check"] == ref["computed_at"].index(counter[ref["best_grad"]])
    else:
        assert ref["best_grad"] == "Vec.zeros(1)"       # the reference would hand back its initial bestGrad; see master.py
    assert state.end is not None and state.updates == 1


def test_async_batch_draw_is_a_permutation():
    """The async worker draws a batch as the first B images of a keyed permutation of [0, n) (csrc/dsgd_feistel.h, the same
    source nvcc compiles into k_async_worker): every position once, whatever n and key -- `shuffle take batchSize`
    (core/Slave.scala:86-88) never repeats a sample inside a batch."""
    from distributed_sgd_b200.native import host_lib
    h = host_lib()
    for n, key in [(1, 5), (2, 1), (3, 77), (17, 123456789), (256, 2**63 + 11), (1000, 42), (4097, 7), (70000, 99)]:
        img = np.array([h.dsgd_feistel_pos(x, n, key) for x in range(n)], dtype=np.int64)
        assert img.min() == 0 and img.max() == n - 1 and len(np.unique(img)) == n, (n, key)
    # different keys give different orders; the first few images are not the identity
    a = [h.dsgd_feistel_pos(x, 560000, 1) for x in range(64)]
    b = [h.dsgd_feistel_pos(x, 560000, 2) for x in range(64)]
    assert a != b and a != list(range(64)) and len(set(a)) == 64
    # rough uniformity of the first image over keys
    first = np.array([h.dsgd_feistel_pos(0, 1000, k) for k in range(4000)])
    hist = np.bincount(first // 100, minlength=10)
    assert hist.min() > 300 and hist.max() < 500, hist
