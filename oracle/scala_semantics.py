"""TEST INFRASTRUCTURE ONLY -- literal, map-based restatement of the reference's Scala arithmetic.

This file is the *semantic anchor* of the oracle: it mirrors the reference's immutable
`Map[Int, Number]` vectors one operation at a time (same filters, same fold order, same
scalar short-cuts), in pure Python floats (IEEE binary64 == what spire.math.Number holds
on this path, SURVEY.md 2.3).  It is slow by construction and is only run on small cases:
  * it is pinned against the only known answers the reference's own tests hold for this
    path (VecTests.scala:12-41, see tests/test_oracle_known_answers.py), and
  * the fast array-based C oracle (oracle/dsgd_oracle.c) is validated against it on
    random small problems (tests/test_oracle_c_vs_literal.py).

Nothing under distributed_sgd_b200/ may import this module (the product path must never
route through the oracle).  PARITY STATUS: "parity unpinned" for SparseSVM / Slave /
Master (the reference has zero tests there, SURVEY.md 8c); pinned only for the L0 vector
algebra by VecTests.

Citations are path:line under src/main/scala/epfl/distributed/ of the reference.
"""
from __future__ import annotations

import math
from typing import Callable, Dict, Iterable, List, Optional, Sequence, Tuple

EPSILON = 1e-20  # math/Sparse.scala:104


class Sparse:
    """math/Sparse.scala:5 + math/Vec.scala:8-85 -- immutable sparse vector.

    `map` never holds an entry with abs(v) <= 1e-20 (constructor filter,
    math/Sparse.scala:108-118); missing keys read as 0 (withDefaultValue).
    """

    __slots__ = ("map", "size")

    def __init__(self, m: Dict[int, float], size: int):
        if len(m) > size:  # math/Sparse.scala:109
            raise ValueError("The sparse vector contains more elements than its defined size")
        for v in m.values():  # math/Vec.scala:14 (NaN guard; `== NaN` is always false on the JVM, kept as a no-op)
            pass
        self.map = {k: float(v) for k, v in m.items() if abs(v) > EPSILON}
        self.size = size

    # -- construction helpers -------------------------------------------------
    @staticmethod
    def zeros(size: int) -> "Sparse":  # math/Sparse.scala:125
        return Sparse({}, size)

    def zeros_like(self) -> "Sparse":  # math/Vec.scala:60-63
        return Sparse.zeros(self.size)

    def get(self, idx: int) -> float:
        return self.map.get(idx, 0.0)

    def apply(self, idx: int) -> float:  # math/Sparse.scala:61-68 (note: idx == size is legal, quirk Q11)
        if idx < 0 or idx > self.size:
            raise IndexError(f"Illegal index '{idx}'")
        return self.get(idx)

    # -- element-wise machinery -----------------------------------------------
    def _elementwise(self, other: "Sparse", op: Callable[[float, float], float],
                     zero_if_one_arg_zero: bool = False) -> "Sparse":
        # math/Sparse.scala:15-41
        if other.size != self.size:
            raise ValueError("Can't perform element-wise operation on vectors of different length")
        if zero_if_one_arg_zero:
            if len(self.map) < len(other.map):  # iterate the smaller map (Sparse.scala:21-25)
                return Sparse({i: op(v, other.get(i)) for i, v in self.map.items()}, self.size)
            return Sparse({i: op(self.get(i), v) for i, v in other.map.items()}, self.size)
        keys = set(self.map) | set(other.map)  # Sparse.scala:33
        return Sparse({i: op(self.get(i), other.get(i)) for i in keys}, self.size)

    def map_values(self, op: Callable[[float], float]) -> "Sparse":
        # math/Sparse.scala:48-57.  The dense branch (default value changes) is unreachable on
        # the hot path (only * and / by non-zero scalars are used, both keep 0 -> 0).
        if abs(op(0.0)) <= EPSILON:
            return Sparse({i: op(v) for i, v in self.map.items()}, self.size)
        raise NotImplementedError("mapValues that moves the default value densifies; off the hot path")

    def __add__(self, other):  # math/Vec.scala:32,34
        if isinstance(other, Sparse):
            return self._elementwise(other, lambda a, b: a + b)
        return self if other == 0 else self.map_values(lambda v: v + other)

    def __sub__(self, other):  # math/Vec.scala:36,38
        if isinstance(other, Sparse):
            return self._elementwise(other, lambda a, b: a - b)
        return self if other == 0 else self.map_values(lambda v: v - other)

    def __mul__(self, other):  # math/Sparse.scala:46 (vec) ; math/Vec.scala:42 (scalar)
        if isinstance(other, Sparse):
            return self._elementwise(other, lambda a, b: a * b, zero_if_one_arg_zero=True)
        return self.zeros_like() if other == 0 else self.map_values(lambda v: v * other)

    __rmul__ = __mul__  # math/Vec.scala:89-106 (RichNumber / RichInt / RichDouble)

    def __truediv__(self, scalar):  # math/Vec.scala:46-47
        if scalar == 0:
            raise ValueError("Division by zero")  # IllegalArgumentException in the reference
        return self.map_values(lambda v: v / scalar)

    # -- reductions -----------------------------------------------------------
    def sum(self) -> float:  # math/Vec.scala:53  (fold in map order; order is not reproducible, see SURVEY 2.3)
        s = 0.0
        for v in self.map.values():
            s = s + v
        return s

    def norm_squared(self) -> float:  # math/Vec.scala:55
        s = 0.0
        for v in self.map.values():
            s = s + v ** 2
        return s

    def norm(self) -> float:  # math/Vec.scala:56
        return math.sqrt(self.norm_squared())

    def dot(self, other: "Sparse") -> float:  # math/Vec.scala:58
        return (self * other).sum()

    def value_like(self, value: float) -> "Sparse":  # math/Vec.scala:65-75
        if value == 0:
            return self.zeros_like()
        return Sparse({i: value for i in self.map}, self.size)

    def non_zero_count(self, epsilon: float = 1e-20) -> int:  # math/Sparse.scala:83-92
        if abs(epsilon) >= EPSILON:
            return len(self.map)
        return sum(1 for v in self.map.values() if abs(v) > epsilon)

    def sparsity(self, epsilon: float = 1e-20) -> float:  # math/Vec.scala:79
        return 1 - self.non_zero_count(epsilon) / self.size

    def __eq__(self, other):  # math/Sparse.scala:96-99
        return isinstance(other, Sparse) and other.size == self.size and other.map == self.map

    def __repr__(self):
        return f"Sparse({dict(sorted(self.map.items()))}, {self.size})"

    def to_dense(self) -> List[float]:
        return [self.get(i) for i in range(self.size + 1)]  # +1: key == size is legal (Q11)


def vec_sum(vecs: Sequence[Sparse]) -> Sparse:  # math/Vec.scala:128-131
    if len(vecs) == 0:
        raise ValueError("Cannot sum an empty list of vectors")  # quirk Q7
    acc = vecs[0]
    for v in vecs[1:]:
        acc = acc + v
    return acc


def vec_mean(vecs: Sequence[Sparse]) -> Sparse:  # math/Vec.scala:139
    return vec_sum(vecs) / len(vecs)


def signum(x: float) -> float:
    return (x > 0) - (x < 0)


Sample = Tuple[Sparse, int]


class SparseSVM:
    """core/ml/SparseSVM.scala:11-33."""

    def __init__(self, lam: float, dim_sparsity: Sparse):
        self.lam = lam
        self.dim_sparsity = dim_sparsity

    def forward(self, w: Sparse, x: Sparse) -> float:  # SparseSVM.scala:14
        return signum(x.dot(w)) * -1.0

    def loss_pred(self, pred: float, y: int) -> float:  # SparseSVM.scala:16
        return max(0.0, 1.0 - y * pred)

    def loss_sample(self, w: Sparse, x: Sparse, y: int) -> float:  # SparseSVM.scala:18
        return self.loss_pred(self.forward(w, x), y)

    def loss(self, w: Sparse, samples: Sequence[Sample]) -> float:  # SparseSVM.scala:20-23
        total = None
        for x, y in samples:  # reduce(_ + _): left fold without a zero element
            l = self.loss_sample(w, x, y)
            total = l if total is None else total + l
        return self.lam * w.norm_squared() + total / len(samples)

    def backward(self, w: Sparse, x: Sparse, y: int) -> Sparse:  # SparseSVM.scala:26-29
        activity = y * x.dot(w)
        return w.zeros_like() if activity < 0 else x * y

    def regularize(self, grad: Sparse, w: Sparse) -> Sparse:  # SparseSVM.scala:31
        return grad + grad.value_like(self.lam * 2.0 * w.dot(self.dim_sparsity))


def slave_gradient(model: SparseSVM, data: Sequence[Sample], w: Sparse, samples_idx: Sequence[int]) -> Sparse:
    """core/Slave.scala:142-157 -- SUM over the batch, then regularize."""
    grads = [model.backward(w, data[i][0], data[i][1]) for i in samples_idx]
    return model.regularize(vec_sum(grads), w)


def slave_forward(model: SparseSVM, data: Sequence[Sample], w: Sparse, samples_idx: Sequence[int]) -> List[float]:
    """core/Slave.scala:129-140."""
    return [model.forward(w, data[i][0]) for i in samples_idx]


def master_sync_step(model: SparseSVM, data: Sequence[Sample], w: Sparse,
                     batches: Sequence[Sequence[int]], lr: float) -> Sparse:
    """core/Master.scala:184-197 -- K gradient requests, MEAN over workers, SGD update.

    `batches[k]` is what the reference obtains from shuffling worker k's index range and
    slicing (Master.scala:184-187); the draw itself is an input at the boundary (SURVEY H6).
    """
    res = [slave_gradient(model, data, w, b) for b in batches]
    grad = vec_mean(res)  # Master.scala:194
    return w - lr * grad  # Master.scala:197


def async_worker_delta(model: SparseSVM, data: Sequence[Sample], w_snapshot: Sparse,
                       samples_idx: Sequence[int], lr: float) -> Sparse:
    """core/Slave.scala:92-99 -- MEAN over the batch, regularize against the snapshot, scale by lr."""
    grads = [model.backward(w_snapshot, data[i][0], data[i][1]) for i in samples_idx]
    return lr * model.regularize(vec_mean(grads), w_snapshot)


def local_accuracy(model: SparseSVM, w: Sparse, data: Sequence[Sample]) -> float:
    """core/Master.scala:100-103."""
    return sum(1 for x, y in data if model.forward(w, x) == y) / len(data)


def local_loss(model: SparseSVM, w: Sparse, data: Sequence[Sample]) -> float:
    """core/Master.scala:105-107."""
    return model.loss(w, data)


def dim_sparsity(train: Sequence[Sample]) -> Sparse:
    """Main.scala:54-65 -- inverse (document frequency + 1), keys shifted by -1 (quirk Q3).

    Feature ids in `train` are the reference's 1-based RCV1 keys.
    """
    dim = train[0][0].size
    buff = [0.0] * dim
    for v, _ in train:
        for idx in v.map.keys():
            buff[idx - 1] += 1
    inv = {i: 1.0 / (c + 1) for i, c in enumerate(buff) if c != 0}
    return Sparse(inv, dim)


def split_vanilla(n: int, n_slaves: int) -> List[List[int]]:
    """core/ml/SplitStrategy.scala:13-14 -- `indices.grouped(ceil(n / K))`."""
    size = int(math.ceil(n / float(n_slaves)))
    return [list(range(s, min(s + size, n))) for s in range(0, n, size)]


def early_stopping_target(target: float) -> Callable[[Sequence[float]], bool]:
    """core/ml/EarlyStopping.scala:11."""
    return lambda losses: (len(losses) > 0) and (losses[0] <= target)


def early_stopping_no_improvement(patience: int = 5, min_delta: float = 1e-3,
                                  min_steps: Optional[int] = None) -> Callable[[Sequence[float]], bool]:
    """core/ml/EarlyStopping.scala:13-46 -- `losses` is newest-first."""
    abs_min_delta = abs(min_delta)

    def find_min(seq):  # EarlyStopping.scala:18-28
        mn, idx_min = 1.7976931348623157e308, -1
        for index, num in enumerate(seq):
            if (num - mn) <= abs_min_delta:
                mn, idx_min = num, index
        return mn, idx_min

    def check(losses):  # EarlyStopping.scala:30-42
        _, idx_min = find_min(losses)
        if idx_min == 0:
            return False
        return idx_min >= patience

    def crit(losses):  # EarlyStopping.scala:44
        if len(losses) == 0:
            return False
        if min_steps is None:
            return check(losses)
        return False if min_steps < len(losses) else check(losses)

    return crit


class MasterAsyncLossChecker:
    """core/MasterAsync.scala:66-177, the master side of an async run, replayed over a RECORDED stream.

    The reference interleaves two activities on shared state: `updateGrad` (one call per delta a slave sends, :164-177) and
    the polling task `startLossChecking.loop` (:96-162).  What the loop sees is fully described by the sequence of its
    polls: at each poll the update counter `innerGradState.updates` and -- if it decides to compute -- the test loss and test
    accuracy of `innerGradState.grad`.  `replay(polls)` restates the loop over such a sequence:
      polls: iterable of (updates, test_loss, test_acc, weights_tag); test_loss / test_acc are only read when the loop
             computes at that poll (pass None otherwise); weights_tag identifies the weight snapshot of the poll.
    and returns the lists the reference would have built plus the state `endComputation` hands back.
    """

    def __init__(self, n_data: int, max_epochs: int, stopping_criterion: Callable[[Sequence[float]], bool],
                 min_steps_between_checks: int, leak_coef: float):
        if not (0 <= leak_coef <= 1):  # :97
            raise ValueError("leaking coefficient must be between 0 and 1")
        self.max_steps = n_data * max_epochs  # initState, :83
        self.stop = stopping_criterion
        self.min_steps = min_steps_between_checks
        self.leak = leak_coef

    def replay(self, polls: Iterable[Tuple[int, Optional[float], Optional[float], object]]) -> dict:
        best_loss = 1.7976931348623157e308  # Number(Double.MaxValue), :69
        best_grad: object = "Vec.zeros(1)"  # :68
        last_step = -self.min_steps  # loop(-minStepsBetweenChecks, ...), :161
        test_losses: List[float] = []  # newest first, like the Scala lists
        test_accs: List[float] = []
        computed_at: List[int] = []
        ended_by = None
        for updates, loss_t, acc_t, tag in polls:
            if updates >= self.max_steps:  # updateGrad reached maxSteps before this poll: endComputation, :171-174
                ended_by = "max_steps"
                break
            if updates - last_step < self.min_steps:  # :110 "Latest step was too close"
                continue
            # :116-125 (only the test-set numbers are live code)
            loss_s = self.leak * loss_t + (1 - self.leak) * (test_losses[0] if test_losses else loss_t)
            acc_s = self.leak * acc_t + (1 - self.leak) * (test_accs[0] if test_accs else acc_t)
            if best_loss > loss_s:  # :132-139  `case oldLoss if oldLoss > lossTest => lossTest`
                best_loss, best_grad = loss_s, tag
            test_losses.insert(0, loss_s)  # :142-145
            test_accs.insert(0, acc_s)
            computed_at.append(updates)
            if self.stop(test_losses):  # :147
                ended_by = "converged"
                break
            last_step = updates  # loop(innerGradState.updates, ...), :156
        return {"test_losses": test_losses, "test_accs": test_accs, "computed_at": computed_at, "best_loss": best_loss,
                "best_grad": best_grad, "ended_by": ended_by}
