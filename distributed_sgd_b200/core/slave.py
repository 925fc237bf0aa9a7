"""core/Slave.scala -- one worker.  Here: one GPU, one dsgd_ctx.

The reference Slave owns the whole training array and answers `forward` / `gradient` /
`startAsync` / `updateGrad` / `stopAsync` RPCs (core/Slave.scala:113-197).  This class keeps that
surface (same method names and argument meaning, snake_case) and hands every one of them to the CUDA
library through the C ABI; there is no arithmetic in this file.
"""
from __future__ import annotations

from typing import Optional, Sequence, Union

import numpy as np

from ..ml.calibration import IsotonicCalibration
from ..ml.class_weight import resolve_class_weight
from ..ml.sparse_logistic import SparseLogistic
from ..ml.sparse_margin import SparseModifiedHuber, SparseSquaredHinge, model_name
from ..ml.sparse_svm import SparseSVM
from ..native import NativeCtx
from ..utils.dataset import SAMPLE_WEIGHT_ASYNC, Data, Topics, has_sample_weights, sample_weights_of


def topics_of(data: Data, test_data: Optional[Data]) -> Optional[Topics]:
    """The topics of the train rows followed by the test rows, the layout of the device rows; None when no part carries
    any.  Both parts must carry topics with the same names, or neither."""
    parts = [data] if test_data is None else [data, test_data]
    if all(p.topics is None for p in parts):
        return None
    if any(p.topics is None for p in parts):
        raise ValueError("topics: the train and the test rows must both carry topics, or neither")
    if test_data is None:
        return data.topics
    a, b = data.topics, test_data.topics
    if a.names != b.names:
        raise ValueError("topics: the train and the test rows carry different topic names")
    return Topics(np.concatenate([a.ptr, b.ptr[1:] + a.ptr[-1]]), np.concatenate([a.ids, b.ids]), a.names)


class Slave:
    def __init__(self, node: int, master: int, data: Data, model: Union[SparseSVM, SparseLogistic, SparseSquaredHinge, SparseModifiedHuber],
                 is_async: bool = False, *,
                 world: int = 1, device: Optional[int] = None, test_data: Optional[Data] = None,
                 ctx: Optional[NativeCtx] = None):
        """`new Slave(node, master, data, model, async)` (core/Slave.scala:20; Main.scala:138,149).

        node = this worker's rank; master = the master's rank (kept for recognisability; the master logic
        runs SPMD on every rank).  `data` is the FULL training array, addressed by global row id (quirk
        Q13).  test_data (extension): rows appended after the training rows so the same device context can
        serve Master.localLoss(testData) -- they are never sampled.  ctx (extension): a device context that already
        holds exactly these rows (train rows followed by the test rows) and its dimSparsity.
        model: SparseSVM, or SparseLogistic, SparseSquaredHinge or SparseModifiedHuber (sync mode only).
        """
        name = model_name(model)
        if name != "svm" and is_async:
            raise ValueError(f"{type(model).__name__}: asynchronous (Hogwild) training supports SparseSVM only")
        if model.l1 and is_async:
            raise ValueError("l1: the L1 penalty is a step of sync training; asynchronous (Hogwild) training has none")
        self.intercept = bool(getattr(model, "fit_intercept", False))
        if self.intercept and is_async:
            raise ValueError("fit_intercept: the intercept is fitted by sync training; asynchronous (Hogwild) training has none")
        # (w_pos, w_neg) of the model's class_weight; "balanced" counts the labels of the train rows
        self.class_weight = resolve_class_weight(getattr(model, "class_weight", None), data.label)
        weighted = self.class_weight != (1.0, 1.0)
        if weighted and is_async:
            raise ValueError("class_weight: class weights belong to sync training; asynchronous (Hogwild) training has none")
        # per-row sample weights of the train and test rows (a part without them weighs 1 per row)
        self.sample_weighted = has_sample_weights(data, test_data)
        if self.sample_weighted and is_async:
            raise ValueError(SAMPLE_WEIGHT_ASYNC)
        # the topics of a multi-label set (one-vs-rest training, Master.local_topic_report), train rows then test rows
        self.topics = topics_of(data, test_data)
        if self.topics is not None and is_async:
            raise ValueError("topics: one-vs-rest training belongs to sync training; asynchronous (Hogwild) training has none")
        self.node, self.master, self.model, self.is_async, self.world = node, master, model, is_async, world
        self.n_train = data.n_rows
        self.n_test = test_data.n_rows if test_data is not None else 0
        self.dim = data.dim
        if ctx is not None:
            if ctx.n_rows != self.n_train + self.n_test or ctx.dim != data.dim:
                raise ValueError("Slave: the given device context does not hold these rows")
            if getattr(ctx, "model", "logistic" if getattr(ctx, "logistic", False) else "svm") != name:
                raise ValueError("Slave: the given device context was created for another model")
            if getattr(ctx, "intercept", False) != self.intercept:
                raise ValueError("Slave: the given device context does not match the model's fit_intercept")
            self.ctx = ctx
            if model.dim_sparsity is None:
                model.dim_sparsity = ctx.compute_dim_sparsity(self.n_train)
            if model.l1:
                ctx.set_l1(model.l1)
            if weighted:
                ctx.set_class_weights(*self.class_weight)
            if self.sample_weighted:
                ctx.set_sample_weights(sample_weights_of(data, test_data))
            if self.topics is not None:
                ctx.load_topics(self.topics.ptr, self.topics.ids, self.topics.n_topics)
            return
        self.ctx = NativeCtx(node if device is None else device, data.dim, model.lam, rank=node, world=world,
                             is_async=is_async, model=name, intercept=self.intercept)
        if test_data is not None:
            row_ptr = np.concatenate([data.row_ptr, test_data.row_ptr[1:] + data.row_ptr[-1]])
            col = np.concatenate([data.col[:data.nnz], test_data.col[:test_data.nnz]])
            val = np.concatenate([data.val[:data.nnz], test_data.val[:test_data.nnz]])
            label = np.concatenate([data.label, test_data.label])
            self.ctx.load_csr(row_ptr, col, val, label)
        else:
            self.ctx.load_csr(data.row_ptr, data.col, data.val, data.label)
        if model.dim_sparsity is None:
            model.dim_sparsity = self.ctx.compute_dim_sparsity(self.n_train)  # Main.scala:54-65 on the device
        else:
            self.ctx.set_dim_sparsity(model.dim_sparsity)
        if model.l1:
            self.ctx.set_l1(model.l1)
        if weighted:
            self.ctx.set_class_weights(*self.class_weight)
        if self.sample_weighted:
            self.ctx.set_sample_weights(sample_weights_of(data, test_data))
        if self.topics is not None:
            self.ctx.load_topics(self.topics.ptr, self.topics.ids, self.topics.n_topics)

    def stop(self):  # Slave.stop (core/Slave.scala:68-77): releases the device context
        self.ctx.close()

    # ---- SlaveImpl -----------------------------------------------------------------------------------
    def forward(self, samples_idx: Sequence[int], weights: Optional[np.ndarray] = None) -> np.ndarray:
        """SlaveImpl.forward (core/Slave.scala:129-140): predictions -signum(x.w) for the listed rows."""
        self._train_ids(samples_idx)
        return self.ctx.forward(samples_idx, weights)

    def margins(self, samples_idx: Sequence[int], weights: Optional[np.ndarray] = None) -> np.ndarray:
        """Extension: the margins x.w in fp64 of the listed rows (forward reports -signum of these)."""
        self._train_ids(samples_idx)
        return self.ctx.margins(samples_idx, weights)

    def topics_topk(self, samples_idx: Sequence[int], weights: np.ndarray, k: int):
        """Extension: (ids int32[n, k], margins float64[n, k]), the k highest-scored topics of each listed row under the
        [T, wdim] weights (score -x . w_t, ties to the lower t; NaN scores left out, -1 and NaN in their slots)."""
        self._train_ids(samples_idx)
        return self.ctx.topics_topk(samples_idx, weights, k)

    def probabilities(self, samples_idx: Sequence[int], weights: Optional[np.ndarray] = None) -> np.ndarray:
        """Extension, SparseLogistic and SparseModifiedHuber only (other models raise DsgdState): P(y = +1 | x) of the listed
        rows, sigmoid(-x.w) or (clip(-x.w, -1, 1) + 1) / 2."""
        self._train_ids(samples_idx)
        return self.ctx.probabilities(samples_idx, weights)

    def calibrated_probabilities(self, samples_idx: Sequence[int], calibration,
                                 weights: Optional[np.ndarray] = None) -> np.ndarray:
        """Extension, any model: P(y = +1 | x) of the listed rows under `calibration` (from Master.calibrate): a Calibration
        gives 1 / (1 + exp(a x.w + b)), an IsotonicCalibration numpy.interp(-x.w, x, y)."""
        self._train_ids(samples_idx)
        if isinstance(calibration, IsotonicCalibration):
            return self.ctx.isotonic_probabilities(samples_idx, calibration.x, calibration.y, weights)
        return self.ctx.calibrated_probabilities(samples_idx, calibration.a, calibration.b, weights)

    def gradient(self, weights: Optional[np.ndarray], samples_idx: Sequence[int]) -> np.ndarray:
        """SlaveImpl.gradient (core/Slave.scala:142-157): regularize(sum of backward over the batch)."""
        self._train_ids(samples_idx)
        return self.ctx.gradient(samples_idx, weights)

    def start_async(self, weights: np.ndarray, samples: Sequence[int], batch_size: int, learning_rate: float, *,
                    concurrency: int = 1, max_updates: int = 0, seed: int = 0):
        """SlaveImpl.startAsync (core/Slave.scala:159-175)."""
        self._train_ids(samples)
        self.ctx.start_async(weights, samples, batch_size, learning_rate, concurrency, max_updates, seed)

    def update_grad(self, grad_update):
        """SlaveImpl.updateGrad (core/Slave.scala:177-185): weights -= gradUpdate.  Accepts a dense vector or
        an (indices, values) pair."""
        if isinstance(grad_update, tuple):
            idx, val = grad_update
        else:
            dense = np.asarray(grad_update, dtype=np.float64)
            idx = np.flatnonzero(dense).astype(np.int32)
            val = dense[idx]
        self.ctx.update_grad(idx, val)

    def stop_async(self):
        """SlaveImpl.stopAsync (core/Slave.scala:187-195)."""
        self.ctx.stop_async()

    # ---- helpers ---------------------------------------------------------------------------------------
    def _train_ids(self, idx):
        idx = np.asarray(idx)
        if idx.size and (idx.min() < 0 or idx.max() >= self.n_train):
            raise IndexError("sample id outside the training rows")  # data(idx) on the reference's array
