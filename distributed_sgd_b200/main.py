"""Main.scala -- the reference's entry point, as a calling sequence over this package.

    python -m distributed_sgd_b200.main [--conf application.conf] [--synthetic-rows N]
    torchrun --nproc-per-node K -m distributed_sgd_b200.main ...

Mirrors `Main.scenario` (Main.scala:70-120): load the `dsgd` configuration (file and/or DSGD_* variables,
Main.scala:36), load the data (Main.scala:47-49; RCV1 text files from `data-path`, or RCV1-shaped synthetic rows when
`--synthetic-rows` is given because no RCV1 copy ships here), 80/20 split by position (:52), dimSparsity (:54-65, on
the device), model (:68), initial distributed loss / accuracy (:75-78), fit (:80-112), final test loss / accuracy
(:115-118).  One process per GPU; `node-count` reference workers are spread over the GPUs as logical workers
(node-count must be a multiple of the number of processes).  Prints one JSON report (the reference logs text).
"""
from __future__ import annotations

import argparse
import dataclasses
import json
import os
import time
from typing import Optional

import numpy as np


def scenario(cfg, data, *, rank: int = 0, world: int = 1, device: Optional[int] = None, seed: int = 0, log=print,
             async_concurrency: int = 64, jvm_exact: bool = False, inspect=None) -> dict:
    """Main.scenario (Main.scala:70-120).  inspect (tests): called as inspect("master", master) once the master exists
    and as inspect("done", (master, state)) before the device context is released."""
    from . import EarlyStopping, Master, Slave, SparseLogistic, SparseModifiedHuber, SparseSquaredHinge, SparseSVM
    from .core import Group

    if cfg.model != "svm" and cfg.is_async:
        raise ValueError(f"model = {cfg.model}: asynchronous (Hogwild) training supports the svm model only")
    if cfg.average_from >= 0 and cfg.is_async:
        raise ValueError("average-from: averaged SGD is a sync-mode option; asynchronous (Hogwild) training does not average")
    if cfg.learning_rate_decay != 0.0 and cfg.is_async:
        raise ValueError("learning-rate-decay: the decaying learning rate is a sync-mode option; asynchronous (Hogwild) "
                         "training keeps its constant rate")
    if cfg.l1 != 0.0 and cfg.is_async:
        raise ValueError("l1: the L1 penalty is a step of sync training; asynchronous (Hogwild) training has none")
    if cfg.fit_intercept and cfg.is_async:
        raise ValueError("fit-intercept: the intercept is fitted by sync training; asynchronous (Hogwild) training has none")
    from .ml.class_weight import parse_class_weight
    class_weight = parse_class_weight(cfg.class_weight)
    if class_weight is not None and cfg.is_async:
        raise ValueError("class-weight: class weights belong to sync training; asynchronous (Hogwild) training has none")
    from .utils.dataset import SAMPLE_WEIGHT_ASYNC, load_sample_weights
    if cfg.sample_weight and cfg.is_async:
        raise ValueError(SAMPLE_WEIGHT_ASYNC)
    if cfg.calibration_weighted and cfg.is_async:
        raise ValueError("calibration-weighted: row weights belong to sync training; an asynchronous (Hogwild) context "
                         "has none to calibrate by")
    if cfg.bootstrap_weighted and cfg.is_async:
        raise ValueError("bootstrap-weighted: row weights belong to sync training; an asynchronous (Hogwild) context "
                         "has none to resample by")
    from .ml.one_vs_rest import parse_topic_rank_k, parse_topic_thresholds, parse_topics
    topics = parse_topics(cfg.topics)
    if topics is not None and cfg.is_async:
        raise ValueError("topics: one-vs-rest training belongs to sync training; asynchronous (Hogwild) training has none")
    rank_k = parse_topic_rank_k(cfg.topic_rank_k, topics)
    thr_mode, thr_fbr = parse_topic_thresholds(cfg.topic_thresholds, cfg.topic_threshold_fbr, topics)
    if topics is None:   # the binary run alone, with the rows as they always were
        data = dataclasses.replace(data, topics=None)
    elif data.topics is None:
        raise ValueError("topics: the data carries no topics (RCV1 is read with them when the key is set; "
                         "--synthetic-topics N plants them on synthetic rows)")
    elif topics != "all":
        data = dataclasses.replace(data, topics=data.topics.select(topics))
    if rank_k and rank_k > data.topics.n_topics:
        raise ValueError(f"topic-rank-k: {rank_k} exceeds the {data.topics.n_topics} topics")
    if cfg.sample_weight:   # one weight per loaded row; the split below carries them
        data = dataclasses.replace(data, weight=load_sample_weights(cfg.sample_weight, data.n_rows))
    train, test = data.split_at(int(data.n_rows * 0.8))                       # Main.scala:52
    # Main.scala:67-68 ("could use another model"); dimSparsity: computed by the Slave on the device
    model_class = {"logistic": SparseLogistic, "squared_hinge": SparseSquaredHinge,
                   "modified_huber": SparseModifiedHuber}.get(cfg.model, SparseSVM)
    model = model_class(cfg.lam, l1=cfg.l1, class_weight=class_weight, fit_intercept=cfg.fit_intercept)
    slave = Slave(rank, 0, train, model, cfg.is_async, world=world, device=device, test_data=test)
    master = Master.create(rank, train, test, model, cfg.is_async, cfg.node_count, slave=slave, group=Group(), seed=seed,
                           log=(log if rank == 0 else None), jvm_exact=jvm_exact)
    if inspect:
        inspect("master", master)
    w0 = np.zeros(data.dim + (1 if cfg.fit_intercept else 0))                 # data(0)._1.zerosLike (Main.scala:74)
    report = {"config": {k: getattr(cfg, k) for k in ("batch_size", "learning_rate", "lam", "node_count", "is_async",
                                                      "max_epochs", "check_every", "leaky_loss", "patience", "conv_delta",
                                                      "model", "learning_rate_decay", "learning_rate_power", "l1",
                                                      "fit_intercept")},
              "rows": {"train": train.n_rows, "test": test.n_rows}, "world": world}
    report["initial_loss"] = master.distributed_loss(w0)                      # Main.scala:75-76
    report["initial_accuracy"] = master.distributed_accuracy(w0)              # Main.scala:77-78
    stop = EarlyStopping.no_improvement(patience=cfg.patience, min_delta=cfg.conv_delta, min_steps=None)
    t0 = time.perf_counter()
    if cfg.is_async:                                                          # Main.scala:82-96
        state = master.fit(w0, cfg.max_epochs, cfg.batch_size, cfg.learning_rate, stop, check_every=cfg.check_every,
                           leak_loss_coef=cfg.leaky_loss, concurrency=async_concurrency, seed=seed)
    else:                                                                      # Main.scala:97-109
        if cfg.node_count % world:
            raise ValueError(f"node-count {cfg.node_count} is not a multiple of the {world} GPU processes")
        state = master.fit(w0, cfg.max_epochs, cfg.batch_size, cfg.learning_rate, stop,
                           virtual_workers=cfg.node_count // world,
                           average_from=cfg.average_from if cfg.average_from >= 0 else None,
                           learning_rate_decay=cfg.learning_rate_decay, learning_rate_power=cfg.learning_rate_power)
    report["fit_seconds"] = time.perf_counter() - t0                          # Measure.durationLog(log, "fit") (Main.scala:80)
    w1 = state.grad
    report["history"] = {k: [float(x) for x in v] for k, v in getattr(master, "history", {}).items()
                         if isinstance(v, list) and all(isinstance(x, (int, float)) for x in v)}
    report["final_test_loss"], report["final_test_accuracy"] = master.local_loss_accuracy(w1, test_data=True)  # :115-118
    report["final_weights_nonzero"] = int(np.count_nonzero(w1[:data.dim]))
    if cfg.fit_intercept:
        report["intercept"] = float(w1[data.dim])   # the learned intercept, the last entry of the weights
        if rank == 0:
            log(f"intercept: {w1[data.dim]:.6g}")
    report["updates"] = state.updates
    if class_weight is not None:
        report["class_weight"] = list(slave.class_weight)   # as resolved over the train rows
        if rank == 0:
            log(f"class weights: w_pos = {slave.class_weight[0]:.6g}, w_neg = {slave.class_weight[1]:.6g}")
        report["test_class_report"] = cr = master.local_class_report(w1, test_data=True)
        if rank == 0:
            log(f"test rows by class: recall+ {cr['recall_pos']:.4f} ({cr['n_pos']} rows), recall- {cr['recall_neg']:.4f} "
                f"({cr['n_neg']} rows), balanced accuracy {cr['balanced_accuracy']:.4f}, weighted loss {cr['weighted_loss']:.6f}")
    if cfg.sample_weight:
        report["test_weighted_report"] = wr = master.local_weighted_report(w1, test_data=True)
        if rank == 0:
            log(f"sample weights: test weight sum {wr['weight_sum']:.6g} over {wr['n']} rows, weighted loss "
                f"{wr['weighted_loss']:.6f}, weighted accuracy {wr['weighted_accuracy']:.4f}")
    if "averaged_steps" in getattr(master, "history", {}):
        report["averaged_steps"] = int(master.history["averaged_steps"])   # the returned weights are their mean
    if cfg.calibrate and cfg.calibration_method == "isotonic":
        # an isotonic map fitted on the train rows, judged on the test rows
        wkw = {"weighted": True} if cfg.calibration_weighted else {}   # unweighted: the calls as they always were
        iso = master.calibrate(w1, method="isotonic", **wkw)
        q = master.local_calibration(iso, w1, test_data=True, **wkw)
        report["calibration"] = {"method": "isotonic", "blocks": iso.blocks, "points": iso.points,
                                 "distinct_scores": iso.distinct_scores, "test_brier": q["brier"],
                                 "test_log_loss": q["log_loss"], "test_ece": q["ece"],
                                 "test_infinite_log_loss_rows": q["infinite_log_loss_rows"]}
        if rank == 0:
            log(f"calibration (isotonic): {iso.blocks} blocks over {iso.distinct_scores} distinct train scores; "
                f"test Brier {q['brier']:.6f}, log loss {q['log_loss']:.6f}, ECE {q['ece']:.6f}")
    elif cfg.calibrate:
        # a Platt sigmoid fitted on the train rows, judged on the test rows; for the logistic model also against the
        # model's own probability, the identity link
        from .ml import Calibration
        wkw = {"weighted": True} if cfg.calibration_weighted else {}   # unweighted: the calls as they always were
        cal = master.calibrate(w1, **wkw)
        q = master.local_calibration(cal, w1, test_data=True, **wkw)
        report["calibration"] = {"method": "sigmoid", "a": cal.a, "b": cal.b, "iterations": cal.iterations, "status": cal.status,
                                 "test_brier": q["brier"], "test_log_loss": q["log_loss"], "test_ece": q["ece"]}
        if cfg.calibration_weighted:
            report["calibration"].update(weighted=True, weight_pos=cal.weight_pos, weight_neg=cal.weight_neg,
                                         test_weight=q["weight"])
        if cfg.model == "logistic":
            q0 = master.local_calibration(Calibration.identity(), w1, test_data=True)
            report["calibration"]["identity"] = {"test_brier": q0["brier"], "test_log_loss": q0["log_loss"],
                                                 "test_ece": q0["ece"]}
        if rank == 0:
            log(f"calibration: A = {cal.a:.6g}, B = {cal.b:.6g} ({cal.iterations} Newton iterations, status {cal.status}); "
                f"test Brier {q['brier']:.6f}, log loss {q['log_loss']:.6f}, ECE {q['ece']:.6f}"
                + (f"; identity link: Brier {q0['brier']:.6f}, log loss {q0['log_loss']:.6f}, ECE {q0['ece']:.6f}"
                   if cfg.model == "logistic" else ""))
    if cfg.bootstrap > 0:
        # Poisson-bootstrap 95 % intervals of the final test metrics (the replicates themselves are not reported)
        bkw = {"weighted": True} if cfg.bootstrap_weighted else {}   # unweighted: the calls as they always were
        bs = master.local_bootstrap(w1, test_data=True, n_boot=cfg.bootstrap, **bkw)
        report["test_bootstrap"] = {m: {k: v for k, v in r.items() if k != "replicates"} for m, r in bs.items()}
        report["test_bootstrap"]["replicates"] = cfg.bootstrap
        if cfg.bootstrap_weighted:
            report["test_bootstrap"]["weighted"] = True
        if rank == 0:
            log(f"bootstrap ({cfg.bootstrap} replicates, 95 %): " + ", ".join(
                f"{m} {bs[m]['estimate']:.4f} [{bs[m]['lo']:.4f}, {bs[m]['hi']:.4f}]" for m in ("auc", "ap", "accuracy", "loss")))
    if topics is not None:
        # one-vs-rest: every topic fitted with the settings of the binary run, then all judged on the test rows in one pass
        t1 = time.perf_counter()
        ovr = master.fit_one_vs_rest(w0, cfg.max_epochs, cfg.batch_size, cfg.learning_rate, stop,
                                     virtual_workers=cfg.node_count // world,
                                     average_from=cfg.average_from if cfg.average_from >= 0 else None,
                                     learning_rate_decay=cfg.learning_rate_decay,
                                     learning_rate_power=cfg.learning_rate_power)
        fit_s = time.perf_counter() - t1
        tr = master.local_topic_report(ovr, test_data=True)
        report["topic_report"] = {"topics": len(ovr.topics), "fit_seconds": fit_s,
                                  "epochs": [len(h["losses"]) for h in ovr.histories], **tr}
        if rank == 0:
            log(f"one-vs-rest ({len(ovr.topics)} topics, {fit_s:.1f} s): test micro F1 {tr['micro_f1']:.4f}, macro F1 "
                f"{tr['macro_f1']:.4f} over {tr['macro_f1_topics']} topics, subset accuracy {tr['subset_accuracy']:.4f}, "
                f"Hamming loss {tr['hamming_loss']:.5f}, top-1 accuracy {tr['top1_accuracy']:.4f}")
        if rank_k:
            rr = master.local_topic_ranking_report(ovr, rank_k, test_data=True)
            report["topic_ranking"] = rr
            if rank == 0:
                log(f"topic ranking (k = {rank_k}, {rr['ranked_rows']} ranked test rows): precision@{rank_k} "
                    f"{rr['precision_at'][rank_k]:.4f}, recall@{rank_k} {rr['recall_at'][rank_k]:.4f}, LRAP "
                    f"{rr['lrap']:.4f}, coverage error {rr['coverage_error']:.3f}, ranking loss {rr['ranking_loss']:.5f}")
        if thr_mode == "scut":
            # SCut: each topic's F1-optimal margin threshold on the train rows, then the test rows judged at them
            t1 = time.perf_counter()
            tuned, summary = master.tune_topic_thresholds(ovr, test_data=False, fbr=thr_fbr)
            tune_s = time.perf_counter() - t1
            tt = master.local_topic_report(tuned, test_data=True)
            report["topic_thresholds"] = {"mode": thr_mode, "fbr": thr_fbr, "tune_seconds": tune_s,
                                          "thresholds": [float(x) for x in tuned.thresholds], "tuning": summary, "test": tt}
            if rank == 0:
                log(f"topic thresholds (scut, fbr {thr_fbr}, {tune_s:.2f} s on the train rows): test micro F1 "
                    f"{tr['micro_f1']:.4f} -> {tt['micro_f1']:.4f}, macro F1 {tr['macro_f1']:.4f} -> {tt['macro_f1']:.4f}, "
                    f"subset accuracy {tr['subset_accuracy']:.4f} -> {tt['subset_accuracy']:.4f}, Hamming loss "
                    f"{tr['hamming_loss']:.5f} -> {tt['hamming_loss']:.5f}")
    if inspect:
        inspect("done", (master, state))
    slave.stop()
    return report


def main(argv=None) -> int:
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--conf", default=None, help="application.conf (HOCON `dsgd { }` block); DSGD_* variables override")
    ap.add_argument("--synthetic-rows", type=int, default=0, help="use RCV1-shaped synthetic rows instead of data-path")
    ap.add_argument("--synthetic-topics", type=int, default=0,
                    help="with --synthetic-rows: plant this many topics on the rows (utils.synthetic_topics) for `topics`")
    ap.add_argument("--seed", type=int, default=0)                            # Random.setSeed(0) (Main.scala:32)
    ap.add_argument("--jvm-exact", action="store_true",
                    help="sync mode: draw the batches from java.util.Random(seed) + Scala's Random.shuffle like the reference")
    args = ap.parse_args(argv)
    from .utils import load_config, rcv1, synthetic_rcv1, synthetic_topics

    rank = int(os.environ.get("RANK", "0"))
    world = int(os.environ.get("WORLD_SIZE", "1"))
    local_rank = int(os.environ.get("LOCAL_RANK", "0"))
    if world > 1:
        import torch.distributed as dist
        dist.init_process_group(backend="gloo", rank=rank, world_size=world)
    cfg = load_config(args.conf)
    from .ml.one_vs_rest import parse_topics
    if args.synthetic_rows:
        data = synthetic_rcv1(n_rows=args.synthetic_rows, seed=args.seed)
        if args.synthetic_topics:
            data = dataclasses.replace(data, topics=synthetic_topics(data, args.synthetic_topics, seed=args.seed))
    else:   # every qrels line is read only when one-vs-rest training asks for it
        data = rcv1(cfg.data_path, full=cfg.full, topics=parse_topics(cfg.topics) is not None)
    report = scenario(cfg, data, rank=rank, world=world, device=local_rank, seed=args.seed,
                      log=lambda s: print(s, flush=True), jvm_exact=args.jvm_exact)
    if rank == 0:
        print(json.dumps(report))
    if world > 1:
        import torch.distributed as dist
        dist.destroy_process_group()
    return 0


if __name__ == "__main__":
    raise SystemExit(main())
