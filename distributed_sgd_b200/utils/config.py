"""utils/Config.scala:3-21 + resources/application.conf:1-52 -- the `dsgd { ... }` parameter contract.

Same keys, same defaults, same DSGD_* environment overrides.  The reference resolves them with
pureconfig over HOCON; here a minimal reader handles the subset of HOCON that application.conf uses
(`key = value` lines inside `dsgd { }`, `${?ENV}` optional substitutions, `#` comments).
"""
from __future__ import annotations

import os
import re
from dataclasses import dataclass, fields
from typing import Dict, Optional


@dataclass
class Config:  # field order and names: utils/Config.scala:3-21 (kebab-case in the file)
    host: str = "127.0.0.1"
    port: int = 4000
    master_host: Optional[str] = None
    master_port: Optional[int] = None
    batch_size: int = 100
    learning_rate: float = 0.5
    lam: float = 0.00001          # `lambda`
    node_count: int = 3
    full: bool = False
    is_async: bool = False        # `async`
    record: bool = False
    data_path: str = "data"
    max_epochs: int = 10
    check_every: int = 100
    leaky_loss: float = 0.9
    conv_delta: float = 0.01
    patience: int = 5
    model: str = "svm"            # extension: "svm" (SparseSVM), or "logistic", "squared_hinge" or "modified_huber"
                                  # (SparseLogistic, SparseSquaredHinge, SparseModifiedHuber; sync mode only)
    average_from: int = -1        # extension: averaged SGD from this epoch (0-based) on, sync mode only; -1: off
    learning_rate_decay: float = 0.0   # extension: step t uses learning-rate / (1 + decay * t)^power, sync mode only
    learning_rate_power: float = 1.0   # extension: 0 decay is the reference's constant rate
    l1: float = 0.0               # extension: L1 penalty l1 * ||w||_1 (lasso; elastic net with lambda), sync mode only
    class_weight: str = "none"    # extension: none, balanced or w_pos,w_neg -- one weight per label, sync mode only
    calibrate: bool = False       # extension: after fit, fit a calibration on the train rows and report its test-set quality
    calibration_method: str = "sigmoid"   # extension: the calibration `calibrate` fits: sigmoid (Platt) or isotonic
    calibration_weighted: bool = False    # extension: `calibrate` fits and judges with every row counted by its weight
    sample_weight: str = ""       # extension: path of a .npy of one weight per loaded row (before the split), sync mode only
    fit_intercept: bool = False   # extension: fit an unregularised intercept (weights dim + 1 long), sync mode only
    bootstrap: int = 0            # extension: Poisson-bootstrap replicates of the final test metrics' intervals; 0: off
    bootstrap_weighted: bool = False   # extension: the bootstrap counts every row by its weight (class x sample weight)
    topics: str = ""              # extension: one-vs-rest training of a multi-label set after the binary run: empty (off),
                                  # all, or a comma-separated list of topic names; sync mode only
    topic_rank_k: int = 0         # extension: with `topics`, rank every test row's topics and report precision and recall at
                                  # 1..k, LRAP, coverage error and ranking loss; 0: off, else 1..32
    topic_thresholds: str = "none"   # extension: with `topics`, scut tunes every topic's F1-optimal margin threshold on the
                                     # train rows after the fit and reports the test topics at them; none: every threshold 0
    topic_threshold_fbr: float = 0.0   # extension: with scut, a topic whose best train F1 is below this keeps only its
                                       # top-scored rows (SCutFBR.1); in [0, 1], 0: off


# application.conf key -> (Config field, DSGD_* variable)   (resources/application.conf:2-50)
_KEYS = {
    "data-path": ("data_path", "DSGD_DATA_PATH"), "host": ("host", "DSGD_NODE_HOST"), "port": ("port", "DSGD_NODE_PORT"),
    "master-host": ("master_host", "DSGD_MASTER_HOST"), "master-port": ("master_port", "DSGD_MASTER_PORT"),
    "batch-size": ("batch_size", "DSGD_BATCH_SIZE"), "learning-rate": ("learning_rate", "DSGD_LEARNING_RATE"),
    "lambda": ("lam", "DSGD_LAMBDA"), "full": ("full", "DSGD_FULL"), "node-count": ("node_count", "DSGD_NODE_COUNT"),
    "async": ("is_async", "DSGD_ASYNC"), "record": ("record", "DSGD_RECORD"), "max-epochs": ("max_epochs", "DSGD_MAX_EPOCHS"),
    "check-every": ("check_every", "DSGD_CHECK_EVERY"), "leaky-loss": ("leaky_loss", "DSGD_LEAKY_LOSS"),
    "patience": ("patience", "DSGD_PATIENCE"), "conv-delta": ("conv_delta", "DSGD_CONV_DELTA"),
    "model": ("model", "DSGD_MODEL"), "average-from": ("average_from", "DSGD_AVERAGE_FROM"),
    "learning-rate-decay": ("learning_rate_decay", "DSGD_LEARNING_RATE_DECAY"),
    "learning-rate-power": ("learning_rate_power", "DSGD_LEARNING_RATE_POWER"),
    "l1": ("l1", "DSGD_L1"), "class-weight": ("class_weight", "DSGD_CLASS_WEIGHT"), "calibrate": ("calibrate", "DSGD_CALIBRATE"),
    "calibration-method": ("calibration_method", "DSGD_CALIBRATION_METHOD"),
    "calibration-weighted": ("calibration_weighted", "DSGD_CALIBRATION_WEIGHTED"),
    "sample-weight": ("sample_weight", "DSGD_SAMPLE_WEIGHT"),
    "fit-intercept": ("fit_intercept", "DSGD_FIT_INTERCEPT"),
    "bootstrap": ("bootstrap", "DSGD_BOOTSTRAP"),
    "bootstrap-weighted": ("bootstrap_weighted", "DSGD_BOOTSTRAP_WEIGHTED"),
    "topics": ("topics", "DSGD_TOPICS"),
    "topic-rank-k": ("topic_rank_k", "DSGD_TOPIC_RANK_K"),
    "topic-thresholds": ("topic_thresholds", "DSGD_TOPIC_THRESHOLDS"),
    "topic-threshold-fbr": ("topic_threshold_fbr", "DSGD_TOPIC_THRESHOLD_FBR"),
}
MODELS = ("svm", "logistic", "squared_hinge", "modified_huber")
_TYPES = {f.name: f.type for f in fields(Config)}


def _coerce(field: str, raw: str):
    raw = raw.strip().strip('"')
    t = str(_TYPES[field])
    if "bool" in t:
        if raw.lower() in ("true", "yes", "on"):
            return True
        if raw.lower() in ("false", "no", "off"):
            return False
        raise ValueError(f"{field}: expected a boolean, got {raw!r}")
    if "int" in t:
        return int(raw)
    if "float" in t:
        return float(raw)
    return raw


def _parse_block(text: str, env: Dict[str, str]) -> Dict[str, str]:
    """Returns key -> raw value for the `dsgd { }` block; later assignments win, `${?X}` only if X is set."""
    m = re.search(r"\bdsgd\s*\{", text)
    if not m:
        return {}
    depth, i = 1, m.end()
    while i < len(text) and depth:
        depth += {"{": 1, "}": -1}.get(text[i], 0)
        i += 1
    out: Dict[str, str] = {}
    for line in text[m.end():i - 1].splitlines():
        line = line.split("#", 1)[0].strip()
        if not line or "=" not in line:
            continue
        key, raw = (s.strip() for s in line.split("=", 1))
        sub = re.fullmatch(r"\$\{\?(\w+)\}", raw)
        if sub:
            if sub.group(1) in env:
                out[key] = env[sub.group(1)]
            continue
        out[key] = raw
    return out


def load_config(path: Optional[str] = None, env: Optional[Dict[str, str]] = None) -> Config:
    """`pureconfig.loadConfigOrThrow[Config]("dsgd")` (Main.scala:36).  Without a file the defaults of
    resources/application.conf apply; DSGD_* variables override either."""
    env = dict(os.environ if env is None else env)
    cfg = Config()
    raw: Dict[str, str] = {}
    if path is not None:
        with open(path) as f:
            raw = _parse_block(f.read(), env)
    else:
        for key, (_, var) in _KEYS.items():
            if var in env:
                raw[key] = env[var]
    for key, value in raw.items():
        if key not in _KEYS:
            raise KeyError(f"unknown key dsgd.{key}")
        field = _KEYS[key][0]
        setattr(cfg, field, _coerce(field, value))
    if cfg.model not in MODELS:
        raise ValueError(f"model: expected one of {', '.join(MODELS)}, got {cfg.model!r}")
    if cfg.average_from < -1:
        raise ValueError(f"average-from: expected an epoch >= 0, or -1 for off, got {cfg.average_from}")
    if not cfg.learning_rate_decay >= 0.0:
        raise ValueError(f"learning-rate-decay: expected a value >= 0, got {cfg.learning_rate_decay}")
    if not cfg.learning_rate_power > 0.0:
        raise ValueError(f"learning-rate-power: expected a value > 0, got {cfg.learning_rate_power}")
    if not (cfg.l1 >= 0.0 and cfg.l1 != float("inf")):
        raise ValueError(f"l1: expected a finite value >= 0, got {cfg.l1}")
    from ..ml.class_weight import parse_class_weight
    parse_class_weight(cfg.class_weight)   # raises on a malformed value
    from ..ml.calibration import METHODS as CALIBRATION_METHODS
    if cfg.calibration_method not in CALIBRATION_METHODS:
        raise ValueError(f"calibration-method: expected one of {', '.join(CALIBRATION_METHODS)}, "
                         f"got {cfg.calibration_method!r}")
    if cfg.bootstrap < 0:
        raise ValueError(f"bootstrap: expected a number of replicates >= 0 (0: off), got {cfg.bootstrap}")
    if cfg.sample_weight and not cfg.sample_weight.endswith(".npy"):
        raise ValueError(f"sample-weight: expected the path of a .npy file, or empty for off, got {cfg.sample_weight!r}")
    from ..ml.one_vs_rest import parse_topic_rank_k, parse_topic_thresholds, parse_topics
    topics = parse_topics(cfg.topics)
    parse_topic_rank_k(cfg.topic_rank_k, topics)   # raises on a malformed value of any of these
    parse_topic_thresholds(cfg.topic_thresholds, cfg.topic_threshold_fbr, topics)
    return cfg
