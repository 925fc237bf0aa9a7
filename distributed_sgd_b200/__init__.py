"""distributed_sgd_b200 -- H100-native data-parallel SGD hot path behind the surface of
zifeo/distributed-sgd's Slave / Master / SparseSVM (see DESIGN.md, INTEGRATION.md, include/dsgd.h).

(The directory is named with an underscore because `distributed-sgd_b200` is not an importable
Python package name.)
"""
from . import native  # noqa: F401
from .core import Master, MasterAsync, MasterSync, Slave  # noqa: F401
from .ml import (EarlyStopping, GradState, SparseLogistic, SparseModifiedHuber, SparseSquaredHinge, SparseSVM,  # noqa: F401
                 SplitStrategy)
from .utils import Config, Data, load_config, rcv1, synthetic_rcv1  # noqa: F401

__all__ = ["native", "Master", "MasterAsync", "MasterSync", "Slave", "EarlyStopping", "GradState", "SparseLogistic",
           "SparseModifiedHuber", "SparseSquaredHinge", "SparseSVM", "SplitStrategy", "Config", "Data", "load_config", "rcv1", "synthetic_rcv1"]
