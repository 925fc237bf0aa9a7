from . import early_stopping as EarlyStopping  # noqa: F401,N812
from . import split_strategy as SplitStrategy  # noqa: F401,N812
from .calibration import Calibration, IsotonicCalibration  # noqa: F401
from .grad_state import GradState  # noqa: F401
from .lr_schedule import learning_rates  # noqa: F401
from .one_vs_rest import OneVsRest  # noqa: F401
from .sparse_logistic import SparseLogistic  # noqa: F401
from .sparse_margin import SparseModifiedHuber, SparseSquaredHinge  # noqa: F401
from .sparse_svm import SparseSVM  # noqa: F401
