from .config import Config, load_config  # noqa: F401
from .dataset import Data, Topics, rcv1, synthetic_rcv1, synthetic_topics, write_rcv1  # noqa: F401
