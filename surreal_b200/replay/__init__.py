from .base import Replay  # noqa: F401
from .fifo_replay import FIFOReplay  # noqa: F401
from .uniform_replay import UniformReplay, PyRandomStream  # noqa: F401
from .prioritized_replay import PrioritizedReplay  # noqa: F401
