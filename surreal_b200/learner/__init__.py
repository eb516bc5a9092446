from .base import Learner  # noqa: F401
from .ppo import PPOLearner  # noqa: F401
from .aggregator import SSARAggregator, MultistepAggregatorWithInfo  # noqa: F401
from .ddpg import DDPGLearner  # noqa: F401
from .dqn import DQNLearner  # noqa: F401
