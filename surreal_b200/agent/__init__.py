from .base import Agent, AGENT_MODES  # noqa: F401
from .ppo_agent import PPOAgent  # noqa: F401
from .ddpg_agent import DDPGAgent  # noqa: F401
from .q_agent import QAgent  # noqa: F401
