"""surreal_b200 -- H100-native actor -> HBM replay -> PPO / DDPG learner hot path behind
SurrealAI/surreal's Agent / Replay / Learner plugin surface (see DESIGN.md)."""
__version__ = '0.1.0'
