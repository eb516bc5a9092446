from .synthetic import SyntheticEnv, SyntheticPixelEnv, DiscreteSyntheticEnv  # noqa: F401
from .classic import CartPoleEnv, PendulumEnv, make_classic_env  # noqa: F401
from .exp_sender_wrapper import (ExpSenderWrapperMultiStepMovingWindowWithInfo,  # noqa: F401
                                 ExpSenderWrapperSSARNStepBootstrap)
