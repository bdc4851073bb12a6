"""pearl_b200 — H100-native (sm_90a) learner hot path of facebookresearch/Pearl:
`ReplayBuffer.sample -> PolicyLearner.learn()` behind Pearl's own plugin API.

    from pearl_b200 import B200ReplayBuffer, B200DeepQLearning, B200DoubleDQN

Hand-written CUDA in libpearlb200.so (C ABI: include/pearl_b200.h), called through
ctypes; PyTorch only allocates memory and provides streams.  No CPU fallback.
"""
from ._compat import CNNQValueMultiHeadNetwork, CNNQValueNetwork  # noqa: F401
from ._compat import (HAVE_PEARL, DuelingQValueNetwork, OneHotActionTensorRepresentationModule, TransitionBatch,  # noqa: F401
                      VanillaQValueMultiHeadNetwork)
from .dqn import B200DeepQLearning, B200DeepSARSA, B200DoubleDQN, B200LearnerGroup  # noqa: F401
from .replay_buffer import B200ReplayBuffer  # noqa: F401
from .sarsa_buffer import B200SARSAReplayBuffer  # noqa: F401
from .per import B200PrioritizedReplayBuffer  # noqa: F401
from .her import B200HindsightExperienceReplayBuffer  # noqa: F401
from .ppo import gae_and_lambda_returns  # noqa: F401
# subclasses of the reference's ContinuousSoftActorCritic / SoftActorCritic / ProximalPolicyOptimization / TD3 / DDPG / TD3BC /
# ImplicitQLearning / QuantileRegressionDeepQLearning / REINFORCE when Pearl is importable, the stand-alone CUDA learners (same keyword arguments) otherwise
from .actor_critic import (B200ContinuousSoftActorCritic, B200DeepDeterministicPolicyGradient,  # noqa: F401
                           B200ImplicitQLearning, B200ProximalPolicyOptimization, B200QuantileRegressionDeepQLearning,
                           B200REINFORCE, B200SoftActorCritic, B200TD3, B200TD3BC)
from .bandit import B200LinearBandit  # noqa: F401
from .neural_linear import B200NeuralLinearBandit  # noqa: F401
from .neural_bandit import B200NeuralBandit  # noqa: F401
# a subclass of the reference's RCSafetyModuleCostCriticContinuousAction when Pearl is importable, stand-alone otherwise
from .rc_safety import B200RCSafetyModuleCostCriticContinuousAction  # noqa: F401
from ._compat import BinaryActionTensorRepresentationModule, UCBExploration  # noqa: F401
from ._compat import FastCBExploration, LossType, NoExploration, SquareCBExploration  # noqa: F401
from ._compat import ThompsonSamplingExplorationLinear  # noqa: F401
# subclasses of the reference's DisjointBanditContainer / DisjointLinearBandit when Pearl is importable
from .disjoint_bandit import B200DisjointBanditContainer, B200DisjointLinearBandit  # noqa: F401
from ._compat import DisjointUCBExploration, ThompsonSamplingExplorationLinearDisjoint  # noqa: F401
from .dist import B200Communicator, all_gather_bytes, shard_owner  # noqa: F401

__all__ = ["B200ReplayBuffer", "B200DeepQLearning", "B200DoubleDQN", "TransitionBatch",
           "OneHotActionTensorRepresentationModule", "HAVE_PEARL", "B200Communicator", "B200LearnerGroup", "B200PrioritizedReplayBuffer", "gae_and_lambda_returns", "B200ContinuousSoftActorCritic", "B200SoftActorCritic", "B200ProximalPolicyOptimization",
           "B200TD3", "B200DeepDeterministicPolicyGradient", "B200HindsightExperienceReplayBuffer", "B200ImplicitQLearning",
           "B200QuantileRegressionDeepQLearning", "B200REINFORCE", "DuelingQValueNetwork", "VanillaQValueMultiHeadNetwork",
           "B200DeepSARSA", "B200SARSAReplayBuffer", "B200TD3BC", "B200LinearBandit", "B200NeuralLinearBandit", "UCBExploration",
           "BinaryActionTensorRepresentationModule", "B200RCSafetyModuleCostCriticContinuousAction", "B200NeuralBandit",
           "SquareCBExploration", "FastCBExploration", "NoExploration", "LossType", "ThompsonSamplingExplorationLinear",
           "B200DisjointBanditContainer", "B200DisjointLinearBandit", "DisjointUCBExploration",
           "ThompsonSamplingExplorationLinearDisjoint", "CNNQValueNetwork", "CNNQValueMultiHeadNetwork"]
