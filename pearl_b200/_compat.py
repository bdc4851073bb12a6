"""Base classes for the drop-in plugins.

When facebookresearch/Pearl is importable, `B200ReplayBuffer` subclasses
`pearl.replay_buffers.replay_buffer.ReplayBuffer` and the learners subclass
`pearl...DeepQLearning` / `DoubleDQN`, so `pearl.pearl_agent.PearlAgent` accepts
them unchanged.  When it is not installed (e.g. the GPU test box) equivalent
stand-alone bases with the same attribute names are used; the CUDA path is
identical in both cases.  Nothing here computes anything.
"""
from __future__ import annotations

from abc import ABC, abstractmethod
from dataclasses import dataclass, fields
from typing import Any, Optional

import torch
from torch import nn

try:  # pragma: no cover - depends on the environment
    from pearl.action_representation_modules.one_hot_action_representation_module import (
        OneHotActionTensorRepresentationModule,
    )
    from pearl.policy_learners.sequential_decision_making.deep_q_learning import (
        DeepQLearning as _RefDeepQLearning,
    )
    from pearl.neural_networks.sequential_decision_making.q_value_networks import DuelingQValueNetwork
    from pearl.neural_networks.sequential_decision_making.q_value_networks import VanillaQValueMultiHeadNetwork
    from pearl.neural_networks.sequential_decision_making.q_value_networks import CNNQValueMultiHeadNetwork, CNNQValueNetwork
    from pearl.policy_learners.sequential_decision_making.double_dqn import DoubleDQN as _RefDoubleDQN
    from pearl.policy_learners.sequential_decision_making.deep_sarsa import DeepSARSA as _RefDeepSARSA
    from pearl.policy_learners.exploration_modules.common.epsilon_greedy_exploration import EGreedyExploration
    from pearl.replay_buffers.replay_buffer import ReplayBuffer
    from pearl.replay_buffers.transition import TransitionBatch

    HAVE_PEARL = True
except Exception:  # ModuleNotFoundError (pearl or gymnasium missing)
    HAVE_PEARL = False

    class ReplayBuffer(ABC):  # mirrors pearl/replay_buffers/replay_buffer.py:18-91
        def __init__(self) -> None:
            super().__init__()
            self._is_action_continuous: bool = False
            self._has_cost_available: bool = False

        @property
        @abstractmethod
        def device_for_batches(self) -> torch.device: ...

        @abstractmethod
        def push(self, state, action, reward, terminated, truncated, curr_available_actions=None,
                 next_state=None, next_available_actions=None, max_number_actions=None,
                 cost=None) -> None: ...

        @abstractmethod
        def sample(self, batch_size: int): ...

        @abstractmethod
        def clear(self) -> None: ...

        @abstractmethod
        def __len__(self) -> int: ...

        @property
        def is_action_continuous(self) -> bool:
            return self._is_action_continuous

        @is_action_continuous.setter
        def is_action_continuous(self, value: bool) -> None:
            self._is_action_continuous = value

    @dataclass
    class TransitionBatch:  # field names of pearl/replay_buffers/transition.py:89-130
        state: torch.Tensor
        action: torch.Tensor
        reward: torch.Tensor
        terminated: Optional[torch.Tensor] = None
        truncated: Optional[torch.Tensor] = None
        next_state: Optional[torch.Tensor] = None
        next_action: Optional[torch.Tensor] = None
        curr_available_actions: Optional[torch.Tensor] = None
        curr_unavailable_actions_mask: Optional[torch.Tensor] = None
        next_available_actions: Optional[torch.Tensor] = None
        next_unavailable_actions_mask: Optional[torch.Tensor] = None
        weight: Optional[torch.Tensor] = None
        time_diff: Optional[torch.Tensor] = None
        cost: Optional[torch.Tensor] = None

        def __post_init__(self) -> None:
            n = self.reward.shape[0]
            if self.terminated is None:
                self.terminated = torch.ones(n, dtype=torch.bool, device=self.reward.device)
            if self.truncated is None:
                self.truncated = torch.zeros(n, dtype=torch.bool, device=self.reward.device)

        def to(self, device):
            for f in fields(self):
                v = getattr(self, f.name)
                if v is not None:
                    setattr(self, f.name, torch.as_tensor(v, device=device))
            return self

        @property
        def device(self) -> torch.device:
            return self.state.device

        def __len__(self) -> int:
            return self.reward.shape[0]

    class OneHotActionTensorRepresentationModule(nn.Module):
        def __init__(self, max_number_actions: int) -> None:
            super().__init__()
            self._max_number_actions = max_number_actions

        def forward(self, x: torch.Tensor) -> torch.Tensor:
            if x.dim() == 1:
                x = x.unsqueeze(-1)
            return torch.nn.functional.one_hot(x.long(), self._max_number_actions).squeeze(-2).float()

        @property
        def max_number_actions(self) -> int:
            return self._max_number_actions

        @property
        def representation_dim(self) -> int:
            return self._max_number_actions

    class _QNet(nn.Module):
        """Same module tree (hence state_dict keys) as VanillaQValueNetwork built by
        mlp_block: `_model.{i}.0` = Linear (pearl/neural_networks/common/utils.py:75-152)."""

        def __init__(self, state_dim: int, action_dim: int, hidden_dims, output_dim: int = 1) -> None:
            super().__init__()
            dims = [state_dim + action_dim] + list(hidden_dims) + [output_dim]
            layers = [nn.Sequential(nn.Linear(dims[i], dims[i + 1]), nn.ReLU()) for i in range(len(dims) - 2)]
            layers.append(nn.Sequential(nn.Linear(dims[-2], dims[-1])))
            self._model = nn.Sequential(*layers)
            self._state_dim, self._action_dim = state_dim, action_dim

    class _ValueMLP(nn.Module):
        """Same module tree as VanillaValueNetwork: `_model` = mlp_block (Linear+ReLU per hidden layer, then Linear)."""

        def __init__(self, input_dim: int, hidden_dims, output_dim: int) -> None:
            super().__init__()
            self._model = _QNet(input_dim, 0, hidden_dims, output_dim)._model

    class DuelingQValueNetwork(nn.Module):
        """Same constructor, module tree and state_dict keys as DuelingQValueNetwork
        (pearl/neural_networks/sequential_decision_making/q_value_networks.py:352-400): `{state,value,advantage}_arch`."""

        def __init__(self, state_dim: int, action_dim: int, hidden_dims, output_dim: int = 1, value_hidden_dims=None,
                     advantage_hidden_dims=None, state_hidden_dims=None) -> None:
            super().__init__()
            self._state_dim, self._action_dim = state_dim, action_dim
            F = hidden_dims[-1]
            self.state_arch = _ValueMLP(state_dim, hidden_dims if state_hidden_dims is None else state_hidden_dims, F)
            self.value_arch = _ValueMLP(F, hidden_dims if value_hidden_dims is None else value_hidden_dims, output_dim)
            self.advantage_arch = _ValueMLP(F + action_dim, hidden_dims if advantage_hidden_dims is None else advantage_hidden_dims,
                                            output_dim)

        @property
        def state_dim(self) -> int:
            return self._state_dim

        @property
        def action_dim(self) -> int:
            return self._action_dim

    class VanillaQValueMultiHeadNetwork(nn.Module):
        """Same constructor, module tree and state_dict keys as VanillaQValueMultiHeadNetwork
        (pearl/neural_networks/sequential_decision_making/q_value_networks.py:185-241): `_model` = mlp_block(state_dim,
        hidden_dims, output_dim), one Q value per action; `use_layer_norm` puts a LayerNorm after each hidden Linear, as
        mlp_block does."""

        def __init__(self, state_dim: int, action_dim: int, hidden_dims, output_dim: int, use_layer_norm: bool = False) -> None:
            super().__init__()
            self._state_dim, self._action_dim, self._output_dim = state_dim, action_dim, output_dim
            dims = [state_dim] + list(hidden_dims) + [output_dim]
            blocks = [nn.Sequential(*([nn.Linear(dims[i], dims[i + 1])] + ([nn.LayerNorm(dims[i + 1])] if use_layer_norm else [])
                                      + [nn.ReLU()])) for i in range(len(dims) - 2)]
            blocks.append(nn.Sequential(nn.Linear(dims[-2], dims[-1])))
            self._model = nn.Sequential(*blocks)

        def forward(self, x: torch.Tensor) -> torch.Tensor:
            return self._model(x)

        @property
        def state_dim(self) -> int:
            return self._state_dim

        @property
        def action_dim(self) -> int:
            return self._action_dim

    class _CNNQBase(nn.Module):
        """Same constructor, module tree and state_dict keys as CNNQValueNetwork / CNNQValueMultiHeadNetwork
        (pearl/neural_networks/sequential_decision_making/q_value_networks.py:713-917): `_model_cnn` = conv_block (Conv2d
        then ReLU per layer, BatchNorm2d after the Conv2d with use_batch_norm_conv), `_model_fc` = mlp_block on the
        flattened conv output (plus the one-hot action for CNNQValueNetwork)."""
        _with_action = True

        def __init__(self, input_width: int, input_height: int, input_channels_count: int, kernel_sizes, output_channels_list,
                     strides, paddings, action_dim: int, hidden_dims_fully_connected=None, output_dim: int = 1,
                     use_batch_norm_conv: bool = False, use_batch_norm_fully_connected: bool = False) -> None:
            super().__init__()
            self._input_channels, self._input_height, self._input_width = input_channels_count, input_height, input_width
            self._output_channels, self._kernel_sizes = output_channels_list, kernel_sizes
            self._strides, self._paddings = strides, paddings
            self._hidden_dims_fully_connected = [] if hidden_dims_fully_connected is None else hidden_dims_fully_connected
            self._use_batch_norm_conv = use_batch_norm_conv
            self._use_batch_norm_fully_connected = use_batch_norm_fully_connected
            self._output_dim = output_dim
            layers, c, h, w = [], input_channels_count, input_height, input_width
            for oc, k, s, p in zip(output_channels_list, kernel_sizes, strides, paddings):
                layers.append(nn.Conv2d(c, oc, k, stride=s, padding=p))
                if use_batch_norm_conv:
                    layers.append(nn.BatchNorm2d(oc))
                layers.append(nn.ReLU())
                c = oc
                h, w = (h + 2 * p - k) // s + 1, (w + 2 * p - k) // s + 1
            self._model_cnn = nn.Sequential(*layers)
            self._mlp_input_dims = c * h * w + (action_dim if self._with_action else 0)
            dims = [self._mlp_input_dims] + list(self._hidden_dims_fully_connected) + [output_dim]
            blocks = [nn.Sequential(*([nn.Linear(dims[i], dims[i + 1]), nn.ReLU()]
                                      + ([nn.BatchNorm1d(dims[i + 1])] if use_batch_norm_fully_connected else [])))
                      for i in range(len(dims) - 2)]
            blocks.append(nn.Sequential(nn.Linear(dims[-2], dims[-1])))
            self._model_fc = nn.Sequential(*blocks)
            self._state_dim = input_channels_count * input_height * input_width
            self._action_dim = action_dim

        @property
        def state_dim(self) -> int:
            return self._state_dim

        @property
        def action_dim(self) -> int:
            return self._action_dim

    class CNNQValueNetwork(_CNNQBase):
        _with_action = True

    class CNNQValueMultiHeadNetwork(_CNNQBase):
        _with_action = False

    class _RefDeepQLearning(nn.Module):
        """Attribute-compatible stand-in for DeepQLearning's constructor
        (deep_q_learning.py:40-59, deep_td_learning.py:60-185)."""

        def __init__(self, action_space=None, hidden_dims=None, exploration_module=None,
                     learning_rate: float = 0.001, discount_factor: float = 0.99,
                     training_rounds: int = 10, batch_size: int = 128, target_update_freq: int = 10,
                     soft_update_tau: float = 0.75, is_conservative: bool = False,
                     conservative_alpha: Optional[float] = 2.0, state_dim: Optional[int] = None,
                     network_type=None, action_representation_module=None, network_instance=None,
                     optimizer=None, **kwargs: Any) -> None:
            super().__init__()
            import copy
            assert state_dim is not None and hidden_dims is not None
            assert action_representation_module is not None
            self._action_space = action_space
            self._training_rounds, self._batch_size = training_rounds, batch_size
            self._training_steps = 0
            self._learning_rate, self._discount_factor = learning_rate, discount_factor
            self._target_update_freq, self._soft_update_tau = target_update_freq, soft_update_tau
            self._is_conservative, self._conservative_alpha = is_conservative, conservative_alpha
            self._is_action_continuous = False
            self.on_policy = False
            self.exploration_module = exploration_module
            self._action_representation_module = action_representation_module
            A = action_representation_module.representation_dim
            if network_instance is not None:
                self._Q = network_instance
            elif network_type is DuelingQValueNetwork:   # deep_td_learning.py make_specified_network
                self._Q = DuelingQValueNetwork(state_dim=state_dim, action_dim=A, hidden_dims=hidden_dims, output_dim=1)
            elif network_type is VanillaQValueMultiHeadNetwork:
                self._Q = VanillaQValueMultiHeadNetwork(state_dim=state_dim, action_dim=A, hidden_dims=hidden_dims,
                                                        output_dim=action_representation_module.max_number_actions)
            else:
                self._Q = _QNet(state_dim, A, hidden_dims)
            self._Q_target = copy.deepcopy(self._Q)
            self._optimizer = optimizer if optimizer is not None else torch.optim.AdamW(
                self._Q.parameters(), lr=learning_rate, amsgrad=True)

        @property
        def action_representation_module(self):
            return self._action_representation_module

        @property
        def requires_tensors(self) -> bool:
            return True

        @property
        def batch_size(self) -> int:
            return self._batch_size

        @property
        def optimizer(self):
            return self._optimizer

        def set_history_summarization_module(self, value) -> None:
            self._history_summarization_module = value

        def reset(self, action_space) -> None:
            self._action_space = action_space

    class _RefDoubleDQN(_RefDeepQLearning):
        pass

    class EGreedyExploration:
        """Attribute-compatible stand-in for EGreedyExploration (exploration_modules/common/epsilon_greedy_exploration.py):
        with probability `curr_epsilon` a uniformly drawn action of the space, else the greedy one."""

        def __init__(self, epsilon: float) -> None:
            self.curr_epsilon = epsilon

        def act(self, subjective_state, action_space, exploit_action, values=None, action_availability_mask=None,
                representation=None):
            import random
            if random.random() < self.curr_epsilon:
                return action_space.actions[random.randrange(action_space.n)]
            return exploit_action

    class _RefDeepSARSA(_RefDeepQLearning):
        """Attribute-compatible stand-in for DeepSARSA's constructor (deep_sarsa.py:35-56): on-policy, and
        EGreedyExploration(0.05) unless an exploration module is given, and DeepTDLearning's own defaults (100 training
        rounds, soft_update_tau 0.1) where DeepQLearning sets others."""

        def __init__(self, state_dim=None, action_space=None, exploration_module=None, action_representation_module=None,
                     optimizer=None, **kwargs: Any) -> None:
            kwargs.setdefault("training_rounds", 100)
            kwargs.setdefault("soft_update_tau", 0.1)
            super().__init__(state_dim=state_dim, action_space=action_space,
                             exploration_module=exploration_module if exploration_module is not None else EGreedyExploration(0.05),
                             action_representation_module=action_representation_module, optimizer=optimizer, **kwargs)
            self.on_policy = True


try:  # pragma: no cover - depends on the environment; kept apart so the names above do not depend on it
    from pearl.action_representation_modules.binary_action_representation_module import (
        BinaryActionTensorRepresentationModule,
    )
    from pearl.action_representation_modules.identity_action_representation_module import (
        IdentityActionRepresentationModule,
    )
    from pearl.policy_learners.contextual_bandits.linear_bandit import LinearBandit as _RefLinearBandit
    from pearl.policy_learners.contextual_bandits.neural_linear_bandit import NeuralLinearBandit as _RefNeuralLinearBandit
    from pearl.policy_learners.contextual_bandits.neural_bandit import NeuralBandit as _RefNeuralBandit
    from pearl.policy_learners.exploration_modules.common.no_exploration import NoExploration
    from pearl.policy_learners.exploration_modules.contextual_bandits.squarecb_exploration import (
        FastCBExploration, SquareCBExploration,
    )
    from pearl.neural_networks.common.utils import LossType
    from pearl.policy_learners.exploration_modules.common.tiebreaking_strategy import TiebreakingStrategy
    from pearl.policy_learners.exploration_modules.contextual_bandits.ucb_exploration import (
        DisjointUCBExploration, UCBExploration,
    )
    from pearl.policy_learners.exploration_modules.contextual_bandits.thompson_sampling_exploration import (
        ThompsonSamplingExplorationLinear, ThompsonSamplingExplorationLinearDisjoint,
    )
    from pearl.policy_learners.contextual_bandits.disjoint_bandit import (
        DisjointBanditContainer as _RefDisjointBanditContainer,
    )
    from pearl.policy_learners.contextual_bandits.disjoint_linear_bandit import (
        DisjointLinearBandit as _RefDisjointLinearBandit,
    )

    HAVE_PEARL_BANDITS = True
except Exception:  # ModuleNotFoundError (pearl or gymnasium missing)
    HAVE_PEARL_BANDITS = False


if not HAVE_PEARL_BANDITS:
    from enum import Enum

    class TiebreakingStrategy(Enum):  # exploration_modules/common/tiebreaking_strategy.py
        NO_TIEBREAKING = 0
        PER_ROW_TIEBREAKING = 1
        BATCH_TIEBREAKING = 2

    class UCBExploration:
        """Attribute-compatible stand-in for UCBExploration (exploration_modules/contextual_bandits/ucb_exploration.py):
        scores = values + alpha * sigma."""

        def __init__(self, alpha: float, randomized_tiebreaking: TiebreakingStrategy = TiebreakingStrategy.NO_TIEBREAKING) -> None:
            self._alpha = alpha
            self.randomized_tiebreaking = randomized_tiebreaking

    class ThompsonSamplingExplorationLinear:
        """Attribute-compatible stand-in for ThompsonSamplingExplorationLinear (exploration_modules/contextual_bandits/
        thompson_sampling_exploration.py): scores from coefficients sampled from N(coefs, (A + lambda I)^-1), or with
        enable_efficient_sampling one normal draw per score around mu with sigma as its deviation."""

        def __init__(self, enable_efficient_sampling: bool = False, randomized_tiebreaking: bool = False) -> None:
            self._enable_efficient_sampling = enable_efficient_sampling
            self.randomized_tiebreaking = randomized_tiebreaking

    class DisjointUCBExploration(UCBExploration):
        """Stand-in for DisjointUCBExploration (ucb_exploration.py:122-155): UCB with one model per arm."""

    class ThompsonSamplingExplorationLinearDisjoint(ThompsonSamplingExplorationLinear):
        """Stand-in for the disjoint explorer (thompson_sampling_exploration.py:106-142): one coefficient draw per arm's
        model.  The disjoint CUDA learners use it; the single-ridge learners refuse it."""

        def __init__(self, enable_efficient_sampling: bool = False) -> None:
            super().__init__(enable_efficient_sampling=enable_efficient_sampling)

    class IdentityActionRepresentationModule(nn.Module):
        def __init__(self, max_number_actions: int = -1, representation_dim: int = -1) -> None:
            super().__init__()
            self._max_number_actions, self._representation_dim = max_number_actions, representation_dim

        def forward(self, x: torch.Tensor) -> torch.Tensor:
            return x

        @property
        def max_number_actions(self) -> int:
            return self._max_number_actions

        @property
        def representation_dim(self) -> int:
            return self._representation_dim

    class BinaryActionTensorRepresentationModule(nn.Module):
        """Same as binary_action_representation_module.py: bit p of the action id at column p."""

        def __init__(self, bits_num: int) -> None:
            super().__init__()
            self._bits_num = bits_num
            self._max_number_actions = 2 ** bits_num

        def forward(self, x: torch.Tensor) -> torch.Tensor:
            if x.dim() == 1:
                x = x.unsqueeze(-1)
            mask = 2 ** torch.arange(self._bits_num, device=x.device)
            return x.bitwise_and(mask).ne(0).to(torch.float32)

        @property
        def max_number_actions(self) -> int:
            return self._max_number_actions

        @property
        def representation_dim(self) -> int:
            return self._bits_num

    class _LinearRegression(nn.Module):
        """Same constructor, buffers and state_dict keys as LinearRegression
        (neural_networks/contextual_bandit/linear_regression.py:20-87)."""

        def __init__(self, feature_dim: int, l2_reg_lambda: float = 1.0, gamma: float = 1.0, force_pinv: bool = False,
                     initial_coefs: Optional[torch.Tensor] = None) -> None:
            super().__init__()
            assert 0 < gamma <= 1, f"gamma should be in (0, 1]. Got gamma={gamma} instead"
            self._feature_dim = feature_dim
            self.gamma, self.l2_reg_lambda, self.force_pinv = gamma, l2_reg_lambda, force_pinv
            d = feature_dim + 1
            self.register_buffer("_A", torch.zeros(d, d))
            self.register_buffer("_b", torch.zeros(d))
            self.register_buffer("_sum_weight", torch.zeros(1))
            self.register_buffer("_inv_A", torch.zeros(d, d))
            if initial_coefs is not None:
                assert initial_coefs.shape == (d,), f"initial_coefs shape {initial_coefs.shape} != {(d,)}"
                self.register_buffer("_coefs", initial_coefs.clone())
            else:
                self.register_buffer("_coefs", torch.zeros(d))

    class _RefLinearBandit(nn.Module):
        """Attribute-compatible stand-in for LinearBandit's constructor (policy_learners/contextual_bandits/linear_bandit.py:
        93-121 on top of ContextualBanditBase / PolicyLearner): same arguments, defaults and state_dict keys."""

        def __init__(self, feature_dim: int, exploration_module=None, l2_reg_lambda: float = 1.0, gamma: float = 1.0,
                     apply_discounting_interval: float = 0.0, force_pinv: bool = False, training_rounds: int = 100,
                     batch_size: int = 128, action_representation_module=None, initial_coefs=None) -> None:
            super().__init__()
            self.exploration_module = exploration_module
            self.action_representation_module = (action_representation_module if action_representation_module is not None
                                                 else IdentityActionRepresentationModule())
            self._history_summarization_module = None
            self._training_rounds, self._batch_size, self._training_steps = training_rounds, batch_size, 0
            self.on_policy, self._is_action_continuous = False, False
            self._feature_dim = feature_dim
            self.model = _LinearRegression(feature_dim=feature_dim, l2_reg_lambda=l2_reg_lambda, gamma=gamma, force_pinv=force_pinv,
                                           initial_coefs=initial_coefs)
            self.apply_discounting_interval = apply_discounting_interval
            self.last_sum_weight_when_discounted = 0.0

        @property
        def feature_dim(self) -> int:
            return self._feature_dim

        @property
        def batch_size(self) -> int:
            return self._batch_size

        def set_history_summarization_module(self, value) -> None:
            self._history_summarization_module = value

        def reset(self, action_space) -> None:
            pass

    class _RefDisjointBanditContainer(nn.Module):
        """Attribute-compatible stand-in for DisjointBanditContainer's constructor (policy_learners/contextual_bandits/
        disjoint_bandit.py:44-65): same arguments and state_dict keys (`_arm_bandits.{i}.model._A`, ...)."""

        def __init__(self, feature_dim: int, arm_bandits, exploration_module, training_rounds: int = 100,
                     batch_size: int = 128) -> None:
            super().__init__()
            self.exploration_module = exploration_module
            self.action_representation_module = IdentityActionRepresentationModule()
            self._history_summarization_module = None
            self._training_rounds, self._batch_size, self._training_steps = training_rounds, batch_size, 0
            self.on_policy, self._is_action_continuous = False, False
            self._feature_dim = feature_dim
            self._arm_bandits = nn.ModuleList(arm_bandits)
            self._n_arms = len(arm_bandits)
            self._null_batch = None

        @property
        def n_arms(self) -> int:
            return self._n_arms

        @property
        def models(self):
            return [bandit.model for bandit in self._arm_bandits]

        @property
        def feature_dim(self) -> int:
            return self._feature_dim

        @property
        def batch_size(self) -> int:
            return self._batch_size

        def set_history_summarization_module(self, value) -> None:
            self._history_summarization_module = value

        def reset(self, action_space) -> None:
            pass

    class _RefDisjointLinearBandit(nn.Module):
        """Attribute-compatible stand-in for DisjointLinearBandit's constructor (policy_learners/contextual_bandits/
        disjoint_linear_bandit.py:41-67): same arguments and state_dict keys (`_linear_regressions.{i}._A`, ...)."""

        def __init__(self, feature_dim: int, action_space, exploration_module, l2_reg_lambda: float = 1.0,
                     training_rounds: int = 100, batch_size: int = 128, state_features_only: bool = False) -> None:
            super().__init__()
            self.exploration_module = exploration_module
            self.action_representation_module = IdentityActionRepresentationModule()
            self._history_summarization_module = None
            self._training_rounds, self._batch_size, self._training_steps = training_rounds, batch_size, 0
            self.on_policy, self._is_action_continuous = False, False
            self._feature_dim = feature_dim
            self._linear_regressions_list = [_LinearRegression(feature_dim=feature_dim, l2_reg_lambda=l2_reg_lambda)
                                             for _ in range(action_space.n)]
            self._linear_regressions = nn.ModuleList(self._linear_regressions_list)
            self._discrete_action_space = action_space
            self._state_features_only = state_features_only

        @property
        def feature_dim(self) -> int:
            return self._feature_dim

        @property
        def batch_size(self) -> int:
            return self._batch_size

        def set_history_summarization_module(self, value) -> None:
            self._history_summarization_module = value

        def reset(self, action_space) -> None:
            pass

    class LossType(Enum):  # neural_networks/common/utils.py
        MSE = "mse"
        MAE = "mae"
        CROSS_ENTROPY = "cross_entropy"

    class ResidualWrapper(nn.Module):  # neural_networks/common/residual_wrapper.py: x + module(x)
        def __init__(self, module: nn.Module) -> None:
            super().__init__()
            self.module = module

        def forward(self, x: torch.Tensor) -> torch.Tensor:
            return x + self.module(x)

    class _ValueNetwork(nn.Module):
        """Same module tree as VanillaValueNetwork over mlp_block with ReLU hidden layers and no normalization or dropout
        (neural_networks/common/utils.py mlp_block): `_model.{i}.0` = Linear, or `_model.{i}.module.0` when a layer of
        equal in / out width is wrapped in a ResidualWrapper."""

        def __init__(self, input_dim: int, hidden_dims, output_dim: int, use_skip_connections: bool = False) -> None:
            super().__init__()
            dims = [input_dim] + list(hidden_dims) + [output_dim]
            layers = []
            for i in range(len(dims) - 1):
                block = nn.Sequential(*([nn.Linear(dims[i], dims[i + 1])] + ([nn.ReLU()] if i < len(dims) - 2 else [])))
                layers.append(ResidualWrapper(block) if use_skip_connections and dims[i] == dims[i + 1] else block)
            self._model = nn.Sequential(*layers)

        def forward(self, x: torch.Tensor) -> torch.Tensor:
            return self._model(x)

    class _NeuralLinearRegression(nn.Module):
        """Same module tree and state_dict keys as NeuralLinearRegression (neural_networks/contextual_bandit/
        neural_linear_regression.py): `_nn_layers`, `_linear_regression_layer`, `output_activation`, `linear_layer_e2e`."""

        def __init__(self, feature_dim: int, hidden_dims, l2_reg_lambda_linear: float = 1.0, gamma: float = 1.0,
                     force_pinv: bool = False, output_activation_name: str = "linear", use_skip_connections: bool = True,
                     nn_e2e: bool = True) -> None:
            super().__init__()
            self._feature_dim = feature_dim
            self._nn_layers = _ValueNetwork(feature_dim, hidden_dims, hidden_dims[-1], use_skip_connections)
            self._linear_regression_layer = _LinearRegression(feature_dim=hidden_dims[-1], l2_reg_lambda=l2_reg_lambda_linear,
                                                              gamma=gamma, force_pinv=force_pinv)
            self.output_activation = {"linear": nn.Identity, "sigmoid": nn.Sigmoid}[output_activation_name]()
            self.linear_layer_e2e = nn.Linear(in_features=hidden_dims[-1], out_features=1, bias=False)
            self.nn_e2e = nn_e2e

    class _RefNeuralLinearBandit(nn.Module):
        """Attribute-compatible stand-in for NeuralLinearBandit's constructor (policy_learners/contextual_bandits/
        neural_linear_bandit.py on top of ContextualBanditBase / PolicyLearner): same arguments, defaults and state_dict
        keys, for the configurations the CUDA learner runs (ReLU hidden layers, no normalization or dropout)."""

        def __init__(self, feature_dim: int, hidden_dims, exploration_module=None, action_representation_module=None,
                     training_rounds: int = 100, batch_size: int = 128, learning_rate: float = 0.0003,
                     l2_reg_lambda_linear: float = 1.0, gamma: float = 1.0, apply_discounting_interval: float = 0.0,
                     force_pinv: bool = False, state_features_only: bool = True, loss_type=LossType.MSE,
                     output_activation_name: str = "linear", use_batch_norm: bool = False, use_layer_norm: bool = False,
                     hidden_activation: str = "relu", last_activation=None, dropout_ratio: float = 0.0,
                     use_skip_connections: bool = False, nn_e2e: bool = True, separate_uncertainty: bool = False) -> None:
            super().__init__()
            assert len(hidden_dims) >= 1
            self.exploration_module = exploration_module
            self.action_representation_module = (action_representation_module if action_representation_module is not None
                                                 else IdentityActionRepresentationModule())
            self._history_summarization_module = None
            self._training_rounds, self._batch_size, self._training_steps = training_rounds, batch_size, 0
            self.on_policy, self._is_action_continuous = False, False
            self._feature_dim = feature_dim
            self.model = _NeuralLinearRegression(feature_dim=feature_dim, hidden_dims=hidden_dims,
                                                 l2_reg_lambda_linear=l2_reg_lambda_linear, gamma=gamma, force_pinv=force_pinv,
                                                 output_activation_name=output_activation_name,
                                                 use_skip_connections=use_skip_connections, nn_e2e=nn_e2e)
            self._optimizer = torch.optim.AdamW(self.model.parameters(), lr=learning_rate, amsgrad=True)
            self._state_features_only = state_features_only
            self.loss_type = LossType(loss_type) if isinstance(loss_type, str) else loss_type
            self.apply_discounting_interval = apply_discounting_interval
            self.last_sum_weight_when_discounted = 0.0
            self.separate_uncertainty = separate_uncertainty

        @property
        def feature_dim(self) -> int:
            return self._feature_dim

        @property
        def batch_size(self) -> int:
            return self._batch_size

        @property
        def optimizer(self):
            return self._optimizer

        def set_history_summarization_module(self, value) -> None:
            self._optimizer.add_param_group({"params": value.parameters()})
            self._history_summarization_module = value

        def reset(self, action_space) -> None:
            pass

    class SquareCBExploration:
        """Attribute-compatible stand-in for SquareCBExploration (exploration_modules/contextual_bandits/
        squarecb_exploration.py): the constructor and the attributes the CUDA learner reads."""

        def __init__(self, gamma: float, reward_lb: float = 0.0, reward_ub: float = 1.0, clamp_values: bool = False,
                     randomized_tiebreaking: bool = False) -> None:
            self._gamma = gamma
            self.reward_lb = reward_lb
            self.reward_ub = reward_ub
            self.clamp_values = clamp_values
            self.randomized_tiebreaking = randomized_tiebreaking

    class FastCBExploration(SquareCBExploration):
        """Stand-in for FastCBExploration: SquareCB's attributes with clamping always on."""

        def __init__(self, gamma: float, reward_lb: float = 0.0, reward_ub: float = 1.0) -> None:
            super().__init__(gamma=gamma, reward_lb=reward_lb, reward_ub=reward_ub, clamp_values=True)

    class NoExploration:
        """Stand-in for NoExploration (exploration_modules/common/no_exploration.py): the first maximum of the values."""

        def __init__(self, randomized_tiebreaking: bool = False) -> None:
            self.randomized_tiebreaking = randomized_tiebreaking

    class _RefNeuralBandit(nn.Module):
        """Attribute-compatible stand-in for NeuralBandit's constructor (policy_learners/contextual_bandits/neural_bandit.py
        on top of ContextualBanditBase / PolicyLearner): same arguments, defaults and state_dict keys
        (`model._model.{0,1,2}.0.{weight,bias}`, VanillaValueNetwork's mlp_block)."""

        def __init__(self, feature_dim: int, hidden_dims, exploration_module, output_dim: int = 1, training_rounds: int = 100,
                     batch_size: int = 128, learning_rate: float = 0.001, state_features_only: bool = False,
                     loss_type=LossType.MSE, action_representation_module=None) -> None:
            super().__init__()
            self.exploration_module = exploration_module
            self.action_representation_module = (action_representation_module if action_representation_module is not None
                                                 else IdentityActionRepresentationModule())
            self._history_summarization_module = None
            self._training_rounds, self._batch_size, self._training_steps = training_rounds, batch_size, 0
            self.on_policy, self._is_action_continuous = False, False
            self._feature_dim = feature_dim
            self.model = _ValueNetwork(feature_dim, hidden_dims, output_dim)
            self._optimizer = torch.optim.AdamW(self.model.parameters(), lr=learning_rate, amsgrad=True)
            self._state_features_only = state_features_only
            self.loss_type = LossType(loss_type) if isinstance(loss_type, str) else loss_type

        @property
        def feature_dim(self) -> int:
            return self._feature_dim

        @property
        def batch_size(self) -> int:
            return self._batch_size

        @property
        def optimizer(self):
            return self._optimizer

        def set_history_summarization_module(self, value) -> None:
            self._optimizer.add_param_group({"params": value.parameters()})
            self._history_summarization_module = value

        def reset(self, action_space) -> None:
            pass
