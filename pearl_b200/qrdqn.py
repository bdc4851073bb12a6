"""B200QuantileRegressionDeepQLearning — the learner side of Pearl's QuantileRegressionDeepQLearning
(pearl/policy_learners/sequential_decision_making/quantile_regression_deep_q_learning.py, QR-DQN) on an H100.

`learn(replay_buffer)` runs `training_rounds` x (sample -> one round) on the GPU through `prl_qrdqn_learn`;
`learn_batch(batch)` runs one round on a caller-supplied TransitionBatch through `prl_qrdqn_learn_batch` (how
`agent.learn_batch` and `offline_learning()` drive the agent).  A round evaluates the online quantile network at the
taken action and the target network at every next-action slot, picks the greedy slot under the risk metric
mean - beta * variance, takes one AdamW(amsgrad) step on the pairwise quantile-Huber loss and, every
`target_update_freq` training steps, soft-updates the target with the new parameters (include/pearl_b200.h).  Same
constructor argument names, defaults and report key (`loss`: mean |theta(s, a) - T|) as the reference.

`variance_weighting_coefficient` is beta of QuantileNetworkMeanVarianceSafetyModule; 0 (the default) is
RiskNeutralSafetyModule.  PyTorch holds the flat parameter vectors; no math happens in Python.  No CPU fallback."""
from __future__ import annotations

import ctypes as C
from typing import Any, Iterable, Optional

import torch

from . import _lib
from ._batch import call, check_features, dense_rows, next_available_first
from ._core import FlatCore
from .per import B200PrioritizedReplayBuffer
from .replay_buffer import B200ReplayBuffer, _stream_ptr


class B200QuantileRegressionDeepQLearning(FlatCore):
    _ABI = "prl_qrdqn"

    def __init__(self, state_dim: int, action_space: Any = None, hidden_dims: Optional[Iterable[int]] = None, num_quantiles: int = 10,
                 learning_rate: float = 5 * 0.0001, discount_factor: float = 0.99, training_rounds: int = 100, batch_size: int = 128,
                 target_update_freq: int = 10, soft_update_tau: float = 0.05, *, n_actions: Optional[int] = None,
                 variance_weighting_coefficient: float = 0.0, device: Optional[torch.device | str | int] = None,
                 max_rounds_per_call: int = 1024, seed: Optional[int] = None) -> None:
        self._open(device, training_rounds, batch_size, max_rounds_per_call, seed)
        hidden = list(hidden_dims or [])
        if len(hidden) != 2:
            raise NotImplementedError("the CUDA QR-DQN learner is built for a quantile network with two hidden layers")
        if (action_space is None) == (n_actions is None):
            raise ValueError("give exactly one of action_space (a DiscreteActionSpace) and n_actions")
        self._state_dim = int(state_dim)
        self._n_actions = int(n_actions if n_actions is not None else action_space.n)
        self._hidden_dims = [int(h) for h in hidden]
        self._num_quantiles = int(num_quantiles)
        self._learning_rate, self._discount_factor = float(learning_rate), float(discount_factor)
        self._target_update_freq, self._soft_update_tau = int(target_update_freq), float(soft_update_tau)
        self._variance_weighting_coefficient = float(variance_weighting_coefficient)
        cfg = self._cfg(1)
        n = int(self._lib.prl_qrdqn_param_count(C.byref(cfg)))
        if n < 0:
            raise ValueError(_lib.last_error())
        dev, f32 = self._device, torch.float32
        self.params = torch.empty(n, dtype=f32, device=dev)
        self._init_like_reference()
        self.target_params = self.params.clone()          # the reference's deepcopy of the online net
        self._state = [torch.zeros(n, dtype=f32, device=dev) for _ in range(3)]      # exp_avg, exp_avg_sq, max_exp_avg_sq

    # ------------------------------------------------------------------ parameters
    def _cfg(self, max_batch: int) -> _lib.QrdqnCfg:
        h1, h2 = self._hidden_dims
        return _lib.QrdqnCfg(self._state_dim, self._n_actions, h1, h2, self._num_quantiles, self._target_update_freq, max_batch,
                             self._max_rounds, self._learning_rate, 0.9, 0.999, 1e-8, 0.01, self._discount_factor,
                             self._soft_update_tau)

    def _shapes(self) -> list:
        (h1, h2), D, N = self._hidden_dims, self._state_dim + self._n_actions, self._num_quantiles
        return [(h1, D), (h1,), (h2, h1), (h2,), (N, h2), (N,)]

    def _init_like_reference(self) -> None:
        """torch's default nn.Linear initialisation (QuantileQValueNetwork's mlp_block is not re-initialised): weights and
        biases U(-1/sqrt(fan_in), 1/sqrt(fan_in))."""
        self._fill(self.params, self._shapes(), xavier=False)

    def load_parameters(self, q, q_target=None) -> None:
        """Flat fp32 vectors in `torch.nn.Module.parameters()` order of the reference's QuantileQValueNetwork."""
        self._load((self.params, q), (self.target_params, q if q_target is None else q_target))

    def set_learning_rate(self, learning_rate: float) -> None:
        """New AdamW learning rate from the next call on; the C handle and its captured graphs are kept."""
        self._learning_rate = float(learning_rate)
        if self._handle.value:
            _lib.check(self._lib.prl_qrdqn_set_lr(self._handle, self._learning_rate))

    def _create(self, h, cfg) -> int:
        p = _lib.ptr
        return self._lib.prl_qrdqn_create(C.byref(h), C.byref(cfg), p(self.params), p(self._state[0]), p(self._state[1]),
                                          p(self._state[2]), p(self.target_params), self._adam_steps[0], p(self._workspace))

    def _beta(self) -> float:
        return self._variance_weighting_coefficient

    # ------------------------------------------------------------------ PolicyLearner.learn (policy_learner.py:162-204)
    def learn(self, replay_buffer: B200ReplayBuffer, trace: Optional[dict] = None) -> dict:
        if isinstance(replay_buffer, B200PrioritizedReplayBuffer):
            raise NotImplementedError("QR-DQN samples uniformly, as the reference: a B200PrioritizedReplayBuffer is not supported")
        if not self._accepts(replay_buffer, False, "QR-DQN needs a replay buffer with discrete actions (is_action_continuous=False)"):
            return {}
        B = self._batch(len(replay_buffer))
        self._bind(B)
        beta = self._beta()

        def chunk(r, done, out, idx):
            return self._lib.prl_qrdqn_learn(self._handle, replay_buffer.handle, r, B, self._training_steps, beta, _lib.ptr(out[0]),
                                             _lib.ptr(idx), _stream_ptr(self._device))
        return self._rounds(replay_buffer, B, trace, 1, {"loss": 0}, chunk)

    # ------------------------------------------------------------------ QuantileRegressionDeepTDLearning.learn_batch
    def learn_batch(self, batch) -> dict:
        """One round on a caller-supplied batch (state, action, reward, next_state, terminated and, optionally,
        next_available_actions with next_unavailable_actions_mask; without them every action is available next).  Like
        the reference it does not advance the training-step count."""
        B, A, dev = int(batch.state.shape[0]), self._n_actions, self._device
        check_features(batch, self._state_dim)
        self._bind(B)
        return {"loss": call(self._lib.prl_qrdqn_set_graph, self._lib.prl_qrdqn_learn_batch, self._handle, self.use_cuda_graph, dev,
                             B, *dense_rows(batch, B, A, dev), *next_available_first(batch, B, A, dev), self._training_steps,
                             self._beta())}
