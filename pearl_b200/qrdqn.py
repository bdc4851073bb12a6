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
from .per import B200PrioritizedReplayBuffer
from .replay_buffer import B200ReplayBuffer, _stream_ptr


class B200QuantileRegressionDeepQLearning:
    def __init__(self, state_dim: int, action_space: Any = None, hidden_dims: Optional[Iterable[int]] = None, num_quantiles: int = 10,
                 learning_rate: float = 5 * 0.0001, discount_factor: float = 0.99, training_rounds: int = 100, batch_size: int = 128,
                 target_update_freq: int = 10, soft_update_tau: float = 0.05, *, n_actions: Optional[int] = None,
                 variance_weighting_coefficient: float = 0.0, device: Optional[torch.device | str | int] = None,
                 max_rounds_per_call: int = 1024, seed: Optional[int] = None) -> None:
        self._device = torch.device("cuda", torch.cuda.current_device()) if device is None else torch.device(device)
        if self._device.index is None:
            self._device = torch.device("cuda", torch.cuda.current_device())
        self._lib = _lib.init(self._device.index)
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
        self._training_rounds, self._batch_size = int(training_rounds), int(batch_size)
        self._target_update_freq, self._soft_update_tau = int(target_update_freq), float(soft_update_tau)
        self._variance_weighting_coefficient = float(variance_weighting_coefficient)
        self._max_rounds = max(int(max_rounds_per_call), 1)
        self._training_steps = 0
        self.use_cuda_graph = True       # False: plain stream launches (profilers)
        self._handle = C.c_void_p(0)
        self._bound_batch = 0
        self._gen = torch.Generator(device=self._device)
        if seed is not None:
            self._gen.manual_seed(int(seed))
        cfg = self._cfg(1)
        n = int(self._lib.prl_qrdqn_param_count(C.byref(cfg)))
        if n < 0:
            raise ValueError(_lib.last_error())
        dev, f32 = self._device, torch.float32
        self.params = torch.empty(n, dtype=f32, device=dev)
        self._init_like_reference()
        self.target_params = self.params.clone()          # the reference's deepcopy of the online net
        self._state = [torch.zeros(n, dtype=f32, device=dev) for _ in range(3)]      # exp_avg, exp_avg_sq, max_exp_avg_sq
        self._adam_step = 0

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
        off, fan_in = 0, 1
        for shp in self._shapes():
            n = shp[0] * (shp[1] if len(shp) == 2 else 1)
            if len(shp) == 2:
                fan_in = shp[1]
            self.params[off:off + n].uniform_(-fan_in ** -0.5, fan_in ** -0.5, generator=self._gen)
            off += n
        assert off == self.params.numel()

    def load_parameters(self, q, q_target=None) -> None:
        """Flat fp32 vectors in `torch.nn.Module.parameters()` order of the reference's QuantileQValueNetwork."""
        t = lambda x: torch.as_tensor(x, dtype=torch.float32).reshape(-1).to(self._device)  # noqa: E731
        self.params.copy_(t(q))
        self.target_params.copy_(t(q if q_target is None else q_target))

    def set_learning_rate(self, learning_rate: float) -> None:
        """New AdamW learning rate from the next call on; the C handle and its captured graphs are kept."""
        self._learning_rate = float(learning_rate)
        if self._handle.value:
            _lib.check(self._lib.prl_qrdqn_set_lr(self._handle, self._learning_rate))

    @property
    def batch_size(self) -> int:
        return self._batch_size

    @property
    def training_rounds(self) -> int:
        return self._training_rounds

    def __del__(self):
        try:
            if getattr(self, "_handle", None) and self._handle.value:
                self._lib.prl_qrdqn_destroy(self._handle)
                self._handle = C.c_void_p(0)
        except Exception:
            pass

    def _restart(self, adam_step: int) -> None:
        """Drop the C handle; the next call re-creates it at AdamW step `adam_step` (moments and parameters are ours)."""
        if self._handle.value:
            self._lib.prl_qrdqn_destroy(self._handle)
            self._handle = C.c_void_p(0)
        self._adam_step = int(adam_step)

    def _current_adam_step(self) -> int:
        return int(self._lib.prl_qrdqn_adam_step(self._handle)) if self._handle.value else int(self._adam_step)

    def _bind(self, need_batch: int) -> None:
        if self._handle.value and need_batch <= self._bound_batch:
            return
        self._restart(self._current_adam_step())
        cfg = self._cfg(max(need_batch, self._batch_size if self._batch_size > 0 else need_batch))
        self._workspace = torch.empty(int(self._lib.prl_qrdqn_workspace_bytes(C.byref(cfg))), dtype=torch.uint8, device=self._device)
        h = C.c_void_p(0)
        p = _lib.ptr
        with torch.cuda.device(self._device):
            _lib.check(self._lib.prl_qrdqn_create(C.byref(h), C.byref(cfg), p(self.params), p(self._state[0]), p(self._state[1]),
                                                  p(self._state[2]), p(self.target_params), self._adam_step, p(self._workspace)))
        self._handle, self._bound_batch = h, cfg.max_batch

    def _beta(self) -> float:
        return self._variance_weighting_coefficient

    # ------------------------------------------------------------------ PolicyLearner.learn (policy_learner.py:162-204)
    def learn(self, replay_buffer: B200ReplayBuffer, trace: Optional[dict] = None) -> dict:
        if not isinstance(replay_buffer, B200ReplayBuffer):
            raise TypeError("B200QuantileRegressionDeepQLearning learns from a B200ReplayBuffer (GPU-resident ring)")
        if isinstance(replay_buffer, B200PrioritizedReplayBuffer):
            raise NotImplementedError("QR-DQN samples uniformly, as the reference: a B200PrioritizedReplayBuffer is not supported")
        if len(replay_buffer) == 0:
            return {}
        if bool(replay_buffer.is_action_continuous):
            raise ValueError("QR-DQN needs a replay buffer with discrete actions (is_action_continuous=False)")
        B = len(replay_buffer) if (self._batch_size == -1 or len(replay_buffer) < self._batch_size) else self._batch_size
        self._bind(B)
        R, dev, beta = self._training_rounds, self._device, self._beta()
        losses, idx_all = [], []
        done = 0
        while done < R:
            r = min(self._max_rounds, R - done)
            out = torch.empty(r, dtype=torch.float32, device=dev)
            idx = torch.empty((r, B), dtype=torch.int32, device=dev) if trace is not None else None
            replay_buffer._rng_push()
            with torch.cuda.device(dev):
                _lib.check(self._lib.prl_qrdqn_set_graph(self._handle, int(self.use_cuda_graph)))
                _lib.check(self._lib.prl_qrdqn_learn(self._handle, replay_buffer.handle, r, B, self._training_steps + done, beta,
                                                     _lib.ptr(out), _lib.ptr(idx), _stream_ptr(dev)))
            replay_buffer._rng_pull()
            losses += out.cpu().tolist()
            if idx is not None:
                idx_all.append(idx.cpu())
            done += r
        self._training_steps += R
        if trace is not None:
            trace["idx"] = torch.cat(idx_all)
            trace["launches"] = int(self._lib.prl_qrdqn_last_launches(self._handle))
        return {"loss": losses}

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
