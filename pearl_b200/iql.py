"""B200ImplicitQLearning — the learner side of Pearl's ImplicitQLearning
(pearl/policy_learners/sequential_decision_making/implicit_q_learning.py), the offline-RL actor-critic, on an H100.

`learn(replay_buffer)` runs `training_rounds` x (sample -> one round) on the GPU through `prl_iql_learn`;
`learn_batch(batch)` runs one round on a caller-supplied TransitionBatch through `prl_iql_learn_batch` (this is how the
reference's `offline_learning()` drives the agent).  A round computes the value (expectile), twin-critic and
advantage-weighted actor losses from the parameters as they were before it, then steps all three AdamW(amsgrad)
optimizers and soft-updates the critic targets (include/pearl_b200.h).  Same constructor argument names, defaults and
report keys (`value_loss`, `actor_loss`, `critic_loss`) as the reference.

Each round draws twice from torch's global CPU generator (`torch.randint(0, 2, (1,))`: which target critic the value
loss and then the actor loss use), as the reference does.  The draws are made here, one `torch.randint(0, 2, (r, 2))`
per chunk of r rounds, which yields the same bits and leaves the generator in the same state as 2r single draws; the
kernels take them as an input.  PyTorch holds the flat parameter vectors; no math happens in Python.  No CPU fallback.

Discrete actions (`n_actions=`): VanillaActorNetwork (softmax).  Continuous actions (`low=` / `high=` or a box
`action_space`): VanillaContinuousActorNetwork (tanh scaled to the box).  The Gaussian actor is not supported."""
from __future__ import annotations

import ctypes as C
from typing import Any, Iterable, Optional

import torch

from . import _lib
from ._core import FlatCore, _bounds
from .replay_buffer import B200ReplayBuffer, _stream_ptr


class B200ImplicitQLearning(FlatCore):
    _ABI = "prl_iql"
    _ONE_STEP = "IQL steps its actor, critics and value net once per round: one AdamW step count"

    def __init__(self, state_dim: int, action_space: Any = None, actor_hidden_dims: Optional[Iterable[int]] = None,
                 critic_hidden_dims: Optional[Iterable[int]] = None, value_critic_hidden_dims: Optional[Iterable[int]] = None,
                 value_critic_learning_rate: float = 1e-3, actor_learning_rate: float = 1e-3, critic_learning_rate: float = 1e-3,
                 critic_soft_update_tau: float = 0.05, discount_factor: float = 0.99, training_rounds: int = 5,
                 batch_size: int = 128, expectile: float = 0.5, temperature_advantage_weighted_regression: float = 0.5,
                 advantage_clamp: float = 100.0, *, n_actions: Optional[int] = None, low=None, high=None,
                 device: Optional[torch.device | str | int] = None, max_rounds_per_call: int = 1024, seed: Optional[int] = None) -> None:
        self._open(device, training_rounds, batch_size, max_rounds_per_call, seed)
        dims = [list(d or []) for d in (actor_hidden_dims, critic_hidden_dims, value_critic_hidden_dims)]
        if any(len(d) != 2 for d in dims):
            raise NotImplementedError("the CUDA IQL learner is built for two hidden layers in the actor, each critic and the value net")
        self._actor_hidden_dims, self._critic_hidden_dims, self._value_hidden_dims = dims
        continuous = action_space is not None or low is not None or high is not None
        if (n_actions is not None) == continuous:
            raise ValueError("give exactly one of n_actions (discrete actions) and low / high or a box action_space (continuous)")
        self._state_dim = int(state_dim)
        self._discrete = n_actions is not None
        if self._discrete:
            self._n_actions, self._action_dim = int(n_actions), 0
            self._low = self._high = None
        else:
            self._low, self._high = _bounds(action_space, low, high, self._device)
            self._n_actions, self._action_dim = 0, int(self._low.numel())
        self._actor_learning_rate, self._critic_learning_rate = float(actor_learning_rate), float(critic_learning_rate)
        self._value_learning_rate = float(value_critic_learning_rate)
        self._critic_soft_update_tau, self._discount_factor = float(critic_soft_update_tau), float(discount_factor)
        self._expectile = float(expectile)
        self._temperature = float(temperature_advantage_weighted_regression)
        self._advantage_clamp = float(advantage_clamp)
        cfg = self._cfg(1)
        pa, pc, pv = (int(self._lib.prl_iql_actor_param_count(C.byref(cfg))), int(self._lib.prl_iql_critic_param_count(C.byref(cfg))),
                      int(self._lib.prl_iql_value_param_count(C.byref(cfg))))
        if min(pa, pc, pv) < 0:
            raise ValueError(_lib.last_error())
        dev, f32 = self._device, torch.float32
        self.actor_params = torch.empty(pa, dtype=f32, device=dev)
        self.critic_params = torch.empty(2 * pc, dtype=f32, device=dev)
        self.value_params = torch.empty(pv, dtype=f32, device=dev)
        self._init_like_reference()
        self.critic_target_params = self.critic_params.clone()
        self._actor_state = [torch.zeros(pa, dtype=f32, device=dev) for _ in range(3)]      # exp_avg, exp_avg_sq, max_exp_avg_sq
        self._critic_state = [torch.zeros(2 * pc, dtype=f32, device=dev) for _ in range(3)]
        self._value_state = [torch.zeros(pv, dtype=f32, device=dev) for _ in range(3)]

    # ------------------------------------------------------------------ parameters
    def _cfg(self, max_batch: int) -> _lib.IqlCfg:
        (a1, a2), (c1, c2), (v1, v2) = self._actor_hidden_dims, self._critic_hidden_dims, self._value_hidden_dims
        return _lib.IqlCfg(self._state_dim, self._n_actions, self._action_dim, a1, a2, c1, c2, v1, v2, max_batch, self._max_rounds,
                           self._actor_learning_rate, self._critic_learning_rate, self._value_learning_rate, 0.9, 0.999, 1e-8, 0.01,
                           self._discount_factor, self._critic_soft_update_tau, self._expectile, self._temperature,
                           self._advantage_clamp)

    def _shapes(self):
        O, N = self._state_dim, self._n_actions or self._action_dim
        (a1, a2), (c1, c2), (v1, v2) = self._actor_hidden_dims, self._critic_hidden_dims, self._value_hidden_dims
        return ([(a1, O), (a1,), (a2, a1), (a2,), (N, a2), (N,)], [(c1, O + N), (c1,), (c2, c1), (c2,), (1, c2), (1,)],
                [(v1, O), (v1,), (v2, v1), (v2,), (1, v2), (1,)])

    def _init_like_reference(self) -> None:
        """Actor and critics: Xavier-uniform weights, biases 0.01 (neural_networks/common/utils.py xavier_init_weights, as
        actor_critic_base.py and twin_critic.py apply it).  Value net: torch's default nn.Linear initialisation
        (VanillaValueNetwork is not re-initialised): weights and biases U(-1/sqrt(fan_in), 1/sqrt(fan_in))."""
        sa, sc, sv = self._shapes()
        self._fill(self.actor_params, sa)
        self._fill(self.critic_params, 2 * sc)
        self._fill(self.value_params, sv, xavier=False)

    def load_parameters(self, actor, q1, q2, value, q1_target=None, q2_target=None) -> None:
        """Flat fp32 vectors in `torch.nn.Module.parameters()` order of the reference networks (VanillaActorNetwork or
        VanillaContinuousActorNetwork, VanillaQValueNetwork over state || action, VanillaValueNetwork)."""
        pc, c, t = self.critic_params.numel() // 2, self.critic_params, self.critic_target_params
        self._load((self.actor_params, actor), (c[:pc], q1), (c[pc:], q2), (self.value_params, value),
                   (t[:pc], q1 if q1_target is None else q1_target), (t[pc:], q2 if q2_target is None else q2_target))

    def set_learning_rates(self, actor_learning_rate: float, critic_learning_rate: float, value_critic_learning_rate: float) -> None:
        """New AdamW learning rates from the next call on; the C handle and its captured graphs are kept."""
        self._actor_learning_rate, self._critic_learning_rate = float(actor_learning_rate), float(critic_learning_rate)
        self._value_learning_rate = float(value_critic_learning_rate)
        if self._handle.value:
            _lib.check(self._lib.prl_iql_set_lr(self._handle, self._actor_learning_rate, self._critic_learning_rate,
                                                self._value_learning_rate))

    def _create(self, h, cfg) -> int:
        p = _lib.ptr
        return self._lib.prl_iql_create(
            C.byref(h), C.byref(cfg), p(self.actor_params), p(self._actor_state[0]), p(self._actor_state[1]), p(self._actor_state[2]),
            p(self.critic_params), p(self._critic_state[0]), p(self._critic_state[1]), p(self._critic_state[2]),
            p(self.critic_target_params), p(self.value_params), p(self._value_state[0]), p(self._value_state[1]),
            p(self._value_state[2]), p(self._low), p(self._high), self._adam_steps[0], p(self._workspace))

    def _bits(self, rounds: int) -> torch.Tensor:
        """The round's two `torch.randint(0, 2, (1,))` draws of the reference (value loss, then actor loss), in one draw."""
        return torch.randint(0, 2, (rounds, 2)).to(device=self._device, dtype=torch.int32)

    # the rows of prl_iql_learn's outputs each report key reads
    _ROWS = {"value_loss": 0, "actor_loss": 2, "critic_loss": 1}

    # ------------------------------------------------------------------ PolicyLearner.learn (policy_learner.py:162-204)
    def learn(self, replay_buffer: B200ReplayBuffer, trace: Optional[dict] = None) -> dict:
        if not self._accepts(replay_buffer, not self._discrete,
                             f"IQL configured for {'discrete' if self._discrete else 'continuous'} actions needs a replay buffer "
                             f"with is_action_continuous={not self._discrete}"):
            return {}
        B = self._batch(len(replay_buffer))
        self._bind(B)

        def chunk(r, done, out, idx):
            bits = self._bits(r)
            return self._lib.prl_iql_learn(self._handle, replay_buffer.handle, r, B, _lib.ptr(bits), _lib.ptr(out[0]), _lib.ptr(out[1]),
                                           _lib.ptr(out[2]), _lib.ptr(idx), _stream_ptr(self._device))
        return self._rounds(replay_buffer, B, trace, 3, self._ROWS, chunk)

    def _action_ids(self, a: torch.Tensor) -> torch.Tensor:
        """Action ids from the one-hot rows the reference's preprocess_batch produces, or from raw ids ([B] or [B, 1])."""
        if a.is_floating_point() and a.dim() >= 2 and a.shape[-1] == self._n_actions and self._n_actions > 1:
            return a.argmax(-1)
        if a.dim() >= 2 and a.shape[-1] == 1:
            a = a.squeeze(-1)
        return a.long()

    # ------------------------------------------------------------------ ImplicitQLearning.learn_batch
    def learn_batch(self, batch) -> dict:
        """One round on a caller-supplied batch (state, action, reward, next_state, terminated).  Like the reference it does
        not advance the training-step count."""
        B, dev = int(batch.state.shape[0]), self._device
        if int(batch.state.shape[-1]) != self._state_dim:
            raise ValueError(f"batch.state has {int(batch.state.shape[-1])} features, the learner {self._state_dim}")
        self._bind(B)
        f32 = lambda t: t.to(device=dev, dtype=torch.float32).contiguous()  # noqa: E731
        state, next_state, reward = f32(batch.state), f32(batch.next_state), f32(batch.reward.reshape(B))
        term = batch.terminated.reshape(B).to(device=dev, dtype=torch.uint8).contiguous()
        act = aid = None
        if self._discrete:
            aid = self._action_ids(batch.action.to(dev)).reshape(B).to(torch.int32).contiguous()
            if bool(((aid < 0) | (aid >= self._n_actions)).any()):
                raise ValueError(f"action ids must lie in [0, {self._n_actions})")
        else:
            act = f32(batch.action.reshape(B, -1))
            if act.shape[1] != self._action_dim:
                raise ValueError(f"batch.action has {act.shape[1]} dimensions, the learner {self._action_dim}")
        bits = self._bits(1)
        out = torch.empty((3, 1), dtype=torch.float32, device=dev)
        with torch.cuda.device(dev):
            _lib.check(self._lib.prl_iql_set_graph(self._handle, int(self.use_cuda_graph)))
            _lib.check(self._lib.prl_iql_learn_batch(self._handle, B, _lib.ptr(state), _lib.ptr(act), _lib.ptr(aid), _lib.ptr(reward),
                                                     _lib.ptr(next_state), _lib.ptr(term), _lib.ptr(bits), _lib.ptr(out[0]),
                                                     _lib.ptr(out[1]), _lib.ptr(out[2]), _stream_ptr(dev)))
        host = out.cpu()
        return {k: host[row].tolist()[0] for k, row in self._ROWS.items()}
