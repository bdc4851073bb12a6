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
from .replay_buffer import B200ReplayBuffer, _stream_ptr
from .sac import _bounds


class B200ImplicitQLearning:
    def __init__(self, state_dim: int, action_space: Any = None, actor_hidden_dims: Optional[Iterable[int]] = None,
                 critic_hidden_dims: Optional[Iterable[int]] = None, value_critic_hidden_dims: Optional[Iterable[int]] = None,
                 value_critic_learning_rate: float = 1e-3, actor_learning_rate: float = 1e-3, critic_learning_rate: float = 1e-3,
                 critic_soft_update_tau: float = 0.05, discount_factor: float = 0.99, training_rounds: int = 5,
                 batch_size: int = 128, expectile: float = 0.5, temperature_advantage_weighted_regression: float = 0.5,
                 advantage_clamp: float = 100.0, *, n_actions: Optional[int] = None, low=None, high=None,
                 device: Optional[torch.device | str | int] = None, max_rounds_per_call: int = 1024, seed: Optional[int] = None) -> None:
        self._device = torch.device("cuda", torch.cuda.current_device()) if device is None else torch.device(device)
        if self._device.index is None:
            self._device = torch.device("cuda", torch.cuda.current_device())
        self._lib = _lib.init(self._device.index)
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
        self._training_rounds, self._batch_size = int(training_rounds), int(batch_size)
        self._expectile = float(expectile)
        self._temperature = float(temperature_advantage_weighted_regression)
        self._advantage_clamp = float(advantage_clamp)
        self._max_rounds = max(int(max_rounds_per_call), 1)
        self._training_steps = 0
        self.use_cuda_graph = True       # False: plain stream launches (profilers)
        self._handle = C.c_void_p(0)
        self._bound_batch = 0
        self._gen = torch.Generator(device=self._device)
        if seed is not None:
            self._gen.manual_seed(int(seed))
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
        self._adam_step = 0

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
        def fill(vec, shapes, xavier):
            off, fan_in = 0, 1
            for shp in shapes:
                n = shp[0] * (shp[1] if len(shp) == 2 else 1)
                if len(shp) == 2:
                    fan_in = shp[1]
                    bound = (6.0 / (shp[0] + shp[1])) ** 0.5 if xavier else fan_in ** -0.5
                    vec[off:off + n].uniform_(-bound, bound, generator=self._gen)
                elif xavier:
                    vec[off:off + n].fill_(0.01)
                else:
                    vec[off:off + n].uniform_(-fan_in ** -0.5, fan_in ** -0.5, generator=self._gen)
                off += n
            assert off == vec.numel()
        sa, sc, sv = self._shapes()
        fill(self.actor_params, sa, True)
        pc = self.critic_params.numel() // 2
        fill(self.critic_params[:pc], sc, True)
        fill(self.critic_params[pc:], sc, True)
        fill(self.value_params, sv, False)

    def load_parameters(self, actor, q1, q2, value, q1_target=None, q2_target=None) -> None:
        """Flat fp32 vectors in `torch.nn.Module.parameters()` order of the reference networks (VanillaActorNetwork or
        VanillaContinuousActorNetwork, VanillaQValueNetwork over state || action, VanillaValueNetwork)."""
        t = lambda x: torch.as_tensor(x, dtype=torch.float32).reshape(-1).to(self._device)  # noqa: E731
        pc = self.critic_params.numel() // 2
        self.actor_params.copy_(t(actor))
        self.critic_params[:pc].copy_(t(q1))
        self.critic_params[pc:].copy_(t(q2))
        self.value_params.copy_(t(value))
        self.critic_target_params[:pc].copy_(t(q1 if q1_target is None else q1_target))
        self.critic_target_params[pc:].copy_(t(q2 if q2_target is None else q2_target))

    def set_learning_rates(self, actor_learning_rate: float, critic_learning_rate: float, value_critic_learning_rate: float) -> None:
        """New AdamW learning rates from the next call on; the C handle and its captured graphs are kept."""
        self._actor_learning_rate, self._critic_learning_rate = float(actor_learning_rate), float(critic_learning_rate)
        self._value_learning_rate = float(value_critic_learning_rate)
        if self._handle.value:
            _lib.check(self._lib.prl_iql_set_lr(self._handle, self._actor_learning_rate, self._critic_learning_rate,
                                                self._value_learning_rate))

    @property
    def batch_size(self) -> int:
        return self._batch_size

    @property
    def training_rounds(self) -> int:
        return self._training_rounds

    def __del__(self):
        try:
            if getattr(self, "_handle", None) and self._handle.value:
                self._lib.prl_iql_destroy(self._handle)
                self._handle = C.c_void_p(0)
        except Exception:
            pass

    def _bind(self, need_batch: int) -> None:
        if self._handle.value and need_batch <= self._bound_batch:
            return
        if self._handle.value:
            self._adam_step = int(self._lib.prl_iql_adam_step(self._handle))
            self._lib.prl_iql_destroy(self._handle)
            self._handle = C.c_void_p(0)
        cfg = self._cfg(max(need_batch, self._batch_size if self._batch_size > 0 else need_batch))
        self._workspace = torch.empty(int(self._lib.prl_iql_workspace_bytes(C.byref(cfg))), dtype=torch.uint8, device=self._device)
        h = C.c_void_p(0)
        p = _lib.ptr
        with torch.cuda.device(self._device):
            _lib.check(self._lib.prl_iql_create(
                C.byref(h), C.byref(cfg), p(self.actor_params), p(self._actor_state[0]), p(self._actor_state[1]), p(self._actor_state[2]),
                p(self.critic_params), p(self._critic_state[0]), p(self._critic_state[1]), p(self._critic_state[2]),
                p(self.critic_target_params), p(self.value_params), p(self._value_state[0]), p(self._value_state[1]),
                p(self._value_state[2]), p(self._low), p(self._high), self._adam_step, p(self._workspace)))
        self._handle, self._bound_batch = h, cfg.max_batch

    def _bits(self, rounds: int) -> torch.Tensor:
        """The round's two `torch.randint(0, 2, (1,))` draws of the reference (value loss, then actor loss), in one draw."""
        return torch.randint(0, 2, (rounds, 2)).to(device=self._device, dtype=torch.int32)

    @staticmethod
    def _report(host: torch.Tensor) -> dict:
        return {"value_loss": host[0].tolist(), "actor_loss": host[2].tolist(), "critic_loss": host[1].tolist()}

    # ------------------------------------------------------------------ PolicyLearner.learn (policy_learner.py:162-204)
    def learn(self, replay_buffer: B200ReplayBuffer, trace: Optional[dict] = None) -> dict:
        if not isinstance(replay_buffer, B200ReplayBuffer):
            raise TypeError("B200ImplicitQLearning learns from a B200ReplayBuffer (GPU-resident ring)")
        if len(replay_buffer) == 0:
            return {}
        if bool(replay_buffer.is_action_continuous) == self._discrete:
            raise ValueError(f"IQL configured for {'discrete' if self._discrete else 'continuous'} actions needs a replay buffer with "
                             f"is_action_continuous={not self._discrete}")
        B = len(replay_buffer) if (self._batch_size == -1 or len(replay_buffer) < self._batch_size) else self._batch_size
        self._bind(B)
        R, dev = self._training_rounds, self._device
        report = {"value_loss": [], "actor_loss": [], "critic_loss": []}
        idx_all = []
        done = 0
        while done < R:
            r = min(self._max_rounds, R - done)
            bits = self._bits(r)
            out = torch.empty((3, r), dtype=torch.float32, device=dev)
            idx = torch.empty((r, B), dtype=torch.int32, device=dev) if trace is not None else None
            replay_buffer._rng_push()
            with torch.cuda.device(dev):
                _lib.check(self._lib.prl_iql_set_graph(self._handle, int(self.use_cuda_graph)))
                _lib.check(self._lib.prl_iql_learn(self._handle, replay_buffer.handle, r, B, _lib.ptr(bits), _lib.ptr(out[0]),
                                                   _lib.ptr(out[1]), _lib.ptr(out[2]), _lib.ptr(idx) if idx is not None else None,
                                                   _stream_ptr(dev)))
            replay_buffer._rng_pull()
            for k, v in self._report(out.cpu()).items():
                report[k] += v
            if idx is not None:
                idx_all.append(idx.cpu())
            done += r
        self._training_steps += R
        if trace is not None:
            trace["idx"] = torch.cat(idx_all)
            trace["launches"] = int(self._lib.prl_iql_last_launches(self._handle))
        return report

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
        return {k: v[0] for k, v in self._report(out.cpu()).items()}
