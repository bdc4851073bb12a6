"""B200REINFORCE — the learner side of Pearl's REINFORCE with a state-value baseline
(pearl/policy_learners/sequential_decision_making/reinforce.py, use_critic=True, on top of actor_critic_base.py:309-366) on
an H100: `learn(replay_buffer)` runs the return pass (the critic at the newest transition's next_state, then every stored
reward added newest -> oldest) and `training_rounds` x (sample -> actor step -> critic step) on the GPU through
`prl_reinforce_*` (include/pearl_b200.h).  Same constructor argument names and reporting keys (`actor_loss`,
`critic_loss`) as the reference.  PyTorch holds the flat parameter vectors; no math happens in Python.  No CPU fallback.

What the reference computes, and this learner with it (DESIGN.md §3): every stored transition ends up holding ONE return R
(the reference's in-place `cum_reward +=` stores the same tensor in each), with no discount and no reset at episode ends;
and the actor loss broadcasts (B,) against (B, 1), so it is B * sum_j nlp_j (R - v_j).
"""
from __future__ import annotations

import ctypes as C
from typing import Iterable, Optional

import torch

from . import _lib
from .replay_buffer import B200ReplayBuffer, _stream_ptr


class B200REINFORCE:
    def __init__(self, state_dim: int, actor_hidden_dims: Optional[Iterable[int]] = None, use_critic: bool = True,
                 critic_hidden_dims: Optional[Iterable[int]] = None, action_space=None, actor_learning_rate: float = 1e-4,
                 critic_learning_rate: float = 1e-4, discount_factor: float = 0.99, training_rounds: int = 8,
                 batch_size: int = 64, *, n_actions: Optional[int] = None, device: Optional[torch.device | str | int] = None,
                 max_rounds_per_call: int = 1024, seed: Optional[int] = None) -> None:
        if not use_critic:
            raise NotImplementedError("the CUDA REINFORCE learner implements use_critic=True (the reference's learn() needs a "
                                      "critic for its bootstrap value)")
        self._device = torch.device("cuda", torch.cuda.current_device()) if device is None else torch.device(device)
        if self._device.index is None:
            self._device = torch.device("cuda", torch.cuda.current_device())
        self._lib = _lib.init(self._device.index)
        if n_actions is None:
            if action_space is None or not hasattr(action_space, "n"):
                raise ValueError("REINFORCE needs a discrete action space (`action_space.n`) or n_actions")
            n_actions = int(action_space.n)
        actor_hidden_dims, critic_hidden_dims = list(actor_hidden_dims or []), list(critic_hidden_dims or [])
        if len(actor_hidden_dims) != 2 or len(critic_hidden_dims) != 2:
            raise NotImplementedError("the CUDA REINFORCE learner is built for two hidden layers in the actor and in the critic")
        self._state_dim, self._n_actions = int(state_dim), int(n_actions)
        self._actor_hidden_dims, self._critic_hidden_dims = actor_hidden_dims, critic_hidden_dims
        self._actor_learning_rate, self._critic_learning_rate = float(actor_learning_rate), float(critic_learning_rate)
        self._discount_factor = float(discount_factor)      # accepted and unused, as in the reference's learn()
        self._training_rounds, self._batch_size = int(training_rounds), int(batch_size)
        self._max_rounds = max(int(max_rounds_per_call), 1)
        self._training_steps = 0
        self.use_cuda_graph = True       # False: plain stream launches (profilers)
        self._handle = C.c_void_p(0)
        self._bound_batch = 0
        self._adam_step = 0
        self._gen = torch.Generator(device=self._device)
        if seed is not None:
            self._gen.manual_seed(int(seed))
        cfg = self._cfg(1)
        pa, pc = int(self._lib.prl_reinforce_actor_param_count(C.byref(cfg))), int(self._lib.prl_reinforce_critic_param_count(C.byref(cfg)))
        if pa < 0 or pc < 0:
            raise ValueError(_lib.last_error())
        dev, f32 = self._device, torch.float32
        self.actor_params = torch.empty(pa, dtype=f32, device=dev)
        self.critic_params = torch.empty(pc, dtype=f32, device=dev)
        self._init_like_reference()
        self._actor_state = [torch.zeros(pa, dtype=f32, device=dev) for _ in range(3)]      # exp_avg, exp_avg_sq, max_exp_avg_sq
        self._critic_state = [torch.zeros(pc, dtype=f32, device=dev) for _ in range(3)]
        self._returns = torch.zeros(2, dtype=f32, device=dev)                               # [R, bootstrap term]

    def _cfg(self, max_batch: int) -> _lib.ReinforceCfg:
        return _lib.ReinforceCfg(self._state_dim, self._n_actions, self._actor_hidden_dims[0], self._actor_hidden_dims[1],
                                 self._critic_hidden_dims[0], self._critic_hidden_dims[1], max_batch, self._max_rounds,
                                 self._actor_learning_rate, self._critic_learning_rate, 0.9, 0.999, 1e-8, 0.01)

    def _shapes(self, hidden, out):
        O, (h1, h2) = self._state_dim, hidden
        return [(h1, O), (h1,), (h2, h1), (h2,), (out, h2), (out,)]

    def _init_like_reference(self) -> None:
        """Actor: Xavier-uniform weights, biases 0.01 (actor_critic_base.py); critic: nn.Linear's default init
        (VanillaValueNetwork is not re-initialised)."""
        def fill(vec, shapes, xavier):
            off, fan_in = 0, 1
            for shp in shapes:
                n = shp[0] * (shp[1] if len(shp) == 2 else 1)
                if len(shp) == 2:
                    fan_in = shp[1]
                    bound = (6.0 / (shp[0] + shp[1])) ** 0.5 if xavier else (1.0 / fan_in) ** 0.5
                    vec[off:off + n].uniform_(-bound, bound, generator=self._gen)
                elif xavier:
                    vec[off:off + n].fill_(0.01)
                else:
                    vec[off:off + n].uniform_(-(1.0 / fan_in) ** 0.5, (1.0 / fan_in) ** 0.5, generator=self._gen)
                off += n
            assert off == vec.numel()
        fill(self.actor_params, self._shapes(self._actor_hidden_dims, self._n_actions), True)
        fill(self.critic_params, self._shapes(self._critic_hidden_dims, 1), False)

    def load_parameters(self, actor, critic) -> None:
        """Flat fp32 vectors in `parameters()` order of the reference's VanillaActorNetwork / VanillaValueNetwork."""
        self.actor_params.copy_(torch.as_tensor(actor, dtype=torch.float32).reshape(-1).to(self._device))
        self.critic_params.copy_(torch.as_tensor(critic, dtype=torch.float32).reshape(-1).to(self._device))

    def set_learning_rates(self, actor_learning_rate: float, critic_learning_rate: float) -> None:
        """New AdamW learning rates from the next `learn()` on; the C handle and its captured graph are kept."""
        self._actor_learning_rate, self._critic_learning_rate = float(actor_learning_rate), float(critic_learning_rate)
        if self._handle.value:
            _lib.check(self._lib.prl_reinforce_set_lr(self._handle, self._actor_learning_rate, self._critic_learning_rate))

    @property
    def last_return(self) -> float:
        """R of the last `learn()`: the return every stored transition held."""
        return float(self._returns[0].item())

    @property
    def last_bootstrap(self) -> float:
        """The term R started from: critic(next_state of the newest transition) * (1 - terminated)."""
        return float(self._returns[1].item())

    @property
    def batch_size(self) -> int:
        return self._batch_size

    @property
    def training_rounds(self) -> int:
        return self._training_rounds

    def __del__(self):
        try:
            if getattr(self, "_handle", None) and self._handle.value:
                self._lib.prl_reinforce_destroy(self._handle)
                self._handle = C.c_void_p(0)
        except Exception:
            pass

    def _bind(self, need_batch: int) -> None:
        if self._handle.value and need_batch <= self._bound_batch:
            return
        if self._handle.value:
            self._adam_step = int(self._lib.prl_reinforce_adam_step(self._handle))
            self._lib.prl_reinforce_destroy(self._handle)
            self._handle = C.c_void_p(0)
        cfg = self._cfg(max(need_batch, self._batch_size if self._batch_size > 0 else need_batch))
        self._workspace = torch.empty(int(self._lib.prl_reinforce_workspace_bytes(C.byref(cfg))), dtype=torch.uint8, device=self._device)
        h, p = C.c_void_p(0), _lib.ptr
        with torch.cuda.device(self._device):
            _lib.check(self._lib.prl_reinforce_create(
                C.byref(h), C.byref(cfg), p(self.actor_params), p(self._actor_state[0]), p(self._actor_state[1]),
                p(self._actor_state[2]), p(self.critic_params), p(self._critic_state[0]), p(self._critic_state[1]),
                p(self._critic_state[2]), self._adam_step, p(self._workspace)))
        self._handle, self._bound_batch = h, cfg.max_batch

    # ------------------------------------------------------------------ REINFORCE.learn (reinforce.py:179-208)
    def learn(self, replay_buffer: B200ReplayBuffer, trace: Optional[dict] = None) -> dict:
        if not isinstance(replay_buffer, B200ReplayBuffer):
            raise TypeError("B200REINFORCE learns from a B200ReplayBuffer (GPU-resident rollout)")
        n = len(replay_buffer)
        if n == 0:
            return {}
        if replay_buffer.is_action_continuous:
            raise ValueError("REINFORCE needs a replay buffer of discrete actions (is_action_continuous=False)")
        B = n if (self._batch_size == -1 or n < self._batch_size) else self._batch_size
        self._bind(B)
        R, dev = self._training_rounds, self._device
        with torch.cuda.device(dev):
            _lib.check(self._lib.prl_reinforce_returns(self._handle, replay_buffer.handle, _lib.ptr(self._returns), _stream_ptr(dev)))
        report = {"actor_loss": [], "critic_loss": []}
        idx_all, done = [], 0
        while done < R:
            r = min(self._max_rounds, R - done)
            out = torch.empty((2, r), dtype=torch.float32, device=dev)
            idx = torch.empty((r, B), dtype=torch.int32, device=dev) if trace is not None else None
            replay_buffer._rng_push()
            with torch.cuda.device(dev):
                _lib.check(self._lib.prl_reinforce_set_graph(self._handle, int(self.use_cuda_graph)))
                _lib.check(self._lib.prl_reinforce_learn(self._handle, replay_buffer.handle, r, B, _lib.ptr(self._returns),
                                                         _lib.ptr(out[0]), _lib.ptr(out[1]), _lib.ptr(idx) if idx is not None else None,
                                                         _stream_ptr(dev)))
            replay_buffer._rng_pull()
            host = out.cpu()
            report["actor_loss"] += host[0].tolist()
            report["critic_loss"] += host[1].tolist()
            if idx is not None:
                idx_all.append(idx.cpu())
            done += r
        self._training_steps += R
        if trace is not None:
            trace["idx"] = torch.cat(idx_all)
            trace["launches"] = int(self._lib.prl_reinforce_last_launches(self._handle))
        return report
