"""B200ContinuousSoftActorCritic — the learner side of Pearl's ContinuousSoftActorCritic
(pearl/policy_learners/sequential_decision_making/soft_actor_critic_continuous.py:42-231 on top of
actor_critic_base.py:309-366) on a B200: `learn(replay_buffer)` runs `training_rounds` x
(sample -> actor step -> critic step -> soft target update -> entropy-coefficient step) on the GPU through
`prl_sac_learn` (include/pearl_b200.h).  Same constructor argument names and the same reporting keys as the
reference (`actor_loss`, `critic_loss`, `entropy_coef`).  PyTorch holds the flat parameter vectors and draws
the reparameterisation noise (the reference's `Normal.rsample`); no math happens in Python.  No CPU fallback.
"""
from __future__ import annotations

import ctypes as C
from typing import Any, Iterable, Optional

import torch

from . import _lib
from ._core import FlatCore, _bounds
from .replay_buffer import B200ReplayBuffer, _stream_ptr


class B200ContinuousSoftActorCritic(FlatCore):
    _ABI = "prl_sac"
    _ONE_STEP = "SAC steps its actor and critics once per round: one AdamW step count"

    def __init__(self, state_dim: int, action_space: Any = None, actor_hidden_dims: Optional[Iterable[int]] = None,
                 critic_hidden_dims: Optional[Iterable[int]] = None, actor_learning_rate: float = 1e-3,
                 critic_learning_rate: float = 1e-3, critic_soft_update_tau: float = 0.005, discount_factor: float = 0.99,
                 training_rounds: int = 100, batch_size: int = 256, entropy_coef: float = 0.2, entropy_autotune: bool = True,
                 *, low=None, high=None, device: Optional[torch.device | str | int] = None, max_rounds_per_call: int = 1024,
                 seed: Optional[int] = None) -> None:
        self._open(device, training_rounds, batch_size, max_rounds_per_call, seed)
        actor_hidden_dims, critic_hidden_dims = list(actor_hidden_dims or []), list(critic_hidden_dims or [])
        if len(actor_hidden_dims) != 2 or len(critic_hidden_dims) != 2:
            raise NotImplementedError("the CUDA SAC learner is built for two hidden layers in the actor and in each critic")
        self._state_dim = int(state_dim)
        self._low, self._high = _bounds(action_space, low, high, self._device)
        self._action_dim = int(self._low.numel())
        self._actor_hidden_dims, self._critic_hidden_dims = actor_hidden_dims, critic_hidden_dims
        self._actor_learning_rate, self._critic_learning_rate = float(actor_learning_rate), float(critic_learning_rate)
        self._critic_soft_update_tau, self._discount_factor = float(critic_soft_update_tau), float(discount_factor)
        self._entropy_autotune = bool(entropy_autotune)
        cfg = self._cfg(1)
        pa, pc = int(self._lib.prl_sac_actor_param_count(C.byref(cfg))), int(self._lib.prl_sac_critic_param_count(C.byref(cfg)))
        dev, f32 = self._device, torch.float32
        self.actor_params = torch.empty(pa, dtype=f32, device=dev)
        self.critic_params = torch.empty(2 * pc, dtype=f32, device=dev)
        self._init_like_reference()
        self.critic_target_params = self.critic_params.clone()
        self._actor_state = [torch.zeros(pa, dtype=f32, device=dev) for _ in range(3)]      # exp_avg, exp_avg_sq, max_exp_avg_sq
        self._critic_state = [torch.zeros(2 * pc, dtype=f32, device=dev) for _ in range(3)]
        self._log_entropy = torch.zeros(4, dtype=f32, device=dev)                              # value + its AdamW state
        self._entropy_coef = torch.full((1,), 1.0 if entropy_autotune else float(entropy_coef), dtype=f32, device=dev)

    # ------------------------------------------------------------------ parameters
    def _cfg(self, max_batch: int) -> _lib.SacCfg:
        return _lib.SacCfg(self._state_dim, self._action_dim, self._actor_hidden_dims[0], self._actor_hidden_dims[1],
                           self._critic_hidden_dims[0], self._critic_hidden_dims[1], int(self._entropy_autotune), max_batch,
                           self._max_rounds, self._actor_learning_rate, self._critic_learning_rate, 0.9, 0.999, 1e-8, 0.01,
                           self._discount_factor, self._critic_soft_update_tau)

    def _actor_shapes(self):
        O, A, (h1, h2) = self._state_dim, self._action_dim, self._actor_hidden_dims
        return [(h1, O), (h1,), (h2, h1), (h2,), (A, h2), (A,), (A, h2), (A,)]

    def _critic_shapes(self):
        D, (c1, c2) = self._state_dim + self._action_dim, self._critic_hidden_dims
        return [(c1, D), (c1,), (c2, c1), (c2,), (1, c2), (1,)]

    def _init_like_reference(self) -> None:
        """Xavier-uniform weights, biases 0.01 (neural_networks/common/utils.py:201-205, applied to the actor at
        actor_critic_base.py:154 and to both critics at twin_critic.py:36-60)."""
        self._fill(self.actor_params, self._actor_shapes())
        self._fill(self.critic_params, 2 * self._critic_shapes())

    def load_parameters(self, actor, q1, q2, q1_target=None, q2_target=None) -> None:
        """Flat fp32 vectors in `torch.nn.Module.parameters()` order of the reference networks (actor: body, fc_mu,
        fc_std; critics: VanillaQValueNetwork)."""
        pc, c, t = self.critic_params.numel() // 2, self.critic_params, self.critic_target_params
        self._load((self.actor_params, actor), (c[:pc], q1), (c[pc:], q2), (t[:pc], q1 if q1_target is None else q1_target),
                   (t[pc:], q2 if q2_target is None else q2_target))

    @property
    def entropy_coef(self) -> float:
        return float(self._entropy_coef.item())

    def _create(self, h, cfg) -> int:
        p = _lib.ptr
        return self._lib.prl_sac_create(
            C.byref(h), C.byref(cfg), p(self.actor_params), p(self._actor_state[0]), p(self._actor_state[1]), p(self._actor_state[2]),
            p(self.critic_params), p(self._critic_state[0]), p(self._critic_state[1]), p(self._critic_state[2]),
            p(self.critic_target_params), p(self._log_entropy), p(self._entropy_coef), p(self._low), p(self._high),
            self._adam_steps[0], p(self._workspace))

    # ------------------------------------------------------------------ PolicyLearner.learn (policy_learner.py:162-204)
    def learn(self, replay_buffer: B200ReplayBuffer, noise: Optional[torch.Tensor] = None, trace: Optional[dict] = None) -> dict:
        if not self._accepts(replay_buffer, True, "continuous SAC needs a replay buffer with is_action_continuous=True"):
            return {}
        B = self._batch(len(replay_buffer))
        self._bind(B)
        A, dev = self._action_dim, self._device

        def chunk(r, done, out, idx):
            if noise is not None:
                nz = noise[done:done + r].to(device=dev, dtype=torch.float32).contiguous()
                if tuple(nz.shape) != (r, 2, B, A):
                    raise ValueError(f"noise must be [rounds, 2, {B}, {A}]")
            else:
                nz = torch.randn((r, 2, B, A), dtype=torch.float32, device=dev, generator=self._gen)
            return self._lib.prl_sac_learn(self._handle, replay_buffer.handle, r, B, _lib.ptr(nz), _lib.ptr(out[0]), _lib.ptr(out[1]),
                                           _lib.ptr(out[2]), _lib.ptr(idx), _stream_ptr(dev))
        rows = {"actor_loss": 0, "critic_loss": 1, "entropy_coef": 2} if self._entropy_autotune else {"actor_loss": 0, "critic_loss": 1}
        return self._rounds(replay_buffer, B, trace, 3, rows, chunk)
