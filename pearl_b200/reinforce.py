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
from ._core import FlatCore
from .replay_buffer import B200ReplayBuffer, _stream_ptr


class B200REINFORCE(FlatCore):
    _ABI = "prl_reinforce"
    _ONE_STEP = "REINFORCE steps actor and critic once per round: one AdamW step count"

    def __init__(self, state_dim: int, actor_hidden_dims: Optional[Iterable[int]] = None, use_critic: bool = True,
                 critic_hidden_dims: Optional[Iterable[int]] = None, action_space=None, actor_learning_rate: float = 1e-4,
                 critic_learning_rate: float = 1e-4, discount_factor: float = 0.99, training_rounds: int = 8,
                 batch_size: int = 64, *, n_actions: Optional[int] = None, device: Optional[torch.device | str | int] = None,
                 max_rounds_per_call: int = 1024, seed: Optional[int] = None) -> None:
        if not use_critic:
            raise NotImplementedError("the CUDA REINFORCE learner implements use_critic=True (the reference's learn() needs a "
                                      "critic for its bootstrap value)")
        self._open(device, training_rounds, batch_size, max_rounds_per_call, seed)
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
        self._fill(self.actor_params, self._shapes(self._actor_hidden_dims, self._n_actions))
        self._fill(self.critic_params, self._shapes(self._critic_hidden_dims, 1), xavier=False)

    def load_parameters(self, actor, critic) -> None:
        """Flat fp32 vectors in `parameters()` order of the reference's VanillaActorNetwork / VanillaValueNetwork."""
        self._load((self.actor_params, actor), (self.critic_params, critic))

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

    def _create(self, h, cfg) -> int:
        p = _lib.ptr
        return self._lib.prl_reinforce_create(
            C.byref(h), C.byref(cfg), p(self.actor_params), p(self._actor_state[0]), p(self._actor_state[1]), p(self._actor_state[2]),
            p(self.critic_params), p(self._critic_state[0]), p(self._critic_state[1]), p(self._critic_state[2]), self._adam_steps[0],
            p(self._workspace))

    # ------------------------------------------------------------------ REINFORCE.learn (reinforce.py:179-208)
    def learn(self, replay_buffer: B200ReplayBuffer, trace: Optional[dict] = None) -> dict:
        if not self._accepts(replay_buffer, False, "REINFORCE needs a replay buffer of discrete actions (is_action_continuous=False)",
                             "rollout"):
            return {}
        B = self._batch(len(replay_buffer))
        self._bind(B)
        dev = self._device
        with torch.cuda.device(dev):
            _lib.check(self._lib.prl_reinforce_returns(self._handle, replay_buffer.handle, _lib.ptr(self._returns), _stream_ptr(dev)))

        def chunk(r, done, out, idx):
            return self._lib.prl_reinforce_learn(self._handle, replay_buffer.handle, r, B, _lib.ptr(self._returns), _lib.ptr(out[0]),
                                                 _lib.ptr(out[1]), _lib.ptr(idx), _stream_ptr(dev))
        return self._rounds(replay_buffer, B, trace, 2, {"actor_loss": 0, "critic_loss": 1}, chunk)
