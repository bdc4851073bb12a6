"""B200TD3 / B200DeepDeterministicPolicyGradient — the learner side of Pearl's TD3
(pearl/policy_learners/sequential_decision_making/td3.py:43-202) and DeepDeterministicPolicyGradient (ddpg.py:41-157, on
actor_critic_base.py:309-366) on a B200: `learn(replay_buffer)` runs `training_rounds` x (sample -> [delayed] actor step ->
twin-critic step -> [delayed] soft target updates) on the GPU through `prl_td3_learn` (include/pearl_b200.h).  Same constructor
argument names and the same report keys (`actor_loss`, `critic_loss`) as the reference.  PyTorch holds the flat parameter
vectors and draws the target-policy noise (the reference's `torch.normal`); no math happens in Python.  No CPU fallback.
`learn_batch(batch)` runs one round on a caller-supplied batch (`prl_td3_learn_batch`), as PearlAgent.learn_batch and
offline_learning() call it.  B200TD3BC is Pearl's TD3BC (td3.py:241-318): the same round with a behaviour-cloning term in
the actor loss.  With a reward-constrained safety module's multiplier (`lambda_constraint`, or `safety_module.lambda_constraint`)
`learn` trains on reward - lambda * cost, as ActorCriticBase.preprocess_batch does (actor_critic_base.py:368-383)."""
from __future__ import annotations

import ctypes as C
from typing import Any, Iterable, Optional

import torch

from . import _lib
from ._core import FlatCore, _bounds
from .replay_buffer import B200ReplayBuffer, _stream_ptr


class B200TD3(FlatCore):
    _ABI = "prl_td3"
    _STEPS = ("_actor_adam_step", "_critic_adam_step")
    _default_freq, _default_noise, _default_clip = 2, 0.2, 0.5

    def __init__(self, state_dim: int, action_space: Any = None, actor_hidden_dims: Optional[Iterable[int]] = None,
                 critic_hidden_dims: Optional[Iterable[int]] = None, actor_learning_rate: float = 1e-3,
                 critic_learning_rate: float = 1e-3, actor_soft_update_tau: float = 0.005, critic_soft_update_tau: float = 0.005,
                 discount_factor: float = 0.99, training_rounds: int = 1, batch_size: int = 256,
                 actor_update_freq: Optional[int] = None, actor_update_noise: Optional[float] = None,
                 actor_update_noise_clip: Optional[float] = None, *, low=None, high=None,
                 device: Optional[torch.device | str | int] = None, max_rounds_per_call: int = 1024, seed: Optional[int] = None,
                 lambda_constraint: Optional[float] = None, safety_module: Any = None) -> None:
        self._open(device, training_rounds, batch_size, max_rounds_per_call, seed)
        actor_hidden_dims, critic_hidden_dims = list(actor_hidden_dims or []), list(critic_hidden_dims or [])
        if len(actor_hidden_dims) != 2 or len(critic_hidden_dims) != 2:
            raise NotImplementedError("the CUDA TD3 / DDPG learner is built for two hidden layers in the actor and in each critic")
        self._state_dim = int(state_dim)
        self._low, self._high = _bounds(action_space, low, high, self._device)
        self._action_dim = int(self._low.numel())
        self._actor_hidden_dims, self._critic_hidden_dims = actor_hidden_dims, critic_hidden_dims
        self._actor_learning_rate, self._critic_learning_rate = float(actor_learning_rate), float(critic_learning_rate)
        self._actor_soft_update_tau, self._critic_soft_update_tau = float(actor_soft_update_tau), float(critic_soft_update_tau)
        self._discount_factor = float(discount_factor)
        self._actor_update_freq = int(self._default_freq if actor_update_freq is None else actor_update_freq)
        self._actor_update_noise = float(self._default_noise if actor_update_noise is None else actor_update_noise)
        self._actor_update_noise_clip = float(self._default_clip if actor_update_noise_clip is None else actor_update_noise_clip)
        self._last_actor_loss = 0.0    # what rounds without an actor update report (td3.py:104,122)
        # the reward-constrained multiplier: `lambda_constraint` when set, else the safety module's, else no shaping
        self.lambda_constraint = None if lambda_constraint is None else float(lambda_constraint)
        self.safety_module = safety_module
        cfg = self._cfg(1)
        pa, pc = int(self._lib.prl_td3_actor_param_count(C.byref(cfg))), int(self._lib.prl_td3_critic_param_count(C.byref(cfg)))
        dev, f32 = self._device, torch.float32
        self.actor_params = torch.empty(pa, dtype=f32, device=dev)
        self.critic_params = torch.empty(2 * pc, dtype=f32, device=dev)
        self._init_like_reference()
        self.actor_target_params = self.actor_params.clone()
        self.critic_target_params = self.critic_params.clone()
        self._actor_state = [torch.zeros(pa, dtype=f32, device=dev) for _ in range(3)]      # exp_avg, exp_avg_sq, max_exp_avg_sq
        self._critic_state = [torch.zeros(2 * pc, dtype=f32, device=dev) for _ in range(3)]

    def _cfg(self, max_batch: int) -> _lib.Td3Cfg:
        return _lib.Td3Cfg(self._state_dim, self._action_dim, self._actor_hidden_dims[0], self._actor_hidden_dims[1],
                           self._critic_hidden_dims[0], self._critic_hidden_dims[1], self._actor_update_freq, max_batch, self._max_rounds,
                           self._actor_learning_rate, self._critic_learning_rate, 0.9, 0.999, 1e-8, 0.01, self._discount_factor,
                           self._actor_soft_update_tau, self._critic_soft_update_tau, self._actor_update_noise_clip)

    def _shapes(self):
        O, A, (h1, h2), (c1, c2) = self._state_dim, self._action_dim, self._actor_hidden_dims, self._critic_hidden_dims
        return [(h1, O), (h1,), (h2, h1), (h2,), (A, h2), (A,)], [(c1, O + A), (c1,), (c2, c1), (c2,), (1, c2), (1,)]

    def _init_like_reference(self) -> None:
        """Xavier-uniform weights, biases 0.01 (neural_networks/common/utils.py:201-205, actor_critic_base.py:154, twin_critic.py:36-60)."""
        sa, sc = self._shapes()
        self._fill(self.actor_params, sa)
        self._fill(self.critic_params, 2 * sc)

    def load_parameters(self, actor, q1, q2, actor_target=None, q1_target=None, q2_target=None) -> None:
        """Flat fp32 vectors in `torch.nn.Module.parameters()` order of the reference networks."""
        pc, c, t = self.critic_params.numel() // 2, self.critic_params, self.critic_target_params
        self._load((self.actor_params, actor), (self.actor_target_params, actor if actor_target is None else actor_target),
                   (c[:pc], q1), (c[pc:], q2), (t[:pc], q1 if q1_target is None else q1_target),
                   (t[pc:], q2 if q2_target is None else q2_target))

    def _create(self, h, cfg) -> int:
        p = _lib.ptr
        _lib.check(self._create_with(h, cfg, (
            p(self.actor_params), p(self._actor_state[0]), p(self._actor_state[1]), p(self._actor_state[2]), p(self.actor_target_params),
            p(self.critic_params), p(self._critic_state[0]), p(self._critic_state[1]), p(self._critic_state[2]),
            p(self.critic_target_params), p(self._low), p(self._high), self._adam_steps[0], self._adam_steps[1], p(self._workspace))))
        # a handle re-created mid-training reports the learner's last actor loss, not 0, until its next actor update
        return self._lib.prl_td3_set_last_actor_loss(h, float(self._last_actor_loss))

    def _create_with(self, h, cfg, args) -> int:
        return self._lib.prl_td3_create(C.byref(h), C.byref(cfg), *args)

    def set_learning_rates(self, actor_lr: float, critic_lr: float) -> None:
        """New AdamW learning rates: the handle is re-created with them at the current step counts (parameters, moments and
        the last actor loss live outside it)."""
        self.restart()
        self._actor_learning_rate, self._critic_learning_rate = float(actor_lr), float(critic_lr)

    def set_last_actor_loss(self, value: float) -> None:
        """The actor loss that rounds without an actor update report (the reference's `_last_actor_loss`)."""
        self._last_actor_loss = float(value)
        if self._handle.value:
            with torch.cuda.device(self._device):
                _lib.check(self._lib.prl_td3_set_last_actor_loss(self._handle, self._last_actor_loss))

    def _before_call(self) -> None:
        pass

    def _cost_lambda(self) -> Optional[float]:
        """The multiplier learn() shapes rewards with (None: none), read on every call."""
        if self.lambda_constraint is not None:
            return float(self.lambda_constraint)
        lam = getattr(self.safety_module, "lambda_constraint", None)
        return None if lam is None else float(lam)

    def _noise(self, noise: Optional[torch.Tensor], r: int, B: int, start: int = 0) -> Optional[torch.Tensor]:
        """[r, B, A] target-policy noise: rows start.. of `noise`, or torch.normal(0, actor_update_noise) draws (td3.py:155-160)."""
        if self._actor_update_noise <= 0.0:
            return None
        A, dev = self._action_dim, self._device
        if noise is not None:
            nz = noise[start:start + r].to(device=dev, dtype=torch.float32).contiguous()
            if tuple(nz.shape) != (r, B, A):
                raise ValueError(f"noise must be [rounds, {B}, {A}]")
            return nz
        return torch.randn((r, B, A), dtype=torch.float32, device=dev, generator=self._gen) * self._actor_update_noise

    # ------------------------------------------------------------------ PolicyLearner.learn (policy_learner.py:162-204)
    def learn(self, replay_buffer: B200ReplayBuffer, noise: Optional[torch.Tensor] = None, trace: Optional[dict] = None) -> dict:
        if not self._accepts(replay_buffer, True, "TD3 / DDPG need a replay buffer with is_action_continuous=True"):
            return {}
        lam = self._cost_lambda()
        if lam is not None and not replay_buffer.has_cost:
            raise ValueError("a reward-constrained multiplier is set but the replay buffer stores no costs (the reference "
                             "fails on batch.cost = None)")
        B = self._batch(len(replay_buffer))
        self._bind(B)
        self._before_call()
        with torch.cuda.device(self._device):
            _lib.check(self._lib.prl_td3_set_cost_lambda(self._handle, int(lam is not None), 0.0 if lam is None else lam))

        def chunk(r, done, out, idx):
            nz = self._noise(noise, r, B, done)
            return self._lib.prl_td3_learn(self._handle, replay_buffer.handle, r, B, int(self._training_steps), _lib.ptr(nz),
                                           _lib.ptr(out[0]), _lib.ptr(out[1]), _lib.ptr(idx), _stream_ptr(self._device))
        report = self._rounds(replay_buffer, B, trace, 2, {"actor_loss": 0, "critic_loss": 1}, chunk)
        self._last_actor_loss = float(report["actor_loss"][-1])
        return report

    # ------------------------------------------------------------------ TD3.learn_batch (td3.py:106-147)
    def learn_batch(self, batch, noise: Optional[torch.Tensor] = None) -> dict:
        """One round on a caller-supplied batch (state, action, reward, next_state, terminated; CPU or GPU tensors,
        `terminated` bool or uint8).  Like the reference it does not advance the training-step count: the actor and the
        targets are updated when `_training_steps % actor_update_freq == 0`.  `noise`: [B, A] or [1, B, A] target-policy
        noise draws, else drawn from the learner's generator."""
        B, dev = int(batch.state.shape[0]), self._device
        if batch.state.dim() != 2 or int(batch.state.shape[1]) != self._state_dim:
            raise ValueError(f"batch.state must be [B, {self._state_dim}], got {tuple(batch.state.shape)}")
        f32 = lambda t: t.to(device=dev, dtype=torch.float32).contiguous()  # noqa: E731
        act = f32(batch.action)
        if act.dim() != 2 or tuple(act.shape) != (B, self._action_dim):
            raise ValueError(f"batch.action must be [{B}, {self._action_dim}] continuous actions, got {tuple(batch.action.shape)}")
        if tuple(batch.next_state.shape) != tuple(batch.state.shape):
            raise ValueError(f"batch.next_state must be [B, {self._state_dim}], got {tuple(batch.next_state.shape)}")
        state, next_state, reward = f32(batch.state), f32(batch.next_state), f32(batch.reward.reshape(B))
        term = batch.terminated.reshape(B).to(device=dev, dtype=torch.uint8).contiguous()
        self._bind(B)
        self._before_call()
        nz = self._noise(None if noise is None else noise.reshape(1, *noise.shape[-2:]), 1, B)
        out = torch.empty((2, 1), dtype=torch.float32, device=dev)
        with torch.cuda.device(dev):
            _lib.check(self._lib.prl_td3_set_graph(self._handle, int(self.use_cuda_graph)))
            _lib.check(self._lib.prl_td3_learn_batch(self._handle, B, _lib.ptr(state), _lib.ptr(act), _lib.ptr(reward), _lib.ptr(next_state),
                                                     _lib.ptr(term), int(self._training_steps), _lib.ptr(nz), _lib.ptr(out[0]),
                                                     _lib.ptr(out[1]), _stream_ptr(dev)))
        host = out.cpu()
        self._last_actor_loss = float(host[0, 0])
        return {"actor_loss": float(host[0, 0]), "critic_loss": float(host[1, 0])}

    @property
    def graph_captures(self) -> int:
        return int(self._lib.prl_td3_graph_captures(self._handle)) if self._handle.value else 0


class B200DeepDeterministicPolicyGradient(B200TD3):
    """DDPG = the same step with an actor update every round and no target-policy noise (ddpg.py:41-157)."""
    _default_freq, _default_noise, _default_clip = 1, 0.0, 0.0

    def __init__(self, *args, **kwargs) -> None:
        for k in ("actor_update_freq", "actor_update_noise", "actor_update_noise_clip"):
            if kwargs.get(k) is not None:
                raise TypeError(f"DeepDeterministicPolicyGradient has no `{k}` (use B200TD3)")
        super().__init__(*args, **kwargs)


class B200TD3BC(B200TD3):
    """TD3BC (td3.py:241-318): TD3 whose actor loss is mean((a - b)^2) - alpha_bc / mean|Q1(s, a)| * mean(Q1(s, a)), with
    b = behavior_policy(s), a VanillaContinuousActorNetwork called through forward(): its raw tanh output, not scaled to
    the box.  `behavior_params` holds the behaviour network's flat W1 b1 W2 b2 W3 b3; `behavior_hidden_dims` are its two
    hidden widths (they may differ from the actor's).  `alpha_bc` is read on every call."""

    def __init__(self, *args, behavior_hidden_dims: Optional[Iterable[int]] = None, alpha_bc: float = 2.5, **kwargs) -> None:
        super().__init__(*args, **kwargs)
        dims = list(behavior_hidden_dims if behavior_hidden_dims is not None else self._actor_hidden_dims)
        if len(dims) != 2 or min(dims) <= 0:
            raise NotImplementedError("the CUDA TD3BC learner is built for a behaviour network with two hidden layers")
        self._behavior_hidden_dims = [int(d) for d in dims]
        self.alpha_bc = float(alpha_bc)
        O, A, (h1, h2) = self._state_dim, self._action_dim, self._behavior_hidden_dims
        self.behavior_params = torch.zeros(h1 * O + h1 + h2 * h1 + h2 + A * h2 + A, dtype=torch.float32, device=self._device)

    def _bc_cfg(self) -> _lib.Td3bcCfg:
        return _lib.Td3bcCfg(*self._behavior_hidden_dims)

    def _workspace_bytes(self, cfg) -> int:
        return int(self._lib.prl_td3bc_workspace_bytes(C.byref(cfg), C.byref(self._bc_cfg())))

    def _create_with(self, h, cfg, args) -> int:
        return self._lib.prl_td3bc_create(C.byref(h), C.byref(cfg), C.byref(self._bc_cfg()), _lib.ptr(self.behavior_params), *args)

    def _before_call(self) -> None:
        with torch.cuda.device(self._device):
            _lib.check(self._lib.prl_td3_set_alpha_bc(self._handle, float(self.alpha_bc)))

    def load_parameters(self, actor, q1, q2, actor_target=None, q1_target=None, q2_target=None, behavior=None) -> None:
        """As B200TD3.load_parameters; `behavior`: the behaviour network's flat parameters (parameters() order)."""
        super().load_parameters(actor, q1, q2, actor_target, q1_target, q2_target)
        if behavior is not None:
            b = torch.as_tensor(behavior, dtype=torch.float32).reshape(-1)
            if b.numel() != self.behavior_params.numel():
                raise ValueError(f"behavior has {b.numel()} parameters, the behaviour network {self.behavior_params.numel()}")
            self.behavior_params.copy_(b.to(self._device))
