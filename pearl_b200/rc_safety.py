"""B200RCSafetyModuleCostCriticContinuousAction — Pearl's reward-constrained safety module
(pearl/safety_modules/reward_constrained_safety_module.py:34-216) for the CUDA TD3 / DDPG / TD3BC learners.

`learn(replay_buffer, policy_learner)` runs once per `PearlAgent.learn()`, after the policy learner's rounds
(pearl_agent.py:213-220): one sampled batch (continuing the buffer's MT19937 stream), the twin cost critic's step towards
cost + cost_discount_factor * min(Qc1', Qc2')(s', actor(s')), the soft update of its target, and the projected step of
the Lagrange multiplier `lambda_constraint` from cq = mean(max(Qc1, Qc2)(s, actor(s))) of the updated critic — all in one
CUDA graph (`prl_rcsafety_learn`, include/pearl_b200.h).  The policy learner then trains on reward - lambda * cost on its
next call.  `lambda_constraint` is a host Python float and the source of truth: a value set by hand is what the next call
uses.  One small device-to-host copy per call reads back lambda, the cost-critic loss and cq (the reference's `.item()`).

When Pearl is importable this class subclasses the reference class with `learn()` replaced: `cost_critic`,
`target_of_cost_critic` and `cost_critic_optimizer.state` become views into the flat vectors of the CUDA step on the first
call.  Without Pearl it is a stand-alone module with the same constructor (`low` / `high` stand in for the action space)
and the same attributes.  No CPU path."""
from __future__ import annotations

import ctypes as C
from typing import Any, Iterable, Optional

import torch

from . import _lib
from ._core import Handle, _bounds, fill_like_reference
from .replay_buffer import B200ReplayBuffer, _stream_ptr
from .td3 import B200TD3

try:  # pragma: no cover - depends on the environment
    from pearl.safety_modules.reward_constrained_safety_module import RCSafetyModuleCostCriticContinuousAction as _RefRC

    HAVE_REFERENCE_RC = True
except Exception:
    HAVE_REFERENCE_RC = False


def _td3_core(policy_learner) -> B200TD3:
    """The CUDA TD3 / DDPG / TD3BC learner behind `policy_learner` (the stand-alone class or a plugin's core)."""
    if isinstance(policy_learner, B200TD3):
        return policy_learner
    if callable(getattr(policy_learner, "_ensure_core", None)):
        core = getattr(policy_learner, "_b200", None) or policy_learner._ensure_core()
        if isinstance(core, B200TD3):
            return core
    raise NotImplementedError("the CUDA reward-constrained safety module works with the CUDA TD3 / DDPG / TD3BC learners "
                              f"(pearl_b200), not {type(policy_learner).__name__}")


class _CostStep(Handle):
    """The CUDA cost-critic step: flat twin cost critic, its target, AdamW vectors and the C handle."""
    _ABI = "prl_rcsafety"

    def __init__(self, state_dim: int, action_dim: int, critic_hidden_dims, *, critic_learning_rate: float, cost_discount_factor: float,
                 critic_soft_update_tau: float, device: torch.device, seed: Optional[int] = None) -> None:
        self._device = device
        self._lib = _lib.init(device.index)
        dims = [int(d) for d in critic_hidden_dims]
        if len(dims) != 2:
            raise NotImplementedError("the CUDA cost critic is built for two hidden layers")
        self._state_dim, self._action_dim, self._hidden = int(state_dim), int(action_dim), dims
        self.critic_learning_rate = float(critic_learning_rate)
        self.cost_discount_factor, self.critic_soft_update_tau = float(cost_discount_factor), float(critic_soft_update_tau)
        self.use_cuda_graph = True
        self._handle = C.c_void_p(0)
        self._bound = (0, 0, 0)               # (max_batch, actor_h1, actor_h2) of the handle
        self._adam_steps = (0,)
        pc = int(self._lib.prl_rcsafety_param_count(C.byref(self._cfg(1, 1, 1))))
        f32 = torch.float32
        self.params = torch.empty(2 * pc, dtype=f32, device=device)
        gen = torch.Generator(device=device)
        if seed is not None:
            gen.manual_seed(int(seed))
        O, A, (c1, c2) = self._state_dim, self._action_dim, dims
        # Xavier-uniform weights, biases 0.01, as the reference's VanillaQValueNetwork
        fill_like_reference(self.params, 2 * [(c1, O + A), (c1,), (c2, c1), (c2,), (1, c2), (1,)], gen)
        self.target_params = self.params.clone()
        self.state = [torch.zeros(2 * pc, dtype=f32, device=device) for _ in range(3)]   # exp_avg, exp_avg_sq, max_exp_avg_sq
        self._out = torch.zeros(3, dtype=torch.float64, device=device)

    def _cfg(self, max_batch: int, h1: int, h2: int) -> _lib.RcsafetyCfg:
        return _lib.RcsafetyCfg(self._state_dim, self._action_dim, h1, h2, self._hidden[0], self._hidden[1], max_batch,
                                self.critic_learning_rate, 0.9, 0.999, 1e-8, 0.01, self.cost_discount_factor, self.critic_soft_update_tau)

    @property
    def adam_step(self) -> int:
        return self.adam_steps()[0]

    def _bind(self, batch: int, h1: int, h2: int) -> None:
        if self._handle.value and batch <= self._bound[0] and (h1, h2) == self._bound[1:]:
            return
        self.restart()
        cfg = self._cfg(batch, h1, h2)
        self._workspace = torch.empty(int(self._lib.prl_rcsafety_workspace_bytes(C.byref(cfg))), dtype=torch.uint8, device=self._device)
        h, p = C.c_void_p(0), _lib.ptr
        with torch.cuda.device(self._device):
            _lib.check(self._lib.prl_rcsafety_create(C.byref(h), C.byref(cfg), p(self.params), p(self.state[0]), p(self.state[1]),
                                                     p(self.state[2]), p(self.target_params), self._adam_steps[0], p(self._workspace)))
        self._handle, self._bound = h, (batch, h1, h2)

    def run(self, replay_buffer: B200ReplayBuffer, core: B200TD3, batch: int, lam: float, constraint_value: float, lr_lambda: float,
            ub: float, trace: Optional[dict] = None) -> tuple:
        """One call; returns (lambda, cost-critic loss, cq) as Python floats."""
        if (core._state_dim, core._action_dim) != (self._state_dim, self._action_dim):
            raise ValueError(f"the policy learner maps {core._state_dim} state features to {core._action_dim} actions; the cost "
                             f"critic is built for {self._state_dim} and {self._action_dim}")
        self._bind(batch, *core._actor_hidden_dims)
        p = _lib.ptr
        step = _lib.RcsafetyStep(core.actor_params.data_ptr(), core._low.data_ptr(), core._high.data_ptr(), float(lam),
                                 float(constraint_value), float(lr_lambda), float(ub), self._out.data_ptr())
        idx = torch.empty(batch, dtype=torch.int32, device=self._device) if trace is not None else None
        dev = self._device
        replay_buffer._rng_push()
        with torch.cuda.device(dev):
            _lib.check(self._lib.prl_rcsafety_set_graph(self._handle, int(self.use_cuda_graph)))
            _lib.check(self._lib.prl_rcsafety_learn(self._handle, replay_buffer.handle, batch, C.byref(step),
                                                    p(idx) if idx is not None else None, _stream_ptr(dev)))
        replay_buffer._rng_pull()
        if trace is not None:
            trace["idx"] = idx.cpu()
        lam_new, loss, cq = self._out.tolist()
        return lam_new, loss, cq

    @property
    def graph_captures(self) -> int:
        return int(self._lib.prl_rcsafety_graph_captures(self._handle)) if self._handle.value else 0

    @property
    def last_launches(self) -> int:
        return int(self._lib.prl_rcsafety_last_launches(self._handle)) if self._handle.value else 0


def _batch_size(module_batch: int, n: int) -> int:
    return n if (module_batch == -1 or n < module_batch) else module_batch


class _B200RCLearnMixin:
    """learn() of the reward-constrained module on the CUDA step; `_step_of(core)` gives the bound _CostStep."""

    def _step_of(self, core: B200TD3, policy_learner) -> _CostStep:
        raise NotImplementedError

    def learn(self, replay_buffer, policy_learner, trace: Optional[dict] = None) -> None:
        if len(replay_buffer) == 0:
            return
        core = _td3_core(policy_learner)
        if not isinstance(replay_buffer, B200ReplayBuffer):
            raise TypeError(f"{type(self).__name__} learns from a B200ReplayBuffer (GPU-resident ring)")
        if not replay_buffer.has_cost:
            raise ValueError("the replay buffer stores no costs: the reference fails on batch.cost = None")
        step = self._step_of(core, policy_learner)
        lam, loss, cq = step.run(replay_buffer, core, _batch_size(int(self._batch_size), len(replay_buffer)), float(self.lambda_constraint),
                                 float(self.constraint_value), float(self.lr_lambda), float(self.lambda_constraint_ub_value), trace)
        self.lambda_constraint = lam
        self.last_cost_critic_loss, self.last_cost_q = loss, cq
        self._after_step(step)

    def _after_step(self, step: _CostStep) -> None:
        pass

    def learn_batch(self, batch, policy_learner=None) -> None:
        """The reference's learn_batch does nothing (offline safety learning is not supported there)."""
        return None


class B200RCSafetyModule(_B200RCLearnMixin):
    """The stand-alone module: the reference's constructor arguments, `low` / `high` for the action box when there is no
    Pearl action space.  `cost_critic_params` / `cost_critic_target_params` hold the twin (q1 then q2, flat in parameters()
    order), `cost_critic_state` the AdamW vectors."""

    def __init__(self, constraint_value: float, state_dim: int, action_space: Any = None, critic_hidden_dims: Optional[Iterable[int]] = None,
                 lambda_constraint_ub_value: float = 20.0, lambda_constraint_init_value: float = 0.0, cost_discount_factor: float = 0.5,
                 lr_lambda: float = 1e-2, critic_learning_rate: float = 1e-3, critic_soft_update_tau: float = 0.005, batch_size: int = 256,
                 use_twin_critic: bool = True, *, low=None, high=None, device: Optional[torch.device | str | int] = None,
                 seed: Optional[int] = None) -> None:
        if not use_twin_critic:
            raise NotImplementedError("the reference's cost-critic step asserts a TwinCritic: use_twin_critic=False does not run")
        dev = torch.device("cuda", torch.cuda.current_device()) if device is None else torch.device(device)
        if dev.index is None:
            dev = torch.device("cuda", torch.cuda.current_device())
        lo, _ = _bounds(action_space, low, high, dev)
        self.constraint_value, self.lr_lambda = float(constraint_value), float(lr_lambda)
        self.lambda_constraint_ub_value = float(lambda_constraint_ub_value)
        self.lambda_constraint = float(lambda_constraint_init_value)
        self._batch_size = int(batch_size)
        self.state_dim, self.action_dim = int(state_dim), int(lo.numel())
        self.hidden_dims = list(critic_hidden_dims or [])
        self.critic_learning_rate, self.cost_discount_factor = float(critic_learning_rate), float(cost_discount_factor)
        self.critic_soft_update_tau = float(critic_soft_update_tau)
        self.use_twin_critic = True
        self.last_cost_critic_loss = self.last_cost_q = None
        self._step = _CostStep(self.state_dim, self.action_dim, self.hidden_dims, critic_learning_rate=self.critic_learning_rate,
                               cost_discount_factor=self.cost_discount_factor, critic_soft_update_tau=self.critic_soft_update_tau,
                               device=dev, seed=seed)

    @property
    def cost_critic_params(self) -> torch.Tensor:
        return self._step.params

    @property
    def cost_critic_target_params(self) -> torch.Tensor:
        return self._step.target_params

    @property
    def cost_critic_state(self) -> list:
        return self._step.state

    @property
    def use_cuda_graph(self) -> bool:
        return self._step.use_cuda_graph

    @use_cuda_graph.setter
    def use_cuda_graph(self, v: bool) -> None:
        self._step.use_cuda_graph = bool(v)

    @property
    def graph_captures(self) -> int:
        return self._step.graph_captures

    @property
    def last_launches(self) -> int:
        return self._step.last_launches

    def set_critic_learning_rate(self, lr: float) -> None:
        """A new AdamW learning rate: the handle is re-created with it at the current step count."""
        self.critic_learning_rate = float(lr)
        self._step.critic_learning_rate = float(lr)
        self._step.restart()

    def load_parameters(self, q1, q2, q1_target=None, q2_target=None) -> None:
        """Flat fp32 vectors in `parameters()` order of the two cost critics (and of their targets)."""
        t = lambda x: torch.as_tensor(x, dtype=torch.float32).reshape(-1).to(self._step._device)  # noqa: E731
        pc = self._step.params.numel() // 2
        self._step.params[:pc].copy_(t(q1)); self._step.params[pc:].copy_(t(q2))
        self._step.target_params[:pc].copy_(t(q1 if q1_target is None else q1_target))
        self._step.target_params[pc:].copy_(t(q2 if q2_target is None else q2_target))

    def _step_of(self, core, policy_learner):
        return self._step

    def __str__(self) -> str:
        return "RCSafetyModuleCostCriticContinuousAction"


def _check_reference_module(m) -> list:
    """The cost critics of a reference module the CUDA step implements: [hidden1, hidden2]; raises NotImplementedError."""
    from .actor_critic import _mlp3, _shapes
    name = lambda x: type(x).__name__  # noqa: E731
    if not getattr(m, "use_twin_critic", False):
        raise NotImplementedError("the reference's cost-critic step asserts a TwinCritic: use_twin_critic=False does not run")
    for net in (m.cost_critic, m.target_of_cost_critic):
        if (name(net), name(getattr(net, "_critic_1", None)), name(getattr(net, "_critic_2", None))) != \
                ("TwinCritic", "VanillaQValueNetwork", "VanillaQValueNetwork"):
            raise NotImplementedError("the CUDA cost critic is built for TwinCritic(VanillaQValueNetwork)")
    sc = _shapes(m.cost_critic)
    if len(sc) != 12 or sc[6:] != sc[:6]:
        raise NotImplementedError("the CUDA cost critic is built for two hidden layers in each critic")
    din, c1, c2, one = _mlp3(sc[:6], "cost critic")
    if din != int(m.state_dim) + int(m.action_dim) or one != 1:
        raise NotImplementedError("unexpected cost-critic shapes")
    return [c1, c2]


def _check_policy_learner(pl) -> None:
    """The policy learner's history summarization must be the identity: the CUDA step reads states as they are stored."""
    hsm = getattr(pl, "_history_summarization_module", None)
    if hsm is not None and type(hsm).__name__ != "IdentityHistorySummarizationModule":
        raise NotImplementedError("the CUDA reward-constrained safety module reads states as they are stored: "
                                  "IdentityHistorySummarizationModule only")


if HAVE_REFERENCE_RC:  # pragma: no cover - depends on the environment

    class B200RCSafetyModuleCostCriticContinuousAction(_B200RCLearnMixin, _RefRC):
        """Drop-in for `pearl...reward_constrained_safety_module.RCSafetyModuleCostCriticContinuousAction`, with `learn()` on
        the GPU for the CUDA TD3 / DDPG / TD3BC learners."""

        def __init__(self, *args: Any, seed: Optional[int] = None, **kwargs: Any) -> None:
            super().__init__(*args, **kwargs)
            self._b200 = None
            self._b200_seed = seed
            self.last_cost_critic_loss = self.last_cost_q = None

        def _step_of(self, core, policy_learner):
            from .actor_critic import _adamw_lr, _adopt, _bind_optimizer, _is_adopted, _is_bound
            _check_policy_learner(policy_learner)
            dev = next(self.cost_critic.parameters()).device
            if dev.type != "cuda":
                raise RuntimeError(f"{type(self).__name__}: the cost critic is on {dev}; move it to a CUDA device "
                                   "(PearlAgent(device_id=0) does this) - pearl_b200 has no CPU path")
            step = self._b200
            if step is None or step._device != dev:
                step = _CostStep(int(self.state_dim), int(self.action_dim), _check_reference_module(self),
                                 critic_learning_rate=_adamw_lr(self.cost_critic_optimizer, "cost critic optimizer"),
                                 cost_discount_factor=float(self.cost_discount_factor),
                                 critic_soft_update_tau=float(self.critic_soft_update_tau), device=dev, seed=self._b200_seed)
                self._b200 = step
            pc = step.params.numel() // 2
            pairs = [(self.cost_critic._critic_1, step.params[:pc]), (self.cost_critic._critic_2, step.params[pc:]),
                     (self.target_of_cost_critic._critic_1, step.target_params[:pc]),
                     (self.target_of_cost_critic._critic_2, step.target_params[pc:])]
            if not all(_is_adopted(m, flat) for m, flat in pairs):
                for m, flat in pairs:
                    _adopt(m, flat)
            # a learning-rate (or discount / tau) change: a new handle at the current step count
            hp = (_adamw_lr(self.cost_critic_optimizer, "cost critic optimizer"), float(self.cost_discount_factor),
                  float(self.critic_soft_update_tau))
            if hp != (step.critic_learning_rate, step.cost_discount_factor, step.critic_soft_update_tau):
                step.critic_learning_rate, step.cost_discount_factor, step.critic_soft_update_tau = hp
                step.restart()
            if not _is_bound(self.cost_critic_optimizer, self.cost_critic, step.state):
                cur = step.adam_step
                got = _bind_optimizer(self.cost_critic_optimizer, self.cost_critic, step.state, cur)
                if got != cur:
                    step.restart((got,))
            return step

        def _after_step(self, step):
            from .actor_critic import _set_steps
            _set_steps(self.cost_critic_optimizer, step.adam_step)

else:
    B200RCSafetyModuleCostCriticContinuousAction = B200RCSafetyModule
