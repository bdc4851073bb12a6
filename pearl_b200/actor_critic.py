"""Actor-critic plugins that SUBCLASS the reference classes (SURVEY.md §8 rows a1 / a14-a16, f3):

    B200ContinuousSoftActorCritic   (ContinuousSoftActorCritic, soft_actor_critic_continuous.py:42-231)
    B200SoftActorCritic             (SoftActorCritic, soft_actor_critic.py: discrete actions)
    B200ProximalPolicyOptimization  (ProximalPolicyOptimization, ppo.py:96-293)
    B200REINFORCE                   (REINFORCE, reinforce.py: use_critic=True)
    B200TD3 / B200DeepDeterministicPolicyGradient  (td3.py:43-202, ddpg.py:41-157)
    B200ImplicitQLearning           (ImplicitQLearning, implicit_q_learning.py: offline RL; learn_batch runs on the GPU too)
    B200QuantileRegressionDeepQLearning  (QuantileRegressionDeepQLearning, QR-DQN; not an actor-critic, but bound the same
                                    way: `_Q`, `_Q_target` and the optimizer state are views; learn_batch runs on the GPU too)

When facebookresearch/Pearl is importable these are the reference classes with `learn()` replaced: the reference
constructor runs unchanged (same arguments, same networks, same optimizers, same exploration module), so
`pearl.pearl_agent.PearlAgent` accepts them as they are, `act()` / `reset()` / `compare()` / `state_dict()` are the
reference's own code.  On the first `learn()` (after PearlAgent moved the learner to its CUDA device) the parameters of
`_actor`, `_critic` (and their targets) are re-pointed at views into the flat fp32 vectors of the CUDA learner
(`pearl_b200.sac / sac_discrete / ppo / td3`), and `optimizer.state` at views into its flat AdamW vectors: the kernels and torch see the
same memory, nothing is copied per call, `get_extra_state` / `set_extra_state` (actor_critic_base.py:411-428) checkpoint
the live state, and a state loaded with `load_state_dict` is picked up on the next `learn()`.

When Pearl is not installed (the GPU test box) the same public names are the stand-alone CUDA learners, which take the
same keyword arguments.  Nothing here computes anything; there is no CPU path."""
from __future__ import annotations

import ctypes as C
from typing import Any

import torch

from .iql import B200ImplicitQLearning as IqlCore
from .ppo import B200ProximalPolicyOptimization as PpoCore
from .qrdqn import B200QuantileRegressionDeepQLearning as QrdqnCore
from .reinforce import B200REINFORCE as RfCore
from .sac import B200ContinuousSoftActorCritic as SacCore
from .sac_discrete import B200SoftActorCritic as SacdCore
from .td3 import B200DeepDeterministicPolicyGradient as DdpgCore
from .td3 import B200TD3 as Td3Core

try:  # pragma: no cover - depends on the environment
    from pearl.policy_learners.sequential_decision_making.ddpg import DeepDeterministicPolicyGradient as _RefDDPG
    from pearl.policy_learners.sequential_decision_making.soft_actor_critic import SoftActorCritic as _RefSACD
    from pearl.policy_learners.sequential_decision_making.ppo import ProximalPolicyOptimization as _RefPPO
    from pearl.policy_learners.sequential_decision_making.soft_actor_critic_continuous import (
        ContinuousSoftActorCritic as _RefSAC,
    )
    from pearl.policy_learners.sequential_decision_making.td3 import TD3 as _RefTD3

    HAVE_REFERENCE = True
except Exception:  # ModuleNotFoundError (pearl or gymnasium missing)
    HAVE_REFERENCE = False

try:  # pragma: no cover - depends on the environment; kept apart so the classes above do not depend on it
    from pearl.policy_learners.sequential_decision_making.implicit_q_learning import ImplicitQLearning as _RefIQL

    HAVE_REFERENCE_IQL = True
except Exception:
    HAVE_REFERENCE_IQL = False

try:  # pragma: no cover - depends on the environment; kept apart so the classes above do not depend on it
    from pearl.policy_learners.sequential_decision_making.reinforce import REINFORCE as _RefREINFORCE

    HAVE_REFERENCE_REINFORCE = True
except Exception:
    HAVE_REFERENCE_REINFORCE = False

try:  # pragma: no cover - depends on the environment; kept apart so the classes above do not depend on it
    from pearl.policy_learners.sequential_decision_making.quantile_regression_deep_q_learning import (
        QuantileRegressionDeepQLearning as _RefQRDQN,
    )

    HAVE_REFERENCE_QRDQN = True
except Exception:
    HAVE_REFERENCE_QRDQN = False


def _adamw_lr(opt: torch.optim.Optimizer, what: str) -> float:
    """The CUDA learners implement torch.optim.AdamW(amsgrad=True) with torch's default betas / eps / weight decay
    (what the reference constructs, actor_critic_base.py:157-166, 200-209)."""
    g = opt.param_groups[0] if isinstance(opt, torch.optim.AdamW) and len(opt.param_groups) == 1 else None
    if (g is None or not g.get("amsgrad", False) or g.get("maximize", False) or tuple(g["betas"]) != (0.9, 0.999)
            or float(g["eps"]) != 1e-8 or float(g["weight_decay"]) != 0.01):
        raise NotImplementedError(f"{what}: the fused update implements torch.optim.AdamW(amsgrad=True) with default "
                                  "betas / eps / weight_decay in one parameter group")
    return float(g["lr"])


def _adam_lr_eps(opt: torch.optim.Optimizer) -> tuple:
    """(lr, eps) of the discrete SAC entropy optimizer, which must be torch.optim.Adam without weight decay or amsgrad
    and with default betas (soft_actor_critic.py constructs Adam(lr=critic lr, eps=1e-4))."""
    g = opt.param_groups[0] if type(opt) is torch.optim.Adam and len(opt.param_groups) == 1 else None
    if (g is None or g.get("amsgrad", False) or g.get("maximize", False) or float(g.get("weight_decay", 0.0)) != 0.0
            or tuple(g["betas"]) != (0.9, 0.999)):
        raise NotImplementedError("entropy optimizer: the CUDA learner implements torch.optim.Adam (no weight decay, no amsgrad, "
                                  "default betas) in one parameter group")
    return float(g["lr"]), float(g["eps"])


def _shapes(module: torch.nn.Module) -> list:
    return [tuple(p.shape) for p in module.parameters()]


def _adopt(module: torch.nn.Module, flat: torch.Tensor) -> None:
    """Copy the module's parameters into `flat` (torch's parameters() order) and re-point them at views of it."""
    off = 0
    for p in module.parameters():
        n = p.numel()
        if off + n > flat.numel():
            break
        flat[off:off + n].copy_(p.detach().reshape(-1).to(device=flat.device, dtype=torch.float32))
        p.data = flat[off:off + n].view(p.shape)
        off += n
    if off != flat.numel() or off != sum(p.numel() for p in module.parameters()):
        raise NotImplementedError(f"{type(module).__name__}: parameter layout is not the one the CUDA learner is built for")


def _is_adopted(module: torch.nn.Module, flat: torch.Tensor) -> bool:
    return next(module.parameters()).data_ptr() == flat.data_ptr()


def _bind_optimizer(opt: torch.optim.Optimizer, module: torch.nn.Module, state3: list, step: int) -> int:
    """Make `opt.state` views into the flat AdamW vectors.  State that is already there and is NOT ours (built by torch,
    or just loaded from a checkpoint) is imported first; returns the AdamW step count to continue from."""
    params = list(module.parameters())
    st = opt.state
    if all(p in st and "exp_avg" in st[p] for p in params) and st[params[0]]["exp_avg"].data_ptr() != state3[0].data_ptr():
        dev = state3[0].device
        cat = lambda key: torch.cat([st[p][key].detach().reshape(-1).to(dev, torch.float32) for p in params])  # noqa: E731
        state3[0].copy_(cat("exp_avg"))
        state3[1].copy_(cat("exp_avg_sq"))
        state3[2].copy_(cat("max_exp_avg_sq") if all("max_exp_avg_sq" in st[p] for p in params) else cat("exp_avg_sq"))
        step = int(float(st[params[0]]["step"]))
    off = 0
    for p in params:
        n = p.numel()
        st[p] = dict(step=torch.tensor(float(step), dtype=torch.float32), exp_avg=state3[0][off:off + n].view(p.shape),
                     exp_avg_sq=state3[1][off:off + n].view(p.shape), max_exp_avg_sq=state3[2][off:off + n].view(p.shape))
        off += n
    return step


def _is_bound(opt: torch.optim.Optimizer, module: torch.nn.Module, state3: list) -> bool:
    p0 = next(module.parameters())
    return p0 in opt.state and "exp_avg" in opt.state[p0] and opt.state[p0]["exp_avg"].data_ptr() == state3[0].data_ptr()


def _set_steps(opt: torch.optim.Optimizer, step: int) -> None:
    for s in opt.state.values():
        if "step" in s:
            s["step"].fill_(float(step))


class _B200ActorCriticMixin:
    """In front of a reference ActorCriticBase subclass.  Subclasses say how to build the CUDA learner from the
    reference object (`_make_core`) and which (module, flat vector) / (optimizer, module, AdamW vectors) pairs exist."""

    def __init__(self, *args: Any, max_rounds_per_call: int = 1024, seed: int | None = None, **kwargs: Any) -> None:
        super().__init__(*args, **kwargs)
        self._b200_opts = dict(max_rounds_per_call=max_rounds_per_call, seed=seed)
        self._b200 = None

    # ---- per algorithm
    def _make_core(self, device: torch.device):
        raise NotImplementedError

    def _module_pairs(self, core) -> list:      # [(module, flat vector)]
        raise NotImplementedError

    def _optimizer_triples(self, core) -> list:  # [(optimizer, module, [exp_avg, exp_avg_sq, max_exp_avg_sq])]
        return [(self._actor_optimizer, self._actor, core._actor_state), (self._critic_optimizer, self._critic, core._critic_state)]

    def _core_steps(self, core) -> tuple:        # AdamW step counts (actor, critic) the CUDA learner is at
        raise NotImplementedError

    def _restart_core(self, core, steps: tuple) -> None:   # drop the C handle; the next learn() re-creates it at `steps`
        raise NotImplementedError

    def _bind_extras(self, core) -> None:   # idempotent: runs on every learn()
        pass

    def _apply_learning_rates(self, core, lrs: tuple) -> None:
        """New (actor, critic) learning rates: by default the C handle is re-created with them at the current AdamW step
        counts (moments and parameters live in the core's vectors)."""
        steps = self._core_steps(core)
        core._actor_learning_rate, core._critic_learning_rate = lrs
        self._restart_core(core, steps)

    # ---- binding
    def _device_of_parameters(self) -> torch.device:
        dev = next(self._actor.parameters()).device
        if dev.type != "cuda":
            raise RuntimeError(f"{type(self).__name__}: parameters are on {dev}; move the learner to a CUDA device "
                               "(PearlAgent(device_id=0) does this) - pearl_b200 has no CPU path")
        return dev

    def _ensure_core(self):
        dev = self._device_of_parameters()
        core = self._b200
        if core is None or core._device != dev:
            core = self._make_core(dev)
            self._b200 = core
        pairs = self._module_pairs(core)
        if not all(_is_adopted(m, flat) for m, flat in pairs):
            for m, flat in pairs:
                _adopt(m, flat)
        self._bind_extras(core)
        # learning rates changed since the CUDA learner was configured (a scheduler, or the user editing param_groups): the C
        # handle is re-created with the new rates at the current AdamW step counts (moments and parameters live in our vectors)
        lrs = (_adamw_lr(self._actor_optimizer, "actor optimizer"), _adamw_lr(self._critic_optimizer, "critic optimizer"))
        if lrs != (core._actor_learning_rate, core._critic_learning_rate):
            self._apply_learning_rates(core, lrs)
        triples = self._optimizer_triples(core)
        if not all(_is_bound(o, m, s3) for o, m, s3 in triples):
            cur = self._core_steps(core)
            steps = tuple(_bind_optimizer(o, m, s3, c) for (o, m, s3), c in zip(triples, cur))
            if steps != cur:
                self._restart_core(core, steps)
        return core

    # ---- PolicyLearner.learn (policy_learner.py:162-204)
    def learn(self, replay_buffer) -> dict:
        if len(replay_buffer) == 0:
            return {}
        core = self._ensure_core()
        core._training_rounds, core._batch_size = int(self._training_rounds), int(self._batch_size)
        core._training_steps = int(self._training_steps)
        report = core.learn(replay_buffer)
        self._training_steps = int(core._training_steps)
        for (opt, _, _), step in zip(self._optimizer_triples(core), self._core_steps(core)):
            _set_steps(opt, step)
        self._after_learn(core)
        return report

    def _after_learn(self, core) -> None:
        pass

    def learn_batch(self, batch) -> dict:
        raise NotImplementedError(f"{type(self).__name__} trains from a B200ReplayBuffer through learn(); a step on a "
                                  "caller-supplied batch is not part of the CUDA learner")


def _mlp3(shapes: list, what: str) -> tuple:
    """(in, h1, h2, out) of a two-hidden-layer MLP from its parameter shapes [W1, b1, W2, b2, W3, b3, ...]."""
    if len(shapes) < 6 or any(len(s) != (2 if i % 2 == 0 else 1) for i, s in enumerate(shapes)):
        raise NotImplementedError(f"{what}: the CUDA learners are built for MLPs with two hidden layers")
    (h1, din), (h2, h1b), (out, h2b) = shapes[0], shapes[2], shapes[4]
    if h1b != h1 or h2b != h2:
        raise NotImplementedError(f"{what}: unexpected layer shapes {shapes}")
    return din, h1, h2, out


if HAVE_REFERENCE:

    class B200ContinuousSoftActorCritic(_B200ActorCriticMixin, _RefSAC):
        """Drop-in for `pearl...soft_actor_critic_continuous.ContinuousSoftActorCritic`."""

        def _make_core(self, device):
            sa, sc = _shapes(self._actor), _shapes(self._critic)
            if len(sa) != 8 or len(sc) != 12:
                raise NotImplementedError("the CUDA SAC learner is built for GaussianActorNetwork + TwinCritic(VanillaQValueNetwork) "
                                          "with two hidden layers each")
            obs, h1, h2, act = _mlp3(sa, "actor")
            dq, c1, c2, one = _mlp3(sc[:6], "critic")
            if sa[6] != (act, h2) or dq != obs + act or one != 1 or sc[6:] != sc[:6]:
                raise NotImplementedError("unexpected SAC network shapes")
            space = getattr(self._actor, "_action_space", None) or self._action_space   # the box the actor scales its output to
            return SacCore(state_dim=obs, actor_hidden_dims=[h1, h2], critic_hidden_dims=[c1, c2],
                           actor_learning_rate=_adamw_lr(self._actor_optimizer, "actor optimizer"),
                           critic_learning_rate=_adamw_lr(self._critic_optimizer, "critic optimizer"),
                           critic_soft_update_tau=float(self._critic_soft_update_tau), discount_factor=float(self._discount_factor),
                           training_rounds=int(self._training_rounds), batch_size=int(self._batch_size),
                           entropy_coef=float(self._entropy_coef), entropy_autotune=bool(self._entropy_autotune),
                           low=space.low, high=space.high, device=device, **self._b200_opts)

        def _module_pairs(self, core):
            return [(self._actor, core.actor_params), (self._critic, core.critic_params), (self._critic_target, core.critic_target_params)]

        def _core_steps(self, core):
            s = int(core._lib.prl_sac_adam_step(core._handle)) if core._handle.value else int(core._adam_step)
            return (s, s)

        def _restart_core(self, core, steps):
            if steps[0] != steps[1]:
                raise NotImplementedError("SAC steps its actor and critics once per round: one AdamW step count")
            if core._handle.value:
                core._lib.prl_sac_destroy(core._handle)
                core._handle = C.c_void_p(0)
            core._adam_step = int(steps[0])

        def _bind_extras(self, core):
            """Entropy coefficient: `_log_entropy` (Parameter) and its AdamW state are the 4 floats of the CUDA learner's
            log-entropy block, `_entropy_coef` (buffer, shape kept) a view of its coefficient.  A state loaded into the
            entropy optimizer since the last call is imported."""
            coef = core._entropy_coef
            if self._entropy_coef.data_ptr() != coef.data_ptr():
                coef.copy_(self._entropy_coef.detach().reshape(1).to(coef))
                self._entropy_coef = coef.view(self._entropy_coef.shape)
            if not self._entropy_autotune:
                return
            blk, p, st = core._log_entropy, self._log_entropy, self._entropy_optimizer.state
            if p.data_ptr() != blk.data_ptr():
                _adamw_lr(self._entropy_optimizer, "entropy optimizer")
                blk[0:1].copy_(p.detach().reshape(1).to(blk))
                p.data = blk[0:1]
            if p in st and "exp_avg" in st[p] and st[p]["exp_avg"].data_ptr() == blk[1:2].data_ptr():
                return
            if p in st and "exp_avg" in st[p]:
                blk[1:2].copy_(st[p]["exp_avg"].reshape(1))
                blk[2:3].copy_(st[p]["exp_avg_sq"].reshape(1))
                blk[3:4].copy_(st[p].get("max_exp_avg_sq", st[p]["exp_avg_sq"]).reshape(1))
            st[p] = dict(step=torch.tensor(float(self._core_steps(core)[0])), exp_avg=blk[1:2], exp_avg_sq=blk[2:3],
                         max_exp_avg_sq=blk[3:4])

        def _after_learn(self, core):
            if self._entropy_autotune:
                _set_steps(self._entropy_optimizer, self._core_steps(core)[0])

    class B200SoftActorCritic(_B200ActorCriticMixin, _RefSACD):
        """Drop-in for `pearl...soft_actor_critic.SoftActorCritic` (discrete actions): VanillaActorNetwork and
        TwinCritic(VanillaQValueNetwork) with two hidden layers each, one-hot action representation.  The actor lr that
        `reset()`'s ExponentialLR changes every episode reaches the CUDA learner through `prl_sacd_set_lr`: same handle,
        same captured graph.  Current action sets are not stored by B200ReplayBuffer: the actor loss always runs over
        every action."""

        def _make_core(self, device):
            sa, sc = _shapes(self._actor), _shapes(self._critic)
            nets = (type(self._actor).__name__, type(self._critic).__name__,
                    type(getattr(self._critic, "_critic_1", None)).__name__, type(getattr(self._critic, "_critic_2", None)).__name__)
            if nets != ("VanillaActorNetwork", "TwinCritic", "VanillaQValueNetwork", "VanillaQValueNetwork") or len(sa) != 6 or len(sc) != 12:
                raise NotImplementedError("the CUDA discrete SAC learner is built for VanillaActorNetwork + TwinCritic(VanillaQValueNetwork) "
                                          "with two hidden layers each")
            obs, h1, h2, n_act = _mlp3(sa, "actor")
            dq, c1, c2, one = _mlp3(sc[:6], "critic")
            arm = getattr(self, "_action_representation_module", None) or getattr(self, "action_representation_module", None)
            if type(arm).__name__ != "OneHotActionTensorRepresentationModule":
                raise NotImplementedError("the CUDA discrete SAC learner folds a one-hot action representation into the critic")
            if dq != obs + n_act or one != 1 or sc[6:] != sc[:6]:
                raise NotImplementedError("unexpected discrete SAC network shapes")
            core = SacdCore(state_dim=obs, n_actions=n_act, actor_hidden_dims=[h1, h2], critic_hidden_dims=[c1, c2],
                            actor_learning_rate=_adamw_lr(self._actor_optimizer, "actor optimizer"),
                            critic_learning_rate=_adamw_lr(self._critic_optimizer, "critic optimizer"),
                            critic_soft_update_tau=float(self._critic_soft_update_tau), discount_factor=float(self._discount_factor),
                            training_rounds=int(self._training_rounds), batch_size=int(self._batch_size),
                            entropy_coef=float(self._entropy_coef), entropy_autotune=bool(self._entropy_autotune), device=device,
                            **self._b200_opts)
            if self._entropy_autotune:
                core._target_entropy = float(self._target_entropy)
                core._entropy_learning_rate, core._entropy_eps = _adam_lr_eps(self._entropy_optimizer)
            return core

        def _module_pairs(self, core):
            return [(self._actor, core.actor_params), (self._critic, core.critic_params), (self._critic_target, core.critic_target_params)]

        def _core_steps(self, core):
            s = int(core._lib.prl_sacd_adam_step(core._handle)) if core._handle.value else int(core._adam_step)
            return (s, s)

        def _restart_core(self, core, steps):
            if steps[0] != steps[1]:
                raise NotImplementedError("discrete SAC steps its actor and critics once per round: one AdamW step count")
            if core._handle.value:
                core._lib.prl_sacd_destroy(core._handle)
                core._handle = C.c_void_p(0)
            core._adam_step = int(steps[0])

        def _apply_learning_rates(self, core, lrs):
            core.set_learning_rates(*lrs)

        def _bind_extras(self, core):
            """`_entropy_coef` (buffer, shape kept) is a view of the core's coefficient; with autotune, `_log_entropy`
            (Parameter) and the entropy optimizer's Adam state are the [log alpha | exp_avg | exp_avg_sq] block of the
            core.  A state loaded into the entropy optimizer since the last call is imported."""
            coef = core._entropy_coef
            if self._entropy_coef.data_ptr() != coef.data_ptr():
                coef.copy_(self._entropy_coef.detach().reshape(1).to(coef))
                self._entropy_coef = coef.view(self._entropy_coef.shape)
            if not self._entropy_autotune:
                return
            hp = _adam_lr_eps(self._entropy_optimizer)
            if hp != (core._entropy_learning_rate, core._entropy_eps):      # fixed in the handle's configuration
                core._entropy_learning_rate, core._entropy_eps = hp
                self._restart_core(core, self._core_steps(core))
            blk, p, st = core._log_entropy, self._log_entropy, self._entropy_optimizer.state
            if p.data_ptr() != blk.data_ptr():
                blk[0:1].copy_(p.detach().reshape(1).to(blk))
                p.data = blk[0:1]
            if p in st and "exp_avg" in st[p] and st[p]["exp_avg"].data_ptr() == blk[1:2].data_ptr():
                return
            if p in st and "exp_avg" in st[p]:
                blk[1:2].copy_(st[p]["exp_avg"].reshape(1))
                blk[2:3].copy_(st[p]["exp_avg_sq"].reshape(1))
            st[p] = dict(step=torch.tensor(float(self._core_steps(core)[0])), exp_avg=blk[1:2], exp_avg_sq=blk[2:3])

        def _after_learn(self, core):
            if self._entropy_autotune:
                _set_steps(self._entropy_optimizer, self._core_steps(core)[0])

    class B200ProximalPolicyOptimization(_B200ActorCriticMixin, _RefPPO):
        """Drop-in for `pearl...ppo.ProximalPolicyOptimization` (discrete actions, as the reference's `_actor_loss`)."""

        def _make_core(self, device):
            sa, sc = _shapes(self._actor), _shapes(self._critic)
            if len(sa) != 6 or len(sc) != 6:
                raise NotImplementedError("the CUDA PPO learner is built for VanillaActorNetwork + VanillaValueNetwork with two hidden layers")
            obs, h1, h2, n_act = _mlp3(sa, "actor")
            oc, c1, c2, one = _mlp3(sc, "critic")
            if oc != obs or one != 1:
                raise NotImplementedError("unexpected PPO network shapes")
            return PpoCore(state_dim=obs, n_actions=n_act, actor_hidden_dims=[h1, h2], critic_hidden_dims=[c1, c2],
                           actor_learning_rate=_adamw_lr(self._actor_optimizer, "actor optimizer"),
                           critic_learning_rate=_adamw_lr(self._critic_optimizer, "critic optimizer"),
                           discount_factor=float(self._discount_factor), training_rounds=int(self._training_rounds),
                           batch_size=int(self._batch_size), epsilon=float(self._epsilon),
                           trace_decay_param=float(self._trace_decay_param), entropy_bonus_scaling=float(self._entropy_bonus_scaling),
                           device=device, **self._b200_opts)

        def _module_pairs(self, core):
            return [(self._actor, core.actor_params), (self._critic, core.critic_params)]

        def _core_steps(self, core):
            s = int(core._lib.prl_ppo_adam_step(core._handle)) if core._handle.value else int(core._adam_step)
            return (s, s)

        def _restart_core(self, core, steps):
            if steps[0] != steps[1]:
                raise NotImplementedError("PPO steps actor and critic once per round: one AdamW step count")
            if core._handle.value:
                core._lib.prl_ppo_destroy(core._handle)
                core._handle = C.c_void_p(0)
            core._adam_step = int(steps[0])

        def preprocess_replay_buffer(self, replay_buffer, process_group=None):
            """ppo.py:201-293 on the GPU; `learn()` calls it itself (as the reference's `learn` does)."""
            core = self._ensure_core()
            core._batch_size = int(self._batch_size)
            return core.preprocess_replay_buffer(replay_buffer, process_group=process_group)

    class _DeterministicMixin(_B200ActorCriticMixin):
        _core_cls = Td3Core

        def _core_kwargs(self) -> dict:
            return {}

        def _make_core(self, device):
            sa, sc = _shapes(self._actor), _shapes(self._critic)
            if len(sa) != 6 or len(sc) != 12:
                raise NotImplementedError("the CUDA TD3 / DDPG learner is built for VanillaContinuousActorNetwork + "
                                          "TwinCritic(VanillaQValueNetwork) with two hidden layers each")
            obs, h1, h2, act = _mlp3(sa, "actor")
            dq, c1, c2, one = _mlp3(sc[:6], "critic")
            if dq != obs + act or one != 1 or sc[6:] != sc[:6]:
                raise NotImplementedError("unexpected TD3 / DDPG network shapes")
            space = getattr(self._actor, "_action_space", None) or self._action_space   # the box the actor scales its output to
            return self._core_cls(state_dim=obs, actor_hidden_dims=[h1, h2], critic_hidden_dims=[c1, c2],
                                  actor_learning_rate=_adamw_lr(self._actor_optimizer, "actor optimizer"),
                                  critic_learning_rate=_adamw_lr(self._critic_optimizer, "critic optimizer"),
                                  actor_soft_update_tau=float(self._actor_soft_update_tau),
                                  critic_soft_update_tau=float(self._critic_soft_update_tau), discount_factor=float(self._discount_factor),
                                  training_rounds=int(self._training_rounds), batch_size=int(self._batch_size),
                                  low=space.low, high=space.high, device=device, **self._core_kwargs(), **self._b200_opts)

        def _module_pairs(self, core):
            return [(self._actor, core.actor_params), (self._actor_target, core.actor_target_params),
                    (self._critic, core.critic_params), (self._critic_target, core.critic_target_params)]

        def _core_steps(self, core):
            if core._handle.value:
                return (int(core._lib.prl_td3_actor_adam_step(core._handle)), int(core._lib.prl_td3_critic_adam_step(core._handle)))
            return tuple(int(x) for x in core._adam_steps)

        def _restart_core(self, core, steps):
            if core._handle.value:
                core._lib.prl_td3_destroy(core._handle)
                core._handle = C.c_void_p(0)
            core._adam_steps = (int(steps[0]), int(steps[1]))

    class B200TD3(_DeterministicMixin, _RefTD3):
        """Drop-in for `pearl...td3.TD3`."""

        def _core_kwargs(self):
            return dict(actor_update_freq=int(self._actor_update_freq), actor_update_noise=float(self._actor_update_noise),
                        actor_update_noise_clip=float(self._actor_update_noise_clip))

    class B200DeepDeterministicPolicyGradient(_DeterministicMixin, _RefDDPG):
        """Drop-in for `pearl...ddpg.DeepDeterministicPolicyGradient`."""
        _core_cls = DdpgCore

else:
    B200ContinuousSoftActorCritic = SacCore
    B200SoftActorCritic = SacdCore
    B200ProximalPolicyOptimization = PpoCore
    B200TD3 = Td3Core
    B200DeepDeterministicPolicyGradient = DdpgCore


def _iql_core_kwargs(pl) -> dict:
    """Checks that a reference ImplicitQLearning is the configuration the CUDA learner implements and returns the core's
    network and action-space arguments; raises NotImplementedError otherwise."""
    name = lambda m: type(m).__name__  # noqa: E731
    actor, critic, value = pl._actor, pl._critic, pl._value_network
    continuous = bool(pl._is_action_continuous)
    if name(actor) != ("VanillaContinuousActorNetwork" if continuous else "VanillaActorNetwork"):
        raise NotImplementedError(f"the CUDA IQL learner is built for VanillaActorNetwork (discrete actions) or VanillaContinuousActorNetwork "
                                  f"(continuous actions), not {name(actor)} with {'continuous' if continuous else 'discrete'} actions")
    if (name(critic), name(getattr(critic, "_critic_1", None)), name(getattr(critic, "_critic_2", None))) != \
            ("TwinCritic", "VanillaQValueNetwork", "VanillaQValueNetwork") or name(value) != "VanillaValueNetwork":
        raise NotImplementedError("the CUDA IQL learner is built for TwinCritic(VanillaQValueNetwork) and VanillaValueNetwork")
    if name(getattr(pl, "_history_summarization_module", None)) != "IdentityHistorySummarizationModule":
        raise NotImplementedError("the CUDA IQL learner reads states as they are stored: IdentityHistorySummarizationModule only")
    arm = getattr(pl, "_action_representation_module", None) or getattr(pl, "action_representation_module", None)
    if name(arm) != ("IdentityActionRepresentationModule" if continuous else "OneHotActionTensorRepresentationModule"):
        raise NotImplementedError("the CUDA IQL learner takes a one-hot action representation (discrete) or the identity (continuous)")
    sa, sc, sv = _shapes(actor), _shapes(critic), _shapes(value)
    if len(sa) != 6 or len(sc) != 12 or len(sv) != 6:
        raise NotImplementedError("the CUDA IQL learner is built for two hidden layers in the actor, each critic and the value net")
    obs, h1, h2, n_out = _mlp3(sa, "actor")
    dq, c1, c2, one = _mlp3(sc[:6], "critic")
    ov, v1, v2, onev = _mlp3(sv, "value network")
    if dq != obs + n_out or one != 1 or sc[6:] != sc[:6] or ov != obs or onev != 1:
        raise NotImplementedError("unexpected IQL network shapes")
    kw = dict(state_dim=obs, actor_hidden_dims=[h1, h2], critic_hidden_dims=[c1, c2], value_critic_hidden_dims=[v1, v2])
    if continuous:
        space = getattr(actor, "_action_space", None) or pl._action_space     # the box the actor scales its output to
        kw.update(low=space.low, high=space.high)
    else:
        kw.update(n_actions=n_out)
    return kw


if HAVE_REFERENCE_IQL:

    class B200ImplicitQLearning(_B200ActorCriticMixin, _RefIQL):
        """Drop-in for `pearl...implicit_q_learning.ImplicitQLearning`: VanillaActorNetwork (discrete) or
        VanillaContinuousActorNetwork (continuous), TwinCritic(VanillaQValueNetwork), VanillaValueNetwork, two hidden layers
        each, AdamW(amsgrad) for all three.  `_value_network` and its optimizer's state are views into the CUDA learner like
        the actor and critics.  A change of any of the three learning rates goes through `prl_iql_set_lr` (same handle, same
        graphs).  `learn_batch` runs on the GPU too, so `PearlAgent.learn_batch` and `offline_learning()` do."""

        def _make_core(self, device):
            kw = _iql_core_kwargs(self)
            return IqlCore(actor_learning_rate=_adamw_lr(self._actor_optimizer, "actor optimizer"),
                           critic_learning_rate=_adamw_lr(self._critic_optimizer, "critic optimizer"),
                           value_critic_learning_rate=_adamw_lr(self._value_network_optimizer, "value optimizer"),
                           critic_soft_update_tau=float(self._critic_soft_update_tau), discount_factor=float(self._discount_factor),
                           training_rounds=int(self._training_rounds), batch_size=int(self._batch_size),
                           expectile=float(self._expectile),
                           temperature_advantage_weighted_regression=float(self._temperature_advantage_weighted_regression),
                           advantage_clamp=float(self._advantage_clamp), device=device, **kw, **self._b200_opts)

        def _module_pairs(self, core):
            return [(self._actor, core.actor_params), (self._critic, core.critic_params), (self._critic_target, core.critic_target_params),
                    (self._value_network, core.value_params)]

        def _optimizer_triples(self, core):
            return super()._optimizer_triples(core) + [(self._value_network_optimizer, self._value_network, core._value_state)]

        def _core_steps(self, core):
            s = int(core._lib.prl_iql_adam_step(core._handle)) if core._handle.value else int(core._adam_step)
            return (s, s, s)

        def _restart_core(self, core, steps):
            if len(set(steps)) != 1:
                raise NotImplementedError("IQL steps its actor, critics and value net once per round: one AdamW step count")
            if core._handle.value:
                core._lib.prl_iql_destroy(core._handle)
                core._handle = C.c_void_p(0)
            core._adam_step = int(steps[0])

        def _apply_learning_rates(self, core, lrs):
            core.set_learning_rates(*lrs, core._value_learning_rate)

        def _bind_extras(self, core):
            vlr = _adamw_lr(self._value_network_optimizer, "value optimizer")
            if vlr != core._value_learning_rate:
                core.set_learning_rates(core._actor_learning_rate, core._critic_learning_rate, vlr)

        def learn_batch(self, batch) -> dict:
            """ImplicitQLearning.learn_batch on the GPU (the batch as preprocess_batch leaves it: one-hot or continuous
            actions).  Like the reference it does not advance the training-step count."""
            core = self._ensure_core()
            report = core.learn_batch(batch)
            for (opt, _, _), step in zip(self._optimizer_triples(core), self._core_steps(core)):
                _set_steps(opt, step)
            return report

else:
    B200ImplicitQLearning = IqlCore


def _reinforce_core_kwargs(pl) -> dict:
    """Checks that a reference REINFORCE is the configuration the CUDA learner implements and returns the core's network
    arguments; raises NotImplementedError otherwise.  use_critic=False is refused: the reference's learn() evaluates the
    critic for its bootstrap value and fails without one."""
    name = lambda m: type(m).__name__  # noqa: E731
    if not getattr(pl, "_use_critic", False):
        raise NotImplementedError("the CUDA REINFORCE learner implements use_critic=True (the reference's learn() needs the "
                                  "critic for its bootstrap value)")
    actor, critic = pl._actor, pl._critic
    if name(actor) != "VanillaActorNetwork":
        raise NotImplementedError(f"the CUDA REINFORCE learner is built for VanillaActorNetwork, not {name(actor)}")
    if name(critic) != "VanillaValueNetwork":
        raise NotImplementedError(f"the CUDA REINFORCE learner is built for VanillaValueNetwork, not {name(critic)}")
    hsm = getattr(pl, "_history_summarization_module", None)
    if isinstance(hsm, torch.nn.Module) and any(True for _ in hsm.parameters()):
        raise NotImplementedError("the CUDA REINFORCE learner reads states as they are stored: a history summarization module "
                                  "without parameters only")
    arm = getattr(pl, "_action_representation_module", None) or getattr(pl, "action_representation_module", None)
    if name(arm) != "OneHotActionTensorRepresentationModule":
        raise NotImplementedError("the CUDA REINFORCE learner takes a one-hot action representation")
    if hasattr(getattr(pl, "safety_module", None), "lambda_constraint"):
        raise NotImplementedError("the CUDA REINFORCE learner does not implement the reward-constrained safety module")
    sa, sc = _shapes(actor), _shapes(critic)
    if len(sa) != 6 or len(sc) != 6:
        raise NotImplementedError("the CUDA REINFORCE learner is built for two hidden layers in the actor and in the critic")
    obs, h1, h2, n_act = _mlp3(sa, "actor")
    oc, c1, c2, one = _mlp3(sc, "critic")
    if oc != obs or one != 1:
        raise NotImplementedError("unexpected REINFORCE network shapes")
    return dict(state_dim=obs, n_actions=n_act, actor_hidden_dims=[h1, h2], critic_hidden_dims=[c1, c2])


if HAVE_REFERENCE_REINFORCE:

    class B200REINFORCE(_B200ActorCriticMixin, _RefREINFORCE):
        """Drop-in for `pearl...reinforce.REINFORCE` with use_critic=True: VanillaActorNetwork and VanillaValueNetwork with two
        hidden layers each, one-hot actions, AdamW(amsgrad) for both.  `learn()` runs the return pass and the training rounds
        on the GPU from a B200ReplayBuffer; a learning-rate change goes through `prl_reinforce_set_lr` (same handle, same
        captured graph).  `act()` is the reference's own code (PropensityExploration over the live parameters)."""

        def _make_core(self, device):
            return RfCore(actor_learning_rate=_adamw_lr(self._actor_optimizer, "actor optimizer"),
                          critic_learning_rate=_adamw_lr(self._critic_optimizer, "critic optimizer"),
                          discount_factor=float(self._discount_factor), training_rounds=int(self._training_rounds),
                          batch_size=int(self._batch_size), device=device, **_reinforce_core_kwargs(self), **self._b200_opts)

        def _module_pairs(self, core):
            return [(self._actor, core.actor_params), (self._critic, core.critic_params)]

        def _core_steps(self, core):
            s = int(core._lib.prl_reinforce_adam_step(core._handle)) if core._handle.value else int(core._adam_step)
            return (s, s)

        def _restart_core(self, core, steps):
            if steps[0] != steps[1]:
                raise NotImplementedError("REINFORCE steps actor and critic once per round: one AdamW step count")
            if core._handle.value:
                core._lib.prl_reinforce_destroy(core._handle)
                core._handle = C.c_void_p(0)
            core._adam_step = int(steps[0])

        def _apply_learning_rates(self, core, lrs):
            core.set_learning_rates(*lrs)

else:
    B200REINFORCE = RfCore


def _qrdqn_adamw_lr(opt: torch.optim.Optimizer) -> float:
    """`_adamw_lr` for the QR-DQN optimizer, whose extra parameter groups (the one
    set_history_summarization_module adds for the identity module) must be empty."""
    groups = opt.param_groups if isinstance(opt, torch.optim.AdamW) else []
    if not groups or any(len(g["params"]) for g in groups[1:]):
        raise NotImplementedError("optimizer: the fused update implements torch.optim.AdamW(amsgrad=True) over the quantile "
                                  "network alone")
    g = groups[0]
    if (not g.get("amsgrad", False) or g.get("maximize", False) or tuple(g["betas"]) != (0.9, 0.999) or float(g["eps"]) != 1e-8
            or float(g["weight_decay"]) != 0.01):
        raise NotImplementedError("optimizer: the fused update implements torch.optim.AdamW(amsgrad=True) with default "
                                  "betas / eps / weight_decay")
    return float(g["lr"])


def _qrdqn_beta(safety_module) -> float:
    """Variance weight of the risk metric: 0 for RiskNeutralSafetyModule (PearlAgent's default for distributional
    learners) or no safety module, `_beta` for QuantileNetworkMeanVarianceSafetyModule."""
    name = type(safety_module).__name__
    if safety_module is None or name == "RiskNeutralSafetyModule":
        return 0.0
    if name == "QuantileNetworkMeanVarianceSafetyModule":
        return float(safety_module._beta)
    raise NotImplementedError(f"the CUDA QR-DQN learner implements RiskNeutralSafetyModule and "
                              f"QuantileNetworkMeanVarianceSafetyModule, not {name}")


def _qrdqn_core_kwargs(pl) -> dict:
    """Checks that a reference QuantileRegressionDeepQLearning is the configuration the CUDA learner implements and
    returns the core's network arguments; raises NotImplementedError otherwise."""
    name = lambda m: type(m).__name__  # noqa: E731
    q = pl._Q
    if name(q) != "QuantileQValueNetwork":
        raise NotImplementedError(f"the CUDA QR-DQN learner is built for QuantileQValueNetwork, not {name(q)}")
    if any(isinstance(m, torch.nn.LayerNorm) for m in q.modules()):
        raise NotImplementedError("the CUDA QR-DQN learner is built for QuantileQValueNetwork without use_layer_norm")
    if name(getattr(pl, "_history_summarization_module", None)) != "IdentityHistorySummarizationModule":
        raise NotImplementedError("the CUDA QR-DQN learner reads states as they are stored: IdentityHistorySummarizationModule only")
    arm = getattr(pl, "_action_representation_module", None) or getattr(pl, "action_representation_module", None)
    if name(arm) != "OneHotActionTensorRepresentationModule":
        raise NotImplementedError("the CUDA QR-DQN learner folds a one-hot action representation into the quantile network")
    sq = _shapes(q)
    if len(sq) != 6:
        raise NotImplementedError("the CUDA QR-DQN learner is built for a quantile network with two hidden layers")
    din, h1, h2, n_q = _mlp3(sq, "quantile network")
    obs, A = int(q.state_dim), int(pl._action_space.n)
    if din != obs + A or int(q.action_dim) != A or n_q != int(q.num_quantiles):
        raise NotImplementedError("unexpected QR-DQN network shapes")
    _qrdqn_beta(getattr(pl, "safety_module", None))
    return dict(state_dim=obs, n_actions=A, hidden_dims=[h1, h2], num_quantiles=n_q)


if HAVE_REFERENCE_QRDQN:

    class B200QuantileRegressionDeepQLearning(_RefQRDQN):
        """Drop-in for `pearl...quantile_regression_deep_q_learning.QuantileRegressionDeepQLearning`:
        QuantileQValueNetwork with two hidden layers, one-hot actions, AdamW(amsgrad).  On the first `learn()` /
        `learn_batch()` (after PearlAgent moved the learner to its CUDA device) `_Q`, `_Q_target` and the optimizer's
        state become views into the CUDA learner's flat vectors; a checkpoint loaded with `load_state_dict` is picked up on
        the next call.  The risk coefficient is read from `self.safety_module` and the learning rate from
        `param_groups[0]` on every call (neither re-creates the handle).  `act()` is the reference's own code."""

        def __init__(self, *args: Any, max_rounds_per_call: int = 1024, seed: int | None = None, **kwargs: Any) -> None:
            super().__init__(*args, **kwargs)
            self._b200_opts = dict(max_rounds_per_call=max_rounds_per_call, seed=seed)
            self._b200 = None

        def _ensure_core(self):
            dev = next(self._Q.parameters()).device
            if dev.type != "cuda":
                raise RuntimeError(f"{type(self).__name__}: parameters are on {dev}; move the learner to a CUDA device "
                                   "(PearlAgent(device_id=0) does this) - pearl_b200 has no CPU path")
            core = self._b200
            if core is None or core._device != dev:
                core = QrdqnCore(learning_rate=_qrdqn_adamw_lr(self._optimizer), discount_factor=float(self._discount_factor),
                                 training_rounds=int(self._training_rounds), batch_size=int(self._batch_size),
                                 target_update_freq=int(self._target_update_freq), soft_update_tau=float(self._soft_update_tau),
                                 device=dev, **_qrdqn_core_kwargs(self), **self._b200_opts)
                self._b200 = core
            if not (_is_adopted(self._Q, core.params) and _is_adopted(self._Q_target, core.target_params)):
                _adopt(self._Q, core.params)
                _adopt(self._Q_target, core.target_params)
            lr = _qrdqn_adamw_lr(self._optimizer)
            if lr != core._learning_rate:
                core.set_learning_rate(lr)
            if not _is_bound(self._optimizer, self._Q, core._state):
                cur = core._current_adam_step()
                step = _bind_optimizer(self._optimizer, self._Q, core._state, cur)
                if step != cur:
                    core._restart(step)
            core._variance_weighting_coefficient = _qrdqn_beta(getattr(self, "safety_module", None))
            core._training_rounds, core._batch_size = int(self._training_rounds), int(self._batch_size)
            core._training_steps = int(self._training_steps)
            return core

        def learn(self, replay_buffer) -> dict:
            """PolicyLearner.learn on the GPU (`training_rounds` rounds from a B200ReplayBuffer)."""
            if len(replay_buffer) == 0:
                return {}
            core = self._ensure_core()
            report = core.learn(replay_buffer)
            self._training_steps = int(core._training_steps)
            _set_steps(self._optimizer, core._current_adam_step())
            return report

        def learn_batch(self, batch) -> dict:
            """QuantileRegressionDeepTDLearning.learn_batch on the GPU (the batch as preprocess_batch leaves it).  Like the
            reference it does not advance the training-step count."""
            core = self._ensure_core()
            report = core.learn_batch(batch)
            _set_steps(self._optimizer, core._current_adam_step())
            return report

else:
    B200QuantileRegressionDeepQLearning = QrdqnCore
