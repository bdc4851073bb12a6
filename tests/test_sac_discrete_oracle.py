"""The discrete SAC restatement (oracle/sac_discrete_oracle.py) against the recordings of the reference's
PearlAgent(SoftActorCritic, BasicReplayBuffer).learn() (tests/golden/sacd_*.npz), and the plugin's class relation to
the reference's SoftActorCritic."""
import importlib
import os
import sys
import types

import numpy as np
import pytest
import torch

from conftest import GOLDEN
from oracle.pearl_oracle import flat
from oracle.sac_discrete_oracle import OracleSACDiscrete

CASES = ("sacd_full", "sacd_dynamic", "sacd_reset")


def make_oracle(fx):
    init = {k: fx[f"init_{k}"] for k in ("actor", "q1", "q2", "q1t", "q2t")}
    h = tuple(int(x) for x in fx["hidden"])
    return OracleSACDiscrete(int(fx["obs"]), int(fx["n_actions"]), h, h, actor_lr=float(fx["actor_lr"]), critic_lr=float(fx["critic_lr"]),
                             gamma=float(fx["gamma"]), tau=float(fx["tau"]), entropy_coef=float(fx["entropy_coef"]),
                             autotune=bool(fx["autotune"]), init=init)


def batch_of(fx, idx):
    t = lambda k: torch.from_numpy(np.asarray(fx[k][idx]))  # noqa: E731
    A = int(fx["n_actions"])
    cnt = t("next_count")
    return dict(state=t("state"), action=t("action"), reward=t("reward"), next_state=t("next_state"), terminated=t("terminated"),
                next_ids=t("next_ids").long(), next_mask=torch.arange(A).unsqueeze(0) >= cnt.unsqueeze(1))


@pytest.mark.parametrize("case", CASES)
def test_sac_discrete_oracle_reproduces_reference(case):
    torch.set_num_threads(1)
    fx = np.load(os.path.join(GOLDEN, f"{case}.npz"))
    orc = make_oracle(fx)
    R = int(fx["rounds"])
    for r in range(R * int(fx["calls"])):
        if r and r % R == 0:
            orc.reset()
        if r % R == 0:
            assert orc.opt_actor.param_groups[0]["lr"] == float(fx["call_actor_lr"][r // R])
        out = orc.learn_batch(batch_of(fx, fx["idx"][r]))
        np.testing.assert_allclose(out["actor_loss"], fx["actor_loss"][r], rtol=5e-6, atol=1e-7)
        np.testing.assert_allclose(out["critic_loss"], fx["critic_loss"][r], rtol=5e-6)
        if orc.autotune:
            np.testing.assert_allclose(out["entropy_coef"], fx["entropy_loss"][r], rtol=5e-6, atol=1e-7)
    tol = dict(rtol=5e-6, atol=5e-7)
    np.testing.assert_allclose(flat(orc.actor).numpy(), fx["actor_after"], **tol)
    np.testing.assert_allclose(flat(orc.q[0]).numpy(), fx["q1_after"], **tol)
    np.testing.assert_allclose(flat(orc.q[1]).numpy(), fx["q2_after"], **tol)
    np.testing.assert_allclose(flat(orc.qt[0]).numpy(), fx["q1t_after"], **tol)
    np.testing.assert_allclose(flat(orc.qt[1]).numpy(), fx["q2t_after"], **tol)
    if orc.autotune:
        st = orc.opt_alpha.state[orc.log_alpha]
        np.testing.assert_allclose(orc.log_alpha.detach().numpy(), fx["log_alpha_after"], **tol)
        np.testing.assert_allclose(st["exp_avg"].numpy(), fx["alpha_exp_avg"], **tol)
        np.testing.assert_allclose(st["exp_avg_sq"].numpy(), fx["alpha_exp_avg_sq"], **tol)


def test_entropy_optimizer_must_be_plain_adam():
    """The plugin binds the entropy optimizer's state to the CUDA learner's torch.optim.Adam arithmetic: AdamW, amsgrad
    or weight decay are refused; the reference's Adam(lr, eps=1e-4) is accepted with its lr and eps."""
    from pearl_b200.actor_critic import _adam_lr_eps
    p = torch.nn.Parameter(torch.zeros(1))
    assert _adam_lr_eps(torch.optim.Adam([p], lr=5e-4, eps=1e-4)) == (5e-4, 1e-4)
    for bad in (torch.optim.AdamW([p], lr=5e-4), torch.optim.Adam([p], amsgrad=True), torch.optim.Adam([p], weight_decay=0.01),
                torch.optim.SGD([p], lr=0.1)):
        with pytest.raises(NotImplementedError):
            _adam_lr_eps(bad)


def test_plugin_subclasses_the_reference_when_importable(monkeypatch):
    """With Pearl importable, `B200SoftActorCritic` is a subclass of the reference's SoftActorCritic (and of the CUDA
    plugin mixin).  Pearl is not installed where the suite runs, so stand-in modules with the reference's module paths
    and class names are installed for the duration of the test."""
    import pearl_b200.actor_critic as ac
    base = "pearl.policy_learners.sequential_decision_making."
    classes = {"ddpg": "DeepDeterministicPolicyGradient", "ppo": "ProximalPolicyOptimization",
               "soft_actor_critic_continuous": "ContinuousSoftActorCritic", "td3": "TD3", "soft_actor_critic": "SoftActorCritic"}
    parts = ["pearl", "pearl.policy_learners", base[:-1]]
    for p in parts:
        monkeypatch.setitem(sys.modules, p, types.ModuleType(p))
    for mod, cls in classes.items():
        m = types.ModuleType(base + mod)
        setattr(m, cls, type(cls, (), {}))
        monkeypatch.setitem(sys.modules, base + mod, m)
    try:
        importlib.reload(ac)
        assert ac.HAVE_REFERENCE
        assert issubclass(ac.B200SoftActorCritic, sys.modules[base + "soft_actor_critic"].SoftActorCritic)
        assert issubclass(ac.B200SoftActorCritic, ac._B200ActorCriticMixin)
    finally:
        monkeypatch.undo()
        importlib.reload(ac)
    if not ac.HAVE_REFERENCE:
        from pearl_b200.sac_discrete import B200SoftActorCritic as Core
        assert ac.B200SoftActorCritic is Core
