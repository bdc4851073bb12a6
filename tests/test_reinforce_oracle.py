"""The REINFORCE restatement (oracle/reinforce_oracle.py) against the recordings of the reference's
PearlAgent(REINFORCE, REINFORCEReplayBuffer).learn() (tests/golden/rf_*.npz); the hand-written gradients of the CUDA loss
kernel against autograd of the reference's expressions; the plugin's class relation and refusals; and the host arithmetic
of prl_reinforce_{actor,critic}_param_count / workspace_bytes."""
import ctypes
import importlib
import os
import random
import sys
import types

import numpy as np
import pytest
import torch

from conftest import GOLDEN
from oracle.pearl_oracle import flat
from oracle.reinforce_oracle import OracleREINFORCE, fold_returns, hand_gradients

CASES = ("rf_method", "rf_multi", "rf_lr")


def _calls(fx):
    """Per learn() call: (offset, n) into the concatenated transitions."""
    off = 0
    for n in fx["call_n"].tolist():
        yield off, n
        off += n


@pytest.mark.parametrize("case", CASES)
def test_reinforce_oracle_reproduces_reference(case):
    torch.set_num_threads(1)
    fx = np.load(os.path.join(GOLDEN, f"{case}.npz"))
    h = tuple(int(x) for x in fx["hidden"])
    lr = fx["call_lr"]
    orc = OracleREINFORCE(int(fx["obs"]), int(fx["n_actions"]), h, h, actor_lr=float(lr[0][0]), critic_lr=float(lr[0][1]),
                          init_actor=fx["init_actor"], init_critic=fx["init_critic"])
    R, B = int(fx["rounds"]), int(fx["batch"])
    r = 0
    for c, (off, n) in enumerate(_calls(fx)):
        orc.set_learning_rates(float(lr[c][0]), float(lr[c][1]))
        sl = slice(off, off + n)
        st, act, rew = (torch.from_numpy(fx[k][sl]) for k in ("state", "action", "reward"))
        boot = orc.bootstrap(fx["next_state"][off + n - 1], fx["terminated"][off + n - 1])
        np.testing.assert_allclose(boot.numpy(), fx["bootstrap"][c:c + 1], rtol=1e-6, atol=1e-7)
        ret = fold_returns(fx["bootstrap"][c], rew)
        assert ret.numpy().tobytes() == fx["ret"][c:c + 1].tobytes()          # the fold is exact from the same bootstrap
        random.setstate((3, tuple(int(x) for x in fx["rng_before"][c]), None))
        k = min(B, n)
        for _ in range(R):
            idx = random.sample(range(n), k)
            assert idx == fx["idx"][r].tolist()
            out = orc.learn_batch(st[idx], act[idx], ret)
            np.testing.assert_allclose(out["actor_loss"], fx["actor_loss"][r], rtol=5e-6, atol=1e-6)
            np.testing.assert_allclose(out["critic_loss"], fx["critic_loss"][r], rtol=5e-6)
            r += 1
        assert random.getstate() == (3, tuple(int(x) for x in fx["rng_after"][c]), None)
    tol = dict(rtol=5e-6, atol=5e-7)
    np.testing.assert_allclose(flat(orc.actor).numpy(), fx["actor_after"], **tol)
    np.testing.assert_allclose(flat(orc.critic).numpy(), fx["critic_after"], **tol)
    # The moments average gradients of scale B |R - v| (hundreds to thousands here).  torch's CPU kernels sum in an order
    # that depends on the instruction set they dispatch to, so an element that cancels to near zero carries summation
    # noise of the vector's scale: the absolute floor is one fp32 ulp-sized step (1e-7) of the largest element.
    for which in ("actor", "critic"):
        for key in ("exp_avg", "exp_avg_sq", "max_exp_avg_sq"):
            want = fx[f"{which}_{key}"]
            np.testing.assert_allclose(orc.adam_state(which, key).numpy(), want, rtol=5e-6, atol=1e-7 * float(np.abs(want).max()))


def test_recordings_show_both_quirks():
    """At least one recording has several episodes and a non-terminated newest transition (nonzero bootstrap), and R
    there is the plain sum over every episode; rf_method's newest transition is terminated (R is the reward sum alone)."""
    fx = np.load(os.path.join(GOLDEN, "rf_multi.npz"))
    assert fx["terminated"].sum() >= 3 and not fx["terminated"][-1] and fx["bootstrap"][0] != 0
    assert np.float32(fx["ret"][0]) == fold_returns(fx["bootstrap"][0], fx["reward"]).item()
    fx = np.load(os.path.join(GOLDEN, "rf_method.npz"))
    assert fx["terminated"][-1] and fx["bootstrap"][0] == 0 and int(fx["call_n"][0]) < int(fx["batch"])
    assert fx["idx"].shape == (8, 40)


@pytest.mark.parametrize("B,A", [(1, 1), (7, 2), (64, 5), (33, 16)])
def test_hand_gradients_equal_autograd_of_the_reference_expressions(B, A):
    torch.manual_seed(B * 100 + A)
    logits = (torch.randn(B, A, dtype=torch.float64) * 3).requires_grad_(True)
    v = torch.randn(B, dtype=torch.float64, requires_grad=True)
    action = torch.randint(0, A, (B,))
    R = 1.75
    ret = torch.full((B, 1), R, dtype=torch.float64)
    onehot = torch.nn.functional.one_hot(action, A).double()
    pa = torch.sum(torch.softmax(logits, -1) * onehot, dim=1, keepdim=True).view(-1)
    actor_loss = torch.sum(-torch.log(pa + 1e-8) * (ret - v.detach()))
    critic_loss = torch.nn.MSELoss()(v.reshape_as(ret), ret)
    g_logits, = torch.autograd.grad(actor_loss, logits)
    g_v, = torch.autograd.grad(critic_loss, v)
    dl, dv = hand_gradients(logits.detach(), action, v.detach(), R)
    torch.testing.assert_close(dl, g_logits, rtol=1e-12, atol=1e-12)
    torch.testing.assert_close(dv, g_v, rtol=1e-12, atol=1e-12)


def _reference_stand_ins(monkeypatch):
    base = "pearl.policy_learners.sequential_decision_making."
    classes = {"ddpg": "DeepDeterministicPolicyGradient", "ppo": "ProximalPolicyOptimization",
               "soft_actor_critic_continuous": "ContinuousSoftActorCritic", "td3": "TD3", "soft_actor_critic": "SoftActorCritic",
               "reinforce": "REINFORCE"}
    for p in ["pearl", "pearl.policy_learners", base[:-1]]:
        monkeypatch.setitem(sys.modules, p, types.ModuleType(p))
    for mod, cls in classes.items():
        m = types.ModuleType(base + mod)
        setattr(m, cls, type(cls, (), {}))
        monkeypatch.setitem(sys.modules, base + mod, m)
    return base


def test_plugin_subclasses_the_reference_when_importable(monkeypatch):
    """With Pearl importable, `B200REINFORCE` subclasses the reference's REINFORCE and the plugin mixin.  Pearl is not
    installed where the suite runs, so stand-in modules with the reference's module paths and class names are used."""
    import pearl_b200.actor_critic as ac
    base = _reference_stand_ins(monkeypatch)
    try:
        importlib.reload(ac)
        assert ac.HAVE_REFERENCE_REINFORCE
        assert issubclass(ac.B200REINFORCE, sys.modules[base + "reinforce"].REINFORCE)
        assert issubclass(ac.B200REINFORCE, ac._B200ActorCriticMixin)
        with pytest.raises(NotImplementedError):
            ac.B200REINFORCE.learn_batch(object(), None)
    finally:
        monkeypatch.undo()
        importlib.reload(ac)
    if not ac.HAVE_REFERENCE_REINFORCE:
        from pearl_b200.reinforce import B200REINFORCE as Core
        assert ac.B200REINFORCE is Core


def _named(cls_name, base=torch.nn.Module):
    return type(cls_name, (base,), {})


def _mlp(dims, cls_name):
    from oracle.pearl_oracle import _mlp as mlp
    net = mlp(dims)
    net.__class__ = type(cls_name, (torch.nn.Sequential,), {})
    return net


def _stand_in(**over):
    """A REINFORCE-shaped object: the attributes _reinforce_core_kwargs reads, as the reference configures them."""
    pl = types.SimpleNamespace(
        _use_critic=True, _actor=_mlp([4, 64, 64, 2], "VanillaActorNetwork"), _critic=_mlp([4, 64, 64, 1], "VanillaValueNetwork"),
        _history_summarization_module=_named("IdentityHistorySummarizationModule")(),
        _action_representation_module=_named("OneHotActionTensorRepresentationModule")(), safety_module=None)
    for k, v in over.items():
        setattr(pl, k, v)
    return pl


def test_plugin_core_arguments_and_refusals():
    from pearl_b200.actor_critic import _reinforce_core_kwargs
    assert _reinforce_core_kwargs(_stand_in()) == dict(state_dim=4, n_actions=2, actor_hidden_dims=[64, 64],
                                                       critic_hidden_dims=[64, 64])

    class Lambda:
        lambda_constraint = 0.0

    class WithParams(torch.nn.Module):
        def __init__(self):
            super().__init__()
            self.lstm = torch.nn.Linear(4, 4)
    refused = {
        "use_critic=False": dict(_use_critic=False),
        "dynamic actor": dict(_actor=_mlp([4, 64, 64, 2], "DynamicActionActorNetwork")),
        "other critic": dict(_critic=_mlp([4, 64, 64, 1], "VanillaQValueNetwork")),
        "three hidden layers": dict(_actor=_mlp([4, 64, 64, 64, 2], "VanillaActorNetwork")),
        "one hidden layer": dict(_critic=_mlp([4, 64, 1], "VanillaValueNetwork")),
        "identity actions": dict(_action_representation_module=_named("IdentityActionRepresentationModule")()),
        "history module with parameters": dict(_history_summarization_module=WithParams()),
        "reward-constrained safety": dict(safety_module=Lambda()),
    }
    for what, over in refused.items():
        with pytest.raises(NotImplementedError):
            _reinforce_core_kwargs(_stand_in(**over))
        print("refused:", what)


def test_core_refuses_use_critic_false_and_other_depths():
    from pearl_b200.reinforce import B200REINFORCE
    with pytest.raises(NotImplementedError, match="use_critic"):
        B200REINFORCE(state_dim=4, actor_hidden_dims=[8, 8], critic_hidden_dims=[8, 8], use_critic=False, n_actions=2)


def _cfg(**kw):
    from pearl_b200 import _lib
    d = dict(obs_dim=4, n_actions=2, actor_h1=64, actor_h2=64, critic_h1=64, critic_h2=64, max_batch=64, max_rounds=8,
             actor_lr=1e-4, critic_lr=1e-4, beta1=0.9, beta2=0.999, eps=1e-8, weight_decay=0.01)
    d.update(kw)
    return _lib.ReinforceCfg(**d)


def test_param_count_and_workspace_host_arithmetic():
    from pearl_b200 import _lib
    lib = _lib.load()
    c = _cfg(obs_dim=5, n_actions=3, actor_h1=7, actor_h2=11, critic_h1=13, critic_h2=17)
    assert lib.prl_reinforce_actor_param_count(ctypes.byref(c)) == 7 * 5 + 7 + 11 * 7 + 11 + 3 * 11 + 3
    assert lib.prl_reinforce_critic_param_count(ctypes.byref(c)) == 13 * 5 + 13 + 17 * 13 + 17 + 17 + 1
    small = lib.prl_reinforce_workspace_bytes(ctypes.byref(_cfg()))
    assert 0 < small < 1 << 22
    # the sampled-index arrays are [max_rounds][max_batch] int32 twice: sized in 64-bit arithmetic
    big = lib.prl_reinforce_workspace_bytes(ctypes.byref(_cfg(max_rounds=1 << 30, max_batch=64)))
    assert big >= 2 * 4 * (1 << 30) * 64 + 2 * 8 * (1 << 30)
    for bad in (dict(n_actions=0), dict(n_actions=256), dict(obs_dim=0), dict(critic_h2=0), dict(max_batch=0), dict(max_rounds=0)):
        for fn in (lib.prl_reinforce_actor_param_count, lib.prl_reinforce_critic_param_count, lib.prl_reinforce_workspace_bytes):
            assert fn(ctypes.byref(_cfg(**bad))) == -1, (fn, bad)
    assert lib.prl_reinforce_actor_param_count(ctypes.byref(_cfg(n_actions=255))) > 0
