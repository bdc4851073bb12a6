"""The QR-DQN restatement (oracle/qrdqn_oracle.py) against the recordings of the reference's
PearlAgent(QuantileRegressionDeepQLearning, BasicReplayBuffer) (tests/golden/qrdqn_*.npz), its hand-written gradient
against torch.autograd, and the plugin's class relation to / refusals of reference configurations it does not implement."""
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
from oracle.qrdqn_oracle import OracleQRDQN, quantile_grad, quantile_loss

CASES = ("qrdqn_neutral", "qrdqn_variance", "qrdqn_lr", "qrdqn_batch")


def max_exp_avg_sq(fx):
    """The recording stores max_exp_avg_sq where it differs from exp_avg_sq only."""
    v = fx["adam_exp_avg_sq"].copy()
    v[fx["adam_max_exp_avg_sq_idx"]] = fx["adam_max_exp_avg_sq_val"]
    return v


def batch_of(fx, idx):
    t = lambda k: torch.from_numpy(np.asarray(fx[k][idx]))  # noqa: E731
    A = int(fx["n_actions"])
    return dict(state=t("state"), action=t("action"), reward=t("reward"), next_state=t("next_state"), terminated=t("terminated"),
                next_ids=t("next_ids").long(), next_mask=torch.arange(A).view(1, A) >= t("next_count").view(-1, 1))


def update_flags(fx):
    """Per round: does the reference soft-update the target after the step?  PolicyLearner.learn counts the round before
    learn_batch checks (training_steps + 1) % freq; agent.learn_batch leaves the count at 0."""
    freq, n = int(fx["target_update_freq"]), len(fx["idx"])
    if bool(fx["learn_batch"]):
        return [(0 + 1) % freq == 0] * n
    return [(r + 2) % freq == 0 for r in range(n)]


@pytest.mark.parametrize("case", CASES)
def test_qrdqn_oracle_reproduces_reference(case):
    torch.set_num_threads(1)
    fx = np.load(os.path.join(GOLDEN, f"{case}.npz"))
    n, B, R = int(fx["n"]), int(fx["batch"]), int(fx["rounds"])
    # indices: what CPython's random.sample draws from the recorded state, which it leaves as recorded
    st = random.getstate()
    try:
        random.setstate((3, tuple(int(x) for x in fx["rng_before"]), None))
        assert [random.sample(range(n), B) for _ in range(len(fx["idx"]))] == fx["idx"].tolist()
        assert random.getstate()[1] == tuple(int(x) for x in fx["rng_after"])
    finally:
        random.setstate(st)
    orc = OracleQRDQN(int(fx["obs"]), int(fx["n_actions"]), fx["hidden"].tolist(), int(fx["num_quantiles"]), lr=float(fx["lr"]),
                      gamma=float(fx["gamma"]), tau=float(fx["tau"]), init=fx["init_q"])
    tol = dict(rtol=5e-6, atol=5e-7)
    flags = update_flags(fx)
    per_call = 1 if bool(fx["learn_batch"]) else R
    assert any(flags) and (bool(fx["learn_batch"]) or not all(flags))
    for r in range(len(fx["idx"])):
        if r % per_call == 0:
            orc.set_learning_rate(float(fx["call_lr"][r // per_call]))
        loss = orc.learn_batch(batch_of(fx, fx["idx"][r]), float(fx["beta"]), flags[r])
        np.testing.assert_allclose(loss, fx["loss"][r], rtol=5e-6, atol=1e-7, err_msg=f"round {r}")
        if (r + 1) % per_call == 0:
            c = r // per_call
            np.testing.assert_allclose(flat(orc.q).numpy(), fx["q_calls"][c], err_msg=f"online net after call {c}", **tol)
            np.testing.assert_allclose(flat(orc.qt).numpy(), fx["qt_calls"][c], err_msg=f"target net after call {c}", **tol)
    params = list(orc.q.parameters())
    for k, want in (("exp_avg", fx["adam_exp_avg"]), ("exp_avg_sq", fx["adam_exp_avg_sq"]), ("max_exp_avg_sq", max_exp_avg_sq(fx))):
        got = torch.cat([orc.opt.state[p][k].reshape(-1) for p in params]).numpy()
        np.testing.assert_allclose(got, want, err_msg=k, **tol)
    assert float(orc.opt.state[params[0]]["step"]) == float(fx["adam_step"]) == len(fx["idx"])


def test_variance_recording_exercises_the_risk_metric():
    """In the mean-variance recording beta changes the greedy slot of some rows, and some next slots are masked."""
    fx = np.load(os.path.join(GOLDEN, "qrdqn_variance.npz"))
    assert float(fx["beta"]) == 2.0 and int(fx["flipped"]) > 0
    assert bool(fx["dynamic"]) and (fx["next_count"][fx["idx"]] < int(fx["n_actions"])).any()


@pytest.mark.parametrize("N", [1, 7, 32])
def test_hand_written_gradient_equals_autograd(N):
    """quantile_grad against torch.autograd of the reference's loss, in float64, on inputs that hit both Huber branches
    and exact ties at u = 0."""
    g = torch.Generator().manual_seed(N)
    B = 9
    theta = (torch.randn(B, N, generator=g, dtype=torch.float64) * 1.5)
    target = torch.randn(B, N, generator=g, dtype=torch.float64) * 1.5
    target[0, :] = theta[0, 0]                   # u = 0 for theta_0 against every target of row 0
    target[1, 0] = theta[1, -1]
    theta.requires_grad_(True)
    u = (target.unsqueeze(2) - theta.detach().unsqueeze(1)).abs()
    assert bool((u <= 1).any()) and bool((u > 1).any()) and bool((u == 0).any())
    quantile_loss(theta, target).backward()
    np.testing.assert_allclose(quantile_grad(theta.detach(), target).numpy(), theta.grad.numpy(), rtol=1e-12, atol=1e-15)


def _stand_ins(monkeypatch):
    base = "pearl.policy_learners.sequential_decision_making."
    classes = {"ddpg": "DeepDeterministicPolicyGradient", "ppo": "ProximalPolicyOptimization",
               "soft_actor_critic_continuous": "ContinuousSoftActorCritic", "td3": "TD3", "soft_actor_critic": "SoftActorCritic",
               "implicit_q_learning": "ImplicitQLearning", "quantile_regression_deep_q_learning": "QuantileRegressionDeepQLearning"}
    for p in ["pearl", "pearl.policy_learners", base[:-1]]:
        monkeypatch.setitem(sys.modules, p, types.ModuleType(p))
    for mod, cls in classes.items():
        m = types.ModuleType(base + mod)
        setattr(m, cls, type(cls, (), {}))
        monkeypatch.setitem(sys.modules, base + mod, m)
    return base


def test_plugin_subclasses_the_reference_when_importable(monkeypatch):
    """With Pearl importable, `B200QuantileRegressionDeepQLearning` subclasses the reference's
    QuantileRegressionDeepQLearning and overrides learn and learn_batch.  Stand-in modules with the reference's module
    paths and class names are installed for the duration of the test."""
    import pearl_b200.actor_critic as ac
    base = _stand_ins(monkeypatch)
    try:
        importlib.reload(ac)
        assert ac.HAVE_REFERENCE_QRDQN
        ref = sys.modules[base + "quantile_regression_deep_q_learning"].QuantileRegressionDeepQLearning
        assert issubclass(ac.B200QuantileRegressionDeepQLearning, ref)
        assert "learn" in vars(ac.B200QuantileRegressionDeepQLearning) and "learn_batch" in vars(ac.B200QuantileRegressionDeepQLearning)
    finally:
        monkeypatch.undo()
        importlib.reload(ac)
    if not ac.HAVE_REFERENCE_QRDQN:
        from pearl_b200.qrdqn import B200QuantileRegressionDeepQLearning as Core
        assert ac.B200QuantileRegressionDeepQLearning is Core


def _named(name, base=torch.nn.Module):
    return type(name, (base,), {})


class _QuantileNet(torch.nn.Module):
    def __init__(self, dims, layer_norm=False):
        super().__init__()
        layers = []
        for i in range(len(dims) - 1):
            layers.append(torch.nn.Linear(dims[i], dims[i + 1]))
            if layer_norm and i < len(dims) - 2:
                layers.append(torch.nn.LayerNorm(dims[i + 1]))
        self._model = torch.nn.Sequential(*layers)
        self.state_dim, self.action_dim, self.num_quantiles = dims[0] - 3, 3, dims[-1]


def _fake_learner(net="QuantileQValueNetwork", hidden=(16, 16), layer_norm=False, history="IdentityHistorySummarizationModule",
                  arm="OneHotActionTensorRepresentationModule", optimizer="amsgrad", safety="RiskNeutralSafetyModule"):
    """The attributes of a reference QuantileRegressionDeepQLearning that the plugin inspects (obs 5, 3 actions, N 8)."""
    obs, A, N = 5, 3, 8
    pl = types.SimpleNamespace()
    pl._Q = type(net, (_QuantileNet,), {})([obs + A] + list(hidden) + [N], layer_norm)
    pl._action_space = types.SimpleNamespace(n=A)
    pl._history_summarization_module = _named(history)()
    pl._action_representation_module = _named(arm)()
    pl.safety_module = _named(safety)()
    pl.safety_module._beta = 0.5
    if optimizer == "amsgrad":
        pl._optimizer = torch.optim.AdamW(pl._Q.parameters(), lr=1e-3, amsgrad=True)
        pl._optimizer.add_param_group({"params": []})        # set_history_summarization_module(identity)
    elif optimizer == "adamw":
        pl._optimizer = torch.optim.AdamW(pl._Q.parameters(), lr=1e-3)
    else:
        pl._optimizer = torch.optim.Adam(pl._Q.parameters(), lr=1e-3)
    return pl


def test_plugin_refuses_configurations_it_does_not_implement():
    """Each configuration the CUDA learner does not implement is refused with NotImplementedError before anything reaches
    the GPU; the supported configuration passes the checks and yields the core's arguments."""
    import pearl_b200.actor_critic as ac
    assert ac._qrdqn_core_kwargs(_fake_learner()) == dict(state_dim=5, n_actions=3, hidden_dims=[16, 16], num_quantiles=8)
    assert ac._qrdqn_adamw_lr(_fake_learner()._optimizer) == 1e-3
    assert ac._qrdqn_beta(_fake_learner().safety_module) == 0.0
    assert ac._qrdqn_beta(None) == 0.0
    assert ac._qrdqn_beta(_fake_learner(safety="QuantileNetworkMeanVarianceSafetyModule").safety_module) == 0.5
    refused = [dict(hidden=(16,)), dict(hidden=(16, 16, 16)), dict(layer_norm=True), dict(net="DuelingQValueNetwork"),
               dict(arm="BinaryActionTensorRepresentationModule"), dict(history="LSTMHistorySummarizationModule"),
               dict(safety="IdentitySafetyModule")]
    for kw in refused:
        with pytest.raises(NotImplementedError):
            ac._qrdqn_core_kwargs(_fake_learner(**kw))
    for opt in ("adamw", "adam"):
        with pytest.raises(NotImplementedError, match="AdamW"):
            ac._qrdqn_adamw_lr(_fake_learner(optimizer=opt)._optimizer)
    pl = _fake_learner()
    pl._optimizer.param_groups[1]["params"].append(torch.nn.Parameter(torch.zeros(2)))   # a history module with parameters
    with pytest.raises(NotImplementedError):
        ac._qrdqn_adamw_lr(pl._optimizer)
