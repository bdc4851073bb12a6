"""The IQL restatement (oracle/iql_oracle.py) against the recordings of the reference's
PearlAgent(ImplicitQLearning, BasicReplayBuffer) (tests/golden/iql_*.npz), the batched randint draw the CUDA learner
makes in place of the reference's single draws, and the plugin's class relation to / refusals of reference
configurations it does not implement."""
import importlib
import os
import sys
import types

import numpy as np
import pytest
import torch

from conftest import GOLDEN
from oracle.iql_oracle import OracleIQL
from oracle.pearl_oracle import flat

CASES = ("iql_discrete", "iql_continuous", "iql_lr", "iql_batch")


def make_oracle(fx):
    init = {k: fx[f"init_{k}"] for k in ("actor", "q1", "q2", "q1t", "q2t", "value")}
    h = tuple(int(x) for x in fx["hidden"])
    lrs = [float(x) for x in fx["lrs"]]
    act = dict(n_actions=int(fx["n_actions"])) if bool(fx["discrete"]) else dict(low=fx["low"], high=fx["high"])
    return OracleIQL(int(fx["obs"]), h, h, h, actor_lr=lrs[0], critic_lr=lrs[1], value_lr=lrs[2], gamma=float(fx["gamma"]),
                     tau=float(fx["tau"]), expectile=float(fx["expectile"]), temperature=float(fx["temperature"]),
                     advantage_clamp=float(fx["advantage_clamp"]), init=init, **act)


def batch_of(fx, idx):
    t = lambda k: torch.from_numpy(np.asarray(fx[k][idx]))  # noqa: E731
    return dict(state=t("state"), action=t("action"), reward=t("reward"), next_state=t("next_state"), terminated=t("terminated"))


@pytest.mark.parametrize("case", CASES)
def test_iql_oracle_reproduces_reference(case):
    torch.set_num_threads(1)
    fx = np.load(os.path.join(GOLDEN, f"{case}.npz"))
    orc = make_oracle(fx)
    n_rounds = len(fx["idx"])
    R = int(fx["rounds"])
    tol = dict(rtol=5e-6, atol=5e-7)
    clamped = 0
    for r in range(n_rounds):
        if not bool(fx["learn_batch"]) and r % R == 0:
            orc.set_learning_rates(*[float(x) for x in fx["call_lrs"][r // R]])
        b = batch_of(fx, fx["idx"][r])
        if case == "iql_discrete":
            with torch.no_grad():
                q = orc._qv(orc.qt[int(fx["bits"][r][1])], b["state"], orc._action_input(b["action"]))
                adv = torch.exp((q - orc.value(b["state"]).view(-1)) * orc.temperature)
            clamped += int((adv > orc.clamp).sum())
        out = orc.learn_batch(b, fx["bits"][r])
        for k in ("value_loss", "actor_loss", "critic_loss"):
            np.testing.assert_allclose(out[k], fx[k][r], rtol=5e-6, atol=1e-7, err_msg=f"round {r} {k}")
    if case == "iql_discrete":
        assert 0 < clamped < n_rounds * int(fx["batch"]), "advantage_clamp does not bind on some rows only"
    np.testing.assert_allclose(flat(orc.actor).numpy(), fx["actor_after"], **tol)
    np.testing.assert_allclose(flat(orc.value).numpy(), fx["value_after"], **tol)
    for i in range(2):
        np.testing.assert_allclose(flat(orc.q[i]).numpy(), fx[f"q{i + 1}_after"], **tol)
        np.testing.assert_allclose(flat(orc.qt[i]).numpy(), fx[f"q{i + 1}t_after"], **tol)
    vp = list(orc.value.parameters())
    for k in ("exp_avg", "exp_avg_sq", "max_exp_avg_sq"):
        got = torch.cat([orc.opt_value.state[p][k].reshape(-1) for p in vp]).numpy()
        np.testing.assert_allclose(got, fx[f"value_{k}"], **tol)
    assert float(orc.opt_value.state[vp[0]]["step"]) == float(fx["value_adam_step"]) == n_rounds


@pytest.mark.parametrize("r", [1, 2, 7, 5000])
def test_batched_randint_matches_single_draws(r):
    """The CUDA learner draws a chunk's bits as one torch.randint(0, 2, (r, 2)); the reference draws (1,) twice per round.
    Same bits in the same order, and the CPU generator ends in the same state."""
    g0 = torch.get_rng_state()
    try:
        torch.manual_seed(1234 + r)
        start = torch.get_rng_state()
        single = [int(torch.randint(0, 2, (1,)).item()) for _ in range(2 * r)]
        after_single = torch.get_rng_state()
        torch.set_rng_state(start)
        batched = torch.randint(0, 2, (r, 2)).reshape(-1).tolist()
        assert batched == single
        assert torch.equal(torch.get_rng_state(), after_single)
    finally:
        torch.set_rng_state(g0)


def test_recorded_bits_are_the_reference_draws():
    """The recorded bits are what one (rounds, 2) draw from the recorded CPU generator state yields."""
    for case in CASES:
        fx = np.load(os.path.join(GOLDEN, f"{case}.npz"))
        g0 = torch.get_rng_state()
        try:
            torch.set_rng_state(torch.from_numpy(fx["torch_rng_before"]))
            assert torch.randint(0, 2, (len(fx["bits"]), 2)).numpy().tolist() == fx["bits"].tolist(), case
            assert np.array_equal(torch.get_rng_state().numpy(), fx["torch_rng_after"]), case
        finally:
            torch.set_rng_state(g0)


def _stand_ins(monkeypatch):
    base = "pearl.policy_learners.sequential_decision_making."
    classes = {"ddpg": "DeepDeterministicPolicyGradient", "ppo": "ProximalPolicyOptimization",
               "soft_actor_critic_continuous": "ContinuousSoftActorCritic", "td3": "TD3", "soft_actor_critic": "SoftActorCritic",
               "implicit_q_learning": "ImplicitQLearning"}
    for p in ["pearl", "pearl.policy_learners", base[:-1]]:
        monkeypatch.setitem(sys.modules, p, types.ModuleType(p))
    for mod, cls in classes.items():
        m = types.ModuleType(base + mod)
        setattr(m, cls, type(cls, (), {}))
        monkeypatch.setitem(sys.modules, base + mod, m)
    return base


def test_plugin_subclasses_the_reference_when_importable(monkeypatch):
    """With Pearl importable, `B200ImplicitQLearning` is a subclass of the reference's ImplicitQLearning and of the CUDA
    plugin mixin, and overrides learn_batch.  Stand-in modules with the reference's module paths and class names are
    installed for the duration of the test."""
    import pearl_b200.actor_critic as ac
    base = _stand_ins(monkeypatch)
    try:
        importlib.reload(ac)
        assert ac.HAVE_REFERENCE and ac.HAVE_REFERENCE_IQL
        assert issubclass(ac.B200ImplicitQLearning, sys.modules[base + "implicit_q_learning"].ImplicitQLearning)
        assert issubclass(ac.B200ImplicitQLearning, ac._B200ActorCriticMixin)
        assert ac.B200ImplicitQLearning.learn_batch is not ac._B200ActorCriticMixin.learn_batch
    finally:
        monkeypatch.undo()
        importlib.reload(ac)
    if not ac.HAVE_REFERENCE_IQL:
        from pearl_b200.iql import B200ImplicitQLearning as Core
        assert ac.B200ImplicitQLearning is Core


def _named(name, base=torch.nn.Module):
    return type(name, (base,), {})


def _mlp(name, dims):
    m = _named(name)()
    m._model = torch.nn.Sequential(*[torch.nn.Linear(dims[i], dims[i + 1]) for i in range(len(dims) - 1)])
    return m


def _fake_learner(actor="VanillaActorNetwork", history="IdentityHistorySummarizationModule", value_opt=torch.optim.AdamW):
    """The attributes of a reference ImplicitQLearning that the plugin inspects (obs 5, 3 discrete actions, [16, 16])."""
    obs, A, h = 5, 3, 16
    pl = types.SimpleNamespace()
    pl._actor = _mlp(actor, [obs, h, h, A])
    critic = _named("TwinCritic")()
    critic._critic_1, critic._critic_2 = _mlp("VanillaQValueNetwork", [obs + A, h, h, 1]), _mlp("VanillaQValueNetwork", [obs + A, h, h, 1])
    pl._critic, pl._value_network = critic, _mlp("VanillaValueNetwork", [obs, h, h, 1])
    pl._is_action_continuous = False
    pl._history_summarization_module = _named(history)()
    pl._action_representation_module = _named("OneHotActionTensorRepresentationModule")()
    pl._actor_optimizer = torch.optim.AdamW(pl._actor.parameters(), lr=1e-3, amsgrad=True)
    pl._critic_optimizer = torch.optim.AdamW(critic.parameters(), lr=1e-3, amsgrad=True)
    pl._value_network_optimizer = value_opt(pl._value_network.parameters(), lr=1e-3, **({"amsgrad": True} if value_opt is torch.optim.AdamW else {}))
    return pl


def test_plugin_refuses_configurations_it_does_not_implement(monkeypatch):
    """A Gaussian actor, a non-identity history summarization module and a value optimizer that is not AdamW(amsgrad)
    are each refused with NotImplementedError before anything reaches the GPU; the supported configuration passes the
    checks and yields the core's arguments."""
    import pearl_b200.actor_critic as ac
    kw = ac._iql_core_kwargs(_fake_learner())
    assert kw == dict(state_dim=5, actor_hidden_dims=[16, 16], critic_hidden_dims=[16, 16], value_critic_hidden_dims=[16, 16], n_actions=3)
    with pytest.raises(NotImplementedError, match="GaussianActorNetwork"):
        ac._iql_core_kwargs(_fake_learner(actor="GaussianActorNetwork"))
    with pytest.raises(NotImplementedError, match="IdentityHistorySummarizationModule"):
        ac._iql_core_kwargs(_fake_learner(history="LSTMHistorySummarizationModule"))
    base = _stand_ins(monkeypatch)
    del base
    try:
        importlib.reload(ac)
        pl = ac.B200ImplicitQLearning.__new__(ac.B200ImplicitQLearning)
        for k, v in vars(_fake_learner(value_opt=torch.optim.Adam)).items():
            setattr(pl, k, v)
        pl._critic_soft_update_tau, pl._discount_factor, pl._training_rounds, pl._batch_size = 0.05, 0.99, 5, 128
        pl._expectile, pl._temperature_advantage_weighted_regression, pl._advantage_clamp = 0.5, 0.5, 100.0
        pl._b200_opts = {}
        with pytest.raises(NotImplementedError, match="value optimizer"):
            pl._make_core(torch.device("cpu"))
    finally:
        monkeypatch.undo()
        importlib.reload(ac)
