"""DeepSARSA on the CPU: the restatement (oracle/sarsa_oracle.py) against the recordings of the reference's
PearlAgent(DeepSARSA, SARSAReplayBuffer) (tests/golden/sarsa_*.npz), the product's host-side delayed-push state machine
(pearl_b200.sarsa_buffer.SarsaPushCache) against the recorded push-to-append sequence, the float64 step against
autograd, and the plugin's construction-time refusals."""
import os
import random

import numpy as np
import pytest
import torch

from conftest import GOLDEN
from oracle.pearl_oracle import flat
from oracle.sarsa_fp64 import sarsa_step
from oracle.sarsa_oracle import OracleSARSA, OracleSARSABuffer, one_hot

CASES = ("sarsa_method", "sarsa_steps", "sarsa_lr", "sarsa_batch")


def load(case):
    return np.load(os.path.join(GOLDEN, f"{case}.npz"))


def max_exp_avg_sq(fx):
    v = fx["adam_exp_avg_sq"].copy()
    v[fx["adam_max_exp_avg_sq_idx"]] = fx["adam_max_exp_avg_sq_val"]
    return v


def appended(fx):
    """The recorded appends as (push, state, action, reward, next_state, next_action, terminated, truncated) rows."""
    return [(int(fx["app_push"][j]), fx["app_state"][j].tolist(), int(fx["app_action"][j]), float(fx["app_reward"][j]),
             fx["app_next_state"][j].tolist(), int(fx["app_next_action"][j]), bool(fx["app_terminated"][j]),
             bool(fx["app_truncated"][j])) for j in range(len(fx["app_push"]))]


def push_args(fx, i):
    return (fx["push_state"][i], int(fx["push_action"][i]), float(fx["push_reward"][i]), bool(fx["push_terminated"][i]),
            bool(fx["push_truncated"][i]), fx["push_next_state"][i])


@pytest.mark.parametrize("case", CASES)
def test_sarsa_oracle_reproduces_reference(case):
    torch.set_num_threads(1)
    fx = load(case)
    orc = OracleSARSA(int(fx["obs"]), int(fx["n_actions"]), fx["hidden"].tolist(), lr=float(fx["lr"]), gamma=float(fx["gamma"]),
                      tau=float(fx["tau"]), target_update_freq=int(fx["target_update_freq"]), init_q=fx["init_q"],
                      batch_size=int(fx["batch"]), training_rounds=int(fx["rounds"]))
    buf = OracleSARSABuffer(int(fx["capacity"]))
    learn_after = set(fx["learn_after"].tolist())
    st = random.getstate()
    tol = dict(rtol=5e-6, atol=5e-7)
    losses, got_app, calls = [], [], 0
    try:
        random.setstate((3, tuple(int(x) for x in fx["rng_before"]), None))
        for i in range(len(fx["push_action"])):
            for t in buf.push(*push_args(fx, i)):
                got_app.append((i, t[0].tolist(), t[1], t[2], t[3].tolist(), t[4], t[5], t[6]))
            if i in learn_after:
                orc.opt.param_groups[0]["lr"] = float(fx["call_lr"][calls])
                losses += orc.learn(buf).get("loss", [])
                np.testing.assert_allclose(flat(orc.Q).numpy(), fx["q_calls"][calls], err_msg=f"online after call {calls}", **tol)
                np.testing.assert_allclose(flat(orc.Qt).numpy(), fx["qt_calls"][calls], err_msg=f"target after call {calls}", **tol)
                calls += 1
        for c in range(len(fx["q_calls"]) - calls):          # agent.learn_batch(buf.sample(batch)): no step count
            losses.append(orc.learn_batch(one_hot(buf.sample(int(fx["batch"])), orc.A)))
            np.testing.assert_allclose(flat(orc.Q).numpy(), fx["q_calls"][c], err_msg=f"online after batch {c}", **tol)
            np.testing.assert_allclose(flat(orc.Qt).numpy(), fx["qt_calls"][c], err_msg=f"target after batch {c}", **tol)
        assert random.getstate()[1] == tuple(int(x) for x in fx["rng_after"])
    finally:
        random.setstate(st)
    assert got_app == appended(fx)
    np.testing.assert_allclose(losses, fx["loss"], rtol=5e-6, atol=1e-7)
    params = list(orc.Q.parameters())
    for k, want in (("exp_avg", fx["adam_exp_avg"]), ("exp_avg_sq", fx["adam_exp_avg_sq"]), ("max_exp_avg_sq", max_exp_avg_sq(fx))):
        got = torch.cat([orc.opt.state[p][k].reshape(-1) for p in params]).numpy()
        np.testing.assert_allclose(got, want, err_msg=k, **tol)
    assert float(orc.opt.state[params[0]]["step"]) == float(fx["adam_step"]) == len(fx["loss"])


@pytest.mark.parametrize("case", CASES)
def test_push_cache_reproduces_recorded_appends(case):
    """The product's host-side state machine releases exactly the transitions the reference appended, push by push, in
    order, with their next actions: the stale-cache append of sarsa_steps included."""
    from pearl_b200.sarsa_buffer import SarsaPushCache
    fx = load(case)
    cache, got = SarsaPushCache(), []
    for i in range(len(fx["push_action"])):
        s, a, r, te, tr, ns = push_args(fx, i)
        for t in cache.step(s, a, r, te, tr, ns):
            got.append((i, t["state"].tolist(), t["action"], float(np.float32(t["reward"])), t["next_state"].tolist(),
                        t["next_action"], t["terminated"], t["truncated"]))
    assert got == appended(fx)


def test_recordings_exercise_the_reference_quirks():
    """Target updates inside and across calls; terminated and truncated rows; clamped on-policy batches; the stale
    cache appended again after an episode end; an lr change; learn_batch without a step count."""
    m = load("sarsa_method")
    assert (int(m["obs"]), int(m["n_actions"]), m["hidden"].tolist(), int(m["batch"]), int(m["rounds"])) == (4, 2, [64, 64], 32, 1)
    assert m["app_terminated"].any() and m["app_truncated"].any()
    assert not (m["app_terminated"] & m["app_truncated"]).any()        # truncated rows are stored with terminated False
    steps = [s for s in range(1, len(m["loss"]) + 1) if (s + 1) % int(m["target_update_freq"]) == 0]
    assert steps and len(m["call_batch"]) > 1
    s = load("sarsa_steps")
    assert bool(s["dynamic"]) and s["call_batch"].max() <= 2 and (s["call_batch"] == 0).any()
    pushes = s["app_push"].tolist()
    assert len(pushes) > len(set(pushes))                               # one push released two transitions: the stale cache
    first = [j for j in range(len(pushes)) if pushes.count(pushes[j]) > 1][0]
    p = pushes[first]
    assert np.array_equal(s["app_next_state"][first], s["push_state"][p])
    lr = load("sarsa_lr")
    assert lr["call_lr"][0] != lr["call_lr"][1]
    b = load("sarsa_batch")
    assert bool(b["learn_batch"]) and int(b["target_update_freq"]) == 1


def test_sarsa_step_matches_float64_autograd():
    g = torch.Generator().manual_seed(3)
    obs, A, H, B, gamma = 7, 5, (11, 9), 13, 0.9
    D = obs + A
    P = H[0] * D + H[0] + H[1] * H[0] + H[1] + H[1] + 1
    w, wt = torch.randn(P, generator=g, dtype=torch.float64) * 0.4, torch.randn(P, generator=g, dtype=torch.float64) * 0.4
    batch = dict(state=torch.randn(B, obs, generator=g, dtype=torch.float64), action=torch.randint(0, A, (B,), generator=g),
                 reward=torch.randn(B, generator=g, dtype=torch.float64), terminated=(torch.rand(B, generator=g) < 0.3).double(),
                 next_state=torch.randn(B, obs, generator=g, dtype=torch.float64), next_action=torch.randint(0, A, (B,), generator=g))
    val, _ = sarsa_step(w, wt, batch, obs, A, gamma, H)
    net = OracleSARSA(obs, A, list(H), gamma=gamma)
    net.Q, net.Qt = net.Q.double(), net.Qt.double()
    with torch.no_grad():
        off = 0
        for p in net.Q.parameters():
            p.copy_(w[off:off + p.numel()].view_as(p)); off += p.numel()
        off = 0
        for p in net.Qt.parameters():
            p.copy_(wt[off:off + p.numel()].view_as(p)); off += p.numel()
    oh = lambda x: torch.nn.functional.one_hot(x, A).double()  # noqa: E731
    b = dict(batch, action=oh(batch["action"]), next_action=oh(batch["next_action"]), terminated=batch["terminated"].bool())
    q = net._q_values(net.Q, b["state"], b["action"])
    y = net._next_values(b) * gamma * (1 - b["terminated"].double()) + b["reward"]
    loss = torch.nn.MSELoss()(q, y)
    loss.backward()
    grad = torch.cat([p.grad.reshape(-1) for p in net.Q.parameters()])
    np.testing.assert_allclose(val["grad"].numpy(), grad.numpy(), rtol=1e-12, atol=1e-14)
    np.testing.assert_allclose(float(val["loss"]), float(loss.detach()), rtol=1e-13)
    np.testing.assert_allclose(float(val["mae"]), float((q - y).abs().mean()), rtol=1e-13)


def _space(A):
    class Space:
        n = A
        actions = [torch.tensor([i]) for i in range(A)]
        actions_batch = torch.arange(A).view(A, 1)
    return Space()


def test_sarsa_construction_and_refusals():
    """B200DeepSARSA is on-policy with EGreedyExploration(0.05) by default; the configurations the CUDA learner does not
    run are refused at construction."""
    import pearl_b200
    mk = lambda A=3, **kw: pearl_b200.B200DeepSARSA(  # noqa: E731
        state_dim=4, action_space=_space(A), hidden_dims=[16, 16], batch_size=8,
        action_representation_module=pearl_b200.OneHotActionTensorRepresentationModule(A), **kw)
    pl = mk()
    assert pl.on_policy and pl._sarsa and not pl._conservative and not pl._dueling
    assert type(pl.exploration_module).__name__ == "EGreedyExploration"
    eps = getattr(pl.exploration_module, "curr_epsilon", getattr(pl.exploration_module, "epsilon", None))
    assert eps == 0.05
    with pytest.raises(NotImplementedError, match="tc"):
        mk(engine="tc")
    with pytest.raises(NotImplementedError, match="conservative"):
        mk(is_conservative=True)
    with pytest.raises(NotImplementedError, match="Dueling"):
        mk(network_type=pearl_b200.DuelingQValueNetwork)
    with pytest.raises(NotImplementedError):
        mk(optimizer=torch.optim.SGD(torch.nn.Linear(1, 1).parameters(), lr=0.1))._adam_hparams()
    with pytest.raises(NotImplementedError):
        pearl_b200.B200LearnerGroup([pl], [object()])
    with pytest.raises(NotImplementedError):
        pl.set_communicator(None)
    with pytest.raises(NotImplementedError):
        pearl_b200.B200DeepSARSA(state_dim=4, action_space=_space(3), hidden_dims=[16, 16, 16],
                                 action_representation_module=pearl_b200.OneHotActionTensorRepresentationModule(3))
    with pytest.raises(AssertionError, match="next action"):
        pl.learn_batch(pearl_b200.TransitionBatch(state=torch.zeros(2, 4), action=torch.zeros(2, 1), reward=torch.zeros(2),
                                                  next_state=torch.zeros(2, 4)))
