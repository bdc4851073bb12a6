"""The conservative DQN restatement (oracle/cql_oracle.py) against the recordings of the reference's
PearlAgent(DeepQLearning / DoubleDQN with is_conservative=True, BasicReplayBuffer) (tests/golden/cql_*.npz), its
hand-written CQL gradient against torch.autograd, and the plugin's construction and refusals on the CPU."""
import os
import random

import numpy as np
import pytest
import torch

from conftest import GOLDEN
from oracle.cql_oracle import OracleCQL, cql_grad, cql_term, one_hot_batch
from oracle.pearl_oracle import flat

CASES = ("cql_dqn", "cql_ddqn", "cql_lr", "cql_batch")


def max_exp_avg_sq(fx):
    """The recording stores max_exp_avg_sq where it differs from exp_avg_sq only."""
    v = fx["adam_exp_avg_sq"].copy()
    v[fx["adam_max_exp_avg_sq_idx"]] = fx["adam_max_exp_avg_sq_val"]
    return v


def batch_of(fx, idx):
    """Rows idx as preprocess_batch hands them to learn_batch: one-hot actions, padded one-hot current and next slots."""
    g = lambda k: np.asarray(fx[k][idx])  # noqa: E731
    return one_hot_batch(int(fx["n_actions"]), torch.from_numpy(g("state")), g("action"), torch.from_numpy(g("reward")),
                         torch.from_numpy(g("next_state")), torch.from_numpy(g("terminated")), g("curr_ids").astype(np.int64),
                         g("next_ids").astype(np.int64), g("next_count"))


@pytest.mark.parametrize("case", CASES)
def test_cql_oracle_reproduces_reference(case):
    torch.set_num_threads(1)
    fx = np.load(os.path.join(GOLDEN, f"{case}.npz"))
    n, B, R = int(fx["n"]), int(fx["batch"]), int(fx["rounds"])
    st = random.getstate()
    try:
        random.setstate((3, tuple(int(x) for x in fx["rng_before"]), None))
        assert [random.sample(range(n), B) for _ in range(len(fx["idx"]))] == fx["idx"].tolist()
        assert random.getstate()[1] == tuple(int(x) for x in fx["rng_after"])
    finally:
        random.setstate(st)
    orc = OracleCQL(int(fx["obs"]), int(fx["n_actions"]), fx["hidden"].tolist(), lr=float(fx["lr"]), gamma=float(fx["gamma"]),
                    tau=float(fx["tau"]), double=bool(fx["double"]), target_update_freq=int(fx["target_update_freq"]),
                    init_q=fx["init_q"], alpha=float(fx["alpha"]))
    tol = dict(rtol=5e-6, atol=5e-7)
    per_call = 1 if bool(fx["learn_batch"]) else R
    for r in range(len(fx["idx"])):
        if r % per_call == 0:
            orc.opt.param_groups[0]["lr"] = float(fx["call_lr"][r // per_call])
            orc.alpha = float(fx["call_alpha"][r // per_call])
        if not bool(fx["learn_batch"]):
            orc.training_steps += 1              # PolicyLearner.learn counts the round first; agent.learn_batch does not
        loss = orc.learn_batch(batch_of(fx, fx["idx"][r]))
        np.testing.assert_allclose(loss, fx["loss"][r], rtol=5e-6, atol=1e-7, err_msg=f"round {r}")
        if (r + 1) % per_call == 0:
            c = r // per_call
            np.testing.assert_allclose(flat(orc.Q).numpy(), fx["q_calls"][c], err_msg=f"online net after call {c}", **tol)
            np.testing.assert_allclose(flat(orc.Qt).numpy(), fx["qt_calls"][c], err_msg=f"target net after call {c}", **tol)
    params = list(orc.Q.parameters())
    for k, want in (("exp_avg", fx["adam_exp_avg"]), ("exp_avg_sq", fx["adam_exp_avg_sq"]), ("max_exp_avg_sq", max_exp_avg_sq(fx))):
        got = torch.cat([orc.opt.state[p][k].reshape(-1) for p in params]).numpy()
        np.testing.assert_allclose(got, want, err_msg=k, **tol)
    assert float(orc.opt.state[params[0]]["step"]) == float(fx["adam_step"]) == len(fx["idx"])


def test_recordings_exercise_the_reference_quirks():
    """The target update fires inside and across learn() calls; lr and alpha change in cql_lr; cql_batch samples padded
    current slots; and wherever A > 2 the reference's data term differs from the taken-action term."""
    fx = {c: np.load(os.path.join(GOLDEN, f"{c}.npz")) for c in CASES}
    d = fx["cql_dqn"]
    steps = [s for s in range(1, int(d["rounds"]) * int(d["calls"]) + 1) if (s + 1) % int(d["target_update_freq"]) == 0]
    assert any(s <= int(d["rounds"]) for s in steps) and any(s > int(d["rounds"]) for s in steps)
    assert (int(d["obs"]), int(d["n_actions"]), d["hidden"].tolist(), int(d["batch"]), float(d["alpha"])) == (4, 2, [64, 64], 32, 2.0)
    assert bool(fx["cql_ddqn"]["double"]) and bool(fx["cql_ddqn"]["dynamic"]) and float(fx["cql_ddqn"]["alpha"]) == 8.0
    lr = fx["cql_lr"]
    assert lr["call_lr"][0] != lr["call_lr"][1] and lr["call_alpha"][0] != lr["call_alpha"][1]
    b = fx["cql_batch"]
    assert bool(b["learn_batch"]) and int(b["padded"]) > 0 and (b["curr_count"][b["idx"]] < int(b["n_actions"])).any()
    for c in ("cql_ddqn", "cql_lr", "cql_batch"):
        assert int(fx[c]["n_actions"]) > 2 and float(fx[c]["term_gap"]) > 1e-3


@pytest.mark.parametrize("A", [2, 5])
def test_hand_written_cql_gradient_equals_autograd(A):
    """cql_grad against torch.autograd of alpha * compute_cql_loss's expression, float64; the gradient does not depend on
    the taken action (the one-hot gather reads columns 0 and 1)."""
    g = torch.Generator().manual_seed(A)
    B, alpha = 7, 3.5
    q_all = (torch.randn(B, A, generator=g, dtype=torch.float64) * 2).requires_grad_(True)
    acts = torch.randint(0, A, (B,), generator=g)
    (alpha * cql_term(q_all, torch.nn.functional.one_hot(acts, A).double())).backward()
    np.testing.assert_allclose(cql_grad(q_all.detach(), alpha).numpy(), q_all.grad.numpy(), rtol=1e-12, atol=1e-15)
    other = (acts + 1) % A
    q2 = q_all.detach().clone().requires_grad_(True)
    (alpha * cql_term(q2, torch.nn.functional.one_hot(other, A).double())).backward()
    assert torch.equal(q2.grad, q_all.grad)


def _space(A):
    class Space:
        n = A
        actions = [torch.tensor([i]) for i in range(A)]
        actions_batch = torch.arange(A).view(A, 1)
    return Space()


def _make(cls_name="B200DeepQLearning", A=3, **kw):
    import pearl_b200
    cls = getattr(pearl_b200, cls_name)
    return cls(state_dim=4, action_space=_space(A), hidden_dims=[16, 16], batch_size=8,
               action_representation_module=pearl_b200.OneHotActionTensorRepresentationModule(A), **kw)


@pytest.mark.parametrize("cls_name", ["B200DeepQLearning", "B200DoubleDQN"])
def test_conservative_construction(cls_name):
    """is_conservative=True constructs (it used to raise NotImplementedError) and keeps alpha where learn() reads it; the
    configurations the conservative learner does not run, or the reference rejects, are refused at construction."""
    pl = _make(cls_name, is_conservative=True, conservative_alpha=8.0)
    assert pl._conservative and pl._conservative_alpha == 8.0 and pl._double == (cls_name == "B200DoubleDQN")
    assert not _make(cls_name)._conservative
    with pytest.raises(ValueError, match="conservative_alpha"):
        _make(cls_name, is_conservative=True, conservative_alpha=None)
    with pytest.raises(ValueError, match="2 actions"):
        _make(cls_name, A=1, is_conservative=True)
    with pytest.raises(NotImplementedError, match="tc"):
        _make(cls_name, is_conservative=True, engine="tc")
    _make(cls_name, is_conservative=True, engine="simt")
    import pearl_b200
    with pytest.raises(NotImplementedError):
        pearl_b200.B200LearnerGroup([pl], [object()])
    with pytest.raises(NotImplementedError):
        pl.set_communicator(None)
