"""The dueling DQN restatement (oracle/dueling_oracle.py) against the recordings of the reference's
PearlAgent(DeepQLearning / DoubleDQN with DuelingQValueNetwork, BasicReplayBuffer) (tests/golden/duel_*.npz), its
hand-written advantage-slot gradient against torch.autograd, the stand-in DuelingQValueNetwork's state_dict, and the
plugin's construction and refusals on the CPU."""
import os
import random

import numpy as np
import pytest
import torch

from conftest import GOLDEN
from oracle.dueling_oracle import OracleDueling, get_q_values, one_hot_batch, slot_grad
from oracle.pearl_oracle import flat, load_flat

CASES = ("duel_dqn", "duel_ddqn", "duel_lr", "duel_batch")


def max_exp_avg_sq(fx):
    """The recording stores max_exp_avg_sq where it differs from exp_avg_sq only."""
    v = fx["adam_exp_avg_sq"].copy()
    v[fx["adam_max_exp_avg_sq_idx"]] = fx["adam_max_exp_avg_sq_val"]
    return v


def batch_of(fx, idx, curr=True):
    """Rows idx as preprocess_batch hands them to learn_batch: one-hot actions, padded one-hot current and next slots;
    curr=False: the batch has no current sets."""
    g = lambda k: np.asarray(fx[k][idx])  # noqa: E731
    b = one_hot_batch(int(fx["n_actions"]), torch.from_numpy(g("state")), g("action"), torch.from_numpy(g("reward")),
                      torch.from_numpy(g("next_state")), torch.from_numpy(g("terminated")), g("curr_ids").astype(np.int64),
                      g("next_ids").astype(np.int64), g("next_count"))
    if not curr:
        b["curr_available_actions"] = None
    return b


@pytest.mark.parametrize("case", CASES)
def test_dueling_oracle_reproduces_reference(case):
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
    orc = OracleDueling(int(fx["obs"]), int(fx["n_actions"]), fx["hidden"].tolist(), lr=float(fx["lr"]), gamma=float(fx["gamma"]),
                        tau=float(fx["tau"]), double=bool(fx["double"]), target_update_freq=int(fx["target_update_freq"]),
                        init_q=fx["init_q"])
    tol = dict(rtol=5e-6, atol=5e-7)
    lb = bool(fx["learn_batch"])
    per_call = 1 if lb else R
    for r in range(len(fx["idx"])):
        if r % per_call == 0:
            orc.opt.param_groups[0]["lr"] = float(fx["call_lr"][r // per_call])
        if not lb:
            orc.training_steps += 1              # PolicyLearner.learn counts the round first; agent.learn_batch does not
        loss = orc.learn_batch(batch_of(fx, fx["idx"][r], curr=bool(fx["call_curr"][r]) if lb else True))
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


def test_dueling_oracle_reproduces_act_recording():
    """act(exploit=True) picks the first argmax of get_q_values over the available set, whose advantage mean runs over that
    set only."""
    fx = np.load(os.path.join(GOLDEN, "duel_act.npz"))
    A = int(fx["n_actions"])
    orc = OracleDueling(int(fx["obs"]), A, fx["hidden"].tolist(), init_q=fx["init_q"])
    for i in range(int(fx["n"])):
        m = int(fx["avail_count"][i])
        ids = fx["avail_ids"][i, :m].astype(np.int64)
        q = orc.q_values(torch.from_numpy(fx["state"][i]).view(1, -1), ids.reshape(1, -1))[0]
        np.testing.assert_allclose(q.numpy(), fx["values"][i, :m], rtol=5e-6, atol=5e-7, err_msg=f"row {i}")
        assert int(ids[int(torch.argmax(q))]) == int(fx["chosen"][i])


def test_recordings_exercise_the_reference_quirks():
    """The target update fires inside and across learn() calls; the lr changes in duel_lr; duel_batch samples padded
    current slots and has a call without current sets; the dynamic recordings tell the all-slot advantage mean from the
    available-slot one, and duel_act the available-set mean from the all-action one."""
    fx = {c: np.load(os.path.join(GOLDEN, f"{c}.npz")) for c in CASES + ("duel_act",)}
    d = fx["duel_dqn"]
    steps = [s for s in range(1, int(d["rounds"]) * int(d["calls"]) + 1) if (s + 1) % int(d["target_update_freq"]) == 0]
    assert any(s <= int(d["rounds"]) for s in steps) and any(s > int(d["rounds"]) for s in steps)
    assert (int(d["obs"]), int(d["n_actions"]), d["hidden"].tolist(), int(d["batch"])) == (4, 2, [64, 64], 32)
    assert bool(fx["duel_ddqn"]["double"]) and bool(fx["duel_ddqn"]["dynamic"])
    assert fx["duel_lr"]["call_lr"][0] != fx["duel_lr"]["call_lr"][1]
    b = fx["duel_batch"]
    assert bool(b["learn_batch"]) and int(b["padded"]) > 0 and (b["curr_count"][b["idx"]] < int(b["n_actions"])).any()
    assert b["call_curr"].tolist() == [True, False, True]
    for c in ("duel_ddqn", "duel_batch", "duel_act"):
        assert float(fx[c]["mean_gap"]) > 1e-3


@pytest.mark.parametrize("query_alone", [False, True])
def test_hand_written_slot_gradient_equals_autograd(query_alone):
    """slot_grad against torch.autograd through get_q_values, float64.  The advantage net is made a table Adv(s, a) = w[a]
    (zero feature weights, identity on the one-hot part), so d sum_b dq_b q_b / d w[k] is the slot gradient summed over the
    rows and slots holding action k; the value head's gradient is dq.  Without current sets it is exactly zero."""
    g = torch.Generator().manual_seed(3)
    B, A, obs = 9, 5, 3
    net = torch.nn.Module()
    net.state_arch = torch.nn.Linear(obs, 4).double()
    net.value_arch = torch.nn.Linear(4, 1).double()
    net.advantage_arch = torch.nn.Linear(4 + A, 1, bias=False).double()
    w = torch.randn(A, generator=g, dtype=torch.float64)
    with torch.no_grad():
        net.advantage_arch.weight.zero_()
        net.advantage_arch.weight[0, 4:] = w
    state = torch.randn(B, obs, generator=g, dtype=torch.float64)
    acts = torch.randint(0, A, (B,), generator=g)
    curr = torch.randint(0, A, (B, A), generator=g)
    curr[:, -2:] = 0                                                        # padding (id 0) counts in the mean
    oh = lambda x: torch.nn.functional.one_hot(x, A).double()  # noqa: E731
    dq = torch.randn(B, generator=g, dtype=torch.float64)
    q = get_q_values(net, state, oh(acts), None if query_alone else oh(curr))
    (dq * q).sum().backward()
    taken, slots = slot_grad(dq, A, query_alone)
    want = torch.zeros(A, dtype=torch.float64)
    want.index_add_(0, acts, taken)
    want.index_add_(0, curr.reshape(-1), slots.reshape(-1))
    got = net.advantage_arch.weight.grad[0, 4:]
    np.testing.assert_allclose(got.numpy(), want.numpy(), rtol=1e-12, atol=1e-15)
    if query_alone:
        assert torch.equal(got, torch.zeros(A, dtype=torch.float64))
    np.testing.assert_allclose(float(net.value_arch.bias.grad), float(dq.sum()), rtol=1e-12)


# DuelingQValueNetwork(state_dim=4, action_dim=6, hidden_dims=[64, 64], output_dim=1) as the reference builds it
PEARL_KEYS = [(f"{arch}._model.{i}.0.{p}", shape) for arch, dims in
              (("state_arch", [4, 64, 64, 64]), ("value_arch", [64, 64, 64, 1]), ("advantage_arch", [70, 64, 64, 1]))
              for i in range(3) for p, shape in (("weight", (dims[i + 1], dims[i])), ("bias", (dims[i + 1],)))]


def test_stand_in_network_has_pearls_state_dict():
    import pearl_b200
    net = pearl_b200.DuelingQValueNetwork(state_dim=4, action_dim=6, hidden_dims=[64, 64], output_dim=1)
    assert [(k, tuple(v.shape)) for k, v in net.state_dict().items()] == PEARL_KEYS
    assert sum(p.numel() for p in net.parameters()) == 25794
    assert (net.state_dim, net.action_dim) == (4, 6)


class _Space:
    def __init__(self, A):
        self.n = A
        self.actions = [torch.tensor([i]) for i in range(A)]
        self.actions_batch = torch.arange(A).view(A, 1)


def _make(cls_name="B200DeepQLearning", A=3, hidden=(16, 16), **kw):
    import pearl_b200
    kw.setdefault("network_type", pearl_b200.DuelingQValueNetwork)
    return getattr(pearl_b200, cls_name)(state_dim=4, action_space=_Space(A), hidden_dims=list(hidden), batch_size=8,
                                         action_representation_module=pearl_b200.OneHotActionTensorRepresentationModule(A), **kw)


@pytest.mark.parametrize("cls_name", ["B200DeepQLearning", "B200DoubleDQN"])
def test_dueling_construction_and_refusals(cls_name):
    """network_type=DuelingQValueNetwork (and a network_instance with its own widths) constructs (it used to raise
    NotImplementedError); the configurations the dueling learner does not run are refused."""
    import pearl_b200
    pl = _make(cls_name)
    assert pl._dueling and not pl._conservative and pl._double == (cls_name == "B200DoubleDQN")
    assert pl._obs_dim == 4 and pl._duel_dims == dict(feature_dim=16, state_h1=16, state_h2=16, value_h1=16, value_h2=16,
                                                      adv_h1=16, adv_h2=16)
    net = pearl_b200.DuelingQValueNetwork(state_dim=4, action_dim=3, hidden_dims=[24, 20], output_dim=1, state_hidden_dims=[32, 8],
                                          value_hidden_dims=[12, 10], advantage_hidden_dims=[40, 6])
    pl = _make(cls_name, network_instance=net)
    assert pl._duel_dims == dict(feature_dim=20, state_h1=32, state_h2=8, value_h1=12, value_h2=10, adv_h1=40, adv_h2=6)
    assert not _make(cls_name, network_type=None)._dueling
    with pytest.raises(NotImplementedError, match="conservative"):
        _make(cls_name, is_conservative=True)
    with pytest.raises(NotImplementedError, match="tc"):
        _make(cls_name, engine="tc")
    _make(cls_name, engine="simt")
    with pytest.raises(NotImplementedError):
        _make(cls_name, hidden=(16, 16, 16))                               # three hidden layers
    net = pearl_b200.DuelingQValueNetwork(state_dim=4, action_dim=3, hidden_dims=[16, 16], output_dim=1)
    net.value_arch._model[0].append(torch.nn.LayerNorm(16))
    with pytest.raises(NotImplementedError):                                # an extra module
        _make(cls_name, network_instance=net)
    net = pearl_b200.DuelingQValueNetwork(state_dim=4, action_dim=3, hidden_dims=[16, 16], output_dim=1)
    net.extra = torch.nn.Linear(2, 2)
    with pytest.raises(NotImplementedError):
        _make(cls_name, network_instance=net)
    net = pearl_b200.DuelingQValueNetwork(state_dim=4, action_dim=3, hidden_dims=[16, 16], output_dim=1)
    with pytest.raises(NotImplementedError, match="AdamW"):
        _make(cls_name, network_instance=net, optimizer=torch.optim.SGD(net.parameters(), lr=0.1))
    with pytest.raises(NotImplementedError, match="AdamW"):
        _make(cls_name, network_instance=net, optimizer=torch.optim.AdamW(net.parameters(), lr=0.1))   # amsgrad off
    with pytest.raises(NotImplementedError, match="one-hot"):
        pearl_b200.B200DeepQLearning(state_dim=4, action_space=_Space(3), hidden_dims=[16, 16],
                                     network_type=pearl_b200.DuelingQValueNetwork, action_representation_module=_NotOneHot(3))
    pl = _make(cls_name)
    with pytest.raises(NotImplementedError):
        pearl_b200.B200LearnerGroup([pl], [object()])
    with pytest.raises(NotImplementedError):
        pl.set_communicator(None)
    with pytest.raises(NotImplementedError):
        pl.set_kernel_timing(True)
    pl.set_history_summarization_module(_NotIdentity())
    with pytest.raises(NotImplementedError):
        pl.preprocess_batch(None)


class _NotOneHot(torch.nn.Module):
    def __init__(self, A):
        super().__init__()
        self.max_number_actions = self.representation_dim = A


class _NotIdentity(torch.nn.Module):
    pass
