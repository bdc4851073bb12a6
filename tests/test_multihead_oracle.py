"""The multi-head DQN restatement (oracle/multihead_oracle.py) against the recordings of the reference's
PearlAgent(DeepQLearning / DoubleDQN with a VanillaQValueMultiHeadNetwork, plain or conservative, BasicReplayBuffer)
(tests/golden/mh_*.npz), its hand-written head gradient against torch.autograd, the stand-in network's state_dict keys,
and the plugin's construction and refusals on the CPU."""
import ctypes
import os
import random

import numpy as np
import pytest
import torch

from conftest import GOLDEN
from oracle.multihead_oracle import OracleMultiHead, cql_term, get_q_values, head_grad, one_hot_batch
from oracle.pearl_oracle import flat

CASES = ("mh_dqn", "mh_ddqn", "mh_cql_dqn", "mh_cql_ddqn", "mh_lr", "mh_batch")


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


def oracle_of(fx):
    return OracleMultiHead(int(fx["obs"]), int(fx["n_actions"]), fx["hidden"].tolist(), lr=float(fx["lr"]), gamma=float(fx["gamma"]),
                           tau=float(fx["tau"]), double=bool(fx["double"]), target_update_freq=int(fx["target_update_freq"]),
                           init_q=fx["init_q"], alpha=float(fx["alpha"]) if bool(fx["conservative"]) else None)


@pytest.mark.parametrize("case", CASES)
def test_multihead_oracle_reproduces_reference(case):
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
    orc = oracle_of(fx)
    tol = dict(rtol=5e-6, atol=5e-7)
    per_call = 1 if bool(fx["learn_batch"]) else R
    for r in range(len(fx["idx"])):
        if r % per_call == 0:
            orc.opt.param_groups[0]["lr"] = float(fx["call_lr"][r // per_call])
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


def test_multihead_oracle_reproduces_reference_act():
    """act(exploit=True) over partial available sets picks the first argmax of Q(s)[id] over the available ids (one state
    per forward, as act() runs it)."""
    torch.set_num_threads(1)
    fx = np.load(os.path.join(GOLDEN, "mh_act.npz"))
    orc = OracleMultiHead(int(fx["obs"]), int(fx["n_actions"]), fx["hidden"].tolist(), init_q=fx["init_q"])
    for i in range(int(fx["n"])):
        m = int(fx["avail_count"][i])
        ids = fx["avail_ids"][i, :m].astype(np.int64)
        v = orc.q_values(torch.from_numpy(fx["state"][i:i + 1]))[0, ids]
        np.testing.assert_array_equal(v.numpy(), fx["values"][i, :m])
        assert int(ids[int(torch.argmax(v))]) == int(fx["chosen"][i])
    assert int(fx["differs"]) > 0


def test_recordings_exercise_the_reference_quirks():
    """The target update fires inside and across learn() calls; mh_dqn is the integration test's network; lr changes in
    mh_lr; mh_batch samples current sets that repeat an id; and wherever conservative with A > 2 the reference's data
    term differs from the taken-action term."""
    fx = {c: np.load(os.path.join(GOLDEN, f"{c}.npz")) for c in CASES}
    d = fx["mh_dqn"]
    steps = [s for s in range(1, int(d["rounds"]) * int(d["calls"]) + 1) if (s + 1) % int(d["target_update_freq"]) == 0]
    assert any(s <= int(d["rounds"]) for s in steps) and any(s > int(d["rounds"]) for s in steps)
    assert (int(d["obs"]), int(d["n_actions"]), d["hidden"].tolist(), bool(d["conservative"])) == (4, 2, [64, 64], False)
    assert bool(fx["mh_ddqn"]["double"]) and bool(fx["mh_ddqn"]["dynamic"])
    assert float(fx["mh_cql_dqn"]["alpha"]) == 2.0 and not bool(fx["mh_cql_dqn"]["double"])
    assert float(fx["mh_cql_ddqn"]["alpha"]) == 8.0 and bool(fx["mh_cql_ddqn"]["double"]) and bool(fx["mh_cql_ddqn"]["dynamic"])
    lr = fx["mh_lr"]
    assert lr["call_lr"][0] != lr["call_lr"][1]
    b = fx["mh_batch"]
    assert bool(b["learn_batch"]) and bool(b["conservative"]) and int(b["dup"]) > 0
    assert (b["curr_count"][b["idx"]] < int(b["n_actions"]) - 1).any()          # at least two padded slots in a row
    for c in ("mh_cql_ddqn", "mh_batch"):
        assert int(fx[c]["n_actions"]) > 2 and float(fx[c]["term_gap"]) > 1e-3


@pytest.mark.parametrize("conservative", [False, True])
@pytest.mark.parametrize("A", [2, 5])
def test_hand_written_head_gradient_equals_autograd(A, conservative):
    """head_grad against torch.autograd of the reference's loss through get_q_values (bmm with one-hot slots), float64,
    with current sets that repeat the padding id 0: the repeated slots' CQL gradients add on one head column, and the data
    term reads slot columns 0 and 1 whatever the taken action."""
    g = torch.Generator().manual_seed(A + 10 * conservative)
    B, alpha = 9, 3.5
    head = (torch.randn(B, A, generator=g, dtype=torch.float64) * 2).requires_grad_(True)
    acts = torch.randint(0, A, (B,), generator=g)
    y = torch.randn(B, generator=g, dtype=torch.float64)
    curr = torch.zeros(B, A, dtype=torch.long)
    for b in range(B):
        m = 1 + b % A
        curr[b, :m] = torch.randperm(A, generator=g)[:m].sort().values
    assert any(int((curr[b] == 0).sum()) > 1 for b in range(B))
    oh = lambda x: torch.nn.functional.one_hot(x, A).double()  # noqa: E731
    bmm = lambda slots: torch.bmm(slots, head.unsqueeze(-1)).squeeze(-1)  # noqa: E731
    q = bmm(oh(acts).unsqueeze(1)).squeeze(-1)
    loss = torch.nn.MSELoss()(q, y)
    if conservative:
        loss = alpha * cql_term(bmm(oh(curr)).view(B, -1), oh(acts)) + loss
    loss.backward()
    dq = 2.0 * (q.detach() - y) / B
    want = head.grad.numpy()
    got = head_grad(head.detach(), acts, curr, dq, alpha if conservative else None).numpy()
    np.testing.assert_allclose(got, want, rtol=1e-12, atol=1e-15)


def test_oracle_slot_values_are_the_head_columns():
    torch.manual_seed(0)
    orc = OracleMultiHead(5, 4, (8, 8))
    s = torch.randn(6, 5)
    ids = torch.randint(0, 4, (6, 4))
    with torch.no_grad():
        got = get_q_values(orc.Q, s, torch.nn.functional.one_hot(ids, 4).float())
    assert torch.equal(got, orc.Q(s).detach().gather(1, ids))


def test_stand_in_network_has_pearls_state_dict():
    import pearl_b200
    net = pearl_b200.VanillaQValueMultiHeadNetwork(state_dim=4, action_dim=2, hidden_dims=[64, 64], output_dim=2)
    sd = net.state_dict()
    assert list(sd) == ["_model.0.0.weight", "_model.0.0.bias", "_model.1.0.weight", "_model.1.0.bias", "_model.2.0.weight",
                        "_model.2.0.bias"]
    assert [tuple(v.shape) for v in sd.values()] == [(64, 4), (64,), (64, 64), (64,), (2, 64), (2,)]
    assert net.state_dim == 4 and net.action_dim == 2 and tuple(net(torch.zeros(3, 4)).shape) == (3, 2)
    ln = pearl_b200.VanillaQValueMultiHeadNetwork(state_dim=4, action_dim=2, hidden_dims=[8], output_dim=2, use_layer_norm=True)
    assert list(ln.state_dict()) == ["_model.0.0.weight", "_model.0.0.bias", "_model.0.1.weight", "_model.0.1.bias",
                                     "_model.1.0.weight", "_model.1.0.bias"]
    orc = OracleMultiHead(4, 2, (64, 64))
    net.load_state_dict({k: v for k, v in zip(sd, orc.Q.state_dict().values())})
    assert torch.equal(flat(net), flat(orc.Q))


def _space(A):
    class Space:
        n = A
        actions = [torch.tensor([i]) for i in range(A)]
        actions_batch = torch.arange(A).view(A, 1)
    return Space()


def _make(cls_name="B200DeepQLearning", A=3, hidden=(16, 16), instance=False, **kw):
    import pearl_b200
    cls = getattr(pearl_b200, cls_name)
    net = dict(network_instance=pearl_b200.VanillaQValueMultiHeadNetwork(state_dim=4, action_dim=A, hidden_dims=list(hidden),
                                                                        output_dim=A)) \
        if instance else dict(network_type=pearl_b200.VanillaQValueMultiHeadNetwork)
    net.update(kw)
    return cls(state_dim=4, action_space=_space(A), hidden_dims=list(hidden), batch_size=8,
               action_representation_module=pearl_b200.OneHotActionTensorRepresentationModule(A), **net)


@pytest.mark.parametrize("instance", [False, True])
@pytest.mark.parametrize("A", [1, 2, 7])
@pytest.mark.parametrize("cls_name", ["B200DeepQLearning", "B200DoubleDQN"])
def test_multihead_construction(cls_name, A, instance):
    """network_type= and network_instance= both build the multi-head learner, recognised by class (at A = 1 the shape
    alone would read as a one-hot vanilla net of obs - 1 inputs); the online net has A outputs and the layout's widths."""
    import pearl_b200
    pl = _make(cls_name, A=A, hidden=(16, 12), instance=instance)
    assert isinstance(pl._Q, pearl_b200.VanillaQValueMultiHeadNetwork)
    assert pl._multihead and not pl._dueling and not pl._conservative
    assert (pl._obs_dim, pl._hidden, pl._n_actions, pl._double) == (4, (16, 12), A, cls_name == "B200DoubleDQN")
    assert pl._Q._model[-1][0].out_features == A and pl._Q_target._model[-1][0].out_features == A
    assert pl.use_cuda_graph
    if A >= 2:
        c = _make(cls_name, A=A, instance=instance, is_conservative=True, conservative_alpha=8.0)
        assert c._multihead and c._conservative and c._conservative_alpha == 8.0


def test_multihead_refusals():
    import pearl_b200
    with pytest.raises(NotImplementedError, match="DeepSARSA"):
        _make("B200DeepSARSA")
    with pytest.raises(NotImplementedError, match="tc"):
        _make(engine="tc")
    _make(engine="simt")
    with pytest.raises(ValueError, match="2 actions"):
        _make(A=1, is_conservative=True)
    with pytest.raises(ValueError, match="conservative_alpha"):
        _make(is_conservative=True, conservative_alpha=None)
    with pytest.raises(NotImplementedError, match="two hidden"):
        _make(hidden=(16, 16, 16))
    with pytest.raises(NotImplementedError, match="two hidden"):
        _make(hidden=(16,))
    ln = pearl_b200.VanillaQValueMultiHeadNetwork(state_dim=4, action_dim=3, hidden_dims=[16, 16], output_dim=3, use_layer_norm=True)
    with pytest.raises(NotImplementedError, match="use_layer_norm"):
        _make(network_instance=ln)
    wrong = pearl_b200.VanillaQValueMultiHeadNetwork(state_dim=4, action_dim=3, hidden_dims=[16, 16], output_dim=4)
    with pytest.raises(NotImplementedError, match="one output per action"):
        _make(network_instance=wrong)

    class OtherRepr(pearl_b200.OneHotActionTensorRepresentationModule):
        pass
    with pytest.raises(NotImplementedError, match="one-hot"):
        pearl_b200.B200DeepQLearning(state_dim=4, action_space=_space(3), hidden_dims=[16, 16],
                                     network_type=pearl_b200.VanillaQValueMultiHeadNetwork, action_representation_module=OtherRepr(3))
    net = pearl_b200.VanillaQValueMultiHeadNetwork(state_dim=4, action_dim=3, hidden_dims=[16, 16], output_dim=3)
    for opt in (torch.optim.Adam(net.parameters()), torch.optim.AdamW(net.parameters(), amsgrad=False)):
        with pytest.raises(NotImplementedError, match="AdamW"):
            _make(network_instance=net, optimizer=opt)
    pl = _make()
    with pytest.raises(NotImplementedError):
        pearl_b200.B200LearnerGroup([pl], [object()])
    with pytest.raises(NotImplementedError, match="set_communicator"):
        pl.set_communicator(None)
    with pytest.raises(NotImplementedError, match="kernel timing"):
        pl.set_kernel_timing(True)
    cql = _make(is_conservative=True, conservative_alpha=2.0)
    with pytest.raises(ValueError, match="curr_available_actions"):
        cql.learn_batch(pearl_b200.TransitionBatch(state=torch.zeros(4, 4), action=torch.zeros(4, 1), reward=torch.zeros(4),
                                                   next_state=torch.zeros(4, 4), terminated=torch.zeros(4, dtype=torch.bool)))


def test_one_hot_learners_are_unchanged():
    """Without network_type the plugin still builds the one-hot vanilla learner."""
    import pearl_b200
    pl = pearl_b200.B200DeepQLearning(state_dim=4, action_space=_space(3), hidden_dims=[16, 16],
                                      action_representation_module=pearl_b200.OneHotActionTensorRepresentationModule(3))
    assert not pl._multihead and (pl._obs_dim, pl._hidden) == (4, (16, 16))


def test_configured_maxima_are_refused_past_32_bit_offsets():
    """2 max_batch max(obs, h1, h2, A) must stay below 2^31 and so must the parameter count; A in [1, 255], and 2 <= A
    when conservative.  param_count / workspace_bytes return -1 at and past each limit and the largest batch under it is
    accepted."""
    from pearl_b200 import _lib
    lib = _lib.load()

    def cfg(**kw):
        base = dict(obs_dim=8, n_actions=4, hidden1=512, hidden2=512, double_dqn=0, conservative=0, target_update_freq=10,
                    max_batch=256, max_rounds=4, lr=1e-3, beta1=0.9, beta2=0.999, eps=1e-8, weight_decay=0.01, gamma=0.99, tau=0.1)
        base.update(kw)
        return ctypes.byref(_lib.MhqCfg(**base))
    top = (1 << 31) // (2 * 512)
    assert lib.prl_mhq_param_count(cfg(max_batch=top - 1)) > 0 and lib.prl_mhq_workspace_bytes(cfg(max_batch=top - 1)) > 0
    for bad in (dict(max_batch=top), dict(n_actions=0), dict(n_actions=256), dict(n_actions=1, conservative=1),
                dict(hidden1=0), dict(obs_dim=1 << 20, hidden1=4096, max_batch=1), dict(max_batch=0), dict(target_update_freq=0)):
        assert lib.prl_mhq_param_count(cfg(**bad)) == -1, bad
        assert lib.prl_mhq_workspace_bytes(cfg(**bad)) == -1, bad
    assert lib.prl_mhq_param_count(cfg(n_actions=1)) == 8 * 512 + 512 + 512 * 512 + 512 + 512 + 1
    assert lib.prl_mhq_param_count(cfg(n_actions=255, conservative=1)) > 0
