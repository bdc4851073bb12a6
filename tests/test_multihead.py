"""Multi-head DQN / DoubleDQN on the GPU (B200DeepQLearning / B200DoubleDQN with a VanillaQValueMultiHeadNetwork, plain or
conservative, csrc/multihead.cu) against
(a) the recordings of the reference's PearlAgent(DeepQLearning / DoubleDQN, BasicReplayBuffer) (tests/golden/mh_*.npz:
    learn() with the same indices from CPython's `random.sample`, agent.learn_batch() on sampled batches with partial
    current sets, and act()), parameters and AdamW state round by round from the oracle's re-synchronised state,
    elementwise 1e-4 (tests/_tol.py);
(b) oracle/multihead_oracle.py at a stress shape (obs 128, 16 actions, [256, 256], batch 256, dynamic next sets, partial
    current sets), DQN, DoubleDQN and both conservative variants, under the SIMT and the tensor-core engine;
plus bit-identity (run to run, graph replay, round chunking, learn_batch vs learn vs a foreign buffer), the launch count,
lr and alpha changes on the same handle, the checkpoint views, q_values / act and the rejected inputs."""
import copy
import ctypes as C
import os
import random

import numpy as np
import pytest
import torch

from conftest import GOLDEN
from oracle.multihead_oracle import OracleMultiHead, one_hot_batch
from oracle.pearl_oracle import flat, load_flat

pytestmark = pytest.mark.gpu

from _tol import close as _close, close_params as _close_params  # noqa: E402
from test_iql import _close_net, _relu_boundary  # noqa: E402

LAUNCHES_PER_ROUND = 16     # 11 contractions (3 online, 3 target, 5 backward) + 5 small kernels, every variant (DESIGN.md §3.4)


class _Space:
    def __init__(self, A):
        self.n = A
        self.actions = [torch.tensor([i]) for i in range(A)]
        self.actions_batch = torch.arange(A).view(A, 1)


def _learner(obs, A, hidden, double=False, alpha=None, **kw):
    import pearl_b200
    cls = pearl_b200.B200DoubleDQN if double else pearl_b200.B200DeepQLearning
    extra = dict(is_conservative=True, conservative_alpha=alpha) if alpha is not None else {}
    return cls(state_dim=obs, action_space=_Space(A), hidden_dims=list(hidden), network_type=pearl_b200.VanillaQValueMultiHeadNetwork,
               action_representation_module=pearl_b200.OneHotActionTensorRepresentationModule(A), **extra, **kw).to("cuda:0")


def _buffer(n, d, A, dynamic, **kw):
    import pearl_b200
    buf = pearl_b200.B200ReplayBuffer(n, **kw)
    t = torch.as_tensor
    extra = dict(next_available_ids=t(d["next_ids"]).to(torch.uint8), next_available_count=t(d["next_count"]).to(torch.int32)) \
        if dynamic else {}
    buf.push_batch(t(d["state"]), t(d["action"]).to(torch.int32), t(d["reward"]), t(d["next_state"]), t(d["terminated"]),
                   torch.zeros(n, dtype=torch.bool), max_number_actions=A, **extra)
    return buf


def _oh(d, i, A, curr=True):
    return one_hot_batch(A, *(torch.from_numpy(np.asarray(d[k][i])) for k in ("state", "action", "reward", "next_state", "terminated")),
                         np.asarray(d["curr_ids"][i]).astype(np.int64) if curr else None,
                         np.asarray(d["next_ids"][i]).astype(np.int64), np.asarray(d["next_count"][i]))


def _batch(d, i, A, one_hot=True, curr=False):
    """A TransitionBatch of rows i, as the reference's preprocess_batch leaves it (one-hot actions and slots) or with raw
    ids; next_unavailable_actions_mask from the stored counts; current slots (padded with id 0) when `curr`."""
    import pearl_b200
    b = _oh(d, i, A, curr)
    if not one_hot:
        ids = lambda x: x.argmax(-1, keepdim=True).float()  # noqa: E731
        b.update(action=b["action"].argmax(-1).view(-1, 1), curr_available_actions=ids(b["curr_available_actions"]),
                 next_available_actions=ids(b["next_available_actions"]))
    if not curr:
        b["curr_available_actions"] = None
    return pearl_b200.TransitionBatch(**b)


def _sync(pl, orc):
    """The learner takes the oracle's parameters, target and AdamW moments (the step counts already agree)."""
    load_flat(pl._Q, flat(orc.Q))
    load_flat(pl._Q_target, flat(orc.Qt))
    st, params = pl.adam_state(), list(orc.Q.parameters())
    for key in ("exp_avg", "exp_avg_sq", "max_exp_avg_sq"):
        if params[0] in orc.opt.state:
            st[key].copy_(torch.cat([orc.opt.state[p][key].reshape(-1) for p in params]))


def _max_exp_avg_sq(fx):
    v = fx["adam_exp_avg_sq"].copy()
    v[fx["adam_max_exp_avg_sq_idx"]] = fx["adam_max_exp_avg_sq_val"]
    return v


@pytest.mark.parametrize("graph", [True, False])
@pytest.mark.parametrize("case", ["mh_dqn", "mh_ddqn", "mh_cql_dqn", "mh_cql_ddqn", "mh_lr", "mh_batch"])
def test_multihead_matches_reference_recording(case, graph):
    """Sampled indices and CPython's `random` state bit-exact, losses at 1e-4; every round starts from the oracle's state
    (which tests/test_multihead_oracle.py pins to the recording), and the parameters, target and AdamW state after it agree
    elementwise to 1e-4; the final state against the recording itself."""
    torch.set_num_threads(1)
    fx = np.load(os.path.join(GOLDEN, f"{case}.npz"))
    n, R, B, calls, A = int(fx["n"]), int(fx["rounds"]), int(fx["batch"]), int(fx["calls"]), int(fx["n_actions"])
    cons = bool(fx["conservative"])
    alpha = float(fx["alpha"]) if cons else None
    lb = bool(fx["learn_batch"])
    buf = _buffer(n, fx, A, bool(fx["dynamic"]))
    pl = _learner(int(fx["obs"]), A, fx["hidden"].tolist(), bool(fx["double"]), alpha, learning_rate=float(fx["lr"]),
                  discount_factor=float(fx["gamma"]), training_rounds=1, batch_size=B, target_update_freq=int(fx["target_update_freq"]),
                  soft_update_tau=float(fx["tau"]))
    pl.use_cuda_graph = graph
    orc = OracleMultiHead(int(fx["obs"]), A, fx["hidden"].tolist(), lr=float(fx["lr"]), gamma=float(fx["gamma"]), tau=float(fx["tau"]),
                          double=bool(fx["double"]), target_update_freq=int(fx["target_update_freq"]), init_q=fx["init_q"], alpha=alpha)
    random.setstate((3, tuple(int(x) for x in fx["rng_before"]), None))
    losses, idx, handles = [], [], []
    per_call = 1 if lb else R
    for r in range(len(fx["idx"])):
        lr = float(fx["call_lr"][r // per_call])
        pl.optimizer.param_groups[0]["lr"] = lr
        orc.opt.param_groups[0]["lr"] = lr
        _sync(pl, orc)
        if lb:                              # agent.learn_batch(buf.sample(batch)), partial current sets
            logical, _ = buf.sample_indices(B, 1)
            i = logical[0].cpu().numpy()
            losses.append(pl.learn_batch(_batch(fx, i, A, curr=True))["loss"])
        else:
            rep = pl.learn(buf, trace=True)
            i = rep["idx"][0].cpu().numpy()
            losses += rep["loss"]
            orc.training_steps += 1
        idx.append(i.tolist())
        handles.append(pl._handle.value)
        want = orc.learn_batch(_oh(fx, i, A))
        _close(losses[-1], want, f"round {r} loss")
        _close(pl.flat_parameters.cpu().numpy(), flat(orc.Q).numpy(), f"round {r} online")
        _close(pl.flat_target_parameters.cpu().numpy(), flat(orc.Qt).numpy(), f"round {r} target")
        st, params = pl.adam_state(), list(orc.Q.parameters())
        for k in ("exp_avg", "exp_avg_sq", "max_exp_avg_sq"):
            _close(st[k].cpu().numpy(), torch.cat([orc.opt.state[p][k].reshape(-1) for p in params]).numpy(), f"round {r} {k}", atol=1e-9)
    assert len(set(handles)) == 1, "an lr change re-created the C handle"
    assert pl._training_steps == (0 if lb else R * calls)
    assert idx == fx["idx"].tolist()                                                  # bit-exact sampling
    assert random.getstate()[1] == tuple(int(x) for x in fx["rng_after"])              # CPython's random as the reference left it
    _close(losses, fx["loss"], "loss")
    _close(pl.flat_parameters.cpu().numpy(), fx["q_calls"][-1], "online net at the end")
    _close(pl.flat_target_parameters.cpu().numpy(), fx["qt_calls"][-1], "target net at the end")
    st = pl.adam_state()
    assert st["step"] == int(fx["adam_step"])
    for k, want in (("exp_avg", fx["adam_exp_avg"]), ("exp_avg_sq", fx["adam_exp_avg_sq"]), ("max_exp_avg_sq", _max_exp_avg_sq(fx))):
        _close(st[k].cpu().numpy(), want, f"AdamW {k}", atol=1e-9)


def test_multihead_act_matches_reference_recording():
    fx = np.load(os.path.join(GOLDEN, "mh_act.npz"))
    A = int(fx["n_actions"])
    pl = _learner(int(fx["obs"]), A, fx["hidden"].tolist())
    load_flat(pl._Q, fx["init_q"])
    load_flat(pl._Q_target, fx["init_q"])
    import pearl_b200  # noqa: F401
    for i in range(int(fx["n"])):
        m = int(fx["avail_count"][i])
        ids = fx["avail_ids"][i, :m].astype(np.int64)

        class Space:
            n = m
            actions = [torch.tensor([int(a)]) for a in ids]
            actions_batch = torch.from_numpy(ids).view(m, 1)
        s = torch.from_numpy(fx["state"][i])
        assert int(pl.act(s, Space(), exploit=True)) == int(fx["chosen"][i])
        _close(pl.q_values(s.view(1, -1))[0].cpu().numpy()[ids], fx["values"][i, :m], f"act values row {i}")


def _data(n, obs, A, seed, p_term=0.1):
    rng = np.random.Generator(np.random.PCG64(seed))
    q8 = lambda x: (np.rint(x * 256) / 256).astype(np.float32)  # noqa: E731
    d = dict(state=q8(rng.standard_normal((n, obs))), next_state=q8(rng.standard_normal((n, obs))), reward=q8(rng.standard_normal(n)),
             terminated=rng.random(n) < p_term, action=rng.integers(0, A, size=n).astype(np.int32))
    for key in ("next", "curr"):
        ids, cnt = np.zeros((n, A), np.int64), np.zeros(n, np.int32)
        for k in range(n):
            m = int(rng.integers(1, A + 1))
            ids[k, :m] = np.sort(rng.choice(A, size=m, replace=False))
            cnt[k] = m
        d.update({f"{key}_ids": ids, f"{key}_count": cnt})
    return d


@pytest.mark.parametrize("engine", [0, 2])
@pytest.mark.parametrize("alpha", [None, 2.0])
@pytest.mark.parametrize("double", [False, True])
def test_multihead_stress_shape_against_oracle(double, alpha, engine):
    """obs 128, 16 actions, [256, 256], batch 256, dynamic next sets and partial current sets, one learn_batch round at a
    time from the oracle's state; the loss and the parameters must agree elementwise to 1e-4 up to the counted AdamW
    outliers of `close_params`, and weight rows of hidden units at the ReLU boundary to one AdamW step.  For DoubleDQN a
    next slot whose online value lies within fp32 noise of its row's best is masked on both sides."""
    from pearl_b200 import TransitionBatch, _lib
    torch.manual_seed(7)
    threads = torch.get_num_threads()
    torch.set_num_threads(8)
    obs, A, H, n, B, R, lr = 128, 16, 256, 3000, 256, 4, 1e-3
    d = _data(n, obs, A, seed=11)
    orc = OracleMultiHead(obs, A, (H, H), lr=lr, gamma=0.99, tau=0.1, double=double, target_update_freq=2, alpha=alpha)
    lib = _lib.load()
    prev = lib.prl_get_contraction_engine()
    _lib.check(lib.prl_set_contraction_engine(engine))
    try:
        pl = _learner(obs, A, (H, H), double, alpha, training_rounds=1, batch_size=B, learning_rate=lr, target_update_freq=2,
                      soft_update_tau=0.1)
        rng = np.random.Generator(np.random.PCG64(19))
        for r in range(R):
            _sync(pl, orc)
            i = rng.choice(n, size=B, replace=False)
            b = _oh(d, i, A)
            if double:
                with torch.no_grad():
                    v = orc._q_values(orc.Q, b["next_state"], b["next_available_actions"])
                    v[b["next_unavailable_actions_mask"]] = -float("inf")
                    best, g = v.max(1, keepdim=True)
                    near = (best - v <= 1e-4 * (1.0 + best.abs())) & ~b["next_unavailable_actions_mask"]
                    near[torch.arange(B), g.view(-1)] = False
                b["next_unavailable_actions_mask"] = b["next_unavailable_actions_mask"] | near
            orc.training_steps = pl._training_steps = r
            skip = _relu_boundary(orc.Q, b["state"])
            ids = lambda t: t.argmax(-1, keepdim=True).float()  # noqa: E731
            rep = pl.learn_batch(TransitionBatch(state=b["state"], action=b["action"].argmax(-1).view(-1, 1), reward=b["reward"],
                                                 next_state=b["next_state"], terminated=b["terminated"],
                                                 curr_available_actions=ids(b["curr_available_actions"]),
                                                 next_available_actions=ids(b["next_available_actions"]),
                                                 next_unavailable_actions_mask=b["next_unavailable_actions_mask"]))
            loss = orc.learn_batch(b)
            _close(rep["loss"], loss, f"round {r} loss")
            _close_net(pl.flat_parameters.cpu().numpy(), orc.Q, skip, f"round {r} online", lr)
            _close_params(pl.flat_target_parameters.cpu().numpy(), flat(orc.Qt).numpy(), f"round {r} target", lr, 1)
    finally:
        _lib.check(lib.prl_set_contraction_engine(prev))
        torch.set_num_threads(threads)


def _vecs(pl):
    st = pl.adam_state()
    return [pl.flat_parameters.cpu(), pl.flat_target_parameters.cpu()] + [st[k].cpu() for k in ("exp_avg", "exp_avg_sq", "max_exp_avg_sq")]


@pytest.mark.parametrize("alpha", [None, 3.0])
@pytest.mark.parametrize("double", [False, True])
def test_multihead_is_bit_reproducible(double, alpha):
    """One call of R rounds == R one-round calls == chunks of 4; CUDA-graph replay == plain launches; two runs agree."""
    n, obs, A, B, R = 1500, 24, 6, 128, 9
    d = _data(n, obs, A, seed=23)

    def run(per_call, graph):
        buf = _buffer(n, d, A, True)
        torch.manual_seed(3)
        pl = _learner(obs, A, (64, 64), double, alpha, training_rounds=R, batch_size=B, max_rounds_per_call=per_call,
                      target_update_freq=4)
        pl.use_cuda_graph = graph
        random.seed(29)
        rep = pl.learn(buf)
        rep["batch"] = pl.learn_batch(_batch(d, np.arange(B), A, curr=True))
        return rep, _vecs(pl)

    base_rep, base = run(R, True)
    for per_call, graph in [(1, True), (R, False), (R, True), (4, True)]:
        rep, vecs = run(per_call, graph)
        assert rep == base_rep, (per_call, graph)
        for a, b in zip(vecs, base):
            assert torch.equal(a, b), (per_call, graph)


class _Foreign:
    """A replay buffer that is not a B200ReplayBuffer: its batches go through learn_batch."""

    def __init__(self, batches):
        self.batches, self.n = list(batches), 10 ** 6

    def __len__(self):
        return self.n

    def sample(self, k):
        return self.batches.pop(0)


@pytest.mark.parametrize("alpha", [None, 4.0])
@pytest.mark.parametrize("one_hot", [True, False])
def test_multihead_learn_batch_equals_learn(one_hot, alpha):
    """learn_batch on the rows a one-round learn() gathered (every action current, as the ring reports), at the same
    training-step count, and learn() over a foreign buffer that returns those rows, leave every vector bit-identical to
    learn() (target update included: freq 2, which fires in round 1)."""
    n, obs, A, B = 800, 12, 5, 96
    d = _data(n, obs, A, seed=43)
    d["curr_ids"] = np.tile(np.arange(A), (n, 1))
    buf = _buffer(n, d, A, True)

    def mk():
        torch.manual_seed(5)
        return _learner(obs, A, (64, 64), True, alpha, training_rounds=1, batch_size=B, target_update_freq=2)
    a, b, c = mk(), mk(), mk()
    random.seed(3)
    rep_a = a.learn(buf, trace=True)
    rows = rep_a["idx"][0].cpu().numpy()
    b._training_steps = 1            # learn() counted its round before the update check
    rep_b = b.learn_batch(_batch(d, rows, A, one_hot=one_hot, curr=True))
    rep_c = c.learn(_Foreign([_batch(d, rows, A, one_hot=one_hot, curr=True)]))
    assert rep_a["loss"][0] == rep_b["loss"] == rep_c["loss"][0]
    assert a._training_steps == c._training_steps == 1
    for x, y, z in zip(_vecs(a), _vecs(b), _vecs(c)):
        assert torch.equal(x, y) and torch.equal(x, z)


@pytest.mark.parametrize("double", [False, True])
def test_multihead_launch_count_and_learning_rate_and_alpha_changes(double):
    n, obs, A, B = 600, 8, 4, 64
    d = _data(n, obs, A, seed=31)
    buf = _buffer(n, d, A, False)
    pl = _learner(obs, A, (32, 32), double, 2.0, training_rounds=5, batch_size=B)
    rep = pl.learn(buf, trace=True)
    assert rep["launches"] == 5 * LAUNCHES_PER_ROUND == pl.launch_info()["launches"]
    h = pl._handle.value
    before = pl.flat_parameters.clone()
    pl.optimizer.param_groups[0]["lr"] = 0.0           # lr 0: AdamW moves nothing, decay factor 1
    pl.learn(buf)
    assert pl._handle.value == h
    assert torch.equal(pl.flat_parameters, before)
    pl.optimizer.param_groups[0]["lr"] = 1e-3
    pl.learn(buf)
    assert pl._handle.value == h and not torch.equal(pl.flat_parameters, before)
    # alpha 0 on the same handle: the round is the plain learner's round
    ref = _learner(obs, A, (32, 32), double, training_rounds=1, batch_size=B)
    load_flat(ref._Q, pl.flat_parameters.cpu())
    load_flat(ref._Q_target, pl.flat_target_parameters.cpu())
    ref.optimizer.load_state_dict(copy.deepcopy(pl.optimizer.state_dict()))
    pl._conservative_alpha = 0.0
    batch = _batch(d, np.arange(B), A, curr=True)
    ref._training_steps = pl._training_steps
    rep_ref, rep_pl = ref.learn_batch(batch), pl.learn_batch(batch)
    assert pl._handle.value == h
    assert rep_pl["loss"] == rep_ref["loss"]
    for x, y in zip(_vecs(pl), _vecs(ref)):
        assert torch.equal(x, y)
    after0 = pl.flat_parameters.clone()
    pl._conservative_alpha = 5.0                         # a new alpha reaches the captured round
    pl.learn_batch(batch)
    assert pl._handle.value == h
    ref.learn_batch(batch)
    assert not torch.allclose(pl.flat_parameters - after0, ref.flat_parameters - after0, rtol=1e-3, atol=1e-6)
    assert pl.launch_info()["launches"] == LAUNCHES_PER_ROUND


def test_multihead_checkpoint_views_and_optimizer_load_state_dict():
    """_Q, _Q_target and the AdamW state are views into the learner's flat vectors; a checkpoint restored with
    `load_state_dict` (networks and optimizer) is picked up by the next call, which then repeats the checkpoint's next
    round bit for bit."""
    n, obs, A, B = 400, 6, 3, 32
    d = _data(n, obs, A, seed=53)
    pl = _learner(obs, A, (32, 32), False, 2.0, training_rounds=2, batch_size=B)
    batch = _batch(d, np.arange(B), A, curr=True)
    pl.learn_batch(batch)
    w, m = pl.flat_parameters, pl.adam_state()["exp_avg"]
    params = list(pl._Q.parameters())
    lo, hi = w.data_ptr(), w.data_ptr() + 4 * w.numel()
    assert all(lo <= p.data_ptr() < hi for p in params)
    wt = pl.flat_target_parameters
    assert all(wt.data_ptr() <= p.data_ptr() < wt.data_ptr() + 4 * wt.numel() for p in pl._Q_target.parameters())
    assert pl.optimizer.state[params[0]]["exp_avg"].data_ptr() == m.data_ptr()
    assert list(pl._Q.state_dict()) == ["_model.0.0.weight", "_model.0.0.bias", "_model.1.0.weight", "_model.1.0.bias",
                                        "_model.2.0.weight", "_model.2.0.bias"]
    ck = copy.deepcopy((pl._Q.state_dict(), pl._Q_target.state_dict(), pl.optimizer.state_dict()))
    pl.learn_batch(batch)
    want = _vecs(pl)
    step = pl.adam_state()["step"]
    pl.learn_batch(batch)
    pl._Q.load_state_dict(ck[0])
    pl._Q_target.load_state_dict(ck[1])
    pl.optimizer.load_state_dict(ck[2])
    pl.learn_batch(batch)
    assert pl.adam_state()["step"] == step
    for x, y in zip(_vecs(pl), want):
        assert torch.equal(x, y)
    assert float(pl.optimizer.state[params[0]]["step"]) == step


def test_multihead_q_values_and_act_against_the_oracle():
    n, obs, A = 1000, 10, 7
    d = _data(n, obs, A, seed=61)
    torch.manual_seed(9)
    pl = _learner(obs, A, (48, 40), True, max_rounds_per_call=8, batch_size=64)
    pl.learn_batch(_batch(d, np.arange(64), A))               # the q_values chunks run through a bound workspace
    orc = OracleMultiHead(obs, A, (48, 40), init_q=pl.flat_parameters.cpu(), init_q_target=pl.flat_target_parameters.cpu())
    s = torch.from_numpy(d["state"])
    for rows in (1, 3, 64, 1000):
        for target in (False, True):
            _close(pl.q_values(s[:rows], target=target).cpu().numpy(), orc.q_values(s[:rows], target=target).numpy(),
                   f"q_values rows {rows} target {target}")
    for k in range(40):
        m = int(d["next_count"][k])
        ids = d["next_ids"][k, :m]

        class Space:
            n = m
            actions = [torch.tensor([int(a)]) for a in ids]
            actions_batch = torch.from_numpy(ids).view(m, 1)
        want = int(ids[int(torch.argmax(orc.q_values(s[k:k + 1])[0, torch.from_numpy(ids)]))])
        assert int(pl.act(s[k], Space(), exploit=True)) == want


def test_multihead_rejects_bad_inputs():
    import pearl_b200
    from pearl_b200 import _lib
    from pearl_b200.replay_buffer import _stream_ptr
    n, obs, A, B = 64, 6, 4, 16
    d = _data(n, obs, A, seed=41)
    pl = _learner(obs, A, (16, 16), False, 2.0, training_rounds=2, batch_size=B)
    assert pl.learn(pearl_b200.B200ReplayBuffer(16)) == {}                  # empty buffer: nothing to do
    per = pearl_b200.B200PrioritizedReplayBuffer(n)
    per.push_batch(torch.from_numpy(d["state"]), torch.from_numpy(d["action"]), torch.from_numpy(d["reward"]),
                   torch.from_numpy(d["next_state"]), torch.from_numpy(d["terminated"]), torch.zeros(n, dtype=torch.bool),
                   max_number_actions=A)
    with pytest.raises(NotImplementedError, match="multi-head"):
        pl.learn(per)
    with pytest.raises(NotImplementedError):
        pearl_b200.B200LearnerGroup([pl], [per])
    disc_buf = _buffer(n, d, A, False)
    pl.learn(disc_buf)
    state0 = _vecs(pl) + [pl.adam_state()["step"], pl._training_steps]
    h = pl._handle.value
    rng_disc = disc_buf.get_rng_state()
    pl._conservative_alpha = None                                           # read on every call
    with pytest.raises(ValueError, match="conservative_alpha"):
        pl.learn(disc_buf)
    pl._conservative_alpha = 2.0
    with pytest.raises(ValueError):                                         # action id outside [0, A)
        pl.learn_batch(pearl_b200.TransitionBatch(state=torch.zeros(B, obs), action=torch.full((B, 1), A), reward=torch.zeros(B),
                                                  next_state=torch.zeros(B, obs), terminated=torch.zeros(B, dtype=torch.bool),
                                                  curr_available_actions=torch.zeros(B, A, 1)))
    with pytest.raises(ValueError, match="curr_available_actions"):        # the reference asserts current sets when conservative
        pl.learn_batch(_batch(d, np.arange(B), A))
    with pytest.raises(ValueError, match="features"):
        pl.learn_batch(pearl_b200.TransitionBatch(state=torch.zeros(B, obs + 1), action=torch.zeros(B, 1), reward=torch.zeros(B),
                                                  next_state=torch.zeros(B, obs + 1), terminated=torch.zeros(B, dtype=torch.bool),
                                                  curr_available_actions=torch.zeros(B, A, 1)))
    cont_buf = pearl_b200.B200ReplayBuffer(n)
    cont_buf.is_action_continuous = True
    t = torch.from_numpy
    cont_buf.push_batch(t(d["state"]), torch.zeros(n, 2), t(d["reward"]), t(d["next_state"]), t(d["terminated"]),
                        torch.zeros(n, dtype=torch.bool))
    dz = dict(d, state=np.zeros((n, obs + 1), np.float32), next_state=np.zeros((n, obs + 1), np.float32))
    other_obs = _buffer(n, dz, A, False)
    other_A = _buffer(n, dict(d, action=d["action"] % 3, next_ids=d["next_ids"][:, :3] % 3), A - 1, False)
    dev = pl._device
    out = torch.zeros(4, dtype=torch.float32, device=dev)
    for buf, rounds, batch in ((cont_buf, 1, B), (other_obs, 1, B), (other_A, 1, B), (disc_buf, 1, B + 1), (disc_buf, 4097, B)):
        rng0 = buf.get_rng_state()
        rc = pl._libh.prl_mhq_learn(pl._handle, buf.handle, rounds, batch, 0, 2.0, _lib.ptr(out), C.c_void_p(0), _stream_ptr(dev))
        assert rc == _lib.PRL_EINVAL, _lib.last_error()
        torch.cuda.synchronize()
        assert np.array_equal(buf.get_rng_state(), rng0), "the sampler ran"
    x = torch.zeros((B + 1, obs), device=dev)
    i32 = torch.zeros(B + 1, dtype=torch.int32, device=dev)
    u8 = torch.zeros(B + 1, dtype=torch.uint8, device=dev)
    rc = pl._libh.prl_mhq_learn_batch(pl._handle, B + 1, _lib.ptr(x), _lib.ptr(i32), _lib.ptr(x[:, 0].contiguous()), _lib.ptr(x),
                                      _lib.ptr(u8), None, None, None, 0, 2.0, _lib.ptr(out), _stream_ptr(dev))
    assert rc == _lib.PRL_EINVAL
    sharded = pearl_b200.B200ReplayBuffer(n, rng="device")
    sharded.push_batch_sharded(0, 2, t(d["state"]), t(d["action"]), t(d["reward"]), t(d["next_state"]), t(d["terminated"]),
                               torch.zeros(n, dtype=torch.bool), max_number_actions=A)
    sharded.seed(5)
    rng0 = sharded.get_rng_state()
    with pytest.raises(ValueError, match="shard"):
        pl.learn(sharded)
    torch.cuda.synchronize()
    assert np.array_equal(sharded.get_rng_state(), rng0), "the sampler ran"
    after = _vecs(pl) + [pl.adam_state()["step"], pl._training_steps]
    assert pl._handle.value == h
    for x, y in zip(state0[:5], after[:5]):
        assert torch.equal(x, y), "a refused call changed the learner's vectors"
    assert state0[5:] == after[5:], "a refused call changed the step counts"
    assert np.array_equal(disc_buf.get_rng_state(), rng_disc), "a refused call advanced the sampler"
    # a refused shape at the next bind leaves the bound handle and its vectors as they were
    h, before = pl._handle.value, [pl._flat[k].clone() for k in ("w", "wt", "m", "v", "vmax")]
    hidden, pl._hidden, pl._bound_ptr = pl._hidden, (16, 1 << 30), None    # past the 32-bit limit: the C side refuses it
    with pytest.raises(ValueError):
        pl._bind(B)
    assert pl._handle.value == h and all(torch.equal(pl._flat[k], x) for k, x in zip(("w", "wt", "m", "v", "vmax"), before))
    assert int(pl._c("adam_step")(pl._handle)) == state0[5]
    pl._hidden = hidden
    pl.learn_batch(_batch(d, np.arange(B), A, curr=True))                  # the learner works on after the refusal
