"""Dueling DQN / DoubleDQN on the GPU (B200DeepQLearning / B200DoubleDQN with a DuelingQValueNetwork, csrc/dueling.cu)
against
(a) the recordings of the reference's PearlAgent(DeepQLearning / DoubleDQN with DuelingQValueNetwork, BasicReplayBuffer)
    (tests/golden/duel_*.npz: learn() with the same indices from CPython's `random.sample`, agent.learn_batch() on sampled
    batches with partial current action sets or none, and act() over partial available sets), elementwise 1e-4
    (tests/_tol.py);
(b) oracle/dueling_oracle.py at a stress shape (obs 128, 16 actions, [256, 256], batch 256, dynamic next sets, partial
    current sets), DQN and DoubleDQN, step by step from a re-synchronised state, under the SIMT and the tensor-core engine;
plus bit-identity (run to run, graph replay, round chunking, learn_batch vs learn vs a foreign buffer, padding bytes of
the ring), the launch count, an lr change on the same handle, the checkpoint views, q_values / act over partial sets and
the rejected inputs."""
import copy
import ctypes as C
import os
import random

import numpy as np
import pytest
import torch

from conftest import GOLDEN
from oracle.dueling_oracle import OracleDueling, get_q_values, one_hot_batch
from oracle.pearl_oracle import flat, load_flat

pytestmark = pytest.mark.gpu

from _tol import close as _close, close_params as _close_params  # noqa: E402
from test_cql import _Foreign, _Space, _buffer, _data, _vecs  # noqa: E402
from test_iql import _relu_boundary  # noqa: E402

LAUNCHES_PER_ROUND = {False: 44, True: 54}     # DQN: 33 contractions + 11 small kernels; DoubleDQN: 42 + 12 (DESIGN.md §3.4)


def _learner(obs, A, hidden, double=False, instance=False, **kw):
    import pearl_b200
    cls = pearl_b200.B200DoubleDQN if double else pearl_b200.B200DeepQLearning
    net = dict(network_instance=pearl_b200.DuelingQValueNetwork(state_dim=obs, action_dim=A, hidden_dims=list(hidden), output_dim=1)) \
        if instance else dict(network_type=pearl_b200.DuelingQValueNetwork)
    return cls(state_dim=obs, action_space=_Space(A), hidden_dims=list(hidden),
               action_representation_module=pearl_b200.OneHotActionTensorRepresentationModule(A), **net, **kw).to("cuda:0")


def _batch(d, i, A, curr="full", one_hot=True):
    """A TransitionBatch of rows i as the reference's preprocess_batch leaves it (one-hot) or with raw ids; next slots
    padded with id 0 and masked from the stored counts; current slots: "full" (every action, as the ring reports),
    "data" (the partial, padded sets of `d`) or None (no current sets)."""
    import pearl_b200
    b = one_hot_batch(A, *(torch.from_numpy(np.asarray(d[k][i])) for k in ("state", "action", "reward", "next_state", "terminated")),
                      np.asarray(d["curr_ids"][i]).astype(np.int64) if curr == "data" else None,
                      np.asarray(d["next_ids"][i]).astype(np.int64), np.asarray(d["next_count"][i]))
    if not one_hot:
        ids = lambda x: x.argmax(-1, keepdim=True).float()  # noqa: E731
        b.update(action=b["action"].argmax(-1).view(-1, 1), curr_available_actions=ids(b["curr_available_actions"]),
                 next_available_actions=ids(b["next_available_actions"]))
    if curr is None:
        b["curr_available_actions"] = None
    return pearl_b200.TransitionBatch(**b)


@pytest.mark.parametrize("case", ["duel_dqn", "duel_ddqn", "duel_lr", "duel_batch"])
def test_dueling_matches_reference_recording(case):
    """The whole recorded run on one handle: bit-exact indices and `random` state, per-round losses elementwise 1e-4.  The
    parameters are then checked round by round from the oracle's state (the oracle reproduces every recording,
    tests/test_dueling_oracle.py): in the directions the advantage mean cancels, the reference's gradient is fp32 noise,
    which AdamW turns into steps of +-lr, so an unsynchronised run drifts from the recording there and, through ReLU
    switches, elsewhere after a few rounds."""
    fx = np.load(os.path.join(GOLDEN, f"{case}.npz"))
    n, R, B, calls, A = int(fx["n"]), int(fx["rounds"]), int(fx["batch"]), int(fx["calls"]), int(fx["n_actions"])
    buf = _buffer(n, fx, A, bool(fx["dynamic"]))
    pl = _learner(int(fx["obs"]), A, fx["hidden"].tolist(), bool(fx["double"]), instance=case == "duel_dqn",
                  learning_rate=float(fx["lr"]), discount_factor=float(fx["gamma"]), training_rounds=R, batch_size=B,
                  target_update_freq=int(fx["target_update_freq"]), soft_update_tau=float(fx["tau"]))
    load_flat(pl._Q, fx["init_q"])
    load_flat(pl._Q_target, fx["init_q"])
    random.setstate((3, tuple(int(x) for x in fx["rng_before"]), None))
    losses, idx, handles = [], [], []
    for c in range(calls):
        pl.optimizer.param_groups[0]["lr"] = float(fx["call_lr"][c])
        if bool(fx["learn_batch"]):         # agent.learn_batch(buf.sample(batch)): partial current sets, or none
            logical, _ = buf.sample_indices(B, 1)
            i = logical[0].cpu().numpy()
            idx.append(i.tolist())
            losses.append(pl.learn_batch(_batch(fx, i, A, curr="data" if bool(fx["call_curr"][c]) else None))["loss"])
        else:
            rep = pl.learn(buf, trace=True)
            losses += rep["loss"]
            idx += rep["idx"].tolist()
        handles.append(pl._handle.value)
    assert len(set(handles)) == 1, "an lr change re-created the C handle"
    assert pl._training_steps == (0 if bool(fx["learn_batch"]) else R * calls)
    assert idx == fx["idx"].tolist()                                                  # bit-exact sampling
    assert random.getstate()[1] == tuple(int(x) for x in fx["rng_after"])              # CPython's random as the reference left it
    _close(losses, fx["loss"], "loss")
    assert pl.adam_state()["step"] == int(fx["adam_step"])
    # round by round from the oracle's state, on the recorded rows
    lb = bool(fx["learn_batch"])
    per_call = 1 if lb else R
    orc = OracleDueling(int(fx["obs"]), A, fx["hidden"].tolist(), lr=float(fx["lr"]), gamma=float(fx["gamma"]), tau=float(fx["tau"]),
                        double=bool(fx["double"]), target_update_freq=int(fx["target_update_freq"]), init_q=fx["init_q"])
    pl = _learner(int(fx["obs"]), A, fx["hidden"].tolist(), bool(fx["double"]), learning_rate=float(fx["lr"]),
                  discount_factor=float(fx["gamma"]), training_rounds=1, batch_size=B, target_update_freq=int(fx["target_update_freq"]),
                  soft_update_tau=float(fx["tau"]))
    for r, rows in enumerate(fx["idx"]):
        lr = float(fx["call_lr"][r // per_call])
        orc.opt.param_groups[0]["lr"] = pl.optimizer.param_groups[0]["lr"] = lr
        orc.training_steps = pl._training_steps = 0 if lb else r + 1
        curr = ("data" if bool(fx["call_curr"][r]) else None) if lb else "full"
        b = _batch(fx, rows, A, curr=curr)
        _sync(pl, orc)
        skip = _duel_skip(orc.Q, b)
        rep = pl.learn_batch(b)
        want = orc.learn_batch(dict(state=b.state, action=b.action, reward=b.reward, next_state=b.next_state, terminated=b.terminated,
                                    curr_available_actions=b.curr_available_actions, next_available_actions=b.next_available_actions,
                                    next_unavailable_actions_mask=b.next_unavailable_actions_mask))
        _close(rep["loss"], want, f"round {r} loss")
        _check_round(pl, orc, skip, f"round {r}", lr)


def test_dueling_act_matches_reference_recording():
    """act(exploit=True) and the values it hands the exploration module: the advantage mean over the available set."""
    import pearl_b200
    from pearl_b200 import dueling
    fx = np.load(os.path.join(GOLDEN, "duel_act.npz"))
    A = int(fx["n_actions"])
    pl = _learner(int(fx["obs"]), A, fx["hidden"].tolist())
    load_flat(pl._Q, fx["init_q"])
    for i in range(int(fx["n"])):
        m = int(fx["avail_count"][i])
        ids = torch.from_numpy(fx["avail_ids"][i, :m].astype(np.int64))
        s = torch.from_numpy(fx["state"][i])
        _close(dueling.q_values(pl, s.view(1, -1), False, ids.view(1, -1))[0].cpu().numpy(), fx["values"][i, :m], f"act values row {i}")

        class Space:
            n = m
            actions = [torch.tensor([int(a)]) for a in ids]
            actions_batch = ids.view(m, 1)
        assert int(pl.act(s, Space(), exploit=True)) == int(fx["chosen"][i])

        class Explore:
            def act(self, subjective_state, action_space, exploit_action, values):
                return values
        pl.exploration_module = Explore()
        _close(pl.act(s, Space()).cpu().numpy(), fx["values"][i, :m], f"exploration values row {i}")
        pl.exploration_module = None
    assert isinstance(pl._Q, pearl_b200.DuelingQValueNetwork)


def _sync(pl, orc):
    """The learner takes the oracle's parameters, target and AdamW moments (the step counts already agree)."""
    load_flat(pl._Q, flat(orc.Q))
    load_flat(pl._Q_target, flat(orc.Qt))
    st, params = pl.adam_state(), list(orc.Q.parameters())
    for key in ("exp_avg", "exp_avg_sq", "max_exp_avg_sq"):
        if params[0] in orc.opt.state:
            st[key].copy_(torch.cat([orc.opt.state[p][key].reshape(-1) for p in params]))


def _duel_boundary(net, state, slots):
    """`_relu_boundary` over the three MLPs (flat offsets state, value, advantage): the advantage net sees every (row, slot)
    input [feature || one-hot slot] of the round.  A flagged unit of the value or advantage net reaches the trunk through
    the feature gradient, so the whole trunk is then included (the recordings, at small shapes, hold the trunk
    elementwise)."""
    with torch.no_grad():
        f = net.state_arch(state)
        x = torch.cat([f.unsqueeze(1).expand(-1, slots.shape[1], -1), slots], dim=-1).reshape(-1, f.shape[1] + slots.shape[2])
    n_s, n_v = flat(net.state_arch).numel(), flat(net.value_arch).numel()
    st, va, ad = _relu_boundary(net.state_arch, state), _relu_boundary(net.value_arch, f), _relu_boundary(net.advantage_arch, x)
    parts = [st, va + n_s, ad + n_s + n_v]
    if va.size or ad.size:
        parts.append(np.arange(n_s))
    return np.unique(np.concatenate(parts))


def _duel_skip(net, b):
    """Elements whose gradient the reference computes as fp32 noise or near a ReLU switch, for a round on batch b (one-hot):
    the ReLU-boundary rows of `_duel_boundary` over the round's online inputs, the advantage head's bias (the advantage
    mean cancels it exactly) and the advantage net's layer-2 biases (a unit active or inactive in every slot of a row
    shifts all of the row's advantages alike, which the mean cancels)."""
    curr = b["curr_available_actions"] if isinstance(b, dict) else b.curr_available_actions
    state, action = (b["state"], b["action"]) if isinstance(b, dict) else (b.state, b.action)
    A = action.shape[-1]
    if curr is None:
        curr = torch.zeros(action.shape[0], 0, A)
    slots = torch.cat([curr.float(), action.float().unsqueeze(1)], dim=1)
    off, free = 0, []
    for name, p in net.named_parameters():
        if name in ("advantage_arch.1.0.bias", "advantage_arch.2.0.bias"):
            free.append(np.arange(off, off + p.numel()))
        off += p.numel()
    return np.unique(np.concatenate([_duel_boundary(net, state.float(), slots)] + free))


def _check_round(pl, orc, skip, what, lr):
    """One round from a synchronised state: `close_params` on every element outside `skip`, which is held to the AdamW
    bound of one step; the target net elementwise.  The advantage mean leaves many gradient elements at the 1e-8 level
    (differences of nearly equal slot terms), where AdamW's step, lr g / (|g| + eps), depends on the last bits of g: up to
    1e-3 of the elements may be such outliers, each within the AdamW bound."""
    got, want = pl.flat_parameters.cpu().numpy(), flat(orc.Q).numpy()
    keep = np.ones(want.size, dtype=bool)
    keep[skip] = False
    _close_params(got[keep], want[keep], f"{what} online", lr, 1, max_frac=1e-3)
    err = float(np.abs(got[skip] - want[skip]).max())
    print(f"    {what}: {skip.size} elements in ReLU-boundary rows or mean-cancelled directions, max abs err {err:.3e}")
    assert err <= 2.02 * lr + 2e-6, f"{what}: a skipped element is off by {err:.3e}, beyond one AdamW step"
    _close_params(pl.flat_target_parameters.cpu().numpy(), flat(orc.Qt).numpy(), f"{what} target", lr, 1)


@pytest.mark.parametrize("engine", [0, 2])
@pytest.mark.parametrize("double", [False, True])
def test_dueling_stress_shape_against_oracle(double, engine):
    """obs 128, 16 actions, [256, 256], batch 256, dynamic next sets and partial current sets, one learn_batch round at a
    time (learn() equals learn_batch bit for bit, test_dueling_learn_batch_equals_learn).  Each round starts from the
    oracle's state; the loss and the parameters must agree elementwise to 1e-4 up to the counted AdamW outliers of
    `close_params`, and weight rows of hidden units at the ReLU boundary to one AdamW step.  For DoubleDQN a next slot whose
    online value lies within fp32 noise of its row's best is masked on both sides (it still enters the advantage mean),
    so both pick the same greedy slot."""
    from pearl_b200 import _lib
    torch.manual_seed(7)
    threads = torch.get_num_threads()
    torch.set_num_threads(8)
    obs, A, H, n, B, R, lr = 128, 16, 256, 3000, 256, 3, 1e-3
    d = _data(n, obs, A, seed=11)
    orc = OracleDueling(obs, A, (H, H), lr=lr, gamma=0.99, tau=0.1, double=double, target_update_freq=2)
    lib = _lib.load()
    prev = lib.prl_get_contraction_engine()
    _lib.check(lib.prl_set_contraction_engine(engine))
    masked = 0
    try:
        pl = _learner(obs, A, (H, H), double, training_rounds=1, batch_size=B, learning_rate=lr, target_update_freq=2,
                      soft_update_tau=0.1)
        rng = np.random.Generator(np.random.PCG64(19))
        for r in range(R):
            _sync(pl, orc)
            i = rng.choice(n, size=B, replace=False)
            b = one_hot_batch(A, *(torch.from_numpy(d[k][i]) for k in ("state", "action", "reward", "next_state", "terminated")),
                              d["curr_ids"][i], d["next_ids"][i], d["next_count"][i])
            if double:
                with torch.no_grad():
                    v = get_q_values(orc.Q, b["next_state"], b["next_available_actions"])
                    v[b["next_unavailable_actions_mask"]] = -float("inf")
                    best, g = v.max(1, keepdim=True)
                    near = (best - v <= 1e-4 * (1.0 + best.abs())) & ~b["next_unavailable_actions_mask"]
                    near[torch.arange(B), g.view(-1)] = False
                masked += int(near.sum())
                b["next_unavailable_actions_mask"] = b["next_unavailable_actions_mask"] | near
            orc.training_steps = pl._training_steps = r
            skip = _duel_skip(orc.Q, b)
            ids = lambda t: t.argmax(-1, keepdim=True).float()  # noqa: E731
            from pearl_b200 import TransitionBatch
            rep = pl.learn_batch(TransitionBatch(state=b["state"], action=b["action"].argmax(-1).view(-1, 1), reward=b["reward"],
                                                 next_state=b["next_state"], terminated=b["terminated"],
                                                 curr_available_actions=ids(b["curr_available_actions"]),
                                                 next_available_actions=ids(b["next_available_actions"]),
                                                 next_unavailable_actions_mask=b["next_unavailable_actions_mask"]))
            loss = orc.learn_batch(b)
            _close(rep["loss"], loss, f"round {r} loss")
            _check_round(pl, orc, skip, f"round {r}", lr)
        print(f"    {masked} near-tie next slots masked over {R} rounds")
    finally:
        _lib.check(lib.prl_set_contraction_engine(prev))
        torch.set_num_threads(threads)


@pytest.mark.parametrize("double", [False, True])
def test_dueling_is_bit_reproducible(double):
    """One call of R rounds == R one-round calls (max_rounds_per_call=1) == chunks of 4; CUDA-graph replay == plain
    launches; two runs agree.  Bit for bit: the launch sequence and every summation order are fixed."""
    n, obs, A, B, R = 1500, 24, 6, 128, 9
    d = _data(n, obs, A, seed=23)

    def run(per_call, graph):
        buf = _buffer(n, d, A, True)
        torch.manual_seed(3)
        pl = _learner(obs, A, (64, 64), double, training_rounds=R, batch_size=B, max_rounds_per_call=per_call, target_update_freq=4)
        pl.use_cuda_graph = graph
        random.seed(29)
        rep = pl.learn(buf)
        rep["batch"] = pl.learn_batch(_batch(d, np.arange(B), A, curr="data"))
        rep["no_curr"] = pl.learn_batch(_batch(d, np.arange(B), A, curr=None))
        return rep, _vecs(pl)

    base_rep, base = run(R, True)
    for per_call, graph in [(1, True), (R, False), (R, True), (4, True)]:
        rep, vecs = run(per_call, graph)
        assert rep == base_rep, (per_call, graph)
        for a, b in zip(vecs, base):
            assert torch.equal(a, b), (per_call, graph)


@pytest.mark.parametrize("one_hot", [True, False])
def test_dueling_learn_batch_equals_learn(one_hot):
    """learn_batch on the rows a one-round learn() gathered (every action current, as the ring reports), at the same
    training-step count, and learn() over a foreign buffer that returns those rows, both leave every vector bit-identical
    to learn() (target update included: freq 2, which fires in round 1)."""
    n, obs, A, B = 800, 12, 5, 96
    d = _data(n, obs, A, seed=43)
    buf = _buffer(n, d, A, True)

    def mk():
        torch.manual_seed(5)
        return _learner(obs, A, (64, 64), True, training_rounds=1, batch_size=B, target_update_freq=2)
    a, b, c = mk(), mk(), mk()
    random.seed(3)
    rep_a = a.learn(buf, trace=True)
    rows = rep_a["idx"][0].cpu().numpy()
    b._training_steps = 1            # learn() counted its round before the update check
    rep_b = b.learn_batch(_batch(d, rows, A, one_hot=one_hot))
    rep_c = c.learn(_Foreign([_batch(d, rows, A, one_hot=one_hot)]))
    assert rep_a["loss"][0] == rep_b["loss"] == rep_c["loss"][0]
    assert a._training_steps == c._training_steps == 1
    for x, y, z in zip(_vecs(a), _vecs(b), _vecs(c)):
        assert torch.equal(x, y) and torch.equal(x, z)


def test_dueling_ring_padding_bytes_do_not_matter():
    """Next-action slots at or beyond the stored count read as action 0: a ring pushed with arbitrary bytes there trains
    exactly like one pushed with zeros."""
    n, obs, A, B = 500, 10, 7, 64
    d = _data(n, obs, A, seed=71)
    junk = d["next_ids"].copy()
    pad = np.arange(A)[None, :] >= d["next_count"][:, None]
    junk[pad] = np.random.Generator(np.random.PCG64(1)).integers(1, A, size=int(pad.sum()))
    out = []
    for ids in (d["next_ids"], junk):
        buf = _buffer(n, dict(d, next_ids=ids), A, True)
        torch.manual_seed(13)
        pl = _learner(obs, A, (32, 32), False, training_rounds=4, batch_size=B, target_update_freq=2)
        random.seed(17)
        out.append((pl.learn(buf)["loss"], _vecs(pl)))
    assert out[0][0] == out[1][0]
    assert all(torch.equal(x, y) for x, y in zip(out[0][1], out[1][1]))


@pytest.mark.parametrize("double", [False, True])
def test_dueling_launch_count_and_learning_rate_change(double):
    n, obs, A, B = 600, 8, 4, 64
    d = _data(n, obs, A, seed=31)
    buf = _buffer(n, d, A, False)
    pl = _learner(obs, A, (32, 32), double, training_rounds=5, batch_size=B)
    rep = pl.learn(buf, trace=True)
    assert rep["launches"] == 5 * LAUNCHES_PER_ROUND[double] == pl.launch_info()["launches"]
    h = pl._handle.value
    before = pl.flat_parameters.clone()
    pl.optimizer.param_groups[0]["lr"] = 0.0           # lr 0: AdamW moves nothing, decay factor 1
    pl.learn(buf)
    assert pl._handle.value == h
    assert torch.equal(pl.flat_parameters, before)
    pl.optimizer.param_groups[0]["lr"] = 1e-3
    pl.learn(buf)
    assert pl._handle.value == h and not torch.equal(pl.flat_parameters, before)


def test_dueling_checkpoint_views_and_optimizer_load_state_dict():
    """_Q, _Q_target and the AdamW state are views into the learner's flat vectors, under Pearl's state_dict keys; a
    checkpoint restored with `load_state_dict` (networks and optimizer) is picked up by the next call, which then repeats
    the checkpoint's next round bit for bit."""
    n, obs, A, B = 400, 6, 3, 32
    d = _data(n, obs, A, seed=53)
    pl = _learner(obs, A, (32, 32), False, training_rounds=2, batch_size=B)
    batch = _batch(d, np.arange(B), A, curr="data")
    pl.learn_batch(batch)
    w, m = pl.flat_parameters, pl.adam_state()["exp_avg"]
    params = list(pl._Q.parameters())
    lo, hi = w.data_ptr(), w.data_ptr() + 4 * w.numel()
    assert all(lo <= p.data_ptr() < hi for p in params)
    wt = pl.flat_target_parameters
    assert all(wt.data_ptr() <= p.data_ptr() < wt.data_ptr() + 4 * wt.numel() for p in pl._Q_target.parameters())
    assert pl.optimizer.state[params[0]]["exp_avg"].data_ptr() == m.data_ptr()
    sd = pl._Q.state_dict()
    assert list(sd)[0] == "state_arch._model.0.0.weight" and list(sd)[-1] == "advantage_arch._model.2.0.bias"
    assert torch.equal(torch.cat([v.reshape(-1) for v in sd.values()]), w)
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


def test_dueling_q_values_and_act_against_oracle():
    """q_values over every action, over partial id sets (the mean over the set) and act() against the oracle, online and
    target, after a few rounds (so online and target differ), in chunks larger than the bound batch."""
    from pearl_b200 import dueling
    n, obs, A = 1000, 10, 7
    d = _data(n, obs, A, seed=61)
    buf = _buffer(n, d, A, True)
    torch.manual_seed(9)
    pl = _learner(obs, A, (48, 40), True, training_rounds=3, batch_size=64, target_update_freq=2)
    pl.learn(buf)
    orc = OracleDueling(obs, A, (48, 40), init_q=pl.flat_parameters.cpu(), init_q_target=pl.flat_target_parameters.cpu())
    s = torch.from_numpy(d["state"])
    for rows in (1, 3, 64, 1000):
        for target in (False, True):
            want = orc.q_values(s[:rows], np.tile(np.arange(A), (rows, 1)), target)
            _close(pl.q_values(s[:rows], target=target).cpu().numpy(), want.numpy(), f"q_values rows {rows} target {target}")
    for K in (1, 3, 6):
        rows = np.flatnonzero(d["next_count"] == K)[:50]
        ids = d["next_ids"][rows, :K]
        for target in (False, True):
            _close(dueling.q_values(pl, s[rows], target, torch.from_numpy(ids)).cpu().numpy(),
                   orc.q_values(s[rows], ids, target).numpy(), f"q_values over {K} ids target {target}")
    for k in range(40):
        m = int(d["next_count"][k])
        ids = torch.from_numpy(d["next_ids"][k, :m])

        class Space:
            n = m
            actions = [torch.tensor([int(a)]) for a in ids]
            actions_batch = ids.view(m, 1)
        q = orc.q_values(s[k:k + 1], ids.view(1, -1).numpy())[0]
        assert int(pl.act(s[k], Space(), exploit=True)) == int(ids[int(torch.argmax(q))])


def test_dueling_rejects_bad_inputs():
    import pearl_b200
    from pearl_b200 import _lib
    from pearl_b200.replay_buffer import _stream_ptr
    n, obs, A, B = 64, 6, 4, 16
    d = _data(n, obs, A, seed=41)
    pl = _learner(obs, A, (16, 16), training_rounds=2, batch_size=B)
    assert pl.learn(pearl_b200.B200ReplayBuffer(16)) == {}                  # empty buffer: nothing to do
    with pytest.raises(NotImplementedError):
        _learner(obs, A, (16, 16), is_conservative=True)
    with pytest.raises(NotImplementedError):
        _learner(obs, A, (16, 16), engine="tc")
    per = pearl_b200.B200PrioritizedReplayBuffer(n)
    per.push_batch(torch.from_numpy(d["state"]), torch.from_numpy(d["action"]), torch.from_numpy(d["reward"]),
                   torch.from_numpy(d["next_state"]), torch.from_numpy(d["terminated"]), torch.zeros(n, dtype=torch.bool),
                   max_number_actions=A)
    with pytest.raises(NotImplementedError):
        pl.learn(per)
    with pytest.raises(NotImplementedError):
        pearl_b200.B200LearnerGroup([pl], [per])
    with pytest.raises(NotImplementedError):
        pl.set_communicator(None)
    with pytest.raises(NotImplementedError):
        pl.set_kernel_timing(True)
    with pytest.raises(ValueError):                                         # action id outside [0, A)
        pl.learn_batch(pearl_b200.TransitionBatch(state=torch.zeros(B, obs), action=torch.full((B, 1), A), reward=torch.zeros(B),
                                                  next_state=torch.zeros(B, obs), terminated=torch.zeros(B, dtype=torch.bool)))
    from pearl_b200 import dueling
    with pytest.raises(ValueError):
        dueling.q_values(pl, torch.zeros(2, obs), False, torch.full((2, 2), A))
    disc_buf = _buffer(n, d, A, False)
    cont_buf = pearl_b200.B200ReplayBuffer(n)
    cont_buf.is_action_continuous = True
    t = torch.from_numpy
    cont_buf.push_batch(t(d["state"]), torch.zeros(n, 2), t(d["reward"]), t(d["next_state"]), t(d["terminated"]),
                        torch.zeros(n, dtype=torch.bool))
    dz = dict(d, state=np.zeros((n, obs + 1), np.float32), next_state=np.zeros((n, obs + 1), np.float32))
    other_obs = _buffer(n, dz, A, False)
    other_A = _buffer(n, dict(d, action=d["action"] % 3, next_ids=d["next_ids"][:, :3] % 3), A - 1, False)
    # the C entry point itself refuses these before the sampler or any learner kernel runs
    pl.learn(disc_buf)
    dev = pl._device
    out = torch.zeros(4, dtype=torch.float32, device=dev)
    for buf, rounds, batch in ((cont_buf, 1, B), (other_obs, 1, B), (other_A, 1, B), (disc_buf, 1, B + 1), (disc_buf, 4097, B)):
        before = [pl.flat_parameters.clone(), pl.flat_target_parameters.clone()]
        rng0 = buf.get_rng_state()
        rc = pl._libh.prl_duel_learn(pl._handle, buf.handle, rounds, batch, 0, _lib.ptr(out), C.c_void_p(0), _stream_ptr(dev))
        assert rc == _lib.PRL_EINVAL, _lib.last_error()
        torch.cuda.synchronize()
        assert np.array_equal(buf.get_rng_state(), rng0), "the sampler ran"
        assert all(torch.equal(x, y) for x, y in zip(before, [pl.flat_parameters, pl.flat_target_parameters])), "a learner kernel ran"
    x = torch.zeros((B + 1, obs), device=dev)
    i32 = torch.zeros(B + 1, dtype=torch.int32, device=dev)
    u8 = torch.zeros(B + 1, dtype=torch.uint8, device=dev)
    rc = pl._libh.prl_duel_learn_batch(pl._handle, B + 1, _lib.ptr(x), _lib.ptr(i32), _lib.ptr(x[:, 0].contiguous()), _lib.ptr(x),
                                       _lib.ptr(u8), None, None, None, 0, _lib.ptr(out), _stream_ptr(dev))
    assert rc == _lib.PRL_EINVAL
    cfg = _lib.DuelCfg.from_buffer_copy(pl._cfg)
    for bad in (0, 256):
        cfg.n_actions = bad
        assert pl._libh.prl_duel_param_count(C.byref(cfg)) == -1
    # a shard of a multi-GPU buffer samples global slots: rejected before the sampler or any learner kernel runs
    sharded = pearl_b200.B200ReplayBuffer(n, rng="device")
    sharded.push_batch_sharded(0, 2, t(d["state"]), t(d["action"]), t(d["reward"]), t(d["next_state"]), t(d["terminated"]),
                               torch.zeros(n, dtype=torch.bool), max_number_actions=A)
    sharded.seed(5)
    rng0 = sharded.get_rng_state()
    params0 = pl.flat_parameters.clone()
    with pytest.raises(ValueError, match="shard"):
        pl.learn(sharded)
    torch.cuda.synchronize()
    assert np.array_equal(sharded.get_rng_state(), rng0), "the sampler ran"
    assert torch.equal(params0, pl.flat_parameters), "a learner kernel ran"
