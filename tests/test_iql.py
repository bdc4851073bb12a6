"""Implicit Q-Learning on the GPU (pearl_b200.B200ImplicitQLearning, csrc/iql.cu) against
(a) the recordings of the reference's PearlAgent(ImplicitQLearning, BasicReplayBuffer) (tests/golden/iql_*.npz: learn()
    with the same indices from CPython's `random.sample` and the same torch.randint draws, and agent.learn_batch() on
    sampled batches), elementwise 1e-4 (tests/_tol.py);
(b) oracle/iql_oracle.py at the offline benchmark's shape (continuous obs 17, act 6, [256, 256], batch 256) and at a
    discrete stress shape (obs 128, 16 actions, [256, 256], batch 256), step by step from a re-synchronised state, under
    the SIMT engine and the tensor-core engine;
plus bit-identity (learn_batch vs learn, round chunking, graph replay, run to run), the launch count and the rejected
inputs."""
import os
import random

import numpy as np
import pytest
import torch

from conftest import GOLDEN
from oracle.iql_oracle import OracleIQL
from oracle.pearl_oracle import flat

pytestmark = pytest.mark.gpu

from _tol import close as _close, close_params as _close_params  # noqa: E402


def _buffer(n, state, action, reward, next_state, term, n_actions=None, **kw):
    import pearl_b200
    buf = pearl_b200.B200ReplayBuffer(n, **kw)
    t = torch.as_tensor
    if n_actions is None:
        buf.is_action_continuous = True
        buf.push_batch(t(state), t(action).float(), t(reward), t(next_state), t(term), torch.zeros(n, dtype=torch.bool))
    else:
        buf.push_batch(t(state), t(action).to(torch.int32), t(reward), t(next_state), t(term), torch.zeros(n, dtype=torch.bool),
                       max_number_actions=n_actions)
    return buf


def _learner(obs, hidden, **kw):
    import pearl_b200
    return pearl_b200.B200ImplicitQLearning(state_dim=obs, actor_hidden_dims=list(hidden), critic_hidden_dims=list(hidden),
                                            value_critic_hidden_dims=list(hidden), **kw)


def _act_kw(fx):
    return dict(n_actions=int(fx["n_actions"])) if bool(fx["discrete"]) else dict(low=fx["low"], high=fx["high"])


def _batch(d, i, n_actions=None, one_hot=True):
    """A TransitionBatch of rows i, with actions as the reference's preprocess_batch leaves them (one-hot) or as ids."""
    import pearl_b200
    t = lambda k: torch.from_numpy(np.asarray(d[k][i]))  # noqa: E731
    a = t("action")
    if n_actions is not None:
        a = torch.nn.functional.one_hot(a.long(), n_actions).float() if one_hot else a.long().view(-1, 1)
    return pearl_b200.TransitionBatch(state=t("state"), action=a, reward=t("reward"), next_state=t("next_state"),
                                      terminated=t("terminated"))


@pytest.mark.parametrize("case", ["iql_discrete", "iql_continuous", "iql_lr", "iql_batch"])
def test_iql_matches_reference_recording(case):
    fx = np.load(os.path.join(GOLDEN, f"{case}.npz"))
    n, R, B, calls = int(fx["n"]), int(fx["rounds"]), int(fx["batch"]), int(fx["calls"])
    disc = bool(fx["discrete"])
    A = int(fx["n_actions"]) if disc else None
    buf = _buffer(n, fx["state"], fx["action"], fx["reward"], fx["next_state"], fx["terminated"], A)
    lrs = [float(x) for x in fx["lrs"]]
    pl = _learner(int(fx["obs"]), fx["hidden"].tolist(), training_rounds=R, batch_size=B, actor_learning_rate=lrs[0],
                  critic_learning_rate=lrs[1], value_critic_learning_rate=lrs[2], critic_soft_update_tau=float(fx["tau"]),
                  discount_factor=float(fx["gamma"]), expectile=float(fx["expectile"]),
                  temperature_advantage_weighted_regression=float(fx["temperature"]), advantage_clamp=float(fx["advantage_clamp"]),
                  **_act_kw(fx))
    pl.load_parameters(fx["init_actor"], fx["init_q1"], fx["init_q2"], fx["init_value"], fx["init_q1t"], fx["init_q2t"])
    random.setstate((3, tuple(int(x) for x in fx["rng_before"]), None))
    torch_rng = torch.get_rng_state()
    torch.set_rng_state(torch.from_numpy(fx["torch_rng_before"]))
    losses = {"value_loss": [], "actor_loss": [], "critic_loss": []}
    idx, handles = [], []
    try:
        if bool(fx["learn_batch"]):
            for _ in range(calls):      # offline_learning(): sample a batch, agent.learn_batch(batch)
                logical, _ = buf.sample_indices(B, 1)
                i = logical[0].cpu().numpy()
                idx.append(i.tolist())
                rep = pl.learn_batch(_batch(fx, i, A))
                for k in losses:
                    losses[k].append(rep[k])
            assert pl._training_steps == 0, "learn_batch advanced the training-step count"
        else:
            for c in range(calls):
                pl.set_learning_rates(*[float(x) for x in fx["call_lrs"][c]])
                trace = {}
                rep = pl.learn(buf, trace=trace)
                handles.append(pl._handle.value)
                for k in losses:
                    losses[k] += rep[k]
                idx += trace["idx"].tolist()
            assert len(set(handles)) == 1, "a learning-rate change re-created the C handle"
        assert idx == fx["idx"].tolist()                                                  # bit-exact sampling
        assert random.getstate()[1] == tuple(int(x) for x in fx["rng_after"])              # CPython's random as the reference left it
        assert torch.equal(torch.get_rng_state(), torch.from_numpy(fx["torch_rng_after"]))   # torch's CPU RNG as well
    finally:
        torch.set_rng_state(torch_rng)
    for k, v in losses.items():
        _close(v, fx[k], k)
    pc = pl.critic_params.numel() // 2
    _close(pl.actor_params.cpu().numpy(), fx["actor_after"], "actor")
    _close(pl.critic_params[:pc].cpu().numpy(), fx["q1_after"], "q1")
    _close(pl.critic_params[pc:].cpu().numpy(), fx["q2_after"], "q2")
    _close(pl.critic_target_params[:pc].cpu().numpy(), fx["q1t_after"], "q1 target")
    _close(pl.critic_target_params[pc:].cpu().numpy(), fx["q2t_after"], "q2 target")
    _close(pl.value_params.cpu().numpy(), fx["value_after"], "value")
    for i, k in enumerate(("exp_avg", "exp_avg_sq", "max_exp_avg_sq")):
        _close(pl._value_state[i].cpu().numpy(), fx[f"value_{k}"], f"value {k}", atol=1e-9)


def _data(n, obs, seed, n_actions=None, low=None, high=None, p_term=0.1):
    rng = np.random.Generator(np.random.PCG64(seed))
    q8 = lambda x: (np.rint(x * 256) / 256).astype(np.float32)  # noqa: E731
    d = dict(state=q8(rng.standard_normal((n, obs))), next_state=q8(rng.standard_normal((n, obs))), reward=q8(rng.standard_normal(n)),
             terminated=rng.random(n) < p_term)
    d["action"] = (rng.integers(0, n_actions, size=n).astype(np.int32) if n_actions is not None
                   else q8(rng.uniform(low, high, size=(n, len(low)))))
    return d


def _adam_flat(opt, params, key):
    return torch.cat([opt.state[p][key].reshape(-1) for p in params])


def _sync_from_oracle(pl, orc):
    """Parameters, targets and the AdamW moments of all three networks from the oracle."""
    pl.load_parameters(flat(orc.actor), flat(orc.q[0]), flat(orc.q[1]), flat(orc.value), flat(orc.qt[0]), flat(orc.qt[1]))
    cp = list(orc.q[0].parameters()) + list(orc.q[1].parameters())
    for i, key in enumerate(("exp_avg", "exp_avg_sq", "max_exp_avg_sq")):
        pl._actor_state[i].copy_(_adam_flat(orc.opt_actor, list(orc.actor.parameters()), key))
        pl._critic_state[i].copy_(_adam_flat(orc.opt_critic, cp, key))
        pl._value_state[i].copy_(_adam_flat(orc.opt_value, list(orc.value.parameters()), key))


def _relu_boundary(net, x, tol=1e-5):
    """Flat indices of the weight rows and biases of the hidden units of `net` (an oracle MLP, before its step) whose
    pre-activation lies within `tol` of zero on some row of `x`.  Whether such a unit passes its gradient depends on the
    last bit of its input, so its row of the weight gradient may differ from the reference's by a whole batch row's share;
    so may, through the backward pass, every parameter of the layers below it, which are included as well."""
    idx, off = [], 0
    with torch.no_grad():
        for layer in net:
            lin = layer[0]
            pre = lin(x)
            n_w = lin.weight.numel()
            if len(layer) > 1:                               # a hidden layer (Linear + ReLU)
                flagged = torch.nonzero((pre.abs() < tol).any(0)).view(-1).tolist()
                if flagged and off:
                    idx += list(range(off))
                for j in flagged:
                    idx += list(range(off + j * lin.in_features, off + (j + 1) * lin.in_features)) + [off + n_w + j]
            off += n_w + lin.bias.numel()
            x = layer(x)
    return np.unique(np.asarray(idx, dtype=np.int64))


def _close_net(got, net, skip, what, lr):
    """`close_params` on every element outside the ReLU-boundary rows `skip` (`_relu_boundary` before the step); those rows
    are printed and held to the AdamW bound of one step."""
    want = flat(net).numpy()
    keep = np.ones(want.size, dtype=bool)
    keep[skip] = False
    _close_params(got[keep], want[keep], what, lr, 1)
    if skip.size:
        err = float(np.abs(got[skip] - want[skip]).max())
        print(f"    {what}: {skip.size} elements in ReLU-boundary rows, max abs err {err:.3e}")
        assert err <= 2.02 * lr + 2e-6, f"{what}: ReLU-boundary row off by {err:.3e}, beyond one AdamW step"


@pytest.mark.parametrize("engine", [0, 2])
@pytest.mark.parametrize("shape", ["offline_continuous", "discrete_128x16"])
def test_iql_stress_shape_against_oracle(shape, engine):
    """Each round starts from the oracle's state (parameters and AdamW moments): AdamW's first steps move an element by
    lr * sign(gradient) whatever its magnitude, so an element whose gradient is zero to within fp32 summation noise may
    step the other way (DESIGN.md §4); each round must agree elementwise to 1e-4 up to the counted outliers of
    `close_params`."""
    from pearl_b200 import _lib
    torch.manual_seed(7)
    threads = torch.get_num_threads()
    torch.set_num_threads(8)
    if shape == "offline_continuous":
        obs, A, act = 17, None, dict(low=np.full(6, -1.0, np.float32), high=np.full(6, 1.0, np.float32))
    else:
        obs, A, act = 128, 16, dict(n_actions=16)
    n, B, R, lr = 3000, 256, 8, 3e-4
    d = _data(n, obs, seed=11, n_actions=A, low=act.get("low"), high=act.get("high"))
    buf = _buffer(n, d["state"], d["action"], d["reward"], d["next_state"], d["terminated"], A)
    orc = OracleIQL(obs, (256, 256), (256, 256), (256, 256), actor_lr=lr, critic_lr=lr, value_lr=lr, gamma=0.99, tau=0.005,
                    expectile=0.7, temperature=3.0, advantage_clamp=100.0, **act)
    for m in [orc.actor] + orc.q:
        for mod in m.modules():
            if isinstance(mod, torch.nn.Linear):
                torch.nn.init.xavier_uniform_(mod.weight)
                mod.bias.data.fill_(0.01)
    for i in range(2):
        orc.qt[i].load_state_dict(orc.q[i].state_dict())
    lib = _lib.load()
    prev = lib.prl_get_contraction_engine()
    _lib.check(lib.prl_set_contraction_engine(engine))
    try:
        pl = _learner(obs, (256, 256), training_rounds=1, batch_size=B, actor_learning_rate=lr, critic_learning_rate=lr,
                      value_critic_learning_rate=lr, critic_soft_update_tau=0.005, discount_factor=0.99, expectile=0.7,
                      temperature_advantage_weighted_regression=3.0, **act)
        pl.load_parameters(flat(orc.actor), flat(orc.q[0]), flat(orc.q[1]), flat(orc.value))
        random.seed(19)
        pc = pl.critic_params.numel() // 2
        for r in range(R):
            trace = {}
            g = torch.get_rng_state()
            rep = pl.learn(buf, trace=trace)
            torch.set_rng_state(g)
            bits = torch.randint(0, 2, (1, 2))[0]
            i = trace["idx"][0].numpy()
            t = lambda k: torch.from_numpy(d[k][i])  # noqa: E731
            sa = torch.cat([t("state"), orc._action_input(t("action"))], dim=-1)
            skip = [_relu_boundary(orc.actor.net, t("state")), _relu_boundary(orc.q[0], sa), _relu_boundary(orc.q[1], sa),
                    _relu_boundary(orc.value, t("state"))]
            out = orc.learn_batch(dict(state=t("state"), action=t("action"), reward=t("reward"), next_state=t("next_state"),
                                       terminated=t("terminated")), bits)
            for k in ("value_loss", "critic_loss", "actor_loss"):
                _close(rep[k], [out[k]], f"round {r} {k}")
            _close_net(pl.actor_params.cpu().numpy(), orc.actor.net, skip[0], "actor", lr)
            _close_net(pl.critic_params[:pc].cpu().numpy(), orc.q[0], skip[1], "q1", lr)
            _close_net(pl.critic_params[pc:].cpu().numpy(), orc.q[1], skip[2], "q2", lr)
            _close_params(pl.critic_target_params[:pc].cpu().numpy(), flat(orc.qt[0]).numpy(), "q1 target", lr, 1)
            _close_params(pl.critic_target_params[pc:].cpu().numpy(), flat(orc.qt[1]).numpy(), "q2 target", lr, 1)
            _close_net(pl.value_params.cpu().numpy(), orc.value, skip[3], "value", lr)
            _sync_from_oracle(pl, orc)
    finally:
        _lib.check(lib.prl_set_contraction_engine(prev))
        torch.set_num_threads(threads)


def _vecs(pl):
    return [pl.actor_params.cpu(), pl.critic_params.cpu(), pl.critic_target_params.cpu(), pl.value_params.cpu(),
            pl._actor_state[1].cpu(), pl._critic_state[2].cpu(), pl._value_state[0].cpu()]


@pytest.mark.parametrize("discrete", [True, False])
def test_iql_learn_batch_equals_learn_bit_for_bit(discrete):
    """learn_batch on the rows a one-round learn() gathered, with the same two bits, leaves every vector bit-identical."""
    n, obs, B = 800, 12, 96
    act = dict(n_actions=5) if discrete else dict(low=[-1.0, 0.0, -2.0], high=[1.0, 0.5, 2.0])
    d = _data(n, obs, seed=43, n_actions=act.get("n_actions"), low=act.get("low"), high=act.get("high"))
    buf = _buffer(n, d["state"], d["action"], d["reward"], d["next_state"], d["terminated"], act.get("n_actions"))
    mk = lambda: _learner(obs, (64, 64), training_rounds=1, batch_size=B, seed=5, **act)  # noqa: E731
    a, b = mk(), mk()
    random.seed(3)
    torch.manual_seed(9)
    trace = {}
    rep_a = a.learn(buf, trace=trace)
    torch.manual_seed(9)
    rep_b = b.learn_batch(_batch(d, trace["idx"][0].numpy(), act.get("n_actions"), one_hot=False))
    assert [rep_a[k][0] for k in rep_b] == list(rep_b.values())
    for x, y in zip(_vecs(a), _vecs(b)):
        assert torch.equal(x, y)


@pytest.mark.parametrize("discrete", [True, False])
def test_iql_is_bit_reproducible(discrete):
    """One call of R rounds == R one-round calls (max_rounds_per_call=1); CUDA-graph replay == plain launches; two runs
    agree.  Bit for bit: the launch sequence and every summation order are fixed."""
    n, obs, B, R = 1500, 24, 128, 9
    act = dict(n_actions=6) if discrete else dict(low=[-1.0, -0.5], high=[1.0, 1.5])
    d = _data(n, obs, seed=23, n_actions=act.get("n_actions"), low=act.get("low"), high=act.get("high"))

    def run(per_call, graph):
        buf = _buffer(n, d["state"], d["action"], d["reward"], d["next_state"], d["terminated"], act.get("n_actions"))
        pl = _learner(obs, (64, 64), training_rounds=R, batch_size=B, max_rounds_per_call=per_call, seed=3, **act)
        pl.use_cuda_graph = graph
        random.seed(29)
        torch.manual_seed(31)
        rep = pl.learn(buf)
        rep["batch"] = pl.learn_batch(_batch(d, np.arange(B), act.get("n_actions")))
        return rep, _vecs(pl)

    base_rep, base = run(R, True)
    for per_call, graph in [(1, True), (R, False), (R, True)]:
        rep, vecs = run(per_call, graph)
        assert rep == base_rep, (per_call, graph)
        for a, b in zip(vecs, base):
            assert torch.equal(a, b), (per_call, graph)


def test_iql_launch_count_is_fixed():
    n, obs, B = 600, 8, 64
    for act, per_round in ((dict(n_actions=4), 36), (dict(low=[-1.0, -1.0], high=[1.0, 1.0]), 33)):
        d = _data(n, obs, seed=31, n_actions=act.get("n_actions"), low=act.get("low"), high=act.get("high"))
        buf = _buffer(n, d["state"], d["action"], d["reward"], d["next_state"], d["terminated"], act.get("n_actions"))
        pl = _learner(obs, (32, 32), training_rounds=5, batch_size=B, **act)
        trace = {}
        pl.learn(buf, trace=trace)
        assert trace["launches"] == 5 * per_round      # 25 contractions + 11 (discrete) / 8 small kernels per round (DESIGN.md §3.4)


def test_iql_rejects_bad_inputs():
    import ctypes as C

    import pearl_b200
    from pearl_b200 import _lib
    from pearl_b200.replay_buffer import _stream_ptr
    n, obs, A, B = 64, 6, 4, 16
    d = _data(n, obs, seed=41, n_actions=A)
    dc = _data(n, obs, seed=41, low=[-1.0, -1.0], high=[1.0, 1.0])
    pl = _learner(obs, (16, 16), training_rounds=2, batch_size=B, n_actions=A)
    cl = _learner(obs, (16, 16), training_rounds=2, batch_size=B, low=[-1.0, -1.0], high=[1.0, 1.0])
    assert pl.learn(pearl_b200.B200ReplayBuffer(16)) == {}                  # empty buffer: nothing to do
    with pytest.raises(NotImplementedError):                                # three hidden layers
        _learner(obs, (16, 16, 16), n_actions=A)
    with pytest.raises(ValueError):                                         # both action kinds / neither
        _learner(obs, (16, 16), n_actions=A, low=[-1.0], high=[1.0])
    with pytest.raises(ValueError):
        _learner(obs, (16, 16))
    disc_buf = _buffer(n, d["state"], d["action"], d["reward"], d["next_state"], d["terminated"], A)
    cont_buf = _buffer(n, dc["state"], dc["action"], dc["reward"], dc["next_state"], dc["terminated"])
    other_obs = _buffer(n, np.zeros((n, obs + 1), np.float32), d["action"], d["reward"], np.zeros((n, obs + 1), np.float32),
                        d["terminated"], A)
    with pytest.raises(ValueError):
        cl.learn(disc_buf)
    with pytest.raises(ValueError):
        pl.learn(cont_buf)
    # the C entry point itself refuses the other action kind, other dimensions and oversized batches before any launch
    dev = pl._device
    pl.learn(disc_buf)
    cl.learn(cont_buf)
    bits = torch.zeros((4, 2), dtype=torch.int32, device=dev)
    out = torch.zeros((3, 4), dtype=torch.float32, device=dev)
    p = _lib.ptr
    for h, buf, batch in ((pl, cont_buf, B), (cl, disc_buf, B), (pl, other_obs, B), (pl, disc_buf, B + 1)):
        before = [h.actor_params.clone(), h.critic_params.clone(), h.value_params.clone()]
        rng0 = buf.get_rng_state()
        rc = h._lib.prl_iql_learn(h._handle, buf.handle, 1, batch, p(bits), p(out[0]), p(out[1]), p(out[2]), C.c_void_p(0), _stream_ptr(dev))
        assert rc == _lib.PRL_EINVAL, _lib.last_error()
        torch.cuda.synchronize()
        assert np.array_equal(buf.get_rng_state(), rng0), "the sampler ran"
        assert all(torch.equal(x, y) for x, y in zip(before, [h.actor_params, h.critic_params, h.value_params])), "a learner kernel ran"
    # a shard of a multi-GPU buffer samples global slots: rejected before the sampler or any learner kernel runs
    sharded = pearl_b200.B200ReplayBuffer(n, rng="device")
    t = torch.from_numpy
    sharded.push_batch_sharded(0, 2, t(d["state"]), t(d["action"]), t(d["reward"]), t(d["next_state"]), t(d["terminated"]),
                               torch.zeros(n, dtype=torch.bool), max_number_actions=A)
    sharded.seed(5)
    rng0 = sharded.get_rng_state()
    params0 = [pl.actor_params.clone(), pl.critic_params.clone(), pl.value_params.clone()]
    with pytest.raises(ValueError, match="shard"):
        pl.learn(sharded)
    torch.cuda.synchronize()
    assert np.array_equal(sharded.get_rng_state(), rng0), "the sampler ran"
    assert all(torch.equal(x, y) for x, y in zip(params0, [pl.actor_params, pl.critic_params, pl.value_params])), "a learner kernel ran"
