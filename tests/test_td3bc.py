"""TD3BC, and learn_batch of TD3 / DDPG, on the GPU: against the recordings of the reference (tests/golden/td3bc_*.npz,
{td3,ddpg}_batch.npz: same sampled indices, same `torch.normal` target noise), against oracle/td3bc_oracle.py at Pearl's
offline benchmark shape, and against the learner itself (learn_batch vs learn, one call vs several, graphs vs plain
launches, launch counts, graph re-use).  Tolerance: elementwise 1e-4 (tests/_tol.py)."""
import os
import random

import numpy as np
import pytest
import torch

from _tol import close as _close, close_params as _close_params
from conftest import GOLDEN
from oracle.pearl_oracle import flat
from oracle.td3bc_oracle import OracleTD3BC

pytestmark = pytest.mark.gpu

CASES = ["td3bc_learn", "td3bc_batch", "td3bc_lr", "td3_batch", "ddpg_batch"]


def _classes():
    from pearl_b200.td3 import B200DeepDeterministicPolicyGradient, B200TD3, B200TD3BC
    return dict(td3=B200TD3, ddpg=B200DeepDeterministicPolicyGradient, td3bc=B200TD3BC)


def _buffer(st, ac, rw, ns, term):
    import pearl_b200
    n = st.shape[0]
    buf = pearl_b200.B200ReplayBuffer(n)
    buf.is_action_continuous = True
    buf.push_batch(torch.from_numpy(st), torch.from_numpy(ac), torch.from_numpy(rw), torch.from_numpy(ns), torch.from_numpy(term),
                   torch.zeros(n, dtype=torch.bool))
    return buf


def _batch(d, ix, device=None, term_dtype=torch.bool):
    from pearl_b200 import TransitionBatch
    t = lambda k: torch.from_numpy(np.ascontiguousarray(d[k][ix])).to(device or "cpu")  # noqa: E731
    return TransitionBatch(state=t("state"), action=t("action"), reward=t("reward"), next_state=t("next_state"),
                           terminated=t("terminated").to(term_dtype))


def _learner(fx, graph):
    kind = str(fx["kind"])
    lrs = fx["call_lrs"][0]
    kw = dict(state_dim=int(fx["obs"]), low=fx["low"], high=fx["high"], actor_hidden_dims=[32, 32], critic_hidden_dims=[32, 32],
              training_rounds=int(fx["rounds"]), batch_size=int(fx["batch"]), actor_learning_rate=float(lrs[0]),
              critic_learning_rate=float(lrs[1]), actor_soft_update_tau=float(fx["actor_tau"]),
              critic_soft_update_tau=float(fx["critic_tau"]), discount_factor=float(fx["gamma"]))
    if kind == "td3bc":
        kw.update(behavior_hidden_dims=[int(x) for x in fx["behavior_hidden"]], alpha_bc=float(fx["call_alpha"][0]))
    pl = _classes()[kind](**kw)
    pl.use_cuda_graph = graph
    init = {k[5:]: fx[k] for k in fx.files if k.startswith("init_")}
    pl.load_parameters(init.pop("actor"), init.pop("q1"), init.pop("q2"), init.pop("actor_t"), init.pop("q1t"), init.pop("q2t"), **init)
    return pl


def _vectors(pl):
    v = dict(actor=pl.actor_params, actor_t=pl.actor_target_params, critic=pl.critic_params, critic_t=pl.critic_target_params)
    for i in range(3):
        v[f"actor_state{i}"], v[f"critic_state{i}"] = pl._actor_state[i], pl._critic_state[i]
    return {k: x.cpu().numpy().copy() for k, x in v.items()}


@pytest.mark.parametrize("graph", [True, False])
@pytest.mark.parametrize("case", CASES)
def test_matches_reference_recording(case, graph):
    """Every learn() and learn_batch() call of the recording: learn() samples the recorded indices from the ring,
    learn_batch() gets the recorded rows; learning-rate changes re-create the handle, which keeps the last actor loss."""
    fx = np.load(os.path.join(GOLDEN, f"{case}.npz"))
    pl = _learner(fx, graph)
    buf = _buffer(fx["state"], fx["action"], fx["reward"], fx["next_state"], fx["terminated"])
    random.setstate((3, tuple(int(x) for x in fx["rng_before"]), None))
    R, B, A = int(fx["rounds"]), int(fx["batch"]), int(fx["act"])
    noise = torch.from_numpy(fx["noise"]) if len(fx["noise"]) else None
    al, cl = [], []
    k = j = 0
    for c, kind in enumerate(fx["call_kind"]):
        lrs = tuple(float(x) for x in fx["call_lrs"][c])
        if lrs != (pl._actor_learning_rate, pl._critic_learning_rate):
            pl.set_learning_rates(*lrs)
        if hasattr(pl, "alpha_bc"):
            pl.alpha_bc = float(fx["call_alpha"][c])
        pl._training_steps = int(fx["call_steps"][c])
        if kind == 0:
            trace = {}
            rep = pl.learn(buf, noise=None if noise is None else noise[j:j + R], trace=trace)
            assert np.array_equal(trace["idx"].numpy(), fx["idx"][k:k + R])
            assert pl._training_steps == int(fx["call_steps"][c]) + R
            al += rep["actor_loss"]; cl += rep["critic_loss"]
            k += R; j += R if noise is not None else 0
        else:
            rep = pl.learn_batch(_batch(fx, fx["idx"][k].astype(np.int64), term_dtype=torch.bool if c % 2 else torch.uint8),
                                 noise=None if noise is None else noise[j])
            assert pl._training_steps == int(fx["call_steps"][c])
            al.append(rep["actor_loss"]); cl.append(rep["critic_loss"])
            k += 1; j += 1 if noise is not None else 0
    assert k == len(fx["idx"]) and (noise is None or j == len(noise)) and B * A > 0
    _close(al, fx["actor_loss"], "actor_loss")
    _close(cl, fx["critic_loss"], "critic_loss")
    pc = pl.critic_params.numel() // 2
    _close(pl.actor_params.cpu().numpy(), fx["actor_after"], "actor")
    _close(pl.actor_target_params.cpu().numpy(), fx["actor_t_after"], "actor target")
    _close(pl.critic_params[:pc].cpu().numpy(), fx["q1_after"], "q1")
    _close(pl.critic_params[pc:].cpu().numpy(), fx["q2_after"], "q2")
    _close(pl.critic_target_params[:pc].cpu().numpy(), fx["q1t_after"], "q1 target")
    _close(pl.critic_target_params[pc:].cpu().numpy(), fx["q2t_after"], "q2 target")


def _adam_flat(opt, params, key):
    return torch.cat([opt.state[p][key].reshape(-1) for p in params])


def _relu_boundary(net, x, tol=1e-5):
    """Flat indices of the parameters whose gradient may depend on the last bit of a hidden unit's input: the weight row and
    bias of every ReLU unit whose pre-activation lies within `tol` of zero on some row of `x`, and every parameter of the
    layers below it."""
    idx, off = [], 0
    with torch.no_grad():
        for layer in net:
            lin = layer[0]
            pre = lin(x)
            n_w = lin.weight.numel()
            if len(layer) > 1 and isinstance(layer[1], torch.nn.ReLU):
                flagged = torch.nonzero((pre.abs() < tol).any(0)).view(-1).tolist()
                if flagged and off:
                    idx += list(range(off))
                for j in flagged:
                    idx += list(range(off + j * lin.in_features, off + (j + 1) * lin.in_features)) + [off + n_w + j]
            off += n_w + lin.bias.numel()
            x = layer(x)
    return np.unique(np.asarray(idx, dtype=np.int64))


def _close_net(got, net, skip, what, lr):
    want = flat(net).numpy()
    keep = np.ones(want.size, dtype=bool)
    keep[skip] = False
    _close_params(got[keep], want[keep], what, lr, 1)
    if skip.size:
        err = float(np.abs(got[skip] - want[skip]).max())
        print(f"    {what}: {skip.size} elements in ReLU-boundary rows, max abs err {err:.3e}")
        assert err <= 2.02 * lr + 2e-6, f"{what}: ReLU-boundary row off by {err:.3e}, beyond one AdamW step"


def _offline_data(n, obs, act, seed):
    rng = np.random.Generator(np.random.PCG64(seed))
    low, high = np.full(act, -1.0, np.float32), np.full(act, 1.0, np.float32)
    low[0], high[0] = -0.5, 2.0                     # one asymmetric coordinate: b and a live in different ranges there
    return dict(state=rng.standard_normal((n, obs)).astype(np.float32), next_state=rng.standard_normal((n, obs)).astype(np.float32),
                reward=rng.standard_normal(n).astype(np.float32), terminated=rng.random(n) < 0.03,
                action=rng.uniform(low, high, size=(n, act)).astype(np.float32), low=low, high=high)


@pytest.mark.parametrize("engine", [0, 2])
def test_td3bc_offline_shape_against_oracle(engine):
    """Pearl's offline benchmark shape (obs 17, 6 actions, [256, 256] actor, critics and behaviour net, batch 256), freq 2.
    Each round starts from the oracle's state (parameters, targets and AdamW moments), so AdamW's sign-like first steps on
    gradients that are zero to within fp32 summation noise stay counted outliers of one round (`close_params`)."""
    from pearl_b200 import _lib
    from pearl_b200.td3 import B200TD3BC
    torch.manual_seed(7)
    threads = torch.get_num_threads()
    torch.set_num_threads(8)
    obs, act, n, B, R, lr = 17, 6, 3000, 256, 6, 3e-4
    d = _offline_data(n, obs, act, seed=12)
    buf = _buffer(d["state"], d["action"], d["reward"], d["next_state"], d["terminated"])
    lib = _lib.load()
    prev = lib.prl_get_contraction_engine()
    _lib.check(lib.prl_set_contraction_engine(engine))
    try:
        pl = B200TD3BC(state_dim=obs, low=d["low"], high=d["high"], actor_hidden_dims=[256, 256], critic_hidden_dims=[256, 256],
                       behavior_hidden_dims=[256, 256], training_rounds=1, batch_size=B, actor_learning_rate=lr, critic_learning_rate=lr,
                       seed=5)
        pc = pl.critic_params.numel() // 2
        init = dict(actor=pl.actor_params.cpu().numpy(), actor_t=pl.actor_target_params.cpu().numpy(),
                    q1=pl.critic_params[:pc].cpu().numpy(), q2=pl.critic_params[pc:].cpu().numpy(),
                    q1t=pl.critic_target_params[:pc].cpu().numpy(), q2t=pl.critic_target_params[pc:].cpu().numpy())
        orc = OracleTD3BC(obs, act, (256, 256), (256, 256), d["low"], d["high"], behavior_hidden=(256, 256), actor_lr=lr, critic_lr=lr,
                          init=init)
        pl.load_parameters(init["actor"], init["q1"], init["q2"], init["actor_t"], init["q1t"], init["q2t"], behavior=flat(orc.behavior))
        g = torch.Generator().manual_seed(9)
        random.seed(23)
        for r in range(R):
            noise = torch.randn((1, B, act), generator=g) * 0.2
            trace = {}
            rep = pl.learn(buf, noise=noise, trace=trace)
            i = trace["idx"][0].numpy()
            t = lambda k: torch.from_numpy(d[k][i])  # noqa: E731
            s = t("state")
            sa = torch.cat([s, orc.act(orc.actor, s)], dim=-1)
            skip_a = _relu_boundary(orc.actor, s)
            skip_q = [_relu_boundary(orc.q[z], torch.cat([s, t("action")], dim=-1)) for z in range(2)]
            skip_q[0] = np.union1d(skip_q[0], _relu_boundary(orc.q[0], sa.detach()))
            orc.training_steps += 1
            out = orc.learn_batch(dict(state=s, action=t("action"), reward=t("reward"), next_state=t("next_state"),
                                       terminated=t("terminated")), noise[0])
            _close(rep["actor_loss"], [out["actor_loss"]], f"round {r} actor_loss")
            _close(rep["critic_loss"], [out["critic_loss"]], f"round {r} critic_loss")
            _close_net(pl.actor_params.cpu().numpy(), orc.actor, skip_a, "actor", lr)
            _close_net(pl.critic_params[:pc].cpu().numpy(), orc.q[0], skip_q[0], "q1", lr)
            _close_net(pl.critic_params[pc:].cpu().numpy(), orc.q[1], skip_q[1], "q2", lr)
            _close_params(pl.actor_target_params.cpu().numpy(), flat(orc.actor_t).numpy(), "actor target", lr, 1)
            _close_params(pl.critic_target_params[:pc].cpu().numpy(), flat(orc.qt[0]).numpy(), "q1 target", lr, 1)
            _close_params(pl.critic_target_params[pc:].cpu().numpy(), flat(orc.qt[1]).numpy(), "q2 target", lr, 1)
            # the next round starts from the oracle's state
            pl.load_parameters(flat(orc.actor), flat(orc.q[0]), flat(orc.q[1]), flat(orc.actor_t), flat(orc.qt[0]), flat(orc.qt[1]))
            cp = list(orc.q[0].parameters()) + list(orc.q[1].parameters())
            for z, key in enumerate(("exp_avg", "exp_avg_sq", "max_exp_avg_sq")):
                if orc.opt_actor.state:
                    pl._actor_state[z].copy_(_adam_flat(orc.opt_actor, list(orc.actor.parameters()), key))
                pl._critic_state[z].copy_(_adam_flat(orc.opt_critic, cp, key))
    finally:
        _lib.check(lib.prl_set_contraction_engine(prev))
        torch.set_num_threads(threads)


def _small(kind, graph=True, seed=3, **extra):
    d = _offline_data(400, 9, 3, seed=31)
    kw = dict(state_dim=9, low=d["low"], high=d["high"], actor_hidden_dims=[64, 48], critic_hidden_dims=[64, 32], batch_size=64,
              actor_learning_rate=1e-3, critic_learning_rate=2e-3, seed=seed, **extra)
    if kind == "td3bc":
        kw.update(behavior_hidden_dims=[40, 24])
    pl = _classes()[kind](**kw)
    if kind == "td3bc":
        pl.behavior_params.copy_(torch.randn(pl.behavior_params.numel(), generator=torch.Generator().manual_seed(4)) * 0.2)
    pl.use_cuda_graph = graph
    return pl, d


@pytest.mark.parametrize("kind", ["td3", "ddpg", "td3bc"])
@pytest.mark.parametrize("steps", [0, 1])
def test_learn_batch_on_the_rows_learn_gathered_is_bit_identical(kind, steps):
    """learn() at training step s counts the step first, so learn_batch at s + 1 on the rows learn() sampled, with the same
    noise, is the same round: every vector and both losses agree bit for bit."""
    a, d = _small(kind)
    b, _ = _small(kind)
    buf = _buffer(d["state"], d["action"], d["reward"], d["next_state"], d["terminated"])
    noise = torch.randn((1, 64, 3), generator=torch.Generator().manual_seed(2)) * 0.2
    a._training_steps, b._training_steps = steps, steps + 1
    random.seed(5)
    trace = {}
    ra = a.learn(buf, noise=noise, trace=trace)
    rb = b.learn_batch(_batch(d, trace["idx"][0].numpy().astype(np.int64), device="cuda"), noise=noise[0])
    assert (ra["actor_loss"][0], ra["critic_loss"][0]) == (rb["actor_loss"], rb["critic_loss"])
    va, vb = _vectors(a), _vectors(b)
    for k in va:
        assert np.array_equal(va[k], vb[k]), k


@pytest.mark.parametrize("kind", ["td3", "td3bc"])
def test_rounds_per_call_and_graphs_do_not_change_results(kind):
    """One learn() of R rounds = R learn() calls of one round = the same with plain launches, bit for bit; learn_batch
    likewise with graphs on and off."""
    R = 5
    noise = torch.randn((R, 64, 3), generator=torch.Generator().manual_seed(6)) * 0.2
    runs = []
    for graph, per_call in ((True, R), (True, 1), (False, R)):
        pl, d = _small(kind, graph, training_rounds=per_call)
        buf = _buffer(d["state"], d["action"], d["reward"], d["next_state"], d["terminated"])
        random.seed(8)
        losses = ([], [])
        for c in range(R // per_call):
            rep = pl.learn(buf, noise=noise[c * per_call:(c + 1) * per_call])
            losses[0].extend(rep["actor_loss"]); losses[1].extend(rep["critic_loss"])
        for c in range(3):
            pl._training_steps = c
            rep = pl.learn_batch(_batch(d, np.arange(64 * c, 64 * c + 64)), noise=noise[c])
            losses[0].append(rep["actor_loss"]); losses[1].append(rep["critic_loss"])
        runs.append((losses, _vectors(pl)))
    for losses, vec in runs[1:]:
        assert losses == runs[0][0]
        for k in vec:
            assert np.array_equal(vec[k], runs[0][1][k]), k


def test_launch_counts_and_graph_reuse():
    """A fixed launch count per round for each variant: TD3BC's actor round adds the behaviour net's three contractions,
    its other round is TD3's.  Alternating learn() and learn_batch() over both variants captures each round once."""
    counts = {}
    for kind in ("td3", "td3bc"):
        for graph in (True, False):
            pl, d = _small(kind, graph, training_rounds=1)
            buf = _buffer(d["state"], d["action"], d["reward"], d["next_state"], d["terminated"])
            batch = _batch(d, np.arange(64))
            seen = []
            for it in range(3):
                for steps in (0, 1):
                    pl._training_steps = steps
                    pl.learn_batch(batch)
                    seen.append(("batch", steps, int(pl._lib.prl_td3_last_launches(pl._handle))))
                    pl._training_steps = steps + 1       # learn() counts first: steps + 2 rounds the other variant
                    pl.learn(buf)
                    seen.append(("learn", steps, int(pl._lib.prl_td3_last_launches(pl._handle))))
                if it == 0:
                    warm = pl.graph_captures
            if graph:
                assert warm == 4 and pl.graph_captures == 4
            per = {}
            for what, steps, n in seen:
                per.setdefault((what, steps), set()).add(n)
            assert all(len(v) == 1 for v in per.values()), per
            update = per[("batch", 0)].pop()
            skip = per[("batch", 1)].pop()
            assert per[("learn", 0)] == {update} and per[("learn", 1)] == {skip}
            counts[kind, graph] = (update, skip)
    for graph in (True, False):
        assert counts["td3bc", graph] == (counts["td3", graph][0] + 3, counts["td3", graph][1])
        assert counts["td3", graph] == counts["td3", True]


def test_alpha_bc_is_read_every_call():
    """A new alpha_bc reaches the next round through the same handle and the same captured graph."""
    a, d = _small("td3bc")
    b, _ = _small("td3bc")
    batch = _batch(d, np.arange(64))
    assert a.learn_batch(batch) == b.learn_batch(batch)
    caps, h = a.graph_captures, a._handle.value
    a.alpha_bc = 0.5
    ra, rb = a.learn_batch(batch), b.learn_batch(batch)
    assert a._handle.value == h and a.graph_captures == caps
    assert ra["actor_loss"] != rb["actor_loss"]
    a.alpha_bc = 2.5
    b.alpha_bc = 0.5
    assert a.learn_batch(batch)["actor_loss"] != b.learn_batch(batch)["actor_loss"]


def test_refusals():
    from pearl_b200.td3 import B200TD3BC
    import pearl_b200
    with pytest.raises(NotImplementedError, match="two hidden layers"):
        B200TD3BC(state_dim=4, low=[-1.0], high=[1.0], actor_hidden_dims=[8, 8], critic_hidden_dims=[8, 8], behavior_hidden_dims=[8])
    pl, d = _small("td3bc")
    with pytest.raises(ValueError, match="behavior has"):
        pl.load_parameters(pl.actor_params, pl.critic_params[:pl.critic_params.numel() // 2],
                           pl.critic_params[pl.critic_params.numel() // 2:], behavior=torch.zeros(7))
    good = _batch(d, np.arange(16))
    bad_state = pearl_b200.TransitionBatch(state=good.state[:, :5], action=good.action, reward=good.reward,
                                           next_state=good.next_state[:, :5], terminated=good.terminated)
    with pytest.raises(ValueError, match="batch.state"):
        pl.learn_batch(bad_state)
    ids = pearl_b200.TransitionBatch(state=good.state, action=torch.zeros(16, 1, dtype=torch.long), reward=good.reward,
                                     next_state=good.next_state, terminated=good.terminated)
    with pytest.raises(ValueError, match="continuous actions"):
        pl.learn_batch(ids)
    disc = pearl_b200.B200ReplayBuffer(32)
    disc.push_batch(good.state, torch.zeros(16, dtype=torch.long), good.reward, good.next_state, good.terminated,
                    torch.zeros(16, dtype=torch.bool), max_number_actions=4)
    with pytest.raises(ValueError, match="is_action_continuous"):
        pl.learn(disc)
