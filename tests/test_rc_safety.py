"""The reward-constrained safety module on the GPU: TD3 / DDPG / TD3BC learn() on cost-shaped rewards plus the CUDA cost
critic and lambda step, against the recordings of the reference (tests/golden/rc_*.npz: same sampled indices, same
`torch.normal` target noise) with graphs on and off, against oracle/rc_safety_oracle.py at Pearl's RCTD3 benchmark shape,
and the cost column of the replay ring (round trips, snapshots, dynamic upgrade, refusals), the unchanged behaviour of
learners that get no multiplier, graph re-use across lambda changes and the refusals.  Tolerance: elementwise 1e-4
(tests/_tol.py)."""
import ctypes as C
import os
import random

import numpy as np
import pytest
import torch

from _tol import close as _close, close_params as _close_params
from conftest import GOLDEN
from oracle.pearl_oracle import flat
from oracle.rc_safety_oracle import OracleCostCritic, agent_learn
from oracle.td3_oracle import OracleTD3

pytestmark = pytest.mark.gpu

CASES = ["rc_td3", "rc_ddpg", "rc_zero", "rc_lr", "rc_td3bc"]


def _cost_buffer(st, ac, rw, ns, term, cost, device=False):
    import pearl_b200
    n = st.shape[0]
    buf = pearl_b200.B200ReplayBuffer(n)
    buf.is_action_continuous = True
    t = (lambda x: torch.from_numpy(np.ascontiguousarray(x)).cuda()) if device else torch.from_numpy  # noqa: E731
    buf.push_batch(t(st), t(ac), t(rw), t(ns), t(term), t(np.zeros(n, dtype=bool)), cost=None if cost is None else t(cost))
    return buf


def _learner(fx, graph):
    from pearl_b200.td3 import B200DeepDeterministicPolicyGradient, B200TD3, B200TD3BC
    kind = str(fx["kind"])
    lrs = fx["call_lrs"][0]
    kw = dict(state_dim=int(fx["obs"]), low=fx["low"], high=fx["high"], actor_hidden_dims=[32, 32], critic_hidden_dims=[32, 32],
              training_rounds=int(fx["rounds"]), batch_size=int(fx["batch"]), actor_learning_rate=float(lrs[0]),
              critic_learning_rate=float(lrs[1]), actor_soft_update_tau=float(fx["actor_tau"]),
              critic_soft_update_tau=float(fx["critic_tau"]), discount_factor=float(fx["gamma"]))
    cls = dict(td3=B200TD3, ddpg=B200DeepDeterministicPolicyGradient, td3bc=B200TD3BC)[kind]
    if kind == "td3bc":
        kw.update(behavior_hidden_dims=[int(x) for x in fx["behavior_hidden"]], alpha_bc=float(fx["alpha_bc"]))
    pl = cls(**kw)
    pl.use_cuda_graph = graph
    init = {k[5:]: fx[k] for k in fx.files if k.startswith("init_")}
    extra = dict(behavior=init["behavior"]) if kind == "td3bc" else {}
    pl.load_parameters(init["actor"], init["q1"], init["q2"], init["actor_t"], init["q1t"], init["q2t"], **extra)
    return pl, init


def _module(fx, init, graph):
    from pearl_b200.rc_safety import B200RCSafetyModule
    m = B200RCSafetyModule(constraint_value=float(fx["constraint"]), state_dim=int(fx["obs"]), low=fx["low"], high=fx["high"],
                           critic_hidden_dims=[32, 32], lambda_constraint_ub_value=float(fx["ub"]), cost_discount_factor=float(fx["cost_gamma"]),
                           lr_lambda=float(fx["lr_lambda"]), critic_learning_rate=float(fx["call_cost_lr"][0]),
                           critic_soft_update_tau=float(fx["cost_tau"]), batch_size=int(fx["rc_batch"]))
    m.use_cuda_graph = graph
    m.load_parameters(init["c1"], init["c2"], init["c1t"], init["c2t"])
    return m


def _run_recording(fx, graph):
    pl, init = _learner(fx, graph)
    rc = _module(fx, init, graph)
    pl.safety_module = rc
    buf = _cost_buffer(fx["state"], fx["action"], fx["reward"], fx["next_state"], fx["terminated"], fx["cost"])
    random.setstate((3, tuple(int(x) for x in fx["rng_before"]), None))
    R = int(fx["rounds"])
    noise = torch.from_numpy(fx["noise"]) if len(fx["noise"]) else None
    out = dict(actor_loss=[], critic_loss=[], cost_loss=[], cq=[], lam=[], lam_before=[])
    for c in range(int(fx["calls"])):
        clr = float(fx["call_cost_lr"][c])
        if clr != rc.critic_learning_rate:
            rc.set_critic_learning_rate(clr)
        out["lam_before"].append(rc.lambda_constraint)
        trace = {}
        rep = pl.learn(buf, noise=None if noise is None else noise[c * R:(c + 1) * R], trace=trace)
        base = c * (R + 1)
        assert np.array_equal(trace["idx"].numpy(), fx["idx"][base:base + R])
        t2 = {}
        rc.learn(buf, pl, trace=t2)
        assert np.array_equal(t2["idx"].numpy(), fx["idx"][base + R])
        out["actor_loss"] += rep["actor_loss"]; out["critic_loss"] += rep["critic_loss"]
        out["cost_loss"].append(rc.last_cost_critic_loss); out["cq"].append(rc.last_cost_q); out["lam"].append(rc.lambda_constraint)
    return pl, rc, out


@pytest.mark.parametrize("graph", [True, False])
@pytest.mark.parametrize("case", CASES)
def test_matches_reference_recording(case, graph):
    fx = np.load(os.path.join(GOLDEN, f"{case}.npz"))
    pl, rc, out = _run_recording(fx, graph)
    _close(out["lam_before"], fx["lambda_before"], "lambda before each call")
    _close(out["lam"], fx["lambda_after"], "lambda")
    _close(out["cq"], fx["cq"], "cq")
    _close(out["cost_loss"], fx["cost_loss"], "cost-critic loss")
    _close(out["actor_loss"], fx["actor_loss"], "actor_loss")
    _close(out["critic_loss"], fx["critic_loss"], "critic_loss")
    pc = pl.critic_params.numel() // 2
    got = dict(actor=pl.actor_params, actor_t=pl.actor_target_params, q1=pl.critic_params[:pc], q2=pl.critic_params[pc:],
               q1t=pl.critic_target_params[:pc], q2t=pl.critic_target_params[pc:], c1=rc.cost_critic_params[:pc],
               c2=rc.cost_critic_params[pc:], c1t=rc.cost_critic_target_params[:pc], c2t=rc.cost_critic_target_params[pc:])
    calls = int(fx["calls"])
    for name, v in got.items():
        lr = float(fx["call_cost_lr"].max()) if name.startswith("c") else 6e-4
        _close_params(v.cpu().numpy(), fx[f"{name}_after"], name, lr, calls * int(fx["rounds"]))
    for i, k in enumerate(("exp_avg", "exp_avg_sq", "max_exp_avg_sq")):
        want = fx[f"cost_{k}"]
        _close(rc.cost_critic_state[i].cpu().numpy(), want, f"cost critic {k}", atol=1e-4 * float(np.abs(want).max()))
    assert rc._step.adam_step == int(fx["cost_step"]) == calls


def test_lambda_changes_reuse_the_captured_graphs():
    """lambda travels in the per-call blocks: the TD3 rounds and the cost step capture once whatever lambda does."""
    fx = np.load(os.path.join(GOLDEN, "rc_td3.npz"))
    pl, rc, out = _run_recording(fx, True)
    assert len(set(out["lam"])) >= 3
    assert pl.graph_captures == 2          # with and without the actor update
    assert rc.graph_captures == 1
    assert rc.last_launches > 9


def test_benchmark_shape_against_the_oracle():
    """Pearl's RCTD3 shape (obs 17, act 6, [256, 256] everywhere, batch 256) over several agent.learn() calls."""
    from pearl_b200.rc_safety import B200RCSafetyModule
    from pearl_b200.td3 import B200TD3
    torch.manual_seed(5)
    O, A, n, B, R, calls = 17, 6, 4000, 256, 2, 3
    g = np.random.default_rng(11)
    q8 = lambda x: (np.rint(x * 256) / 256).astype(np.float32)  # noqa: E731
    d = dict(state=q8(g.standard_normal((n, O))), next_state=q8(g.standard_normal((n, O))), reward=q8(g.standard_normal(n)),
             action=q8(g.uniform(-1, 1, (n, A))), terminated=g.random(n) < 0.05, cost=q8(g.uniform(1, 2, n)))
    low, high = -np.ones(A, np.float32), np.ones(A, np.float32)
    pl = B200TD3(state_dim=O, low=low, high=high, actor_hidden_dims=[256, 256], critic_hidden_dims=[256, 256], training_rounds=R,
                 batch_size=B, seed=3)
    rc = B200RCSafetyModule(constraint_value=0.05, state_dim=O, low=low, high=high, critic_hidden_dims=[256, 256], lr_lambda=0.3,
                            lambda_constraint_ub_value=2.0, lambda_constraint_init_value=0.2, batch_size=B, seed=4)
    pl.safety_module = rc
    pc = pl.critic_params.numel() // 2
    orc = OracleTD3(O, A, (256, 256), (256, 256), low, high, actor_tau=0.005, critic_tau=0.005, actor_update_freq=2, noise_clip=0.5,
                    init=dict(actor=pl.actor_params.cpu(), actor_t=pl.actor_target_params.cpu(), q1=pl.critic_params[:pc].cpu(),
                              q2=pl.critic_params[pc:].cpu(), q1t=pl.critic_target_params[:pc].cpu(), q2t=pl.critic_target_params[pc:].cpu()))
    cc = OracleCostCritic(O, A, (256, 256), lr=1e-3, cost_gamma=0.5, tau=0.005, constraint=0.05, lr_lambda=0.3, ub=2.0, lam=0.2,
                          init=dict(c1=rc.cost_critic_params[:pc].cpu(), c2=rc.cost_critic_params[pc:].cpu(),
                                    c1t=rc.cost_critic_target_params[:pc].cpu(), c2t=rc.cost_critic_target_params[pc:].cpu()))
    buf = _cost_buffer(d["state"], d["action"], d["reward"], d["next_state"], d["terminated"], d["cost"], device=True)
    random.seed(21)
    t = torch.from_numpy
    lams, want = [], []
    for c in range(calls):
        noise = torch.randn((R, B, A)) * 0.2
        tr, t2 = {}, {}
        pl.learn(buf, noise=noise, trace=tr)
        rc.learn(buf, pl, trace=t2)
        rows = [{k: t(v[ix.numpy().astype(np.int64)]) for k, v in d.items()} for ix in list(tr["idx"]) + [t2["idx"]]]
        _, _, loss, cq = agent_learn(orc, cc, rows, R, noise)
        _close([rc.last_cost_q], [cq], f"cq, call {c}")
        _close([rc.last_cost_critic_loss], [loss], f"cost loss, call {c}")
        lams.append(rc.lambda_constraint); want.append(cc.lam)
    _close(lams, want, "lambda")
    assert 0 < min(lams) and max(lams) < 2.0 and len(set(lams)) == calls      # interior: the shaping is exercised
    _close_params(pl.actor_params.cpu().numpy(), flat(orc.actor).numpy(), "actor", 1e-3, calls * R)
    _close_params(rc.cost_critic_params[:pc].cpu().numpy(), flat(cc.q[0]).numpy(), "cost critic 1", 1e-3, calls)
    _close_params(rc.cost_critic_target_params[pc:].cpu().numpy(), flat(cc.qt[1]).numpy(), "cost critic 2 target", 1e-3, calls)


# ---------------------------------------------------------------- the cost column of the ring
def _rows(n=300, obs=5, act=2, seed=0):
    g = np.random.default_rng(seed)
    return (g.standard_normal((n, obs)).astype(np.float32), g.uniform(-1, 1, (n, act)).astype(np.float32),
            g.standard_normal(n).astype(np.float32), g.standard_normal((n, obs)).astype(np.float32), g.random(n) < 0.1,
            g.standard_normal(n).astype(np.float32))


@pytest.mark.parametrize("device", [False, True])
def test_cost_pushes_round_trip_through_sample(device):
    st, ac, rw, ns, te, co = _rows()
    buf = _cost_buffer(st, ac, rw, ns, te, co, device=device)
    assert buf.has_cost
    random.seed(3)
    logical, _ = buf.sample_indices(300, 1)
    random.seed(3)
    b = buf.sample(300)
    ix = logical[0].cpu().numpy().astype(np.int64)
    assert b.cost.dtype == torch.float32 and tuple(b.cost.shape) == (300,)
    assert np.array_equal(b.cost.cpu().numpy().view(np.uint32), co[ix].view(np.uint32))
    assert np.array_equal(b.reward.cpu().numpy(), rw[ix]) and np.array_equal(b.state.cpu().numpy(), st[ix])
    plain = _cost_buffer(st, ac, rw, ns, te, None)
    assert not plain.has_cost and plain.sample(4).cost is None


def test_single_pushes_and_snapshots_keep_costs():
    import pearl_b200
    st, ac, rw, ns, te, co = _rows(20)
    buf = pearl_b200.B200ReplayBuffer(32)
    buf.is_action_continuous = True
    for i in range(20):
        buf.push(torch.from_numpy(st[i]), torch.from_numpy(ac[i]), float(rw[i]), bool(te[i]), False, next_state=torch.from_numpy(ns[i]),
                 cost=float(co[i]))
    sd = buf.state_dict()
    assert sd["cost"] is True
    other = pearl_b200.B200ReplayBuffer(32)
    other.load_state_dict(sd)
    assert other.has_cost
    random.seed(9)
    a = buf.sample(20)
    random.seed(9)
    b = other.sample(20)
    assert torch.equal(a.cost, b.cost) and torch.equal(a.state, b.state)
    old = dict(sd)
    old.pop("cost")         # a snapshot without the key loads as a plain buffer ...
    plain = pearl_b200.B200ReplayBuffer(32)
    plain.load_state_dict(_plain_snapshot())
    assert not plain.has_cost
    with pytest.raises(ValueError):
        plain.load_state_dict(old)     # ... so a cost buffer's records without it fail the layout check


def _plain_snapshot():
    import pearl_b200
    st, ac, rw, ns, te, _ = _rows(10)
    buf = pearl_b200.B200ReplayBuffer(32)
    buf.is_action_continuous = True
    buf.push_batch(*(torch.from_numpy(x) for x in (st, ac, rw, ns, te, np.zeros(10, bool))))
    sd = buf.state_dict()
    sd.pop("cost")
    return sd


def test_dynamic_upgrade_keeps_costs():
    import pearl_b200
    g = np.random.default_rng(4)
    n, A = 12, 5
    buf = pearl_b200.B200ReplayBuffer(16)
    st, ns = g.standard_normal((n, 3)).astype(np.float32), g.standard_normal((n, 3)).astype(np.float32)
    co = g.standard_normal(n).astype(np.float32)
    buf.push_batch(torch.from_numpy(st[:8]), torch.arange(8) % A, torch.zeros(8), torch.from_numpy(ns[:8]), torch.zeros(8, dtype=torch.bool),
                   torch.zeros(8, dtype=torch.bool), max_number_actions=A, cost=torch.from_numpy(co[:8]))
    ids = torch.zeros(4, A, dtype=torch.uint8)
    ids[:, :2] = torch.tensor([3, 1], dtype=torch.uint8)
    buf.push_batch(torch.from_numpy(st[8:]), torch.arange(4), torch.zeros(4), torch.from_numpy(ns[8:]), torch.zeros(4, dtype=torch.bool),
                   torch.zeros(4, dtype=torch.bool), next_available_ids=ids, next_available_count=torch.full((4,), 2, dtype=torch.int32),
                   cost=torch.from_numpy(co[8:]))
    g_ = buf._gather_logical(torch.arange(n, dtype=torch.int32, device="cuda"))
    assert np.array_equal(g_["cost"].cpu().numpy(), co)
    assert g_["avail"][8:, :2].cpu().tolist() == [[3.0, 1.0]] * 4


def test_wrong_kind_pushes_multi_and_sharded_refusals():
    import pearl_b200
    from pearl_b200 import _lib
    st, ac, rw, ns, te, co = _rows(10)
    buf = _cost_buffer(st, ac, rw, ns, te, co)
    f = lambda x: torch.from_numpy(x)  # noqa: E731
    with pytest.raises(ValueError):
        buf.push_batch(f(st), f(ac), f(rw), f(ns), f(te), f(np.zeros(10, bool)))
    plain = _cost_buffer(st, ac, rw, ns, te, None)
    with pytest.raises(ValueError):
        plain.push_batch(f(st), f(ac), f(rw), f(ns), f(te), f(np.zeros(10, bool)), cost=f(co))
    with pytest.raises(ValueError):
        buf.set_shard(0, 2, 20)
    lib = _lib.load()
    arr = (C.c_void_p * 1)(buf.handle.value)
    tr = np.zeros(10, np.uint8)
    p = lambda x: C.c_void_p(x.ctypes.data)  # noqa: E731
    rc = lib.prl_buf_push_host_multi(arr, 1, 10, p(st), p(ac), p(rw), p(ns), p(te.astype(np.uint8)), p(tr), None)
    assert rc == _lib.PRL_EINVAL and "PRL_BUF_COST" in _lib.last_error()
    rc = lib.prl_buf_push_host(buf.handle, 10, p(st), p(ac), p(rw), p(ns), p(te.astype(np.uint8)), p(tr), None, None, None)
    assert rc == _lib.PRL_EINVAL
    for cls in (pearl_b200.B200PrioritizedReplayBuffer, pearl_b200.B200SARSAReplayBuffer):
        with pytest.raises(NotImplementedError):
            cls(16).push(torch.zeros(3), 0, 0.0, False, False, next_state=torch.zeros(3), max_number_actions=2, cost=1.0)


# ---------------------------------------------------------------- no multiplier: nothing changes
def _same_bits(a, b, what):
    assert torch.equal(a.view(torch.int32), b.view(torch.int32)), what


def test_td3_and_sac_on_a_cost_buffer_without_multiplier_are_unchanged():
    import pearl_b200
    from pearl_b200.td3 import B200TD3
    st, ac, rw, ns, te, co = _rows(400, obs=6, act=3, seed=8)
    for make in (lambda: B200TD3(state_dim=6, low=[-1] * 3, high=[1] * 3, actor_hidden_dims=[32, 32], critic_hidden_dims=[32, 32],
                                 training_rounds=4, batch_size=64, seed=1),
                 lambda: pearl_b200.actor_critic.SacCore(state_dim=6, low=[-1] * 3, high=[1] * 3, actor_hidden_dims=[32, 32],
                                                         critic_hidden_dims=[32, 32], training_rounds=4, batch_size=64, seed=1)):
        res = []
        for cost in (co, None):
            pl = make()
            buf = _cost_buffer(st, ac, rw, ns, te, cost)
            random.seed(5)
            torch.manual_seed(5)
            pl.learn(buf)
            pl.learn(buf)
            res.append((pl.actor_params.clone(), pl.critic_params.clone()))
        _same_bits(res[0][0], res[1][0], f"{type(pl).__name__} actor")
        _same_bits(res[0][1], res[1][1], f"{type(pl).__name__} critic")


def test_dqn_on_a_discrete_cost_buffer_is_unchanged():
    import pearl_b200

    class _Space:
        def __init__(self, A):
            self.n = A
            self.actions = [torch.tensor([i]) for i in range(A)]
            self.actions_batch = torch.arange(A).view(A, 1)
    g = np.random.default_rng(2)
    n, O, A = 300, 4, 3
    st, ns = torch.from_numpy(g.standard_normal((n, O)).astype(np.float32)), torch.from_numpy(g.standard_normal((n, O)).astype(np.float32))
    act, rw = torch.from_numpy(g.integers(0, A, n)), torch.from_numpy(g.standard_normal(n).astype(np.float32))
    te, co = torch.from_numpy(g.random(n) < 0.1), torch.from_numpy(g.standard_normal(n).astype(np.float32))
    res = []
    for cost in (co, None):
        torch.manual_seed(0)
        pl = pearl_b200.B200DeepQLearning(state_dim=O, action_space=_Space(A), hidden_dims=[32, 32], training_rounds=5, batch_size=32,
                                          action_representation_module=pearl_b200.OneHotActionTensorRepresentationModule(A)).to("cuda")
        buf = pearl_b200.B200ReplayBuffer(n)
        buf.push_batch(st, act, rw, ns, te, torch.zeros(n, dtype=torch.bool), max_number_actions=A, cost=cost)
        random.seed(1)
        pl.learn(buf)
        res.append({k: v.clone() for k, v in pl.state_dict().items() if torch.is_tensor(v) and v.dtype == torch.float32})
    for k in res[0]:
        _same_bits(res[0][k], res[1][k], k)


# ---------------------------------------------------------------- refusals
def test_refusals():
    import pearl_b200
    from pearl_b200.rc_safety import B200RCSafetyModule
    from pearl_b200.td3 import B200TD3
    st, ac, rw, ns, te, co = _rows(100, obs=5, act=2)
    pl = B200TD3(state_dim=5, low=[-1, -1], high=[1, 1], actor_hidden_dims=[16, 16], critic_hidden_dims=[16, 16], batch_size=16)
    rc = B200RCSafetyModule(constraint_value=0.1, state_dim=5, low=[-1, -1], high=[1, 1], critic_hidden_dims=[16, 16], batch_size=16)
    plain = _cost_buffer(st, ac, rw, ns, te, None)
    pl.lambda_constraint = 0.5
    with pytest.raises(ValueError, match="costs"):
        pl.learn(plain)                     # a multiplier on a buffer without costs
    with pytest.raises(ValueError, match="costs"):
        rc.learn(plain, pl)
    pl.lambda_constraint = None
    pl.learn(plain)                         # no multiplier: trains as before
    sac = pearl_b200.actor_critic.SacCore(state_dim=5, low=[-1, -1], high=[1, 1], actor_hidden_dims=[16, 16], critic_hidden_dims=[16, 16])
    with pytest.raises(NotImplementedError):
        rc.learn(_cost_buffer(st, ac, rw, ns, te, co), sac)
    other = B200TD3(state_dim=4, low=[-1, -1], high=[1, 1], actor_hidden_dims=[16, 16], critic_hidden_dims=[16, 16], batch_size=16)
    with pytest.raises(ValueError):
        rc.learn(_cost_buffer(st, ac, rw, ns, te, co), other)      # dimensions differ
    with pytest.raises(NotImplementedError):
        B200RCSafetyModule(constraint_value=0.1, state_dim=5, low=[-1], high=[1], critic_hidden_dims=[16, 16], use_twin_critic=False)
    with pytest.raises(NotImplementedError):
        B200RCSafetyModule(constraint_value=0.1, state_dim=5, low=[-1], high=[1], critic_hidden_dims=[16, 16, 16])
    g = np.random.default_rng(0)
    dbuf = pearl_b200.B200ReplayBuffer(50)
    dbuf.push_batch(torch.zeros(50, 5), torch.zeros(50, dtype=torch.int64), torch.zeros(50), torch.zeros(50, 5),
                    torch.zeros(50, dtype=torch.bool), torch.zeros(50, dtype=torch.bool), max_number_actions=2,
                    cost=torch.from_numpy(g.standard_normal(50).astype(np.float32)))
    with pytest.raises(ValueError):
        rc.learn(dbuf, pl)                  # discrete buffer
