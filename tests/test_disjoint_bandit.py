"""GPU checks of B200DisjointBanditContainer and B200DisjointLinearBandit (csrc/disjoint_bandit.cu) against the eager
oracle (oracle/disjoint_oracle.py) and themselves: learn_batch and agent loops, per-arm discounting marks, the report,
bit-identity run to run, graph vs eager and across round chunking, the launch count, checkpoint views, UCB and Thompson
scores (the arm-major layout included), masked act and the runtime refusals.  Sums elementwise, solved quantities
normwise, as test_bandit.py."""
from __future__ import annotations

import os
import random
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import disjoint_oracle as do  # noqa: E402

pytestmark = pytest.mark.gpu

DEV = "cuda:0"
TOL = 1e-4


class Space:
    def __init__(self, n):
        self.n = n
        self.actions = [torch.tensor([i]) for i in range(n)]
        self.actions_batch = torch.arange(n).view(n, 1)


def close(got, ref, what, normwise=False):
    got, ref = torch.as_tensor(got).double().cpu(), torch.as_tensor(ref).double().cpu()
    assert got.shape == ref.shape, f"{what}: shape {tuple(got.shape)} != {tuple(ref.shape)}"
    if normwise:
        assert float((got - ref).norm()) <= TOL * (1 + float(ref.norm())), f"{what}: normwise distance too large"
    else:
        assert bool(((got - ref).abs() <= TOL * (1 + ref.abs())).all()), f"{what}: elementwise distance too large"


def check_arms(models, oracle, what):
    for k, (m, r) in enumerate(zip(models, oracle.arms)):
        for name, ref, nw in (("_A", r.A, False), ("_b", r.b, False), ("_sum_weight", r.sum_weight, False),
                              ("_inv_A", r.inv_A, True), ("_coefs", r.coefs, True)):
            close(getattr(m, name), ref, f"{what} arm {k} {name}", nw)


LAMS, GAMMAS, INTERVALS = [1.0, 2.0, 0.5, 4.0, 1.5], [0.9, 1.0, 0.5, 0.8, 0.7], [40.0, 0.0, 25.0, 10.0, 30.0]


def make_container(obs=4, b200_arms=(0, 2), **kw):
    import pearl_b200 as P
    from pearl_b200._compat import _RefLinearBandit
    arms = []
    for k in range(5):
        cls = P.B200LinearBandit if k in b200_arms else _RefLinearBandit
        arms.append(cls(feature_dim=obs, l2_reg_lambda=LAMS[k], gamma=GAMMAS[k], apply_discounting_interval=INTERVALS[k],
                        initial_coefs=torch.arange(obs + 1, dtype=torch.float32) if k == 4 else None))
    return P.B200DisjointBanditContainer(feature_dim=obs, arm_bandits=arms, exploration_module=P.DisjointUCBExploration(0.3),
                                         training_rounds=10, batch_size=128, **kw)


def container_oracle(obs=4):
    return do.Disjoint(5, obs + 1, LAMS, GAMMAS, INTERVALS, coefs=[None] * 4 + [torch.arange(obs + 1, dtype=torch.float32)])


def batches(obs=4, calls=6, seed=0):
    g = torch.Generator().manual_seed(seed)
    out = []
    for c in range(calls):
        B = [7, 64, 33, 128, 1, 50][c % 6]
        state = torch.randn(B, 5, obs, generator=g) if c == 2 else torch.randn(B, obs, generator=g)
        action = torch.randint(0, 4, (B, 1), generator=g)         # arm 4 never observed
        if c == 3:
            action[:] = 1                                          # every row to one arm
        reward = torch.randn(B, 1, generator=g)
        weight = torch.rand(B, 1, generator=g) if c % 2 else None
        if c == 5:
            weight[action[:, 0] == 3] = 0.0                        # an all-zero-weight arm
        out.append((state, action, reward, weight))
    return out


@pytest.mark.parametrize("graph", [True, False])
def test_container_learn_batch_matches_the_oracle(graph):
    import pearl_b200 as P
    torch.cuda.set_device(0)
    dc = make_container()
    dc.use_cuda_graph = graph
    ref = container_oracle()
    for c, (state, action, reward, weight) in enumerate(batches()):
        rep = dc.learn_batch(P.TransitionBatch(state=state.to(DEV), action=action.to(DEV), reward=reward.to(DEV),
                                               weight=None if weight is None else weight.to(DEV)))
        want = ref.round(state, action, reward, weight)
        check_arms(dc.models, ref, f"call {c}")
        for k in range(5):
            p, y, w = want[k]
            close(rep[f"arm_{k}_prediction"], p, f"call {c} arm {k} prediction", True)
            assert torch.equal(rep[f"arm_{k}_label"].cpu(), y.float()), f"call {c} arm {k} label"
            assert torch.equal(rep[f"arm_{k}_weight"].cpu(), w.float()), f"call {c} arm {k} weight"
            close(dc._arm_bandits[k].last_sum_weight_when_discounted, ref.arms[k].last, f"call {c} arm {k} last")
    # the unobserved arm's initial_coefs were replaced by inv(lambda I) b = 0 at the first call
    assert float(dc.models[4]._coefs.abs().max()) == 0.0


def run_loop(graph=True, chunk=1024, seed=1, n=300):
    import pearl_b200 as P
    torch.cuda.set_device(0)
    dc = make_container(max_rounds_per_call=chunk)
    dc.use_cuda_graph = graph
    buf = P.B200ReplayBuffer(100000, rng="python")
    random.seed(seed)
    g = torch.Generator().manual_seed(seed)
    S, A, R = torch.randn(n, 4, generator=g), torch.randint(0, 4, (n,), generator=g), torch.randn(n, generator=g)
    space, traces, reports, chosen = Space(5), [], [], []
    for i in range(n):
        buf.push(S[i], int(A[i]), float(R[i]), True, False, next_state=None, max_number_actions=5)
        if i % 100 == 99:
            tr = {}
            reports.append(dc.learn(buf, trace=tr))
            traces.append(tr)
            chosen.append(dc.act(S[i], space).cpu())
    return dc, (S, A, R), traces, reports, chosen


def test_container_agent_loop_matches_the_oracle():
    dc, (S, A, R), traces, reports, _ = run_loop()
    ref = container_oracle()
    for c, (tr, rep) in enumerate(zip(traces, reports)):
        assert tr["launches"] == 7 * 10
        for r, idx in enumerate(tr["idx"]):
            idx = idx.long()
            want = ref.round(S[idx], A[idx].reshape(-1, 1), R[idx])
            assert tr["counts"][r].tolist() == [int((A[idx] == k).sum()) for k in range(5)]
            for k in range(5):
                close(rep[f"arm_{k}_prediction"][r], want[k][0], f"call {c} round {r} arm {k} prediction", True)
                assert torch.equal(rep[f"arm_{k}_label"][r].cpu(), want[k][1].float())
    check_arms(dc.models, ref, "after the loop")          # every stored row has weight 1: the marks are exact counts
    for k in range(5):
        assert dc._arm_bandits[k].last_sum_weight_when_discounted == ref.arms[k].last


def test_bit_identity_graph_eager_and_chunking():
    base = run_loop()
    for kw in (dict(), dict(graph=False), dict(chunk=3)):
        other = run_loop(**kw)
        for m0, m1 in zip(base[0].models, other[0].models):
            for name in ("_A", "_b", "_sum_weight", "_inv_A", "_coefs"):
                assert torch.equal(getattr(m0, name), getattr(m1, name)), f"{kw}: {name} differs"
        assert all(torch.equal(a, b) for a, b in zip(base[4], other[4]))
        for r0, r1 in zip(base[3], other[3]):
            for key in r0:
                assert all(torch.equal(a, b) for a, b in zip(r0[key], r1[key])), f"{kw}: {key} differs"


def test_state_dict_views_and_load():
    import pearl_b200 as P
    dc, *_ = run_loop(n=100)
    keys = set(dc.state_dict().keys())
    want = {f"_arm_bandits.{i}.model.{b}" for i in range(5) for b in ("_A", "_b", "_sum_weight", "_inv_A", "_coefs")}
    assert want <= keys
    flat = dc._dj.flat
    for k, m in enumerate(dc.models):
        assert m._A.data_ptr() == flat["A"][k].data_ptr() and m._coefs.data_ptr() == flat["coefs"][k].data_ptr()
    sd = {k: v.clone() for k, v in dc.state_dict().items()}
    sd["_arm_bandits.1.model._coefs"] = torch.full_like(sd["_arm_bandits.1.model._coefs"], 3.0)
    dc.load_state_dict(sd)
    s = dc.get_scores(torch.zeros(1, 4, device=DEV), Space(5), exploit=True)
    assert float(s[0, 1]) == 3.0
    dc.models[2]._coefs = torch.full((5,), 7.0)          # a reassigned buffer is gathered back before the next call
    s = dc.get_scores(torch.zeros(1, 4, device=DEV), Space(5), exploit=True)
    assert float(s[0, 2]) == 7.0
    assert P.B200DisjointBanditContainer is type(dc)


def test_ucb_scores_exploit_and_masked_act():
    dc, *_ = run_loop(n=200)
    ref = container_oracle()
    for k, r in enumerate(ref.arms):
        m = dc.models[k]
        r.inv_A, r.coefs = m._inv_A.cpu(), m._coefs.cpu()
    states = torch.randn(37, 4, generator=torch.Generator().manual_seed(5))
    got = dc.get_scores(states.to(DEV), Space(5))
    close(got, ref.scores(states, 0.3), "ucb scores", True)
    close(dc.get_scores(states.to(DEV), Space(5), exploit=True), ref.scores(states, 0.3, False), "exploit scores", True)
    mask = torch.rand(37, 5, generator=torch.Generator().manual_seed(6)) > 0.4
    a = dc.act(states.to(DEV), Space(5), action_availability_mask=mask.to(DEV)).cpu().reshape(-1)
    s = got.cpu().masked_fill(~mask, -float("inf"))
    want = torch.where(mask.any(1), s.argmax(1), torch.zeros(37, dtype=torch.long))
    assert torch.equal(a, want)


def test_thompson_draws_layout_and_generator_state():
    import pearl_b200 as P
    dc, *_ = run_loop(n=200)
    dc.exploration_module = P.ThompsonSamplingExplorationLinearDisjoint()
    ref = container_oracle()
    for k, r in enumerate(ref.arms):
        m = dc.models[k]
        r.A, r.coefs = m._A.cpu(), m._coefs.cpu()
    states = torch.randn(6, 4, generator=torch.Generator().manual_seed(7))
    torch.manual_seed(11)
    got = dc.get_scores(states.to(DEV), Space(5)).cpu()
    after = torch.get_rng_state()
    torch.manual_seed(11)
    eps = ref.draws()
    assert torch.equal(torch.get_rng_state(), after), "the draws leave the generator where the reference's do"
    close(got, ref.ts_scores(states, ref.thetas(eps)), "thompson scores (arm-major layout)", True)
    # the layout quirk: 4 identical states, arm means 0 / 100 / 200 / -1000 / -2000 and tiny noise.  The per-arm scores
    # stacked (5, 4) arm-major and read as (4, 5) rows: [0 0 0 0 100], [100 100 100 200 200], [200 200 -1e3 ..],
    # [-1e3 -2e3 ..]
    sd = dc.state_dict()
    for k in range(5):
        sd[f"_arm_bandits.{k}.model._A"] = torch.eye(5) * 1e8
        sd[f"_arm_bandits.{k}.model._coefs"] = torch.tensor([100.0 * k if k < 3 else -1e3 * (k - 2), 0, 0, 0, 0])
    dc.load_state_dict(sd)
    x = torch.ones(4, 4, device=DEV)
    assert dc.act(x, Space(5)).cpu().reshape(-1).tolist() == [4, 3, 0, 0]
    assert dc.act(x[:1], Space(5)).cpu().reshape(-1).tolist() == [2]      # n = 1: the natural layout
    sd["_arm_bandits.1.model._A"] = -torch.eye(5) * 1e3          # not positive definite: the reference raises
    dc.load_state_dict(sd)
    with pytest.raises(ValueError):
        dc.act(x, Space(5))


@pytest.mark.parametrize("sfo", [False, True])
def test_disjoint_linear_bandit_learn_batch_and_act(sfo):
    import pearl_b200 as P
    torch.cuda.set_device(0)
    obs, K = 3, 3
    f = obs if sfo else obs + 1
    lb = P.B200DisjointLinearBandit(feature_dim=f, action_space=Space(K), exploration_module=P.DisjointUCBExploration(0.1),
                                    l2_reg_lambda=2.0, state_features_only=sfo)
    ref = do.Disjoint(K, f + 1, [2.0] * K, linear=True)
    feat = None if sfo else torch.arange(K, dtype=torch.float32).reshape(K, 1)
    g = torch.Generator().manual_seed(3)
    for c in range(4):
        B = [16, 5, 40, 9][c]
        state, reward = torch.randn(B, obs, generator=g), torch.randn(B, 1, generator=g)
        action = torch.randint(0, K, (B, 1), generator=g)
        if c == 1:
            action[action == 2] = 0              # an absent arm: skipped, no solve
        if c == 2:
            action[0] = 7                        # an out-of-range action matches no arm
        weight = torch.rand(B, 1, generator=g) if c == 3 else None
        assert lb.learn_batch(P.TransitionBatch(state=state.to(DEV), action=action.to(DEV), reward=reward.to(DEV),
                                                weight=None if weight is None else weight.to(DEV))) == {}
        ref.round(state, action, reward, weight, feat)
        check_arms(list(lb._linear_regressions), ref, f"call {c}")
    s = torch.randn(1, obs, generator=g)
    a = int(lb.act(s.to(DEV), Space(K)).reshape(-1)[0])
    assert a == int(torch.argmax(ref.scores(s, 0.1, True, feat)[0]))
    with pytest.raises(NotImplementedError):
        lb.get_scores(s, Space(K))


def test_disjoint_linear_bandit_agent_loop_and_launches():
    import pearl_b200 as P
    torch.cuda.set_device(0)
    K = 3
    lb = P.B200DisjointLinearBandit(feature_dim=4, action_space=Space(K), exploration_module=P.DisjointUCBExploration(0.1),
                                    l2_reg_lambda=4.0, training_rounds=2, batch_size=1)
    ref = do.Disjoint(K, 5, [4.0] * K, linear=True)
    feat = torch.arange(K, dtype=torch.float32).reshape(K, 1)
    buf = P.B200ReplayBuffer(1000, rng="python")
    random.seed(0)
    g = torch.Generator().manual_seed(0)
    pushed = []
    for step in range(40):
        s = torch.randn(3, generator=g)
        a = int(lb.act(s.to(DEV), Space(K)).reshape(-1)[0])
        assert a == int(torch.argmax(ref.scores(s.reshape(1, 3), 0.1, True, feat)[0]))
        r = float(s.sum()) * (a + 1) * 0.1
        buf.push(s, a, r, True, False, next_state=None, max_number_actions=K)
        pushed.append((s, a, r))
        tr = {}
        assert lb.learn(buf, trace=tr) == {}
        assert tr["launches"] == 6 * 2
        for idx in tr["idx"]:
            s_, a_, r_ = pushed[int(idx[0])]
            ref.round(s_.reshape(1, 3), torch.tensor([[a_]]), torch.tensor([r_]), None, feat)
        check_arms(list(lb._linear_regressions), ref, f"step {step}")


def test_runtime_refusals():
    import pearl_b200 as P
    torch.cuda.set_device(0)
    dc = make_container()
    bad = P.TransitionBatch(state=torch.randn(4, 4, device=DEV), action=torch.tensor([[0], [1], [5], [0]], device=DEV),
                            reward=torch.randn(4, 1, device=DEV))
    with pytest.raises(AssertionError):
        dc.learn_batch(bad)
    bad.action = bad.action.float()
    with pytest.raises(AssertionError):
        dc.learn_batch(bad)
    neg = P.TransitionBatch(state=torch.randn(4, 4, device=DEV), action=torch.tensor([[0], [1], [2], [0]], device=DEV),
                            reward=torch.randn(4, 1, device=DEV), weight=-torch.ones(4, 1, device=DEV))
    with pytest.raises(NotImplementedError, match="negative weights"):
        dc.learn_batch(neg)
    buf = P.B200ReplayBuffer(100, rng="python")
    buf.push(torch.zeros(4), 6, 0.0, True, False, next_state=None, max_number_actions=7)
    with pytest.raises(ValueError):
        dc.learn(buf)


# ---------------------------------------------------------------------- the reference's recordings (tests/golden/cb_dj_*)
GOLDEN = os.path.join(ROOT, "tests", "golden")


def load(name):
    return dict(np.load(os.path.join(GOLDEN, f"{name}.npz")))


def check_snap(models, fx, c, what, prefix="", lasts=None):
    for k, m in enumerate(models):
        for name, nw in (("A", False), ("b", False), ("sum_weight", False), ("inv_A", True), ("coefs", True)):
            close(getattr(m, "_" + name), fx[f"{prefix}call_{name}"][c][k], f"{what} call {c} arm {k} {name}", nw)
        if lasts is not None:
            close(lasts[k], fx[f"{prefix}call_last"][c][k], f"{what} call {c} arm {k} last")


def golden_container(fx, ex, obs=None):
    import pearl_b200 as P
    from pearl_b200._compat import _RefLinearBandit
    obs = int(fx["obs"]) if obs is None else obs
    arms = [_RefLinearBandit(feature_dim=obs, l2_reg_lambda=float(fx["lams"][k]), gamma=float(fx["gammas"][k]),
                             apply_discounting_interval=float(fx["intervals"][k]),
                             initial_coefs=torch.from_numpy(fx["initial_coefs"]) if k == 3 else None) for k in range(4)]
    return P.B200DisjointBanditContainer(feature_dim=obs, arm_bandits=arms, exploration_module=ex, training_rounds=10,
                                         batch_size=128)


def set_python_rng(words):
    random.setstate((3, tuple(int(x) for x in words), None))


@pytest.mark.parametrize("graph", [True, False])
def test_recorded_disjoint_linear_agent_loop(graph):
    import pearl_b200 as P
    torch.cuda.set_device(0)
    fx = load("cb_dj_agent")
    K, obs = int(fx["n_arms"]), int(fx["obs"])
    lb = P.B200DisjointLinearBandit(feature_dim=obs + 1, action_space=Space(K), exploration_module=P.DisjointUCBExploration(0.1),
                                    batch_size=1, l2_reg_lambda=float(fx["lam"]), training_rounds=int(fx["rounds"]))
    lb.use_cuda_graph = graph
    buf = P.B200ReplayBuffer(1, rng="python")
    set_python_rng(fx["rng_before"])
    idx = []
    for t in range(len(fx["act_chosen"])):
        a = int(lb.act(torch.from_numpy(fx["push_state"][t]).to(DEV), Space(K)).reshape(-1)[0])
        if fx["act_keep"][t]:
            assert a == int(fx["act_chosen"][t]), f"step {t}: choice"
        buf.push(torch.from_numpy(fx["push_state"][t]), int(fx["push_action"][t]), float(fx["push_reward"][t]), True, False,
                 next_state=None, max_number_actions=K)
        tr = {}
        lb.learn(buf, trace=tr)
        idx.append(tr["idx"].numpy().ravel())
        assert tr["launches"] == 6 * int(fx["rounds"])
        check_snap(list(lb._linear_regressions), fx, t, "agent")
    assert np.array_equal(np.concatenate(idx), fx["idx"])
    assert np.array_equal(np.asarray(random.getstate()[1], np.uint64).astype(np.uint32), fx["rng_after"])


@pytest.mark.parametrize("graph", [True, False])
def test_recorded_container_agent_loop(graph):
    import pearl_b200 as P
    torch.cuda.set_device(0)
    fx = load("cb_dj_container")
    dc = golden_container(fx, P.DisjointUCBExploration(float(fx["alpha"])))
    dc.use_cuda_graph = graph
    buf = P.B200ReplayBuffer(100000, rng="python")
    set_python_rng(fx["rng_before"])
    pushed = [0]

    def push(n):
        for i in range(pushed[0], pushed[0] + n):
            buf.push(torch.from_numpy(fx["push_state"][i]), int(fx["push_action"][i]), float(fx["push_reward"][i]), True, False,
                     next_state=None, max_number_actions=4)
        pushed[0] += n
    reports, idx, counts = [], [], []

    def learn(c):
        tr = {}
        reports.append(dc.learn(buf, trace=tr))
        idx.append(tr["idx"].numpy().ravel())
        counts.append(tr["counts"].numpy())
        check_snap(dc.models, fx, c, "container", lasts=[a.last_sum_weight_when_discounted for a in dc._arm_bandits])
    push(int(fx["prefill"]))
    learn(0)
    for t in range(len(fx["act_chosen"])):
        a = int(dc.act(torch.from_numpy(fx["act_state"][t]).to(DEV), Space(4)).reshape(-1)[0])
        if fx["act_keep"][t]:
            assert a == int(fx["act_chosen"][t]), f"step {t}: choice"
        push(20)
        learn(t + 1)
    assert np.array_equal(np.concatenate(idx), fx["idx"])
    assert np.array_equal(np.concatenate(counts), fx["counts"])
    assert np.array_equal(np.asarray(random.getstate()[1], np.uint64).astype(np.uint32), fx["rng_after"])
    pred, label, weight = [], [], []
    for rep in reports:
        for r in range(10):
            for k in range(4):
                pred.append(rep[f"arm_{k}_prediction"][r].cpu().numpy().ravel())
                label.append(rep[f"arm_{k}_label"][r].cpu().numpy().ravel())
                weight.append(rep[f"arm_{k}_weight"][r].cpu().numpy().ravel())
    assert np.array_equal(np.concatenate(label), fx["label"]) and np.array_equal(np.concatenate(weight), fx["weight"])
    o = 0
    for p in pred:
        close(p, fx["pred"][o:o + len(p)], "prediction", True)
        o += len(p)


def test_recorded_learn_batch():
    import pearl_b200 as P
    torch.cuda.set_device(0)
    fx = load("cb_dj_batch")
    obs = int(fx["obs"])
    dc = golden_container(fx, P.DisjointUCBExploration(0.5))
    so = ao = 0
    for c, B in enumerate(fx["c_B"]):
        B = int(B)
        n = B * (4 if fx["c_state3d"][c] else 1) * obs
        state = torch.from_numpy(fx["c_state"][so:so + n]).reshape((B, 4, obs) if fx["c_state3d"][c] else (B, obs))
        act = torch.from_numpy(fx["c_action"][ao:ao + B]).reshape(B, 1)
        w = torch.from_numpy(fx["c_weight"][ao:ao + B]).reshape(B, 1).to(DEV) if fx["c_has_weight"][c] else None
        dc.learn_batch(P.TransitionBatch(state=state.to(DEV), action=act.to(DEV),
                                         reward=torch.from_numpy(fx["c_reward"][ao:ao + B]).reshape(B, 1).to(DEV), weight=w))
        check_snap(dc.models, fx, c, "container learn_batch", "c_", [a.last_sum_weight_when_discounted for a in dc._arm_bandits])
        so, ao = so + n, ao + B
    for sfo in (0, 1):
        p = f"l{sfo}_"
        lb = P.B200DisjointLinearBandit(feature_dim=obs if sfo else obs + 1, action_space=Space(3),
                                        exploration_module=P.DisjointUCBExploration(0.1), l2_reg_lambda=3.0,
                                        state_features_only=bool(sfo))
        o = 0
        for c, B in enumerate(fx[p + "B"]):
            B = int(B)
            sl = slice(o, o + B)
            lb.learn_batch(P.TransitionBatch(state=torch.from_numpy(fx[p + "state"][o * obs:(o + B) * obs]).reshape(B, obs).to(DEV),
                                             action=torch.from_numpy(fx[p + "action"][sl]).reshape(B, 1).to(DEV),
                                             reward=torch.from_numpy(fx[p + "reward"][sl]).reshape(B, 1).to(DEV),
                                             weight=torch.from_numpy(fx[p + "weight"][sl]).reshape(B, 1).to(DEV)))
            check_snap(list(lb._linear_regressions), fx, c, f"DisjointLinearBandit sfo={sfo}", p)
            o += B


def test_recorded_thompson_sampling():
    import pearl_b200 as P
    torch.cuda.set_device(0)
    fx = load("cb_dj_ts")
    # DisjointLinearBandit LinTS loop: the recorded acts, each from the generator state the reference started it in
    K, obs = int(fx["l_n_arms"]), int(fx["l_obs"])
    lb = P.B200DisjointLinearBandit(feature_dim=obs + 1, action_space=Space(K),
                                    exploration_module=P.ThompsonSamplingExplorationLinearDisjoint(), batch_size=int(fx["l_batch"]),
                                    training_rounds=int(fx["l_rounds"]), l2_reg_lambda=float(fx["l_lam"]))
    buf = P.B200ReplayBuffer(100000, rng="python")
    n0 = int(fx["l_prefill"])
    for i in range(n0):
        buf.push(torch.from_numpy(fx["l_push_state"][i]), int(fx["l_push_action"][i]), float(fx["l_push_reward"][i]), True, False,
                 next_state=None, max_number_actions=K)
    set_python_rng(fx["l_rng_before"])
    idx = []
    for t in range(len(fx["l_act_chosen"])):
        torch.set_rng_state(torch.from_numpy(fx["l_torch_before"][t]))
        a = int(lb.act(torch.from_numpy(fx["l_act_state"][t]).to(DEV), Space(K)).reshape(-1)[0])
        assert np.array_equal(torch.get_rng_state().numpy(), fx["l_torch_after"][t]), f"step {t}: generator state"
        assert a == int(fx["l_act_chosen"][t]), f"step {t}: choice"
        i = n0 + t
        buf.push(torch.from_numpy(fx["l_push_state"][i]), int(fx["l_push_action"][i]), float(fx["l_push_reward"][i]), True, False,
                 next_state=None, max_number_actions=K)
        tr = {}
        lb.learn(buf, trace=tr)
        idx.append(tr["idx"].numpy().ravel())
        check_snap(list(lb._linear_regressions), fx, t, "LinTS", "l_")
    assert np.array_equal(np.concatenate(idx), fx["l_idx"])
    assert np.array_equal(np.asarray(random.getstate()[1], np.uint64).astype(np.uint32), fx["l_rng_after"])
    # container: Thompson get_scores over identical and random states (the arm-major layout), then a masked act
    obs = int(fx["c_obs"])
    dc = golden_container(fx, P.ThompsonSamplingExplorationLinearDisjoint(), obs)
    n = len(fx["c_fit_action"])
    dc.learn_batch(P.TransitionBatch(state=torch.from_numpy(fx["c_fit_state"]).to(DEV),
                                     action=torch.from_numpy(fx["c_fit_action"]).reshape(n, 1).to(DEV),
                                     reward=torch.from_numpy(fx["c_fit_reward"]).reshape(n, 1).to(DEV)))
    o = 0
    for i in range(3):
        st = torch.from_numpy(fx[f"c_state{i}"])
        torch.set_rng_state(torch.from_numpy(fx["c_torch_before"][i]))
        s = dc.get_scores(st.to(DEV), Space(4)).cpu()
        assert np.array_equal(torch.get_rng_state().numpy(), fx["c_torch_after"][i])
        close(s.reshape(-1), fx["c_scores"][o:o + s.numel()], f"thompson scores {i}", True)
        o += s.numel()
    mask = torch.from_numpy(fx["m_mask"])
    torch.set_rng_state(torch.from_numpy(fx["m_torch_before"]))
    a = dc.act(torch.from_numpy(fx["c_state1"]).to(DEV), Space(4), action_availability_mask=mask.to(DEV)).cpu().reshape(-1)
    assert np.array_equal(torch.get_rng_state().numpy(), fx["m_torch_after"])
    keep = fx["m_keep"]
    assert np.array_equal(a.numpy()[keep], fx["m_chosen"][keep])


def test_recorded_ucb_scores():
    import pearl_b200 as P
    torch.cuda.set_device(0)
    fx = load("cb_dj_scores")
    dc = golden_container(fx, P.DisjointUCBExploration(float(fx["alpha"])))
    n = len(fx["fit_action"])
    dc.learn_batch(P.TransitionBatch(state=torch.from_numpy(fx["fit_state"]).to(DEV),
                                     action=torch.from_numpy(fx["fit_action"]).reshape(n, 1).to(DEV),
                                     reward=torch.from_numpy(fx["fit_reward"]).reshape(n, 1).to(DEV)))
    st = torch.from_numpy(fx["states"]).to(DEV)
    close(dc.get_scores(st, Space(4)), fx["ucb"], "ucb scores", True)
    close(dc.get_scores(st, Space(4), exploit=True), fx["mu"], "exploit scores", True)
    keep = fx["keep"]
    assert np.array_equal(dc.act(st, Space(4)).cpu().reshape(-1).numpy()[keep], fx["chosen"][keep])
    a = dc.act(st, Space(4), action_availability_mask=torch.from_numpy(fx["mask"]).to(DEV)).cpu().reshape(-1).numpy()
    assert np.array_equal(a[fx["m_keep"]], fx["m_chosen"][fx["m_keep"]])
