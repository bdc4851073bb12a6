"""CPU checks of the disjoint-bandit oracle (oracle/disjoint_oracle.py) on the reference behaviours it restates (the null
batch, the skip rule, per-arm discounting, the Thompson layout), and of the host-side refusals of
B200DisjointBanditContainer / B200DisjointLinearBandit that fire before a device is touched."""
from __future__ import annotations

import os
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import disjoint_oracle as do  # noqa: E402


class Space:
    def __init__(self, actions):
        self.actions = list(actions)
        self.n = len(self.actions)


def test_container_null_batch_replaces_initial_coefs_and_discounts():
    ref = do.Disjoint(2, 3, [1.0, 2.0], [0.5, 0.5], [0.0, 1e-9], coefs=[None, torch.tensor([1.0, 2.0, 3.0])])
    out = ref.round(torch.randn(4, 2), torch.zeros(4, 1, dtype=torch.long), torch.randn(4))
    assert torch.equal(ref.arms[1].coefs, torch.zeros(3))          # inv(lambda I) 0
    p, y, w = out[1]
    assert p.shape == (1, 1) and float(y) == 0.0 and float(w) == 0.0
    assert out[0][0].shape == (4, 1)
    assert ref.arms[1].last == 0.0                                   # 0 - 0 >= 1e-9 is false: no discount


def test_linear_skips_empty_arms_and_drops_unmatched_rows():
    ref = do.Disjoint(3, 3, [1.0] * 3, linear=True)
    before = ref.arms[2].inv_A.clone()
    assert ref.round(torch.randn(5, 2), torch.tensor([[0], [1], [7], [0], [1]]), torch.randn(5)) == {}
    assert torch.equal(ref.arms[2].inv_A, before)                    # no solve: still zeros
    assert float(ref.arms[0].sum_weight) == 2.0 and float(ref.arms[1].sum_weight) == 2.0


def test_thompson_layout_is_arm_major():
    ref = do.Disjoint(3, 2, [1.0] * 3)
    theta = torch.tensor([[0.0, 0.0], [100.0, 0.0], [200.0, 0.0]])
    s = ref.ts_scores(torch.zeros(4, 1), theta)
    assert torch.argmax(s, 1).tolist() == [0, 1, 2, 0]
    assert torch.argmax(ref.ts_scores(torch.zeros(1, 1), theta), 1).tolist() == [2]


def test_draws_are_per_arm():
    ref = do.Disjoint(3, 20, [1.0] * 3)
    torch.manual_seed(0)
    eps = ref.draws()
    torch.manual_seed(0)
    assert torch.equal(eps, torch.stack([torch.empty(20).normal_() for _ in range(3)]))
    torch.manual_seed(0)
    assert not torch.equal(eps.reshape(-1), torch.empty(60).normal_())   # one joint draw is another stream


def _pb():
    import pearl_b200 as P
    from pearl_b200._compat import _RefLinearBandit
    return P, _RefLinearBandit


def test_container_refusals():
    P, Ref = _pb()
    ucb = P.DisjointUCBExploration(0.1)
    with pytest.raises(NotImplementedError, match="Module arm"):
        P.B200DisjointBanditContainer(4, [torch.nn.Module()], ucb)
    with pytest.raises(NotImplementedError, match="force_pinv"):
        P.B200DisjointBanditContainer(4, [Ref(feature_dim=4, force_pinv=True)], ucb)
    with pytest.raises(NotImplementedError, match="l2_reg_lambda"):
        P.B200DisjointBanditContainer(4, [Ref(feature_dim=4, l2_reg_lambda=0.0)], ucb)
    with pytest.raises(NotImplementedError, match="feature_dim=128"):
        P.B200DisjointBanditContainer(128, [Ref(feature_dim=128)], ucb)
    with pytest.raises(NotImplementedError, match="1025 arms"):
        P.B200DisjointBanditContainer(2, [Ref(feature_dim=2) for _ in range(1025)], ucb)
    dc = P.B200DisjointBanditContainer(2, [Ref(feature_dim=2)], P.ThompsonSamplingExplorationLinearDisjoint(True))
    with pytest.raises(NotImplementedError, match="enable_efficient_sampling"):
        dc.act(torch.zeros(2), Space([torch.tensor([0])]))
    dc.exploration_module = P.DisjointUCBExploration(0.1, randomized_tiebreaking=P._compat.TiebreakingStrategy.PER_ROW_TIEBREAKING)
    with pytest.raises(NotImplementedError, match="tie-breaking"):
        dc.act(torch.zeros(2), Space([torch.tensor([0])]))
    dc.exploration_module = P.UCBExploration(0.1)
    with pytest.raises(NotImplementedError, match="UCBExploration"):
        dc.get_scores(torch.zeros(2), Space([torch.tensor([0])]))


def test_disjoint_linear_refusals():
    P, _ = _pb()
    ucb = P.DisjointUCBExploration(0.1)
    with pytest.raises(NotImplementedError, match="action space"):
        P.B200DisjointLinearBandit(4, Space([torch.tensor([1]), torch.tensor([0])]), ucb)
    with pytest.raises(NotImplementedError, match="action space"):
        P.B200DisjointLinearBandit(4, Space([torch.tensor([0, 1])]), ucb)
    with pytest.raises(NotImplementedError, match="feature_dim=200"):
        P.B200DisjointLinearBandit(200, Space([torch.tensor([0])]), ucb)
    with pytest.raises(NotImplementedError, match="l2_reg_lambda"):
        P.B200DisjointLinearBandit(4, Space([torch.tensor([0])]), ucb, l2_reg_lambda=-1.0)
    lb = P.B200DisjointLinearBandit(4, Space([torch.tensor([0])]), P.ThompsonSamplingExplorationLinearDisjoint(True))
    with pytest.raises(NotImplementedError, match="enable_efficient_sampling"):
        lb.act(torch.zeros(3), Space([torch.tensor([0])]))
    lb.exploration_module = ucb
    lb.action_representation_module = P.OneHotActionTensorRepresentationModule(1)
    with pytest.raises(NotImplementedError, match="identity action representation"):
        lb.act(torch.zeros(3), Space([torch.tensor([0])]))
    with pytest.raises(NotImplementedError, match="get_scores"):
        lb.get_scores(torch.zeros(3), Space([torch.tensor([0])]))


# ---------------------------------------------------------------------- the reference's recordings (tests/golden/cb_dj_*)
def load(name):
    return dict(np.load(os.path.join(ROOT, "tests", "golden", f"{name}.npz")))


def agree(ref, fx, c, prefix=""):
    for k, r in enumerate(ref.arms):
        for name, nw in (("A", False), ("b", False), ("sum_weight", False), ("inv_A", True), ("coefs", True)):
            got, want = getattr(r, name).double(), torch.from_numpy(fx[f"{prefix}call_{name}"][c][k]).double()
            if nw:
                assert float((got - want).norm()) <= 1e-4 * (1 + float(want.norm())), f"call {c} arm {k} {name}"
            else:
                assert bool(((got - want).abs() <= 1e-4 * (1 + want.abs())).all()), f"call {c} arm {k} {name}"
        if not ref.linear:
            assert abs(r.last - fx[f"{prefix}call_last"][c][k]) <= 1e-4 * (1 + abs(r.last)), f"call {c} arm {k} last"


def container_of(fx, obs):
    return do.Disjoint(4, obs + 1, fx["lams"], fx["gammas"], fx["intervals"],
                       coefs=[None] * 3 + [torch.from_numpy(fx["initial_coefs"])])


def test_oracle_reproduces_the_recorded_agent_loops():
    fx = load("cb_dj_agent")
    K, obs = int(fx["n_arms"]), int(fx["obs"])
    ref = do.Disjoint(K, obs + 2, [float(fx["lam"])] * K, linear=True)
    feat = torch.arange(K, dtype=torch.float32).reshape(K, 1)
    R = int(fx["rounds"])
    for t in range(len(fx["act_chosen"])):
        assert set(fx["idx"][t * R:(t + 1) * R].tolist()) == {0}        # a one-transition buffer
        for _ in range(R):
            ref.round(torch.from_numpy(fx["push_state"][t:t + 1]), torch.tensor([[int(fx["push_action"][t])]]),
                      torch.from_numpy(fx["push_reward"][t:t + 1]), None, feat)
        agree(ref, fx, t)
    fx = load("cb_dj_container")
    ref = container_of(fx, int(fx["obs"]))
    S, A, Rw = (torch.from_numpy(fx[k]) for k in ("push_state", "push_action", "push_reward"))
    o, r = 0, 0
    for c in range(len(fx["call_A"])):
        for _ in range(10):
            n = int(fx["idx_len"][r])
            i = torch.from_numpy(fx["idx"][o:o + n]).long()
            want = ref.round(S[i], A[i].reshape(-1, 1), Rw[i])
            assert [int((A[i] == k).sum()) for k in range(4)] == fx["counts"][r].tolist()
            o, r = o + n, r + 1
            assert set(want) == {0, 1, 2, 3}
        agree(ref, fx, c)


def test_oracle_reproduces_the_recorded_learn_batch():
    fx = load("cb_dj_batch")
    obs = int(fx["obs"])
    ref = container_of(fx, obs)
    so = ao = 0
    for c, B in enumerate(fx["c_B"]):
        B = int(B)
        n = B * (4 if fx["c_state3d"][c] else 1) * obs
        state = torch.from_numpy(fx["c_state"][so:so + n]).reshape((B, 4, obs) if fx["c_state3d"][c] else (B, obs))
        w = torch.from_numpy(fx["c_weight"][ao:ao + B]) if fx["c_has_weight"][c] else None
        out = ref.round(state, torch.from_numpy(fx["c_action"][ao:ao + B]).reshape(B, 1), torch.from_numpy(fx["c_reward"][ao:ao + B]), w)
        assert out[3][2].shape == (1, 1) and float(out[3][2]) == 0.0       # arm 3 is never named: its null batch
        agree(ref, fx, c, "c_")
        so, ao = so + n, ao + B
    for sfo in (0, 1):
        p = f"l{sfo}_"
        ref = do.Disjoint(3, obs + (1 if sfo else 2), [3.0] * 3, linear=True)
        feat = None if sfo else torch.arange(3, dtype=torch.float32).reshape(3, 1)
        o = 0
        for c, B in enumerate(fx[p + "B"]):
            B = int(B)
            sl = slice(o, o + B)
            ref.round(torch.from_numpy(fx[p + "state"][o * obs:(o + B) * obs]).reshape(B, obs),
                      torch.from_numpy(fx[p + "action"][sl]).reshape(B, 1), torch.from_numpy(fx[p + "reward"][sl]),
                      torch.from_numpy(fx[p + "weight"][sl]), feat)
            agree(ref, fx, c, p)
            o += B


def test_oracle_reproduces_the_recorded_thompson_draws_and_layout():
    fx = load("cb_dj_ts")
    obs = int(fx["c_obs"])
    ref = container_of(fx, obs)
    n = len(fx["c_fit_action"])
    ref.round(torch.from_numpy(fx["c_fit_state"]), torch.from_numpy(fx["c_fit_action"]).reshape(n, 1),
              torch.from_numpy(fx["c_fit_reward"]))
    o = 0
    for i in range(3):
        torch.set_rng_state(torch.from_numpy(fx["c_torch_before"][i]))
        eps = ref.draws()
        assert np.array_equal(torch.get_rng_state().numpy(), fx["c_torch_after"][i])
        assert torch.equal(eps, torch.from_numpy(fx["c_eps"][i]))
        theta = ref.thetas(eps)
        assert float((theta - torch.from_numpy(fx["c_theta"][i])).norm()) <= 1e-5 * (1 + float(theta.norm()))
        s = ref.ts_scores(torch.from_numpy(fx[f"c_state{i}"]), theta).reshape(-1)
        want = torch.from_numpy(fx["c_scores"][o:o + s.numel()])
        assert float((s - want).norm()) <= 1e-4 * (1 + float(want.norm()))
        o += s.numel()


def test_oracle_reproduces_the_recorded_ucb_scores():
    fx = load("cb_dj_scores")
    ref = container_of(fx, int(fx["obs"]))
    n = len(fx["fit_action"])
    ref.round(torch.from_numpy(fx["fit_state"]), torch.from_numpy(fx["fit_action"]).reshape(n, 1), torch.from_numpy(fx["fit_reward"]))
    st = torch.from_numpy(fx["states"])
    assert float((ref.scores(st, float(fx["alpha"])) - torch.from_numpy(fx["ucb"])).abs().max()) <= 1e-4
    assert float((ref.scores(st, 0.0, False) - torch.from_numpy(fx["mu"])).abs().max()) <= 1e-4
