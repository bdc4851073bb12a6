#!/usr/bin/env python
"""Generate tests/golden/cb_dj_*.npz by RUNNING THE REFERENCE's disjoint linear bandits (DisjointBanditContainer of
LinearBandit arms, DisjointLinearBandit) with DisjointUCBExploration and ThompsonSamplingExplorationLinearDisjoint (CPU,
same stubs and import path as oracle/gen_golden.py).

    PYTHONDONTWRITEBYTECODE=1 python oracle/gen_disjoint_golden.py

Cases:
  cb_dj_agent      test_agent.py's DisjointLinearBandit config (obs 3, actions tensor([0..2]), feature_dim 4,
                   DisjointUCBExploration alpha 0.1, batch 1, a one-transition BasicReplayBuffer, training_rounds 100)
                   as an act -> push -> learn() loop; lambda 20 keeps cond(A + lambda I) within 1e4
  cb_dj_container  a container of 4 LinearBandit arms with different lambda / gamma / interval and an initial_coefs arm
                   (3) that no pushed transition names, as an agent loop over a BasicReplayBuffer, batch 128, 10 rounds,
                   discounting inside and across calls; the full per-arm report of every round
  cb_dj_batch      container learn_batch calls (weights, an all-zero-weight arm, a 3-D state) and DisjointLinearBandit
                   learn_batch calls with state_features_only False and True (an absent arm, an out-of-range action)
  cb_dj_ts         disjoint Thompson sampling on both classes as agent loops (the torch generator state before and after
                   every act, the per-arm draws, theta and the choice), then container get_scores / act over several
                   identical and random states (the arm-major layout) and a masked act
  cb_dj_scores     container UCB get_scores with exploit False and True over many states, and a masked act

Recorded: the pushes, the sampled logical indices, CPython's `random` state before and after, and after every learning
call every arm's A, b, sum_weight, inv_A, coefs and last_sum_weight_when_discounted.  The generator asserts
cond(A_k + lambda_k I) <= 1e4 for every arm after every call; that oracle/disjoint_oracle.py reproduces every call (the
null batch, the skip rule, per-arm discounting, the Thompson draws replayed from the generator and the arm-major layout);
and a margin on every choice the tests hold (flagged `keep`; the best available score beats the second by MARGIN relative, and by
CHOICE_SAFETY times the largest change the tests' tolerance on theta can make).  The reference's masked act fails in
`embedding` under the pinned torch, so masked choices are recorded by its first-maximum rule on the scores it computed.
"""
from __future__ import annotations

import os
import random
import sys

import numpy as np

sys.dont_write_bytecode = True
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from oracle.gen_golden import state_words  # noqa: E402  (sets up the reference import path and stubs)
from oracle.gen_neural_linear_golden import save  # noqa: E402
from oracle import disjoint_oracle as do  # noqa: E402

import torch  # noqa: E402
from torch.distributions.multivariate_normal import MultivariateNormal  # noqa: E402
from pearl.policy_learners.contextual_bandits.disjoint_bandit import DisjointBanditContainer  # noqa: E402
from pearl.policy_learners.contextual_bandits.disjoint_linear_bandit import DisjointLinearBandit  # noqa: E402
from pearl.policy_learners.contextual_bandits.linear_bandit import LinearBandit  # noqa: E402
from pearl.policy_learners.exploration_modules.contextual_bandits.thompson_sampling_exploration import (  # noqa: E402
    ThompsonSamplingExplorationLinearDisjoint,
)
from pearl.policy_learners.exploration_modules.contextual_bandits.ucb_exploration import DisjointUCBExploration  # noqa: E402
from pearl.replay_buffers.basic_replay_buffer import BasicReplayBuffer  # noqa: E402
from pearl.replay_buffers.transition import TransitionBatch  # noqa: E402
from pearl.utils.instantiations.spaces.discrete_action import DiscreteActionSpace  # noqa: E402

MARGIN = 1e-3
THETA_TOL = 1e-4       # tests hold theta to THETA_TOL relative, normwise
CHOICE_SAFETY = 4.0
COND_MAX = 1e4
TOL = 1e-4

_thetas: list = []
_orig_sample = MultivariateNormal.sample


def _sample_spy(self, sample_shape=torch.Size()):
    t = _orig_sample(self, sample_shape)
    _thetas.append(t.detach().clone())
    return t


MultivariateNormal.sample = _sample_spy


def space(n):
    return DiscreteActionSpace([torch.tensor([i]) for i in range(n)])


def regs(pl):
    return [a.model for a in pl._arm_bandits] if isinstance(pl, DisjointBanditContainer) else list(pl._linear_regressions)


def snapshot(pl):
    out = {k: [] for k in ("A", "b", "sum_weight", "inv_A", "coefs", "last", "cond")}
    arms = list(pl._arm_bandits) if isinstance(pl, DisjointBanditContainer) else [None] * len(regs(pl))
    for m, arm in zip(regs(pl), arms):
        M = (m._A + m.l2_reg_lambda * torch.eye(m._A.shape[0])).double()
        cond = float(torch.linalg.cond(M))
        assert cond <= COND_MAX, f"cond(A + lambda I) = {cond:.3g}"
        for k, v in (("A", m._A), ("b", m._b), ("sum_weight", m._sum_weight), ("inv_A", m._inv_A), ("coefs", m._coefs)):
            out[k].append(v.detach().numpy().copy())
        out["last"].append(float(arm.last_sum_weight_when_discounted) if arm is not None else 0.0)
        out["cond"].append(cond)
    return {k: np.asarray(v) for k, v in out.items()}


def agree(snap, ref: do.Disjoint, what):
    """The oracle's state equals the reference's within the tests' tolerances."""
    for k, r in enumerate(ref.arms):
        for name, mine, nw in (("A", r.A, False), ("b", r.b, False), ("sum_weight", r.sum_weight, False),
                               ("inv_A", r.inv_A, True), ("coefs", r.coefs, True)):
            got, want = torch.from_numpy(snap[name][k]).double(), mine.double()
            if nw:
                ok = float((got - want).norm()) <= TOL * (1 + float(want.norm()))
            else:
                ok = bool(((got - want).abs() <= TOL * (1 + want.abs())).all())
            assert ok, f"{what}: arm {k} {name} differs from the oracle"
        assert abs(snap["last"][k] - r.last) <= TOL * (1 + abs(r.last)), f"{what}: arm {k} last differs"


def margin_ok(scores, bound=None, mask=None):
    s = scores.double().reshape(-1, scores.shape[-1]).clone()
    if mask is not None:
        s[~mask.bool().reshape(s.shape)] = -float("inf")
    top = torch.topk(s, 2, dim=-1).values
    gap = top[:, 0] - top[:, 1]
    ok = gap > MARGIN * (1.0 + top[:, 0].abs())
    if bound is not None:
        ok &= gap > CHOICE_SAFETY * 2 * bound
    return bool(ok.all())


def theta_bound(x, theta):
    """The largest score change a theta within THETA_TOL (normwise, relative) can make, per row."""
    x1 = torch.cat([torch.ones(x.shape[0], 1), x.float()], 1).double()
    return x1.norm(dim=1) * THETA_TOL * (1 + float(theta.double().norm()))


def ts_act(pl, ref: do.Disjoint, state, sp, feat=None, mask=None):
    """One Thompson act: the draws replayed from the generator, theta and scores checked against the oracle."""
    _thetas.clear()
    before = torch.get_rng_state()
    scores = pl.get_scores(state, sp) if isinstance(pl, DisjointBanditContainer) else None
    if scores is None:
        chosen = int(pl.act(state, sp).reshape(-1)[0])
    after = torch.get_rng_state()
    torch.set_rng_state(before)
    eps = ref.draws()
    assert torch.equal(torch.get_rng_state(), after), "the call does not draw exactly K separate draws of d"
    theta = torch.stack(_thetas)
    x = state.reshape(-1, state.shape[-1])
    want = ref.thetas(eps)
    assert float((want - theta).norm()) <= 1e-5 * (1 + float(theta.norm())), "theta differs from the restatement"
    s = ref.ts_scores(x, theta, feat)
    if scores is not None:
        assert float((s - scores).abs().max()) <= 1e-5 * (1 + float(scores.abs().max())), "scores differ (layout?)"
        chosen = None
    return dict(before=before.numpy().copy(), after=after.numpy().copy(), eps=eps.numpy().copy(), theta=theta.numpy().copy(),
                scores=s, bound=theta_bound(torch.cat([x, feat[:1].expand(x.shape[0], -1)], 1) if feat is not None else x, theta),
                chosen=chosen)


class Loop:
    """An agent loop over a BasicReplayBuffer with the sampled logical indices and the pushes recorded."""

    def __init__(self, capacity):
        self.buf = BasicReplayBuffer(capacity)
        self.idx, self.P = [], dict(state=[], action=[], reward=[])
        orig = self.buf.sample

        def sample_spy(k):
            pos = {id(t): j for j, t in enumerate(self.buf.memory)}
            s0 = random.getstate()
            self.idx.append([pos[id(t)] for t in random.sample(self.buf.memory, k)])   # 0 = the oldest still stored
            random.setstate(s0)
            return orig(k)
        self.buf.sample = sample_spy
        self.capacity = capacity

    @property
    def offset(self):
        return max(0, len(self.P["state"]) - self.capacity)

    def push(self, s, a, r, n_act):
        self.buf.push(state=torch.from_numpy(s), action=torch.tensor([a]), reward=float(r), terminated=True, truncated=False,
                      curr_available_actions=None, next_state=None, next_available_actions=None, max_number_actions=n_act)
        self.P["state"].append(s); self.P["action"].append(a); self.P["reward"].append(np.float32(r))

    def rows(self, idx):
        i = self.offset + np.asarray(idx)
        return (torch.from_numpy(np.stack(self.P["state"])[i]), torch.from_numpy(np.asarray(self.P["action"])[i]).reshape(-1, 1),
                torch.from_numpy(np.asarray(self.P["reward"], np.float32)[i]))


def stack_snaps(snaps, out, prefix=""):
    for k in snaps[0]:
        out[f"{prefix}call_{k}"] = np.stack([s[k] for s in snaps])


def gen_agent():
    seed, obs, K, lam, steps = 0, 3, 3, 20.0, 40
    torch.manual_seed(seed); random.seed(seed); torch.set_num_threads(1)
    rng = np.random.default_rng(seed)
    pl = DisjointLinearBandit(feature_dim=obs + 1, action_space=space(K), exploration_module=DisjointUCBExploration(alpha=0.1),
                              batch_size=1, l2_reg_lambda=lam)
    ref = do.Disjoint(K, obs + 2, [lam] * K, linear=True)
    feat = torch.arange(K, dtype=torch.float32).reshape(K, 1)
    loop, snaps, chosen, act_state, keep = Loop(1), [], [], [], []
    w = rng.standard_normal((K, obs)).astype(np.float32)
    rng_before = state_words(random.getstate())
    for t in range(steps):
        s = rng.standard_normal(obs).astype(np.float32)
        x = torch.from_numpy(s).reshape(1, obs)
        a = int(pl.act(x, space(K)).reshape(-1)[0])
        sc = ref.scores(x, 0.1, True, feat)
        assert a == int(torch.argmax(sc[0]))
        # a choice is held to the recording only where it has a margin (early on, unsolved arms tie exactly); the loop
        # pushes the recorded action either way
        keep.append(margin_ok(sc))
        chosen.append(a); act_state.append(s)
        r = np.float32(np.round((s @ w[a] + 0.1 * rng.standard_normal()) * 256) / 256)
        loop.push(s, a, r, K)
        n0 = len(loop.idx)
        pl.learn(loop.buf)
        for idx in loop.idx[n0:]:
            ref.round(*loop.rows(idx), None, feat)
        snaps.append(snapshot(pl))
        agree(snaps[-1], ref, f"step {t}")
    out = dict(obs=obs, n_arms=K, lam=lam, alpha=0.1, rounds=pl._training_rounds, batch=1, capacity=1,
               push_state=np.stack(loop.P["state"]), push_action=np.asarray(loop.P["action"], np.int64),
               push_reward=np.asarray(loop.P["reward"], np.float32), idx=np.asarray(loop.idx, np.int64).reshape(-1),
               act_chosen=np.asarray(chosen, np.int64), act_keep=np.asarray(keep), rng_before=rng_before,
               rng_after=state_words(random.getstate()))
    assert sum(keep) >= steps // 2, "too few choices with a margin"
    stack_snaps(snaps, out)
    save("cb_dj_agent", out, f"DisjointLinearBandit agent loop, {steps} steps x {pl._training_rounds} rounds")


LAMS, GAMMAS, INTERVALS = [1.0, 2.0, 0.5, 4.0], [0.9, 0.5, 1.0, 0.7], [300.0, 150.0, 0.0, 100.0]


def container(ex, obs):
    arms = [LinearBandit(feature_dim=obs, l2_reg_lambda=LAMS[k], gamma=GAMMAS[k], apply_discounting_interval=INTERVALS[k],
                         initial_coefs=torch.linspace(-1, 1, obs + 1) if k == 3 else None) for k in range(4)]
    return DisjointBanditContainer(feature_dim=obs, arm_bandits=arms, exploration_module=ex, training_rounds=10, batch_size=128)


def container_ref(obs):
    return do.Disjoint(4, obs + 1, LAMS, GAMMAS, INTERVALS, coefs=[None] * 3 + [torch.linspace(-1, 1, obs + 1)])


def gen_container():
    seed, obs, prefill, steps = 1, 6, 200, 12
    torch.manual_seed(seed); random.seed(seed); torch.set_num_threads(1)
    rng = np.random.default_rng(seed)
    pl = container(DisjointUCBExploration(alpha=0.5), obs)
    ref = container_ref(obs)
    loop, snaps, chosen, act_state, preds, labels, weights, counts, keep = Loop(100000), [], [], [], [], [], [], [], []
    w = rng.standard_normal((4, obs)).astype(np.float32)
    rng_before = state_words(random.getstate())

    def push():
        s = rng.standard_normal(obs).astype(np.float32)
        a = int(rng.integers(0, 3))                       # arm 3 is never named: its initial_coefs go at the first call
        loop.push(s, a, np.float32(np.round((s @ w[a] + 0.1 * rng.standard_normal()) * 256) / 256), 4)

    def learn():
        n0 = len(loop.idx)
        rep = pl.learn(loop.buf)
        for r, idx in enumerate(loop.idx[n0:]):
            st, ac, rw = loop.rows(idx)
            want = ref.round(st, ac, rw)
            counts.append([int((ac == k).sum()) for k in range(4)])
            for k in range(4):
                p = rep[f"arm_{k}_prediction"][r]
                assert float((p - want[k][0]).norm()) <= TOL * (1 + float(p.norm())), f"round {r} arm {k} prediction"
                assert torch.equal(rep[f"arm_{k}_label"][r].float().reshape(-1), want[k][1].float().reshape(-1))
                assert torch.equal(rep[f"arm_{k}_weight"][r].float().reshape(-1), want[k][2].float().reshape(-1))
                preds.append(p.detach().numpy().ravel()); labels.append(rep[f"arm_{k}_label"][r].numpy().ravel())
                weights.append(rep[f"arm_{k}_weight"][r].numpy().ravel())
        snaps.append(snapshot(pl))
        agree(snaps[-1], ref, f"learn call {len(snaps)}")

    for _ in range(prefill):
        push()
    learn()
    assert float(snaps[0]["coefs"][3].__abs__().max()) == 0.0, "the null batch replaces initial_coefs"
    for t in range(steps):
        s = rng.standard_normal(obs).astype(np.float32)
        x = torch.from_numpy(s)
        a = int(pl.act(x, space(4)).reshape(-1)[0])
        sc = ref.scores(x.reshape(1, obs), 0.5)
        assert a == int(torch.argmax(sc[0]))
        keep.append(margin_ok(sc))
        chosen.append(a); act_state.append(s)
        for _ in range(20):
            push()
        learn()
    out = dict(obs=obs, n_arms=4, lams=np.asarray(LAMS), gammas=np.asarray(GAMMAS), intervals=np.asarray(INTERVALS),
               initial_coefs=torch.linspace(-1, 1, obs + 1).numpy(), alpha=0.5, rounds=10, batch=128, prefill=prefill,
               push_state=np.stack(loop.P["state"]), push_action=np.asarray(loop.P["action"], np.int64),
               push_reward=np.asarray(loop.P["reward"], np.float32), idx=np.concatenate([np.asarray(i) for i in loop.idx]),
               idx_len=np.asarray([len(i) for i in loop.idx], np.int32), counts=np.asarray(counts, np.int32),
               pred=np.concatenate(preds).astype(np.float32), label=np.concatenate(labels).astype(np.float32),
               weight=np.concatenate(weights).astype(np.float32), act_state=np.stack(act_state),
               act_chosen=np.asarray(chosen, np.int64), act_keep=np.asarray(keep), rng_before=rng_before,
               rng_after=state_words(random.getstate()))
    assert sum(keep) >= steps // 2, "too few choices with a margin"
    stack_snaps(snaps, out)
    assert any(s["last"][0] > 0 for s in snaps) and snaps[-1]["last"][1] > snaps[0]["last"][1], "discounting inside and across calls"
    save("cb_dj_container", out, f"container agent loop, {len(snaps)} learn calls x 10 rounds")


def gen_batch():
    torch.manual_seed(2); torch.set_num_threads(1)
    g = torch.Generator().manual_seed(2)
    obs, out = 5, {}
    pl = container(DisjointUCBExploration(alpha=0.5), obs)
    ref = container_ref(obs)
    snaps, rows = [], dict(state=[], action=[], reward=[], weight=[], has_weight=[], state3d=[], B=[])
    for c in range(5):
        B = [9, 60, 33, 1, 80][c]
        state3d = c == 2
        state = torch.randn(B, 4, obs, generator=g) if state3d else torch.randn(B, obs, generator=g)
        action = torch.randint(0, 3, (B, 1), generator=g)
        reward = torch.round(torch.randn(B, 1, generator=g) * 256) / 256
        weight = torch.rand(B, 1, generator=g) if c in (1, 4) else None
        if c == 4:
            weight[action[:, 0] == 2] = 0.0            # an all-zero-weight arm
        rep = pl.learn_batch(TransitionBatch(state=state, action=action, reward=reward, weight=weight))
        want = ref.round(state, action, reward, weight)
        for k in range(4):
            assert float((rep[f"arm_{k}_prediction"] - want[k][0]).norm()) <= TOL * (1 + float(want[k][0].norm()))
            assert torch.equal(rep[f"arm_{k}_weight"].float().reshape(-1), want[k][2].float().reshape(-1))
        assert rep["arm_3_weight"].shape == (1, 1) and float(rep["arm_3_label"]) == 0.0, "the null batch reports"
        snaps.append(snapshot(pl))
        agree(snaps[-1], ref, f"container call {c}")
        rows["state"].append(state.reshape(-1).numpy()); rows["action"].append(action.numpy().ravel())
        rows["reward"].append(reward.numpy().ravel()); rows["state3d"].append(int(state3d)); rows["B"].append(B)
        rows["weight"].append(weight.numpy().ravel() if weight is not None else np.ones(B, np.float32))
        rows["has_weight"].append(int(weight is not None))
    for k in ("state", "action", "reward", "weight"):
        out[f"c_{k}"] = np.concatenate(rows[k])
    for k in ("state3d", "B", "has_weight"):
        out[f"c_{k}"] = np.asarray(rows[k], np.int32)
    out.update(obs=obs, lams=np.asarray(LAMS), gammas=np.asarray(GAMMAS), intervals=np.asarray(INTERVALS),
               initial_coefs=torch.linspace(-1, 1, obs + 1).numpy())
    stack_snaps(snaps, out, "c_")
    for sfo in (False, True):
        K, f = 3, obs if sfo else obs + 1
        pl = DisjointLinearBandit(feature_dim=f, action_space=space(K), exploration_module=DisjointUCBExploration(0.1),
                                  l2_reg_lambda=3.0, state_features_only=sfo)
        ref = do.Disjoint(K, f + 1, [3.0] * K, linear=True)
        feat = None if sfo else torch.arange(K, dtype=torch.float32).reshape(K, 1)
        snaps, rows = [], dict(state=[], action=[], reward=[], weight=[], B=[])
        for c in range(4):
            B = [12, 7, 40, 5][c]
            state, reward = torch.randn(B, obs, generator=g), torch.round(torch.randn(B, 1, generator=g) * 256) / 256
            action = torch.randint(0, K, (B, 1), generator=g)
            if c == 1:
                action[action == 2] = 0                  # an absent arm: skipped
            if c == 2:
                action[0] = 5                            # out of range: matches no arm
            weight = torch.rand(B, 1, generator=g)
            before = [m._inv_A.clone() for m in pl._linear_regressions]
            assert pl.learn_batch(TransitionBatch(state=state, action=action, reward=reward, weight=weight)) == {}
            if c == 1:
                assert torch.equal(pl._linear_regressions[2]._inv_A, before[2]), "an absent arm is not solved"
            ref.round(state, action, reward, weight, feat)
            snaps.append(snapshot(pl))
            agree(snaps[-1], ref, f"DisjointLinearBandit sfo={sfo} call {c}")
            rows["state"].append(state.numpy().ravel()); rows["action"].append(action.numpy().ravel())
            rows["reward"].append(reward.numpy().ravel()); rows["weight"].append(weight.numpy().ravel()); rows["B"].append(B)
        p = f"l{int(sfo)}_"
        for k in ("state", "action", "reward", "weight"):
            out[p + k] = np.concatenate(rows[k])
        out[p + "B"] = np.asarray(rows["B"], np.int32)
        stack_snaps(snaps, out, p)
    save("cb_dj_batch", out, "container and DisjointLinearBandit learn_batch")


def ts_pack(recs, out, p):
    out[p + "torch_before"] = np.stack([r["before"] for r in recs])
    out[p + "torch_after"] = np.stack([r["after"] for r in recs])
    out[p + "eps"] = np.stack([r["eps"] for r in recs])
    out[p + "theta"] = np.stack([r["theta"] for r in recs])


def gen_ts():
    out = {}
    # DisjointLinearBandit LinTS agent loop (batch 8, 5 rounds)
    seed, obs, K, lam = 3, 3, 3, 20.0
    torch.manual_seed(seed); random.seed(seed); torch.set_num_threads(1)
    rng = np.random.default_rng(seed)
    pl = DisjointLinearBandit(feature_dim=obs + 1, action_space=space(K), exploration_module=ThompsonSamplingExplorationLinearDisjoint(),
                              batch_size=8, training_rounds=5, l2_reg_lambda=lam)
    ref = do.Disjoint(K, obs + 2, [lam] * K, linear=True)
    feat = torch.arange(K, dtype=torch.float32).reshape(K, 1)
    loop, snaps, recs = Loop(100000), [], []
    w = rng.standard_normal((K, obs)).astype(np.float32)
    for _ in range(30):
        a = int(rng.integers(0, K)); s = rng.standard_normal(obs).astype(np.float32)
        loop.push(s, a, np.float32(np.round((s @ w[a]) * 256) / 256), K)
    rng_before = state_words(random.getstate())
    act_state = []
    t = 0
    while len(recs) < 25:
        t += 1
        s = rng.standard_normal(obs).astype(np.float32)
        x = torch.from_numpy(s).reshape(1, obs)
        snap_before = torch.get_rng_state()
        rec = ts_act(pl, ref, x, space(K), feat)
        sc = rec["scores"]
        if not margin_ok(sc, rec["bound"]):
            torch.set_rng_state(snap_before)      # a choice too close to call: this state is not recorded or acted on
            torch.empty(K * (obs + 2)).normal_()  # the same draws the call made, so the stream stays the reference's
            continue
        a = rec["chosen"]
        assert a == int(torch.argmax(sc[0]))
        recs.append(rec); act_state.append(s)
        loop.push(s, a, np.float32(np.round((s @ w[a] + 0.1 * rng.standard_normal()) * 256) / 256), K)
        n0 = len(loop.idx)
        pl.learn(loop.buf)
        for idx in loop.idx[n0:]:
            ref.round(*loop.rows(idx), None, feat)
        snaps.append(snapshot(pl))
        agree(snaps[-1], ref, f"LinTS step {t}")
    ts_pack(recs, out, "l_")
    out.update(l_obs=obs, l_n_arms=K, l_lam=lam, l_batch=8, l_rounds=5, l_push_state=np.stack(loop.P["state"]),
               l_push_action=np.asarray(loop.P["action"], np.int64), l_push_reward=np.asarray(loop.P["reward"], np.float32),
               l_idx=np.concatenate([np.asarray(i) for i in loop.idx]), l_act_state=np.stack(act_state),
               l_act_chosen=np.asarray([r["chosen"] for r in recs], np.int64), l_rng_before=rng_before,
               l_rng_after=state_words(random.getstate()), l_prefill=30)
    stack_snaps(snaps, out, "l_")

    # container: learn_batch to a fitted state, then Thompson get_scores over identical and random states, masked act
    torch.manual_seed(4)
    g = torch.Generator().manual_seed(4)
    obs = 4
    pl = container(ThompsonSamplingExplorationLinearDisjoint(), obs)
    ref = container_ref(obs)
    X, A, R = torch.randn(300, obs, generator=g), torch.randint(0, 4, (300, 1), generator=g), torch.randn(300, 1, generator=g)
    R = R + 3.0 * A.float()
    pl.learn_batch(TransitionBatch(state=X, action=A, reward=R))
    ref.round(X, A, R)
    agree(snapshot(pl), ref, "container fit")
    out.update(c_obs=obs, c_fit_state=X.numpy(), c_fit_action=A.numpy().ravel(), c_fit_reward=R.numpy().ravel(),
               lams=np.asarray(LAMS), gammas=np.asarray(GAMMAS), intervals=np.asarray(INTERVALS),
               initial_coefs=torch.linspace(-1, 1, obs + 1).numpy())
    states = [torch.ones(4, obs), torch.randn(6, obs, generator=g), torch.randn(1, obs, generator=g)]
    crecs, cscores = [], []
    for i, st in enumerate(states):
        rec = ts_act(pl, ref, st, space(4))
        crecs.append(rec); cscores.append(rec["scores"].numpy().ravel())
        out[f"c_state{i}"] = st.numpy()
    # the layout: 4 identical states read arm-major
    s0 = crecs[0]["scores"]
    per_arm = torch.from_numpy(crecs[0]["theta"]) @ torch.cat([torch.ones(1), torch.ones(obs)])
    assert torch.allclose(s0.reshape(-1), per_arm.repeat_interleave(4), rtol=1e-5, atol=1e-5), "arm-major layout"
    ts_pack(crecs, out, "c_")
    out["c_scores"] = np.concatenate(cscores)
    # masked act over the random states: the first maximum over the available arms of the scores the reference made
    mask = torch.rand(6, 4, generator=g) > 0.3
    mask[:, 0] = True
    rec = ts_act(pl, ref, states[1], space(4))
    masked = rec["scores"].masked_fill(~mask, -float("inf"))
    keep = [bool(margin_ok(masked[i:i + 1], rec["bound"][i:i + 1])) for i in range(6)]
    out.update(m_mask=mask.numpy(), m_keep=np.asarray(keep), m_chosen=torch.argmax(masked, 1).numpy(),
               m_torch_before=rec["before"], m_torch_after=rec["after"], m_theta=rec["theta"])
    assert sum(keep) >= 3
    save("cb_dj_ts", out, "disjoint Thompson sampling: DisjointLinearBandit loop and container scores / act")


def gen_scores():
    torch.manual_seed(5)
    g = torch.Generator().manual_seed(5)
    obs = 4
    pl = container(DisjointUCBExploration(alpha=0.7), obs)
    ref = container_ref(obs)
    X, A, R = torch.randn(200, obs, generator=g), torch.randint(0, 3, (200, 1), generator=g), torch.randn(200, 1, generator=g)
    pl.learn_batch(TransitionBatch(state=X, action=A, reward=R))
    ref.round(X, A, R)
    agree(snapshot(pl), ref, "scores fit")
    states = torch.randn(40, obs, generator=g)
    ucb = pl.get_scores(states, space(4))
    mu = pl.get_scores(states, space(4), exploit=True)
    assert ucb.shape == (40, 4) and mu.shape == (40, 4)
    assert float((ucb - ref.scores(states, 0.7)).abs().max()) <= 1e-5 * (1 + float(ucb.abs().max()))
    assert float((mu - ref.scores(states, 0.7, False)).abs().max()) <= 1e-5 * (1 + float(mu.abs().max()))
    acts = pl.act(states, space(4)).reshape(-1)
    assert torch.equal(acts, torch.argmax(ucb, 1))
    mask = torch.rand(40, 4, generator=g) > 0.4
    mask[:, 1] = True
    masked = ucb.masked_fill(~mask, -float("inf"))
    keep = [margin_ok(masked[i:i + 1]) for i in range(40)]
    out = dict(obs=obs, lams=np.asarray(LAMS), gammas=np.asarray(GAMMAS), intervals=np.asarray(INTERVALS),
               initial_coefs=torch.linspace(-1, 1, obs + 1).numpy(), alpha=0.7, fit_state=X.numpy(),
               fit_action=A.numpy().ravel(), fit_reward=R.numpy().ravel(), states=states.numpy(), ucb=ucb.detach().numpy(),
               mu=mu.detach().numpy(), chosen=acts.numpy(), keep=np.asarray([margin_ok(ucb[i:i + 1]) for i in range(40)]),
               mask=mask.numpy(), m_chosen=torch.argmax(masked, 1).numpy(), m_keep=np.asarray(keep))
    save("cb_dj_scores", out, "container UCB get_scores (exploit both ways) and act, masked act")


if __name__ == "__main__":
    gen_agent()
    gen_container()
    gen_batch()
    gen_ts()
    gen_scores()
