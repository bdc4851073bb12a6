#!/usr/bin/env python
"""Generate tests/golden/cb_ts_*.npz by RUNNING THE REFERENCE's Thompson sampling (ThompsonSamplingExplorationLinear) on
LinearBandit and NeuralLinearBandit (CPU, same stubs and import path as oracle/gen_golden.py).

    PYTHONDONTWRITEBYTECODE=1 python oracle/gen_ts_golden.py

Cases:
  cb_ts_neural   the CB benchmark's NeuralTS config (return_neural_lin_ts_config: hidden [64, 16], lr 0.01, batch 128,
                 10 rounds, state_features_only=False, 5-bit binary action code, default sampling) as an agent loop:
                 act -> push -> learn() per step over a BasicReplayBuffer.  The ridge runs with lambda 8 and gamma 0.5 every
                 1000 rows, as cb_nl_agent does, which keeps cond(A + lambda I) within 1e4
  cb_ts_linear   LinTS on LinearBandit with one-hot codes and discounting inside the run, as an agent loop, once with the
                 default sampling (prefix def_) and once with enable_efficient_sampling (prefix eff_)
  cb_ts_scores   NeuralLinearBandit with a sigmoid output: get_scores with separate_uncertainty False and True, act over
                 many states with and without a mask; LinearBandit get_scores and act over many states in both modes

Recorded: the pushes, the sampled logical indices, CPython's `random` state, and after every learn() the ridge buffers
(and the network's parameters); for every Thompson call the torch generator state before and after it, the standard
normals it drew (replayed from the generator: d of them, or n x S with efficient sampling), theta, the scores and the
choices.  The generator asserts cond(A + lambda I) <= 1e4 after every call, that the draws replayed from the generator
leave it where the call left it, that oracle/ts_oracle.py reproduces theta and the scores, and a margin on every recorded
choice: the gap between the best and second-best available score exceeds MARGIN (relative), and exceeds by CHOICE_SAFETY
times the largest score change theta's tolerance THETA_TOL (tests/test_ts_bandits.py) can cause.  The reference's
masked act fails in `embedding` under the pinned torch, so masked choices are recorded by its first-maximum rule on the
scores it computed.
"""
from __future__ import annotations

import os
import random
import sys

import numpy as np

sys.dont_write_bytecode = True
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from oracle.gen_golden import state_words  # noqa: E402  (sets up the reference import path and stubs)
from oracle.gen_neural_linear_golden import flat, save  # noqa: E402
from oracle.gen_bandit_golden import snapshot as lin_snapshot  # noqa: E402
from oracle import ts_oracle  # noqa: E402

import torch  # noqa: E402
from torch.distributions.multivariate_normal import MultivariateNormal  # noqa: E402
from pearl.action_representation_modules.binary_action_representation_module import (  # noqa: E402
    BinaryActionTensorRepresentationModule,
)
from pearl.action_representation_modules.one_hot_action_representation_module import (  # noqa: E402
    OneHotActionTensorRepresentationModule,
)
from pearl.policy_learners.contextual_bandits.linear_bandit import LinearBandit  # noqa: E402
from pearl.policy_learners.contextual_bandits.neural_linear_bandit import NeuralLinearBandit  # noqa: E402
from pearl.policy_learners.exploration_modules.contextual_bandits.thompson_sampling_exploration import (  # noqa: E402
    ThompsonSamplingExplorationLinear,
)
from pearl.replay_buffers.basic_replay_buffer import BasicReplayBuffer  # noqa: E402
from pearl.replay_buffers.transition import TransitionBatch  # noqa: E402
from pearl.utils.instantiations.spaces.discrete_action import DiscreteActionSpace  # noqa: E402

MARGIN = 1e-3          # relative gap between the best and second-best available score of a recorded choice
THETA_TOL = 1e-4       # tests hold theta to |theta - theta_ref| <= THETA_TOL (1 + |theta_ref|), elementwise
CHOICE_SAFETY = 4.0
COND_MAX = 1e4

THETA_ERR = [0.0]      # the largest relative distance of a recorded theta from the float64 sample
_log: list = []        # the Thompson calls of the current learner, appended by the spies below
_orig_sample = MultivariateNormal.sample


def _sample_spy(self, sample_shape=torch.Size()):
    t = _orig_sample(self, sample_shape)
    _log[-1]["theta"] = t.detach().clone()
    return t


MultivariateNormal.sample = _sample_spy


def spy_explorer(ex):
    orig = ex.get_scores

    def get_scores(subjective_state, action_space, values, representation=None, exploit_action=None):
        out = orig(subjective_state=subjective_state, action_space=action_space, values=values, representation=representation)
        _log[-1].update(x=subjective_state.detach().reshape(-1, subjective_state.shape[-1]).clone(), scores=out.detach().clone())
        return out
    ex.get_scores = get_scores
    return ex


def thompson_call(fn, ridge, efficient, n_draws):
    """Run one act / get_scores, then replay its draws from the generator and check them and the result against
    ts_oracle.  Returns the call's record."""
    before = torch.get_rng_state()
    _log.append({})
    out = fn()
    after = torch.get_rng_state()
    rec = _log[-1]
    torch.set_rng_state(before)
    draws = torch.empty(n_draws).normal_()
    assert torch.equal(torch.get_rng_state(), after), "the call does not draw exactly the replayed standard normals"
    rec.update(out=out, torch_before=before.numpy().copy(), torch_after=after.numpy().copy(), draws=draws)
    x = rec["x"]
    if efficient:
        want = ts_oracle.efficient_scores(ridge._inv_A, ridge._coefs, x, draws)
        assert torch.allclose(want.reshape(-1), rec["scores"].reshape(-1), rtol=1e-6, atol=1e-6), "efficient scores differ"
        rec["bound"] = torch.zeros(x.shape[0], dtype=torch.float64)
    else:
        theta = rec["theta"]
        t32 = ts_oracle.sample_theta(ridge._A, ridge.l2_reg_lambda, ridge._coefs, draws)
        assert float((t32 - theta).abs().max()) <= 1e-6 * (1 + float(theta.abs().max())), "theta differs from the restatement"
        # the fp32 reference's own distance from the float64 sample stays well inside the tests' tolerance
        t64 = ts_oracle.sample_theta(ridge._A, ridge.l2_reg_lambda, ridge._coefs, draws, torch.float64)
        err = float((t64 - theta.double()).abs().max()) / (1 + float(t64.abs().max()))
        assert err <= THETA_TOL / CHOICE_SAFETY, f"the fp32 reference's theta is {err:.3g} from the float64 sample"
        THETA_ERR[0] = max(THETA_ERR[0], err)
        assert float((ts_oracle.theta_scores(x, theta).reshape(-1) - rec["scores"].reshape(-1)).abs().max()) <= 1e-5 * (
            1 + float(rec["scores"].abs().max())), "scores differ from [1, x] . theta"
        # the largest score change a theta within the tests' tolerance can cause, per row
        x1 = torch.cat([torch.ones(x.shape[0], 1), x.float()], 1).double()
        rec["bound"] = x1.abs().sum(1) * THETA_TOL * (1 + float(theta.abs().max()))
    return rec


def margin_ok(scores, bound, mask=None):
    s = scores.double().reshape(-1, scores.shape[-1]).clone()
    b = bound.reshape(s.shape[0], -1).max(1).values if bound.numel() > s.shape[0] else bound.reshape(-1)
    if mask is not None:
        s[~mask.bool().reshape(s.shape)] = -float("inf")
    top = torch.topk(s, 2, dim=-1).values
    gap = top[:, 0] - top[:, 1]
    return bool((gap > MARGIN * (1.0 + top[:, 0].abs())).all() and (gap > CHOICE_SAFETY * 2 * b).all())


def ts_records(recs, prefix):
    out = {f"{prefix}torch_before": np.stack([r["torch_before"] for r in recs]),
           f"{prefix}torch_after": np.stack([r["torch_after"] for r in recs])}
    out[f"{prefix}draws"] = np.concatenate([r["draws"].numpy().ravel() for r in recs]).astype(np.float32)
    out[f"{prefix}draws_len"] = np.asarray([r["draws"].numel() for r in recs], np.int32)
    out[f"{prefix}scores"] = np.concatenate([r["scores"].numpy().ravel() for r in recs]).astype(np.float32)
    if "theta" in recs[0]:
        out[f"{prefix}theta"] = np.stack([r["theta"].numpy() for r in recs])
    return out


def nl_snapshot(pl):
    lin = pl.model._linear_regression_layer
    M = ts_oracle.precision(lin._A, lin.l2_reg_lambda).double()
    cond = float(torch.linalg.cond(M))
    assert cond <= COND_MAX, f"cond(A + lambda I) = {cond:.3g} leaves the regime where the fp32 reference is accurate"
    return dict(params=flat(pl), A=lin._A.numpy().copy(), b=lin._b.numpy().copy(), sum_weight=lin._sum_weight.numpy().copy(),
                inv_A=lin._inv_A.numpy().copy(), coefs=lin._coefs.numpy().copy(), last=float(pl.last_sum_weight_when_discounted),
                cond=cond)


def agent(*, kind, efficient=False, obs, n_act, rep, hidden=None, lr=0.01, batch, rounds, prefill, steps, gamma, interval, lam,
          seed, scale=1.0, prefix=""):
    torch.manual_seed(seed)
    random.seed(seed)
    torch.set_num_threads(1)
    rng = np.random.default_rng(seed)
    module = OneHotActionTensorRepresentationModule(n_act) if rep == "one_hot" else BinaryActionTensorRepresentationModule(rep)
    act_dim = module.representation_dim
    space = DiscreteActionSpace([torch.tensor([i]) for i in range(n_act)])
    feats = module(torch.arange(n_act).view(-1, 1)).numpy().reshape(n_act, act_dim)
    ex = spy_explorer(ThompsonSamplingExplorationLinear(enable_efficient_sampling=efficient))
    if kind == "nl":
        pl = NeuralLinearBandit(feature_dim=obs + act_dim, hidden_dims=list(hidden), exploration_module=ex,
                                action_representation_module=module, training_rounds=rounds, batch_size=batch, learning_rate=lr,
                                gamma=gamma, apply_discounting_interval=interval, state_features_only=False,
                                l2_reg_lambda_linear=lam)
        ridge, snapshot, d = pl.model._linear_regression_layer, nl_snapshot, hidden[-1] + 1
    else:
        pl = LinearBandit(feature_dim=obs + act_dim, exploration_module=ex, l2_reg_lambda=lam, gamma=gamma,
                          apply_discounting_interval=interval, training_rounds=rounds, batch_size=batch,
                          action_representation_module=module)
        ridge, snapshot, d = pl.model, lin_snapshot, obs + act_dim + 1
    init = flat(pl) if kind == "nl" else None
    buf = BasicReplayBuffer(100000)
    theta, beta = rng.standard_normal(obs).astype(np.float32) * 0.5, rng.standard_normal(act_dim).astype(np.float32)
    idxs, snaps = [], []
    orig_sample = buf.sample

    def sample_spy(k):
        pos = {id(t): j for j, t in enumerate(buf.memory)}
        s0 = random.getstate()
        idxs.append([pos[id(t)] for t in random.sample(buf.memory, k)])
        random.setstate(s0)
        return orig_sample(k)
    buf.sample = sample_spy
    P = dict(state=[], action=[], reward=[])

    def push(s, a):
        r = np.float32(np.round((np.tanh(s @ theta) + feats[a] @ beta * 0.5 + 0.1 * rng.standard_normal()) * 256) / 256)
        buf.push(state=torch.from_numpy(s), action=torch.tensor([a]), reward=float(r), terminated=True, truncated=False,
                 curr_available_actions=None, next_state=None, next_available_actions=None, max_number_actions=n_act)
        P["state"].append(s); P["action"].append(a); P["reward"].append(r)

    def learn():
        pl.learn(buf)
        snaps.append(snapshot(pl))

    for _ in range(prefill):
        push(np.round(rng.standard_normal(obs) * scale * 64).astype(np.float32) / 64, int(rng.integers(n_act)))
    rs = random.getstate()
    learn()
    torch_start = torch.get_rng_state().numpy().copy()
    chosen, states, recs = [], [], []
    for _ in range(steps):
        s = np.round(rng.standard_normal(obs) * scale * 64).astype(np.float32) / 64
        rec = thompson_call(lambda: pl.act(torch.from_numpy(s), space), ridge, efficient, n_act if efficient else d)
        a = int(rec["out"].reshape(-1)[0])
        assert a == int(torch.argmax(rec["scores"].reshape(-1)))
        assert margin_ok(rec["scores"], rec["bound"]), f"Thompson margin too small for a recorded action (step {len(chosen)})"
        chosen.append(a); states.append(s); recs.append(rec)
        push(s, a)
        learn()
    assert interval == 0 or any(sn["last"] > 0 for sn in snaps)
    p = prefix
    out = {f"{p}push_state": np.stack(P["state"]), f"{p}push_action": np.asarray(P["action"], np.int32),
           f"{p}push_reward": np.asarray(P["reward"], np.float32), f"{p}act_state": np.stack(states),
           f"{p}act_chosen": np.asarray(chosen, np.int32), f"{p}rng_before": state_words(rs),
           f"{p}rng_after": state_words(random.getstate()), f"{p}torch_start": torch_start,
           f"{p}torch_end": torch.get_rng_state().numpy().copy(),
           f"{p}idx": np.asarray([j for r in idxs for j in r], dtype=np.int32),
           f"{p}idx_len": np.asarray([len(r) for r in idxs], np.int32),
           f"{p}keys": np.asarray(list(pl.state_dict().keys()))}
    if init is not None:
        out[f"{p}init"] = init
    out.update({f"{p}call_{k}": np.stack([np.asarray(sn[k]) for sn in snaps]) for k in snaps[0]})
    out.update(ts_records(recs, p))
    return out, snaps


def gen_neural(name, **kw):
    out, snaps = agent(kind="nl", **kw)
    cfg = dict(kw)
    cfg["hidden"] = np.asarray(cfg["hidden"], np.int32)
    cfg["rep"] = f"binary{cfg['rep']}"
    cfg["act_dim"] = int(str(cfg["rep"])[6:])
    save(name, {**cfg, "l2_reg_lambda": kw["lam"], **out},
         f"{len(snaps)} calls, cond <= {max(s['cond'] for s in snaps):.3g}, discounted at {sorted(set(s['last'] for s in snaps))[:4]}")


def gen_linear(name, **kw):
    out = dict(kw)
    out.update(act_dim=kw["n_act"], l2_reg_lambda=kw["lam"])
    for prefix, efficient in (("def_", False), ("eff_", True)):
        o, snaps = agent(kind="lin", efficient=efficient, prefix=prefix, **kw)
        out.update(o)
    save(name, out, f"{len(snaps)} calls per mode, cond <= {max(s['cond'] for s in snaps):.3g}")


def gen_scores(name, *, obs, n_act, hidden, n_states, seed):
    torch.manual_seed(seed)
    torch.set_num_threads(1)
    rng = np.random.default_rng(seed)
    space = DiscreteActionSpace([torch.tensor([i]) for i in range(n_act)])
    module = OneHotActionTensorRepresentationModule(n_act)
    out = dict(seed=seed, obs=obs, n_actions=n_act, hidden=np.asarray(hidden, np.int32), n_states=n_states)
    # NeuralLinearBandit, sigmoid output, state || one-hot action
    ex = spy_explorer(ThompsonSamplingExplorationLinear())
    pl = NeuralLinearBandit(feature_dim=obs + n_act, hidden_dims=list(hidden), exploration_module=ex, batch_size=256,
                            learning_rate=0.01, action_representation_module=module, output_activation_name="sigmoid",
                            state_features_only=False, l2_reg_lambda_linear=4.0)
    s = rng.standard_normal((256, obs)).astype(np.float32)
    a = np.eye(n_act, dtype=np.float32)[rng.integers(n_act, size=256)]
    r = (1 / (1 + np.exp(-(0.5 * s[:, 0] + a @ np.linspace(-3, 3, n_act))))).astype(np.float32)
    for _ in range(3):
        pl.learn_batch(TransitionBatch(state=torch.from_numpy(s), action=torch.from_numpy(a), reward=torch.from_numpy(r)))
    lin = pl.model._linear_regression_layer
    snap = nl_snapshot(pl)
    states = torch.from_numpy(rng.standard_normal((n_states, obs)).astype(np.float32))
    mask = torch.from_numpy(rng.random((n_states, n_act)) < 0.6)
    mask[:, 0] = True
    d = hidden[-1] + 1
    out["nl_torch_start"] = torch.get_rng_state().numpy().copy()
    recs = []
    with torch.no_grad():
        recs.append(thompson_call(lambda: pl.get_scores(states, space), lin, False, d))
        # get_scores applies the sigmoid after the explorer: the explorer's scores are the pre-activation products
        assert torch.allclose(recs[-1]["out"], torch.sigmoid(recs[-1]["scores"]).reshape(n_states, n_act))
        pl.separate_uncertainty = True
        recs.append(thompson_call(lambda: pl.get_scores(states, space), lin, False, d))
        assert torch.equal(recs[-1]["out"], recs[-1]["scores"].reshape(n_states, n_act))
        pl.separate_uncertainty = False
    recs.append(thompson_call(lambda: pl.act(states, space), lin, False, d))
    act_all = recs[-1]["out"].reshape(-1)
    assert margin_ok(recs[-1]["scores"], recs[-1]["bound"]), "Thompson margin too small for a recorded action (nl act)"
    # masked act: the reference fails in `embedding` (float indices) under the pinned torch; its first-maximum rule on the
    # scores it draws is recorded instead
    before = torch.get_rng_state()
    _log.append({})        # what the spies see of the failing call stays out of the records
    try:
        pl.act(states, space, action_availability_mask=mask)
        raise AssertionError("the reference's masked act ran: record its result instead")
    except (RuntimeError, TypeError):
        pass
    torch.set_rng_state(before)
    recs.append(thompson_call(lambda: pl.get_scores(states, space), lin, False, d))   # the same draws and pre-activation scores
    sc = recs[-1]["scores"].reshape(n_states, n_act)
    act_mask = torch.argmax(torch.where(mask, sc, torch.tensor(-float("inf"))), dim=1)
    assert margin_ok(sc, recs[-1]["bound"], mask), "Thompson margin too small for a recorded action (nl masked act)"
    out.update(nl_params=snap["params"], nl_A=snap["A"], nl_b=snap["b"], nl_sum_weight=snap["sum_weight"], nl_inv_A=snap["inv_A"],
               nl_coefs=snap["coefs"], nl_cond=snap["cond"], nl_l2_reg_lambda=4.0, states=states.numpy(), mask=mask.numpy(),
               nl_scores_act=recs[0]["out"].numpy(), nl_scores_sep=recs[1]["out"].numpy(),
               nl_act_all=act_all.numpy().astype(np.int32), nl_act_mask=act_mask.numpy().astype(np.int32),
               nl_keys=np.asarray(list(pl.state_dict().keys())))
    out.update(ts_records(recs, "nl_"))
    # LinearBandit over the same states in both modes: get_scores, then act
    for prefix, efficient in (("lin_def_", False), ("lin_eff_", True)):
        ex = spy_explorer(ThompsonSamplingExplorationLinear(enable_efficient_sampling=efficient))
        lb = LinearBandit(feature_dim=obs + n_act, exploration_module=ex, l2_reg_lambda=2.0, action_representation_module=module)
        lb.learn_batch(TransitionBatch(state=torch.from_numpy(s), action=torch.from_numpy(a), reward=torch.from_numpy(r)))
        snap = lin_snapshot(lb)
        nd = n_states * n_act if efficient else obs + n_act + 1
        out[f"{prefix}torch_start"] = torch.get_rng_state().numpy().copy()
        rs = [thompson_call(lambda: lb.get_scores(states, space), lb.model, efficient, nd),
              thompson_call(lambda: lb.act(states, space), lb.model, efficient, nd)]
        assert margin_ok(rs[1]["scores"], rs[1]["bound"]), f"Thompson margin too small for a recorded action ({prefix})"
        out.update({f"{prefix}{k}": v for k, v in snap.items()})
        out.update({f"{prefix}get_scores": rs[0]["out"].numpy(), f"{prefix}act": rs[1]["out"].reshape(-1).numpy().astype(np.int32),
                    f"{prefix}l2_reg_lambda": 2.0})
        out.update(ts_records(rs, prefix))
    save(name, out, f"{n_states} states x {n_act} actions")


if __name__ == "__main__":
    gen_neural("cb_ts_neural", obs=16, n_act=26, rep=5, hidden=(64, 16), lr=0.01, batch=128, rounds=10, prefill=150, steps=6,
               gamma=0.5, interval=1000.0, lam=8.0, seed=95, scale=0.5)
    gen_linear("cb_ts_linear", obs=10, n_act=6, rep="one_hot", batch=64, rounds=4, prefill=80, steps=10, gamma=0.5,
               interval=600.0, lam=1.0, seed=96)
    gen_scores("cb_ts_scores", obs=12, n_act=7, hidden=(24, 12), n_states=8, seed=132)
    print(f"largest relative distance of a recorded theta from the float64 sample: {THETA_ERR[0]:.3g}")
