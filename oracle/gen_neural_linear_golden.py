#!/usr/bin/env python
"""Generate tests/golden/cb_nl_*.npz by RUNNING THE REFERENCE's NeuralLinearBandit (CPU, same stubs and import path as
oracle/gen_golden.py).

    PYTHONDONTWRITEBYTECODE=1 python oracle/gen_neural_linear_golden.py

Cases:
  cb_nl_agent    the reference's CB benchmark config (return_neural_lin_ucb_config: hidden [64, 16], lr 0.01, batch 128,
                 10 rounds, state_features_only=False, 5-bit binary action code, UCB alpha 1, nn_e2e) as an agent loop:
                 act -> push -> learn() per step over a BasicReplayBuffer.  The ridge runs with lambda 8 and gamma 0.5
                 every 1000 rows, which keeps cond(A + lambda I) within 1e4 over 1280 rows per call
  cb_nl_onehot   nn_e2e=False with one-hot codes, gamma 0.5 with a discounting interval hit inside and across calls, and
                 skip connections with h1 == h2 (the middle and last layers are residual); the first calls move the MLP
                 by weight decay alone (the coefs start at zero)
  cb_nl_batch    learn_batch with weights: MAE for three calls, then an lr change, a load_state_dict round trip, and
                 CROSS_ENTROPY with a sigmoid output on a second learner; each has one all-zero-weight batch mid-run
  cb_nl_scores   state_features_only=True: get_scores with separate_uncertainty False and True, act with and without masks

Recorded: the initial flat parameters, the pushes, the sampled logical indices, CPython's `random` state, the per-round
loss, mu_scores and predictions, and after every call the flat parameters, the AdamW state (exp_avg, exp_avg_sq,
max_exp_avg_sq over the parameters that have state, and the step), the ridge buffers and last_sum_weight_when_discounted;
the actions act() chose; the state_dict key list.  The generator asserts cond(A + lambda I) <= 1e4 after every call, a
margin between the best and second-best UCB score of every recorded choice, |p - y| away from 0 on every MAE row (where
l1's gradient changes sign), and the number of AdamW states (6 without e2e).
"""
from __future__ import annotations

import os
import random
import sys

import numpy as np

sys.dont_write_bytecode = True
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from oracle.gen_golden import GOLDEN, state_words  # noqa: E402  (sets up the reference import path and stubs)

import torch  # noqa: E402
from pearl.action_representation_modules.binary_action_representation_module import (  # noqa: E402
    BinaryActionTensorRepresentationModule,
)
from pearl.action_representation_modules.one_hot_action_representation_module import (  # noqa: E402
    OneHotActionTensorRepresentationModule,
)
from pearl.policy_learners.contextual_bandits.neural_linear_bandit import NeuralLinearBandit  # noqa: E402
from pearl.policy_learners.exploration_modules.contextual_bandits.ucb_exploration import UCBExploration  # noqa: E402
from pearl.replay_buffers.basic_replay_buffer import BasicReplayBuffer  # noqa: E402
from pearl.replay_buffers.transition import TransitionBatch  # noqa: E402
from pearl.utils.instantiations.spaces.discrete_action import DiscreteActionSpace  # noqa: E402

MARGIN = 1e-3
COND_MAX = 1e4
MAE_GAP = 1e-3


def flat(pl):
    return torch.cat([p.detach().reshape(-1) for p in pl.model.parameters()]).numpy().copy()


def adam(pl):
    params = list(pl.model.parameters())
    used = [p for p in params if p in pl.optimizer.state]
    if not used:
        z = np.zeros(sum(p.numel() for p in params[:-1]) if not pl.model.nn_e2e else sum(p.numel() for p in params), np.float32)
        return dict(m=z, v=z, vmax=z, step=0.0, n_state=0)
    st = pl.optimizer.state
    cat = lambda k: torch.cat([st[p][k].reshape(-1) for p in used]).numpy().copy()  # noqa: E731
    return dict(m=cat("exp_avg"), v=cat("exp_avg_sq"), vmax=cat("max_exp_avg_sq"), step=float(st[used[0]]["step"]), n_state=len(used))


def snapshot(pl):
    lin = pl.model._linear_regression_layer
    M = (lin._A + lin.l2_reg_lambda * torch.eye(lin._A.shape[0])).double()
    cond = float(torch.linalg.cond(M))
    assert cond <= COND_MAX, f"cond(A + lambda I) = {cond:.3g} leaves the regime where the fp32 reference is accurate"
    a = adam(pl)
    assert a["n_state"] in (0, 7 if pl.model.nn_e2e else 6), a["n_state"]
    return dict(params=flat(pl), A=lin._A.numpy().copy(), b=lin._b.numpy().copy(), sum_weight=lin._sum_weight.numpy().copy(),
                inv_A=lin._inv_A.numpy().copy(), coefs=lin._coefs.numpy().copy(), last=float(pl.last_sum_weight_when_discounted),
                cond=cond, **{f"adam_{k}": np.asarray(v) for k, v in a.items()})


def margin_ok(scores, mask=None):
    s = scores.double().reshape(-1, scores.shape[-1]).clone()
    if mask is not None:
        s[~mask.bool().reshape(s.shape)] = -float("inf")
    top = torch.topk(s, 2, dim=-1).values
    return bool((top[:, 0] - top[:, 1] > MARGIN * (1.0 + top[:, 0].abs())).all())


def stack(snaps):
    return {f"call_{k}": np.stack([np.asarray(s[k]) for s in snaps]) for k in snaps[0]}


def save(name, out, what):
    path = os.path.join(GOLDEN, f"{name}.npz")
    np.savez_compressed(path, **out)
    print(f"{name}.npz: {os.path.getsize(path) // 1024} KB, {what}")


def gen_agent(name, *, obs, n_act, rep, hidden, lr, batch, rounds, prefill, steps, alpha, gamma, interval, e2e, skip, seed, scale=1.0, lam=1.0):
    torch.manual_seed(seed)
    random.seed(seed)
    torch.set_num_threads(1)
    rng = np.random.default_rng(seed)
    module = OneHotActionTensorRepresentationModule(n_act) if rep == "one_hot" else BinaryActionTensorRepresentationModule(rep)
    act_dim = module.representation_dim
    space = DiscreteActionSpace([torch.tensor([i]) for i in range(n_act)])
    feats = module(torch.arange(n_act).view(-1, 1)).numpy().reshape(n_act, act_dim)
    pl = NeuralLinearBandit(feature_dim=obs + act_dim, hidden_dims=list(hidden), exploration_module=UCBExploration(alpha=alpha),
                            action_representation_module=module, training_rounds=rounds, batch_size=batch, learning_rate=lr,
                            gamma=gamma, apply_discounting_interval=interval, state_features_only=False,
                            use_skip_connections=skip, nn_e2e=e2e, l2_reg_lambda_linear=lam)
    init = flat(pl)
    buf = BasicReplayBuffer(100000)
    theta, beta = rng.standard_normal(obs).astype(np.float32) * 0.5, rng.standard_normal(act_dim).astype(np.float32)
    idxs, preds, losses, mus, snaps = [], [], [], [], []
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
        rep_ = pl.learn(buf)
        preds.extend(p.numpy().ravel() for p in rep_["prediction"])
        losses.extend(float(x) for x in rep_["loss"])
        mus.extend(float(x) for x in rep_["mu_scores"])
        snaps.append(snapshot(pl))

    for _ in range(prefill):
        push(np.round(rng.standard_normal(obs) * scale * 64).astype(np.float32) / 64, int(rng.integers(n_act)))
    rs = random.getstate()
    learn()
    chosen, states = [], []
    for _ in range(steps):
        s = np.round(rng.standard_normal(obs) * scale * 64).astype(np.float32) / 64
        a = int(pl.act(torch.from_numpy(s), space).reshape(-1)[0])
        # act's own scores: UCB on the pre-activation values (the linear output activation makes them get_scores')
        assert margin_ok(pl.get_scores(torch.from_numpy(s), space)), "UCB margin too small for a recorded action"
        chosen.append(a); states.append(s)
        push(s, a)
        learn()
    assert interval == 0 or any(s["last"] > 0 for s in snaps)
    out = dict(seed=seed, obs=obs, n_actions=n_act, rep=rep if isinstance(rep, str) else f"binary{rep}", act_dim=act_dim,
               hidden=np.asarray(hidden, np.int32), lr=lr, batch=batch, rounds=rounds, alpha=alpha, gamma=gamma, interval=interval,
               e2e=e2e, skip=skip, l2_reg_lambda=lam, prefill=prefill, init=init,
               push_state=np.stack(P["state"]), push_action=np.asarray(P["action"], np.int32),
               push_reward=np.asarray(P["reward"], np.float32), act_state=np.stack(states), act_chosen=np.asarray(chosen, np.int32),
               rng_before=state_words(rs), rng_after=state_words(random.getstate()),
               idx=np.asarray([j for r in idxs for j in r], dtype=np.int32), idx_len=np.asarray([len(r) for r in idxs], np.int32),
               pred=np.concatenate(preds).astype(np.float32), loss=np.asarray(losses, np.float32), mu=np.asarray(mus, np.float32),
               keys=np.asarray(list(pl.state_dict().keys())), **stack(snaps))
    save(name, out, f"{len(snaps)} calls, {len(idxs)} rounds, discounted at {sorted(set(s['last'] for s in snaps))[:4]}")


def gen_batch(name, *, obs, act_dim, hidden, batch, calls, seed):
    """Two learners on dense batches: MAE (linear output) and CROSS_ENTROPY (sigmoid output), both e2e."""
    torch.manual_seed(seed)
    torch.set_num_threads(1)
    rng = np.random.default_rng(seed)
    out = dict(seed=seed, obs=obs, act_dim=act_dim, hidden=np.asarray(hidden, np.int32), batch=batch, calls=calls,
               l2_reg_lambda=0.5, gamma=0.9, interval=150.0, lr0=0.005, lr1=0.02, lr_change_at=2, reload_at=2, zero_at=1)
    for tag, loss, act in (("mae", "mae", "linear"), ("ce", "cross_entropy", "sigmoid")):
        pl = NeuralLinearBandit(feature_dim=obs + act_dim, hidden_dims=list(hidden), batch_size=batch, learning_rate=0.005,
                                l2_reg_lambda_linear=0.5, gamma=0.9, apply_discounting_interval=150.0, state_features_only=False,
                                loss_type=loss, output_activation_name=act)
        out[f"{tag}_init"] = flat(pl)
        B = dict(state=[], action=[], reward=[], weight=[])
        preds, losses, mus, snaps = [], [], [], []
        for c in range(calls):
            if c == out["lr_change_at"]:
                for g in pl.optimizer.param_groups:
                    g["lr"] = out["lr1"]
            if c == out["reload_at"]:
                pl.load_state_dict({k: v.clone() for k, v in pl.state_dict().items()})
            s = rng.standard_normal((batch, obs)).astype(np.float32)
            a = rng.uniform(-1, 1, (batch, act_dim)).astype(np.float32)
            z = s.sum(1) * 0.3 + a @ np.linspace(-1, 1, act_dim).astype(np.float32)
            if loss == "mae":
                r = (z + 0.1 * rng.standard_normal(batch)).astype(np.float32)
            else:
                r = (rng.random(batch) < 1 / (1 + np.exp(-z))).astype(np.float32)
            w = rng.uniform(0.25, 2.0, batch).astype(np.float32)
            if c == out["zero_at"]:
                w[:] = 0
            rep_ = pl.learn_batch(TransitionBatch(state=torch.from_numpy(s), action=torch.from_numpy(a), reward=torch.from_numpy(r),
                                                  weight=torch.from_numpy(w)))
            p = rep_["prediction"].numpy().ravel()
            if loss == "mae" and c != out["zero_at"]:
                assert np.abs(p - r).min() > MAE_GAP, "an MAE row sits at |p - y| = 0"
            preds.append(p); losses.append(float(rep_["loss"])); mus.append(float(rep_["mu_scores"]))
            snaps.append(snapshot(pl))
            B["state"].append(s); B["action"].append(a); B["reward"].append(r); B["weight"].append(w)
        assert any(sn["last"] > 0 for sn in snaps)
        assert snaps[out["zero_at"]]["adam_step"] == snaps[out["zero_at"] - 1]["adam_step"]
        out.update({f"{tag}_b_{k}": np.stack(v) for k, v in B.items()})
        out.update({f"{tag}_pred": np.stack(preds), f"{tag}_loss": np.asarray(losses, np.float32),
                    f"{tag}_mu": np.asarray(mus, np.float32)})
        out.update({f"{tag}_{k}": v for k, v in stack(snaps).items()})
    save(name, out, f"{calls} calls x 2 losses")


def gen_scores(name, *, obs, n_act, hidden, n_states, seed):
    """A state-features-only learner fitted by learn_batch, then scored over a batch of states."""
    torch.manual_seed(seed)
    torch.set_num_threads(1)
    rng = np.random.default_rng(seed)
    space = DiscreteActionSpace([torch.tensor([i]) for i in range(n_act)])
    pl = NeuralLinearBandit(feature_dim=obs, hidden_dims=list(hidden), exploration_module=UCBExploration(alpha=2.0), batch_size=256,
                            learning_rate=0.01, action_representation_module=OneHotActionTensorRepresentationModule(n_act),
                            output_activation_name="sigmoid")
    s = rng.standard_normal((256, obs)).astype(np.float32)
    r = (s[:, 0] + 0.1 * rng.standard_normal(256)).astype(np.float32)
    for _ in range(3):
        pl.learn_batch(TransitionBatch(state=torch.from_numpy(s), action=torch.zeros(256, n_act), reward=torch.from_numpy(r)))
    states = torch.from_numpy(rng.standard_normal((n_states, obs)).astype(np.float32))
    mask = torch.from_numpy(rng.random((n_states, n_act)) < 0.6)
    mask[:, 0] = True
    ucb = pl.get_scores(states, space)
    pl.separate_uncertainty = True
    ucb_sep = pl.get_scores(states, space)
    pl.separate_uncertainty = False
    act_all = pl.act(states, space).reshape(-1)
    # every action of a state scores the same: NO_TIEBREAKING picks the first available one.  The reference's masked act
    # fails in `embedding` (float indices) under this torch version, so masked choices follow its first-maximum rule.
    first_max = lambda sc: torch.argmax(torch.where(mask, sc, torch.tensor(-float("inf"))), dim=1)  # noqa: E731
    act_mask = first_max(ucb)
    assert (act_all == 0).all()
    lin = pl.model._linear_regression_layer
    out = dict(seed=seed, obs=obs, n_actions=n_act, hidden=np.asarray(hidden, np.int32), alpha=2.0, params=flat(pl),
               A=lin._A.numpy(), b=lin._b.numpy(), sum_weight=lin._sum_weight.numpy(), inv_A=lin._inv_A.numpy(),
               coefs=lin._coefs.numpy(), states=states.numpy(), mask=mask.numpy(), ucb=ucb.numpy(), ucb_sep=ucb_sep.numpy(),
               act_mask=act_mask.numpy().astype(np.int32), act_all=act_all.numpy().astype(np.int32),
               keys=np.asarray(list(pl.state_dict().keys())))
    save(name, out, f"{n_states} states")


if __name__ == "__main__":
    gen_agent("cb_nl_agent", obs=16, n_act=26, rep=5, hidden=(64, 16), lr=0.01, batch=128, rounds=10, prefill=150, steps=6,
              alpha=1.0, gamma=0.5, interval=1000.0, e2e=True, skip=False, seed=91, scale=0.5, lam=8.0)
    gen_agent("cb_nl_onehot", obs=10, n_act=6, rep="one_hot", hidden=(16, 16), lr=0.01, batch=64, rounds=4, prefill=80, steps=10,
              alpha=1.0, gamma=0.5, interval=600.0, e2e=False, skip=True, seed=92)
    gen_batch("cb_nl_batch", obs=8, act_dim=4, hidden=(32, 8), batch=64, calls=5, seed=93)
    gen_scores("cb_nl_scores", obs=12, n_act=7, hidden=(24, 12), n_states=64, seed=94)
