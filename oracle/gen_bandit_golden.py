#!/usr/bin/env python
"""Generate tests/golden/cb_*.npz by RUNNING THE REFERENCE's LinearBandit (CPU, same stubs and import path as
oracle/gen_golden.py).

    PYTHONDONTWRITEBYTECODE=1 python oracle/gen_bandit_golden.py

Cases:
  cb_lin_method   the agent loop: act -> push -> learn() per step over a BasicReplayBuffer, one-hot actions (obs 16, 10
                  actions, batch 128, 10 rounds, UCB alpha 1), gamma 0.5 with a discounting interval that fires inside and
                  across calls; the buffer starts below the batch size so the clamp is exercised
  cb_lin_binary   the same loop with the binary code of 5 bits over 26 actions, no discounting
  cb_lin_batch    learn_batch on dense action feature vectors (as Pearl's own unit tests call it) with weights (one batch
                  of all-zero weights, one without weights), initial_coefs and discounting
  cb_lin_scores   act / get_scores over a batch of states with availability masks, alpha 0 and alpha 2, and exploit=True

Recorded: the pushes, the sampled logical indices of every round, CPython's `random` state before and after, the
per-round predictions, the state after every call (A, b, sum_weight, inv_A, coefs, last_sum_weight_when_discounted), the
actions act() chose, and the scores.  The generator asserts cond(A + lambda I) <= 1e4 after every call (where the
reference's fp32 inverse is accurate to well inside the 1e-4 contract, DESIGN.md) and a margin between the best and the
second-best available UCB score of every recorded action, so that fp32 rounding cannot flip it.
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
from pearl.policy_learners.contextual_bandits.linear_bandit import LinearBandit  # noqa: E402
from pearl.policy_learners.exploration_modules.contextual_bandits.ucb_exploration import UCBExploration  # noqa: E402
from pearl.replay_buffers.basic_replay_buffer import BasicReplayBuffer  # noqa: E402
from pearl.replay_buffers.transition import TransitionBatch  # noqa: E402
from pearl.utils.instantiations.spaces.discrete_action import DiscreteActionSpace  # noqa: E402

MARGIN = 1e-3      # relative gap between the best and the second-best available score of a recorded action
COND_MAX = 1e4


def snapshot(pl):
    m = pl.model
    M = (m._A + m.l2_reg_lambda * torch.eye(m._A.shape[0])).double()
    cond = float(torch.linalg.cond(M))
    assert cond <= COND_MAX, f"cond(A + lambda I) = {cond:.3g} leaves the regime where the fp32 reference is accurate"
    return dict(A=m._A.numpy().copy(), b=m._b.numpy().copy(), sum_weight=m._sum_weight.numpy().copy(),
                inv_A=m._inv_A.numpy().copy(), coefs=m._coefs.numpy().copy(), last=float(pl.last_sum_weight_when_discounted),
                cond=cond)


def margin_ok(scores, mask=None):
    s = scores.double().clone()
    if mask is not None:
        s[~mask.bool()] = -float("inf")
    top = torch.topk(s, 2, dim=-1).values
    gap = top[..., 0] - top[..., 1]
    return bool((gap > MARGIN * (1.0 + top[..., 0].abs())).all())


def stack(snaps):
    return {f"call_{k}": np.stack([np.asarray(s[k]) for s in snaps]) for k in snaps[0]}


def rewards(rng, theta, beta, s, a_feat):
    r = s @ theta + a_feat @ beta + 0.1 * rng.standard_normal()
    return np.float32(np.round(r * 256) / 256)


def gen_method(name, *, obs, n_act, rep, batch, rounds, prefill, steps, alpha, gamma, interval, seed):
    torch.manual_seed(seed)
    random.seed(seed)
    torch.set_num_threads(1)
    rng = np.random.default_rng(seed)
    module = OneHotActionTensorRepresentationModule(n_act) if rep == "one_hot" else BinaryActionTensorRepresentationModule(rep)
    act_dim = module.representation_dim
    space = DiscreteActionSpace([torch.tensor([i]) for i in range(n_act)])
    feats = module(torch.arange(n_act).view(-1, 1)).numpy().reshape(n_act, act_dim)
    pl = LinearBandit(feature_dim=obs + act_dim, exploration_module=UCBExploration(alpha=alpha), l2_reg_lambda=1.0, gamma=gamma,
                      apply_discounting_interval=interval, training_rounds=rounds, batch_size=batch,
                      action_representation_module=module)
    buf = BasicReplayBuffer(100000)
    theta, beta = rng.standard_normal(obs).astype(np.float32) * 0.5, rng.standard_normal(act_dim).astype(np.float32)
    idxs, preds, snaps = [], [], []
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
        r = rewards(rng, theta, beta, s, feats[a])
        buf.push(state=torch.from_numpy(s), action=torch.tensor([a]), reward=float(r), terminated=True, truncated=False,
                 curr_available_actions=None, next_state=None, next_available_actions=None, max_number_actions=n_act)
        P["state"].append(s); P["action"].append(a); P["reward"].append(r)

    def learn():
        rep_ = pl.learn(buf)
        preds.extend(p.numpy().ravel() for p in rep_["prediction"])
        snaps.append(snapshot(pl))

    for _ in range(prefill):
        push(np.round(rng.standard_normal(obs) * 64).astype(np.float32) / 64, int(rng.integers(n_act)))
    rs = random.getstate()
    learn()
    chosen, states = [], []
    for _ in range(steps):
        s = np.round(rng.standard_normal(obs) * 64).astype(np.float32) / 64
        a = int(pl.act(torch.from_numpy(s), space).reshape(-1)[0])
        assert margin_ok(pl.get_scores(torch.from_numpy(s), space)), "UCB margin too small for a recorded action"
        chosen.append(a); states.append(s)
        push(s, a)
        learn()
    assert any(s["last"] > 0 for s in snaps) or interval == 0
    out = dict(seed=seed, obs=obs, n_actions=n_act, rep=rep if isinstance(rep, str) else f"binary{rep}", act_dim=act_dim,
               batch=batch, rounds=rounds, alpha=alpha, gamma=gamma, interval=interval, l2_reg_lambda=1.0, prefill=prefill,
               push_state=np.stack(P["state"]), push_action=np.asarray(P["action"], np.int32),
               push_reward=np.asarray(P["reward"], np.float32), act_state=np.stack(states), act_chosen=np.asarray(chosen, np.int32),
               rng_before=state_words(rs), rng_after=state_words(random.getstate()),
               idx=np.asarray([j for r in idxs for j in r], dtype=np.int32), idx_len=np.asarray([len(r) for r in idxs], np.int32),
               pred=np.concatenate(preds).astype(np.float32), keys=np.asarray(list(pl.state_dict().keys())), **stack(snaps))
    save(name, out, f"{len(snaps)} calls, {len(idxs)} rounds, discounted at {sorted(set(s['last'] for s in snaps))[:4]}")
    return out


def gen_batch(name, *, obs, act_dim, batch, calls, gamma, interval, seed):
    torch.manual_seed(seed)
    rng = np.random.default_rng(seed)
    init = torch.from_numpy(rng.standard_normal(obs + act_dim + 1).astype(np.float32))
    pl = LinearBandit(feature_dim=obs + act_dim, l2_reg_lambda=0.5, gamma=gamma, apply_discounting_interval=interval,
                      batch_size=batch, initial_coefs=init)
    B = dict(state=[], action=[], reward=[], weight=[], has_weight=[])
    preds, snaps = [], []
    for c in range(calls):
        s = rng.standard_normal((batch, obs)).astype(np.float32)
        a = rng.uniform(-1, 1, (batch, act_dim)).astype(np.float32)
        r = (s.sum(1) * 0.3 + a @ np.arange(act_dim, dtype=np.float32) + 0.1 * rng.standard_normal(batch)).astype(np.float32)
        w = rng.uniform(0.25, 2.0, batch).astype(np.float32)
        if c == 1:
            w[:] = 0
        has_w = c != 2
        rep_ = pl.learn_batch(TransitionBatch(state=torch.from_numpy(s), action=torch.from_numpy(a), reward=torch.from_numpy(r),
                                              weight=torch.from_numpy(w) if has_w else None))
        preds.append(rep_["prediction"].numpy().ravel())
        snaps.append(snapshot(pl))
        B["state"].append(s); B["action"].append(a); B["reward"].append(r); B["weight"].append(w if has_w else np.ones_like(w))
        B["has_weight"].append(has_w)
    assert any(s["last"] > 0 for s in snaps)
    out = dict(seed=seed, obs=obs, act_dim=act_dim, batch=batch, gamma=gamma, interval=interval, l2_reg_lambda=0.5,
               initial_coefs=init.numpy(), **{f"b_{k}": np.stack(v) for k, v in B.items()}, pred=np.stack(preds), **stack(snaps))
    save(name, out, f"{calls} calls, discounted at {sorted(set(s['last'] for s in snaps))}")
    return out


def gen_scores(name, *, obs, n_act, n_states, seed):
    """A LinearBandit fitted by learn_batch on one-hot rows, then scored over a batch of states."""
    torch.manual_seed(seed)
    rng = np.random.default_rng(seed)
    module = OneHotActionTensorRepresentationModule(n_act)
    space = DiscreteActionSpace([torch.tensor([i]) for i in range(n_act)])
    pl = LinearBandit(feature_dim=obs + n_act, exploration_module=UCBExploration(alpha=2.0), batch_size=256,
                      action_representation_module=module)
    s = rng.standard_normal((256, obs)).astype(np.float32)
    a = rng.integers(n_act, size=256)
    r = (s[:, 0] + 0.5 * a + 0.1 * rng.standard_normal(256)).astype(np.float32)
    pl.learn_batch(TransitionBatch(state=torch.from_numpy(s), action=module(torch.from_numpy(a).view(-1, 1)),
                                   reward=torch.from_numpy(r)))
    states = torch.from_numpy(rng.standard_normal((n_states, obs)).astype(np.float32))
    mask = torch.from_numpy(rng.random((n_states, n_act)) < 0.6)
    mask[:, 0] = True
    ucb = pl.get_scores(states, space)
    exploit = pl.get_scores(states, space, exploit=True)
    assert margin_ok(ucb, mask) and margin_ok(ucb), "UCB margin too small"
    # act() with a mask: get_model_action_index_batch's first maximum over the available positions.  Its masked-tensor
    # argmax returns floating-point indices under this torch version, which nn.functional.embedding refuses, so the
    # masked choices are taken by that rule from the reference's own scores.
    first_max = lambda sc: torch.argmax(torch.where(mask, sc, torch.tensor(-float("inf"))), dim=1)  # noqa: E731
    act_mask = first_max(ucb)
    act_all = pl.act(states, space).reshape(-1)
    pl.exploration_module = UCBExploration(alpha=0.0)
    ucb0 = pl.get_scores(states, space)
    assert margin_ok(ucb0, mask)
    act0 = first_max(ucb0)
    m = pl.model
    out = dict(seed=seed, obs=obs, n_actions=n_act, A=m._A.numpy(), b=m._b.numpy(), sum_weight=m._sum_weight.numpy(),
               inv_A=m._inv_A.numpy(), coefs=m._coefs.numpy(), states=states.numpy(), mask=mask.numpy(), alpha=2.0,
               ucb=ucb.numpy(), ucb0=ucb0.numpy(), exploit=exploit.numpy(), act_mask=act_mask.numpy().astype(np.int32),
               act_all=act_all.numpy().astype(np.int32), act0=act0.numpy().astype(np.int32))
    save(name, out, f"{n_states} states")


def save(name, out, what):
    path = os.path.join(GOLDEN, f"{name}.npz")
    np.savez_compressed(path, **out)
    print(f"{name}.npz: {os.path.getsize(path) // 1024} KB, {what}")


if __name__ == "__main__":
    gen_method("cb_lin_method", obs=16, n_act=10, rep="one_hot", batch=128, rounds=10, prefill=120, steps=16, alpha=1.0,
               gamma=0.5, interval=2000.0, seed=81)
    gen_method("cb_lin_binary", obs=16, n_act=26, rep=5, batch=64, rounds=4, prefill=50, steps=12, alpha=1.0, gamma=1.0,
               interval=0.0, seed=82)
    gen_batch("cb_lin_batch", obs=8, act_dim=4, batch=64, calls=6, gamma=0.8, interval=100.0, seed=83)
    gen_scores("cb_lin_scores", obs=12, n_act=7, n_states=64, seed=84)
