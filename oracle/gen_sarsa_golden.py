#!/usr/bin/env python
"""Record tests/golden/sarsa_*.npz by RUNNING THE REFERENCE's DeepSARSA under PearlAgent with a SARSAReplayBuffer
(TEST INFRASTRUCTURE; same set-up and stubs as oracle/gen_golden.py, which provides the import path).

    PYTHONDONTWRITEBYTECODE=1 python oracle/gen_sarsa_golden.py

The pushes are a scripted episode stream (states chain within an episode: a push's state is the previous push's next
state), made with the same calls PearlAgent.observe makes; agent.learn() runs PolicyLearner.learn and then clears the
buffer, since DeepSARSA is on-policy.  Four cases:
  sarsa_method  SARSA_method's shape (obs 4, 2 actions, [64, 64], batch 32, training_rounds 1); several episodes ending
                terminated or truncated, learn() after each; target_update_freq 3 fires inside and across calls
  sarsa_steps   learn() after every push, so the batch is clamped to a buffer of 0-2 transitions; dynamic next-action sets;
                one reset state equals the stale cache's next state, so the reference appends that stale transition again
  sarsa_lr      two learn() calls, the learning rate changed in between
  sarsa_batch   agent.learn_batch on sampled, preprocessed batches; target_update_freq 1, since agent.learn_batch leaves the
                training-step count at 0
Recorded: every push, the transitions each push appended (with their next actions), the pushes after which learn() ran,
the sampled logical indices of every round, CPython's `random` state before and after, per-round losses, the initial
online net (the target is its deepcopy), the online and target nets after every call, and the AdamW state
(max_exp_avg_sq where it differs from exp_avg_sq).
"""
from __future__ import annotations

import os
import random
import sys

import numpy as np

sys.dont_write_bytecode = True
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from oracle.gen_golden import GOLDEN, flat_params, state_words  # noqa: E402  (sets up the reference import path and stubs)

import torch  # noqa: E402
from pearl.action_representation_modules.one_hot_action_representation_module import (  # noqa: E402
    OneHotActionTensorRepresentationModule,
)
from pearl.pearl_agent import PearlAgent  # noqa: E402
from pearl.policy_learners.sequential_decision_making.deep_sarsa import DeepSARSA  # noqa: E402
from pearl.replay_buffers.sequential_decision_making.sarsa_replay_buffer import SARSAReplayBuffer  # noqa: E402
from pearl.utils.instantiations.spaces.discrete_action import DiscreteActionSpace  # noqa: E402


def episodes(obs, A, lengths, ends, seed, dynamic=False, stale_reset=()):
    """The push stream: per episode, states on a 1/256 grid, the last push terminated ('t') or truncated ('u').
    stale_reset: episode numbers whose reset state equals the last state of the episode before (its terminal push's
    state, which is the stale cache's next state)."""
    rng = np.random.Generator(np.random.PCG64(seed))
    q8 = lambda x: (np.rint(x * 256) / 256).astype(np.float32)  # noqa: E731
    P = dict(state=[], action=[], reward=[], next_state=[], terminated=[], truncated=[], next_ids=[], next_count=[])
    prev_last = None
    for e, (L, end) in enumerate(zip(lengths, ends)):
        s = q8(rng.standard_normal((L + 1, obs)))
        if e in stale_reset:
            s[0] = prev_last
        for t in range(L):
            P["state"].append(s[t]); P["next_state"].append(s[t + 1])
            P["action"].append(int(rng.integers(0, A))); P["reward"].append(float(q8(rng.standard_normal())))
            P["terminated"].append(t == L - 1 and end == "t"); P["truncated"].append(t == L - 1 and end == "u")
            ids = np.zeros(A, np.int64)
            m = int(rng.integers(1, A + 1)) if dynamic else A
            ids[:m] = np.sort(rng.choice(A, size=m, replace=False)) if dynamic else np.arange(A)
            P["next_ids"].append(ids); P["next_count"].append(m)
        prev_last = s[L - 1]
    return {k: np.asarray(v) for k, v in P.items()}


def gen(name, *, obs, n_act, hidden, batch, rounds, seed, data_seed, lengths, ends, learn_every="episode", dynamic=False,
        stale_reset=(), lr=1e-3, new_lr=None, freq=10, tau=0.1, gamma=0.99, learn_batch_calls=0, capacity=10000):
    torch.manual_seed(seed)
    random.seed(seed)
    torch.set_num_threads(1)
    full = DiscreteActionSpace(actions=list(torch.arange(n_act).view(-1, 1)))
    pl = DeepSARSA(state_dim=obs, action_space=full, hidden_dims=list(hidden), learning_rate=lr, discount_factor=gamma,
                   training_rounds=rounds, batch_size=batch, target_update_freq=freq, soft_update_tau=tau,
                   action_representation_module=OneHotActionTensorRepresentationModule(n_act))
    assert pl.on_policy
    buf = SARSAReplayBuffer(capacity)
    agent = PearlAgent(policy_learner=pl, replay_buffer=buf, device_id=-1)
    P = episodes(obs, n_act, lengths, ends, data_seed, dynamic, stale_reset)
    n = len(P["action"])
    ends_at = np.cumsum(lengths) - 1
    if learn_every == "episode":
        learn_after = list(ends_at)
    elif learn_every == "step":
        learn_after = list(range(n))
    else:
        learn_after = []
    init = flat_params(pl._Q)
    assert np.array_equal(init, flat_params(pl._Q_target))
    idxs, losses, q_calls, qt_calls, call_lr, call_batch = [], [], [], [], [], []
    app = dict(push=[], state=[], action=[], reward=[], next_state=[], next_action=[], terminated=[], truncated=[])
    orig_sample = buf.sample

    def sample_spy(k):
        pos = {id(t): j for j, t in enumerate(buf.memory)}
        s0 = random.getstate()
        idxs.append([pos[id(t)] for t in random.sample(buf.memory, k)])
        random.setstate(s0)
        return orig_sample(k)
    buf.sample = sample_spy
    space = lambda row, m: DiscreteActionSpace(actions=[torch.tensor([int(a)]) for a in row[:m]])  # noqa: E731
    rs = random.getstate()
    calls = 0
    for i in range(n):
        before = len(buf.memory)
        buf.push(state=torch.from_numpy(P["state"][i]), action=torch.tensor([int(P["action"][i])]), reward=float(P["reward"][i]),
                 terminated=bool(P["terminated"][i]), truncated=bool(P["truncated"][i]), curr_available_actions=full,
                 next_state=torch.from_numpy(P["next_state"][i]),
                 next_available_actions=space(P["next_ids"][i], P["next_count"][i]) if dynamic else full, max_number_actions=n_act)
        for t in list(buf.memory)[before:]:
            app["push"].append(i); app["state"].append(t.state.numpy().ravel()); app["action"].append(int(t.action.reshape(-1)[0]))
            app["reward"].append(float(t.reward)); app["next_state"].append(t.next_state.numpy().ravel())
            app["next_action"].append(int(t.next_action.reshape(-1)[0])); app["terminated"].append(bool(t.terminated))
            app["truncated"].append(bool(t.truncated))
        if i in learn_after:
            if calls and new_lr is not None:
                pl._optimizer.param_groups[0]["lr"] = new_lr
            call_lr.append(pl._optimizer.param_groups[0]["lr"])
            call_batch.append(min(batch, len(buf)))
            losses += [float(x) for x in agent.learn().get("loss", [])]
            assert len(buf) == 0
            q_calls.append(flat_params(pl._Q)); qt_calls.append(flat_params(pl._Q_target))
            calls += 1
    for _ in range(learn_batch_calls):
        call_lr.append(pl._optimizer.param_groups[0]["lr"])
        call_batch.append(batch)
        losses.append(float(agent.learn_batch(buf.sample(batch))["loss"]))
        q_calls.append(flat_params(pl._Q)); qt_calls.append(flat_params(pl._Q_target))
    if learn_batch_calls:
        assert pl._training_steps == 0
    params = list(pl._Q.parameters())
    st = pl._optimizer.state
    adam = {k: np.concatenate([st[p][k].numpy().ravel() for p in params]) for k in ("exp_avg", "exp_avg_sq", "max_exp_avg_sq")}
    vmax = adam.pop("max_exp_avg_sq")
    differs = np.flatnonzero(vmax != adam["exp_avg_sq"]).astype(np.int32)
    adam.update(max_exp_avg_sq_idx=differs, max_exp_avg_sq_val=vmax[differs])
    out = dict(seed=seed, obs=obs, n_actions=n_act, hidden=np.asarray(hidden), batch=batch, rounds=rounds, capacity=capacity,
               learn_batch=bool(learn_batch_calls), lr=lr, call_lr=np.asarray(call_lr), call_batch=np.asarray(call_batch, np.int32),
               target_update_freq=freq, tau=tau, gamma=gamma, dynamic=dynamic, learn_after=np.asarray(learn_after, np.int32),
               push_state=P["state"], push_action=P["action"].astype(np.int32), push_reward=P["reward"].astype(np.float32),
               push_next_state=P["next_state"], push_terminated=P["terminated"], push_truncated=P["truncated"],
               push_next_ids=P["next_ids"].astype(np.uint8), push_next_count=P["next_count"].astype(np.int32),
               **{f"app_{k}": np.asarray(v, dtype=np.float32 if k in ("reward", "state", "next_state") else None)
                  for k, v in app.items()},
               rng_before=state_words(rs), rng_after=state_words(random.getstate()),
               idx=np.asarray([j for r in idxs for j in r], dtype=np.int32), idx_len=np.asarray([len(r) for r in idxs], np.int32),
               loss=np.asarray(losses), init_q=init, q_calls=np.stack(q_calls), qt_calls=np.stack(qt_calls),
               adam_step=float(st[params[0]]["step"]) if params[0] in st else 0.0, **{f"adam_{k}": v for k, v in adam.items()})
    path = os.path.join(GOLDEN, f"{name}.npz")
    np.savez_compressed(path, **out)
    print(f"{name}.npz: {os.path.getsize(path) // 1024} KB, {n} pushes, {len(app['push'])} appended, {calls or learn_batch_calls} "
          f"calls, {len(losses)} rounds, loss", losses[:3])
    return out


if __name__ == "__main__":
    o = gen("sarsa_method", obs=4, n_act=2, hidden=(64, 64), batch=32, rounds=1, seed=71, data_seed=701, freq=3,
            lengths=[40, 25, 50, 12, 33, 45], ends=["t", "u", "t", "t", "u", "t"])
    assert o["app_truncated"].any() and o["app_terminated"].any()
    o = gen("sarsa_steps", obs=5, n_act=4, hidden=(32, 32), batch=8, rounds=2, seed=72, data_seed=702, freq=2, dynamic=True,
            lengths=[4, 3, 5, 1, 4], ends=["t", "u", "t", "t", "u"], stale_reset=(1, 3), learn_every="step")
    pushes = o["app_push"]
    assert len(pushes) > len(set(pushes.tolist())) or len(pushes) > len(o["push_action"]), "no stale-cache append"
    gen("sarsa_lr", obs=6, n_act=3, hidden=(32, 32), batch=16, rounds=3, seed=73, data_seed=703, freq=4, new_lr=3e-3,
        lengths=[30, 28], ends=["t", "u"])
    gen("sarsa_batch", obs=6, n_act=5, hidden=(32, 32), batch=16, rounds=1, seed=74, data_seed=704, freq=1,
        lengths=[60, 70, 50], ends=["t", "u", "t"], learn_every="none", learn_batch_calls=3)
