#!/usr/bin/env python
"""Record tests/golden/cql_*.npz by RUNNING THE REFERENCE's DeepQLearning / DoubleDQN with is_conservative=True under
PearlAgent with a BasicReplayBuffer (TEST INFRASTRUCTURE; same set-up and stubs as oracle/gen_golden.py, which provides
the import path).

    PYTHONDONTWRITEBYTECODE=1 python oracle/gen_cql_golden.py

Four cases:
  cql_dqn    DeepQLearning at CDQN_method's shape (obs 4, 2 actions, [64, 64], batch 32, alpha 2), terminal rows,
             target_update_freq 3, two learn() calls: the target update fires inside a call and across the boundary
  cql_ddqn   DoubleDQN, 6 actions, dynamic next-action sets, alpha 8
  cql_lr     two learn() calls; the learning rate and alpha both change in between
  cql_batch  three agent.learn_batch() calls on sampled batches whose rows have PARTIAL current action sets (padded with
             action id 0, which the reference's CQL term counts); target_update_freq 1, since agent.learn_batch leaves
             the training-step count at 0
learn() cases push the full current action set: B200ReplayBuffer stores none and samples the full set.
Recorded: the transitions (current sets as ids padded with 0 and counts), the sampled logical indices of every round,
CPython's `random` state before and after, per-round losses, the initial online net (the target is its deepcopy), the
online and target nets after every call, and the AdamW state (max_exp_avg_sq where it differs from exp_avg_sq).
The generator asserts, per round: DoubleDQN's best available online next value beats the second best by more than 1e-3;
for A > 2, the reference's data term mean(Q_all.gather(1, one_hot)) differs from the taken-action mean Q(s, a) by more
than 1e-3 (the recording tells the two apart); and, in cql_batch, that padded current slots occur.
"""
from __future__ import annotations

import os
import random
import sys

import numpy as np

sys.dont_write_bytecode = True
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from oracle.gen_golden import GOLDEN, flat_params, state_words  # noqa: E402  (sets up the reference import path and stubs)
from oracle.synth import make_transitions  # noqa: E402

import torch  # noqa: E402
from pearl.action_representation_modules.one_hot_action_representation_module import (  # noqa: E402
    OneHotActionTensorRepresentationModule,
)
from pearl.pearl_agent import PearlAgent  # noqa: E402
from pearl.policy_learners.sequential_decision_making.deep_q_learning import DeepQLearning  # noqa: E402
from pearl.policy_learners.sequential_decision_making.double_dqn import DoubleDQN  # noqa: E402
from pearl.replay_buffers.basic_replay_buffer import BasicReplayBuffer  # noqa: E402
from pearl.utils.instantiations.spaces.discrete_action import DiscreteActionSpace  # noqa: E402

MARGIN = 1e-3


def _round_checks(pl, batch, double, stats):
    with torch.no_grad():
        B, A = batch.state.shape[0], batch.action.shape[-1]
        if double:
            v = pl._Q.get_q_values(batch.next_state, batch.next_available_actions).view(B, -1)
            v[batch.next_unavailable_actions_mask] = -float("inf")
            top = torch.topk(v, 2, dim=-1).values
            two = (~batch.next_unavailable_actions_mask).sum(-1) >= 2
            assert bool((top[two, 0] - top[two, 1] > MARGIN).all()), \
                f"greedy margin below {MARGIN}: {(top[two, 0] - top[two, 1]).min()}"
        q_all = pl._Q.get_q_values(batch.state, batch.curr_available_actions).view(B, -1)
        data_term = float(q_all.gather(1, batch.action.long()).mean())
        taken = float(pl._Q.get_q_values(batch.state, batch.action).mean())
        if A > 2:
            assert abs(data_term - taken) > MARGIN, f"data term {data_term} within {MARGIN} of the taken-action term {taken}"
        stats["term_gap"] = max(stats["term_gap"], abs(data_term - taken))
        stats["padded"] += int(batch.curr_unavailable_actions_mask.sum())


def gen_cql_golden(name, *, obs, n_act, hidden, n, batch, rounds, seed, data_seed, alpha, double=False, dynamic=False,
                   partial_curr=False, p_term=0.1, lr=1e-3, new_lr=None, new_alpha=None, calls=1, freq=10, tau=0.1, gamma=0.99,
                   learn_batch_calls=0):
    torch.manual_seed(seed)
    random.seed(seed)
    torch.set_num_threads(1)
    full = DiscreteActionSpace(actions=list(torch.arange(n_act).view(-1, 1)))
    cls = DoubleDQN if double else DeepQLearning
    pl = cls(state_dim=obs, action_space=full, hidden_dims=list(hidden), learning_rate=lr, discount_factor=gamma,
             training_rounds=rounds, batch_size=batch, target_update_freq=freq, soft_update_tau=tau, is_conservative=True,
             conservative_alpha=alpha, action_representation_module=OneHotActionTensorRepresentationModule(n_act))
    buf = BasicReplayBuffer(n)
    agent = PearlAgent(policy_learner=pl, replay_buffer=buf, device_id=-1)
    data = make_transitions(n, obs, n_act, seed=data_seed, dynamic=dynamic, p_term=p_term)
    ids = data.get("next_avail_ids", np.tile(np.arange(n_act), (n, 1)))
    cnt = data.get("next_avail_n", np.full(n, n_act))
    curr_ids, curr_cnt = np.tile(np.arange(n_act), (n, 1)), np.full(n, n_act)
    if partial_curr:
        rng = np.random.Generator(np.random.PCG64(data_seed + 1))
        curr_ids = np.zeros((n, n_act), np.int64)
        for i in range(n):
            m = int(rng.integers(1, n_act + 1))
            curr_ids[i, :m] = np.sort(rng.choice(n_act, size=m, replace=False))
            curr_cnt[i] = m
    space = lambda row, m: DiscreteActionSpace(actions=[torch.tensor([int(a)]) for a in row[:m]])  # noqa: E731
    for i in range(n):
        buf.push(state=torch.from_numpy(data["state"][i]), action=torch.tensor(int(data["action"][i])),
                 reward=float(data["reward"][i]), terminated=bool(data["terminated"][i]), truncated=False,
                 curr_available_actions=space(curr_ids[i], curr_cnt[i]) if partial_curr else full,
                 next_state=torch.from_numpy(data["next_state"][i]),
                 next_available_actions=space(ids[i], cnt[i]) if dynamic else full, max_number_actions=n_act)
    init = flat_params(pl._Q)
    assert np.array_equal(init, flat_params(pl._Q_target))
    idxs = []
    stats = {"term_gap": 0.0, "padded": 0}
    orig_sample, orig_learn_batch = buf.sample, pl.learn_batch

    def sample_spy(k):
        pos = {id(t): j for j, t in enumerate(buf.memory)}
        s0 = random.getstate()
        idxs.append([pos[id(t)] for t in random.sample(buf.memory, k)])
        random.setstate(s0)
        return orig_sample(k)

    def learn_batch_spy(b):
        _round_checks(pl, b, double, stats)
        return orig_learn_batch(b)
    buf.sample = sample_spy
    pl.learn_batch = learn_batch_spy
    rs = random.getstate()
    losses, call_lr, call_alpha, q_calls, qt_calls = [], [], [], [], []
    for c in range(learn_batch_calls or calls):
        if c and new_lr is not None:
            pl._optimizer.param_groups[0]["lr"] = new_lr
        if c and new_alpha is not None:
            pl._conservative_alpha = new_alpha
        call_lr.append(pl._optimizer.param_groups[0]["lr"])
        call_alpha.append(pl._conservative_alpha)
        if learn_batch_calls:
            losses.append(float(agent.learn_batch(buf.sample(batch))["loss"]))
        else:
            losses += [float(x) for x in agent.learn()["loss"]]
        q_calls.append(flat_params(pl._Q))
        qt_calls.append(flat_params(pl._Q_target))
    if learn_batch_calls:
        assert pl._training_steps == 0
    if partial_curr:
        assert stats["padded"] > 0, "no padded current slot was sampled"
    params = list(pl._Q.parameters())
    st = pl._optimizer.state
    adam = {k: np.concatenate([st[p][k].numpy().ravel() for p in params]) for k in ("exp_avg", "exp_avg_sq", "max_exp_avg_sq")}
    vmax = adam.pop("max_exp_avg_sq")
    differs = np.flatnonzero(vmax != adam["exp_avg_sq"]).astype(np.int32)
    adam.update(max_exp_avg_sq_idx=differs, max_exp_avg_sq_val=vmax[differs])
    out = dict(seed=seed, obs=obs, n_actions=n_act, hidden=np.asarray(hidden), n=n, batch=batch, rounds=rounds, double=double,
               calls=learn_batch_calls or calls, learn_batch=bool(learn_batch_calls), alpha=alpha, call_alpha=np.asarray(call_alpha),
               lr=lr, call_lr=np.asarray(call_lr), target_update_freq=freq, tau=tau, gamma=gamma, dynamic=dynamic,
               partial_curr=partial_curr, state=data["state"], next_state=data["next_state"], reward=data["reward"],
               action=data["action"].astype(np.int32), terminated=data["terminated"], next_ids=ids.astype(np.uint8),
               next_count=cnt.astype(np.int32), curr_ids=curr_ids.astype(np.uint8), curr_count=curr_cnt.astype(np.int32),
               rng_before=state_words(rs), rng_after=state_words(random.getstate()), idx=np.asarray(idxs, dtype=np.int32),
               loss=np.asarray(losses), init_q=init, q_calls=np.stack(q_calls), qt_calls=np.stack(qt_calls),
               adam_step=float(st[params[0]]["step"]), term_gap=stats["term_gap"], padded=stats["padded"],
               **{f"adam_{k}": v for k, v in adam.items()})
    path = os.path.join(GOLDEN, f"{name}.npz")
    np.savez_compressed(path, **out)
    print(f"{name}.npz: {os.path.getsize(path) // 1024} KB, loss", losses[:3], "term gap", stats["term_gap"], "padded", stats["padded"])


def gen_first_passing(name, seed, **kw):
    """Random networks put some rows' two best slots within the margin: try seed, seed + 1000, ... until every round
    passes the checks."""
    for k in range(300):
        try:
            return gen_cql_golden(name, seed=seed + 1000 * k, **kw)
        except AssertionError as e:
            print(f"{name}: seed {seed + 1000 * k} rejected ({e})")
    raise RuntimeError(f"{name}: no seed passed the checks")


if __name__ == "__main__":
    gen_first_passing("cql_dqn", 91, obs=4, n_act=2, hidden=(64, 64), n=300, batch=32, rounds=5, calls=2, freq=3, alpha=2.0,
                      data_seed=901, p_term=0.15)
    gen_first_passing("cql_ddqn", 92, obs=6, n_act=6, hidden=(32, 32), n=300, batch=16, rounds=3, data_seed=902, alpha=8.0,
                      double=True, dynamic=True, freq=2)
    gen_first_passing("cql_lr", 93, obs=5, n_act=3, hidden=(32, 32), n=200, batch=24, rounds=3, calls=2, data_seed=903, alpha=2.0,
                      new_lr=3e-3, new_alpha=0.5, freq=4)
    gen_first_passing("cql_batch", 94, obs=6, n_act=5, hidden=(32, 32), n=240, batch=16, rounds=5, data_seed=904, alpha=4.0,
                      double=True, dynamic=True, partial_curr=True, freq=1, learn_batch_calls=3)
