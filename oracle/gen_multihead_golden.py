#!/usr/bin/env python
"""Record tests/golden/mh_*.npz by RUNNING THE REFERENCE's DeepQLearning / DoubleDQN with a VanillaQValueMultiHeadNetwork,
plain or conservative, under PearlAgent with a BasicReplayBuffer (TEST INFRASTRUCTURE; same set-up and stubs as
oracle/gen_golden.py, which provides the import path).

    PYTHONDONTWRITEBYTECODE=1 python oracle/gen_multihead_golden.py

Cases:
  mh_dqn       DeepQLearning with the network of Pearl's multi-head integration test passed as network_instance (obs 4,
               2 actions, [64, 64]), batch 32, terminal rows, target_update_freq 3, two learn() calls: the target update
               fires inside a call and across the boundary
  mh_ddqn      DoubleDQN (network_type=VanillaQValueMultiHeadNetwork), 6 actions, dynamic next-action sets
  mh_cql_dqn   conservative DeepQLearning at CDQN_method's shape (obs 4, 2 actions, [64, 64], batch 32), alpha 2
  mh_cql_ddqn  conservative DoubleDQN, 6 actions, dynamic next-action sets, alpha 8
  mh_lr        two learn() calls; the learning rate changes in between
  mh_batch     three agent.learn_batch() calls, conservative DoubleDQN, on sampled batches whose rows have PARTIAL current
               action sets (padded with action id 0); target_update_freq 1, since agent.learn_batch leaves the
               training-step count at 0
  mh_act       act(exploit=True) over partial available action sets, and the Q values act() ranks
learn() cases push the full current action set: B200ReplayBuffer stores none and samples the full set.
Recorded: the transitions (current sets as ids padded with 0 and counts), the sampled logical indices of every round,
CPython's `random` state before and after, per-round losses, the initial online net (the target is its deepcopy), the
online and target nets after every call, and the AdamW state (max_exp_avg_sq where it differs from exp_avg_sq).
The generator asserts, per round: DoubleDQN's best available online next value beats the second best by more than 1e-3;
masked next slots occur in the dynamic cases; the slot values of get_q_values equal the head columns of the ids the
slots hold, bit for bit; when conservative with A > 2, the reference's data term mean(Q_all.gather(1, one_hot)) differs
from the taken-action mean by more than 1e-3 (it reads slot columns 0 and 1); and, in mh_batch, that some row's current
slots repeat an id (padding), whose CQL gradients the reference adds on one head column: the recorded gradient of the
head outputs at such a column equals the sum over its slots.
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
from pearl.neural_networks.sequential_decision_making.q_value_networks import VanillaQValueMultiHeadNetwork  # noqa: E402
from pearl.pearl_agent import PearlAgent  # noqa: E402
from pearl.policy_learners.sequential_decision_making.deep_q_learning import DeepQLearning  # noqa: E402
from pearl.policy_learners.sequential_decision_making.double_dqn import DoubleDQN  # noqa: E402
from pearl.replay_buffers.basic_replay_buffer import BasicReplayBuffer  # noqa: E402
from pearl.utils.functional_utils.learning.loss_fn_utils import compute_cql_loss  # noqa: E402
from pearl.utils.instantiations.spaces.discrete_action import DiscreteActionSpace  # noqa: E402

MARGIN = 1e-3


def _round_checks(pl, batch, double, dynamic, stats):
    B, A = batch.state.shape[0], batch.action.shape[-1]
    with torch.no_grad():
        mask = batch.next_unavailable_actions_mask
        head = pl._Q(batch.next_state)
        slots = pl._Q.get_q_values(batch.next_state, batch.next_available_actions).view(B, -1)
        ids = batch.next_available_actions.argmax(-1)
        assert torch.equal(slots, head.gather(1, ids)), "a slot value differs from the head column of its id"
        if double:
            v = slots.clone()
            v[mask] = -float("inf")
            top = torch.topk(v, 2, dim=-1).values
            two = (~mask).sum(-1) >= 2
            assert bool((top[two, 0] - top[two, 1] > MARGIN).all()), \
                f"greedy margin below {MARGIN}: {(top[two, 0] - top[two, 1]).min()}"
        if dynamic:
            assert bool(mask.any()), "no masked next slot in the round"
    if not pl._is_conservative:
        return
    with torch.no_grad():
        q_all = pl._Q.get_q_values(batch.state, batch.curr_available_actions).view(B, -1)
        data_term = float(q_all.gather(1, batch.action.long()).mean())
        taken = float(pl._Q.get_q_values(batch.state, batch.action).mean())
    if A > 2:
        assert abs(data_term - taken) > MARGIN, f"data term {data_term} within {MARGIN} of the taken-action term {taken}"
    stats["term_gap"] = max(stats["term_gap"], abs(data_term - taken))
    cids = batch.curr_available_actions.argmax(-1)
    dup = [(b, int(j)) for b in range(B) for j in torch.unique(cids[b]) if int((cids[b] == j).sum()) > 1]
    stats["dup"] += len(dup)
    if dup:
        # the reference's CQL gradient at the head outputs: slots holding one id add on that id's column
        out = pl._Q(batch.state).detach().requires_grad_(True)
        q_slots = torch.bmm(batch.curr_available_actions, out.unsqueeze(-1)).squeeze(-1)
        g_slots = torch.autograd.grad(torch.logsumexp(q_slots, -1).mean() - q_slots.gather(1, batch.action.long()).mean(), q_slots,
                                      retain_graph=True)[0]
        g_head = torch.autograd.grad(torch.logsumexp(q_slots, -1).mean() - q_slots.gather(1, batch.action.long()).mean(), out)[0]
        for b, j in dup:
            assert torch.allclose(g_head[b, j], g_slots[b][cids[b] == j].sum(), rtol=1e-6, atol=1e-9)
        assert float(compute_cql_loss(pl._Q, batch, B).detach()) == float(torch.logsumexp(q_all, -1).mean() - q_all.gather(1, batch.action.long()).mean())


def _learner(obs, n_act, hidden, double, lr, gamma, rounds, batch, freq, tau, instance, alpha):
    full = DiscreteActionSpace(actions=list(torch.arange(n_act).view(-1, 1)))
    cls = DoubleDQN if double else DeepQLearning
    net = dict(network_instance=VanillaQValueMultiHeadNetwork(state_dim=obs, action_dim=n_act, hidden_dims=list(hidden),
                                                              output_dim=n_act)) \
        if instance else dict(network_type=VanillaQValueMultiHeadNetwork)
    cons = dict(is_conservative=True, conservative_alpha=alpha) if alpha is not None else {}
    return full, cls(state_dim=obs, action_space=full, hidden_dims=list(hidden), learning_rate=lr, discount_factor=gamma,
                     training_rounds=rounds, batch_size=batch, target_update_freq=freq, soft_update_tau=tau,
                     action_representation_module=OneHotActionTensorRepresentationModule(n_act), **net, **cons)


def gen_mh_golden(name, *, obs, n_act, hidden, n, batch, rounds, seed, data_seed, double=False, dynamic=False, alpha=None,
                  partial_curr=False, p_term=0.1, lr=1e-3, new_lr=None, calls=1, freq=10, tau=0.1, gamma=0.99,
                  learn_batch_calls=0, instance=False):
    torch.manual_seed(seed)
    random.seed(seed)
    torch.set_num_threads(1)
    full, pl = _learner(obs, n_act, hidden, double, lr, gamma, rounds, batch, freq, tau, instance, alpha)
    assert isinstance(pl._Q, VanillaQValueMultiHeadNetwork)
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
    stats = {"term_gap": 0.0, "dup": 0}
    orig_sample, orig_learn_batch = buf.sample, pl.learn_batch

    def sample_spy(k):
        pos = {id(t): j for j, t in enumerate(buf.memory)}
        s0 = random.getstate()
        idxs.append([pos[id(t)] for t in random.sample(buf.memory, k)])
        random.setstate(s0)
        return orig_sample(k)

    def learn_batch_spy(b):
        _round_checks(pl, b, double, dynamic, stats)
        return orig_learn_batch(b)
    buf.sample = sample_spy
    pl.learn_batch = learn_batch_spy
    rs = random.getstate()
    losses, call_lr, q_calls, qt_calls = [], [], [], []
    for c in range(learn_batch_calls or calls):
        if c and new_lr is not None:
            pl._optimizer.param_groups[0]["lr"] = new_lr
        call_lr.append(pl._optimizer.param_groups[0]["lr"])
        if learn_batch_calls:
            losses.append(float(agent.learn_batch(buf.sample(batch))["loss"]))
        else:
            losses += [float(x) for x in agent.learn()["loss"]]
        q_calls.append(flat_params(pl._Q))
        qt_calls.append(flat_params(pl._Q_target))
    if learn_batch_calls:
        assert pl._training_steps == 0
    if partial_curr:
        assert stats["dup"] > 0, "no current set with a repeated (padded) id was sampled"
    params = list(pl._Q.parameters())
    st = pl._optimizer.state
    adam = {k: np.concatenate([st[p][k].numpy().ravel() for p in params]) for k in ("exp_avg", "exp_avg_sq", "max_exp_avg_sq")}
    vmax = adam.pop("max_exp_avg_sq")
    differs = np.flatnonzero(vmax != adam["exp_avg_sq"]).astype(np.int32)
    adam.update(max_exp_avg_sq_idx=differs, max_exp_avg_sq_val=vmax[differs])
    out = dict(seed=seed, obs=obs, n_actions=n_act, hidden=np.asarray(hidden), n=n, batch=batch, rounds=rounds, double=double,
               calls=learn_batch_calls or calls, learn_batch=bool(learn_batch_calls), conservative=alpha is not None,
               alpha=0.0 if alpha is None else alpha, lr=lr, call_lr=np.asarray(call_lr), target_update_freq=freq, tau=tau,
               gamma=gamma, dynamic=dynamic, partial_curr=partial_curr, state=data["state"], next_state=data["next_state"],
               reward=data["reward"], action=data["action"].astype(np.int32), terminated=data["terminated"],
               next_ids=ids.astype(np.uint8), next_count=cnt.astype(np.int32), curr_ids=curr_ids.astype(np.uint8),
               curr_count=curr_cnt.astype(np.int32), rng_before=state_words(rs), rng_after=state_words(random.getstate()),
               idx=np.asarray(idxs, dtype=np.int32), loss=np.asarray(losses), init_q=init, q_calls=np.stack(q_calls),
               qt_calls=np.stack(qt_calls), adam_step=float(st[params[0]]["step"]), term_gap=stats["term_gap"], dup=stats["dup"],
               **{f"adam_{k}": v for k, v in adam.items()})
    path = os.path.join(GOLDEN, f"{name}.npz")
    np.savez_compressed(path, **out)
    print(f"{name}.npz: {os.path.getsize(path) // 1024} KB, loss", losses[:3], "term gap", stats["term_gap"], "dup", stats["dup"])


def gen_mh_act(name, *, obs, n_act, hidden, n, seed, data_seed):
    """act(exploit=True) over partial available sets, and the Q values of the available ids act() ranks."""
    torch.manual_seed(seed)
    random.seed(seed)
    torch.set_num_threads(1)
    _, pl = _learner(obs, n_act, hidden, False, 1e-3, 0.99, 1, 1, 10, 0.1, False, None)
    init = flat_params(pl._Q)
    data = make_transitions(n, obs, n_act, seed=data_seed, dynamic=True)
    ids, cnt = data["next_avail_ids"].astype(np.int64), data["next_avail_n"]
    assert (cnt < n_act).any()
    chosen, values = [], np.zeros((n, n_act), np.float32)
    allq = pl._Q(torch.from_numpy(data["state"])).detach()
    differs = 0
    for i in range(n):
        m = int(cnt[i])
        space = DiscreteActionSpace(actions=[torch.tensor([int(a)]) for a in ids[i, :m]])
        s = torch.from_numpy(data["state"][i])
        chosen.append(int(pl.act(s, space, exploit=True)))
        with torch.no_grad():
            q = pl._Q.get_q_values(s.unsqueeze(0), pl.action_representation_module(space.actions_batch).unsqueeze(0))[0]
        values[i, :m] = q.numpy()
        differs += int(chosen[-1] != int(allq[i].argmax()))
    assert differs > 0, "the available-set argmax equals the all-action argmax in every row"
    out = dict(seed=seed, obs=obs, n_actions=n_act, hidden=np.asarray(hidden), n=n, init_q=init, state=data["state"],
               avail_ids=ids.astype(np.uint8), avail_count=cnt.astype(np.int32), chosen=np.asarray(chosen, dtype=np.int32),
               values=values, differs=differs)
    path = os.path.join(GOLDEN, f"{name}.npz")
    np.savez_compressed(path, **out)
    print(f"{name}.npz: {os.path.getsize(path) // 1024} KB, rows whose available argmax differs", differs)


def gen_first_passing(name, seed, **kw):
    """Random networks put some rows' two best slots within the margin: try seed, seed + 1000, ... until every round
    passes the checks."""
    for k in range(300):
        try:
            return gen_mh_golden(name, seed=seed + 1000 * k, **kw)
        except AssertionError as e:
            print(f"{name}: seed {seed + 1000 * k} rejected ({e})")
    raise RuntimeError(f"{name}: no seed passed the checks")


if __name__ == "__main__":
    gen_first_passing("mh_dqn", 111, obs=4, n_act=2, hidden=(64, 64), n=300, batch=32, rounds=5, calls=2, freq=3,
                      data_seed=1101, p_term=0.15, instance=True)
    gen_first_passing("mh_ddqn", 112, obs=6, n_act=6, hidden=(32, 32), n=300, batch=16, rounds=3, data_seed=1102, double=True,
                      dynamic=True, freq=2)
    gen_first_passing("mh_cql_dqn", 113, obs=4, n_act=2, hidden=(64, 64), n=300, batch=32, rounds=5, calls=2, freq=3, alpha=2.0,
                      data_seed=1103, p_term=0.15)
    gen_first_passing("mh_cql_ddqn", 114, obs=6, n_act=6, hidden=(32, 32), n=300, batch=16, rounds=3, data_seed=1104, alpha=8.0,
                      double=True, dynamic=True, freq=2)
    gen_first_passing("mh_lr", 115, obs=5, n_act=3, hidden=(32, 32), n=200, batch=24, rounds=3, calls=2, data_seed=1105,
                      new_lr=3e-3, freq=4)
    gen_first_passing("mh_batch", 116, obs=6, n_act=5, hidden=(32, 32), n=240, batch=16, rounds=5, data_seed=1106, alpha=4.0,
                      double=True, dynamic=True, partial_curr=True, freq=1, learn_batch_calls=3)
    gen_mh_act("mh_act", obs=5, n_act=6, hidden=(32, 32), n=40, seed=117, data_seed=1107)
