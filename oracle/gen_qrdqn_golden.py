#!/usr/bin/env python
"""Record tests/golden/qrdqn_*.npz by RUNNING THE REFERENCE's QuantileRegressionDeepQLearning under PearlAgent with a
BasicReplayBuffer (TEST INFRASTRUCTURE; same set-up and stubs as oracle/gen_golden.py, which provides the import path).

    PYTHONDONTWRITEBYTECODE=1 python oracle/gen_qrdqn_golden.py

Four cases:
  qrdqn_neutral   the default RiskNeutralSafetyModule at QRDQN_method's shape (obs 4, 2 actions, [64, 64], batch 32,
                  N = 10), terminal rows, target_update_freq 3, two learn() calls: the target update fires inside a call
                  and across the boundary
  qrdqn_variance  QuantileNetworkMeanVarianceSafetyModule(2.0), N = 32, 6 actions, dynamic next-action sets (masked
                  slots); asserts that beta changes the greedy slot on some rows
  qrdqn_lr        two learn() calls; the learning rate changes in between
  qrdqn_batch     three agent.learn_batch() calls on sampled batches (target_update_freq 1: agent.learn_batch leaves the
                  training-step count at 0, so the update fires on every call)
Recorded: the transitions, the sampled logical indices of every round (0 = oldest element of the deque), CPython's
`random` state before and after, per-round losses, the initial online net (the target is its deepcopy), the online and
target nets after every call (the last row is the final state), and the AdamW state (max_exp_avg_sq as the elements where
it differs from exp_avg_sq).  For every round the generator asserts that both Huber branches occur and that the best unmasked risk value beats the second best by more than 1e-3, so
an fp32 summation-order difference cannot flip a greedy slot in the tests.
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
from pearl.policy_learners.sequential_decision_making.quantile_regression_deep_q_learning import (  # noqa: E402
    QuantileRegressionDeepQLearning,
)
from pearl.replay_buffers.basic_replay_buffer import BasicReplayBuffer  # noqa: E402
from pearl.safety_modules.risk_sensitive_safety_modules import QuantileNetworkMeanVarianceSafetyModule  # noqa: E402
from pearl.utils.instantiations.spaces.discrete_action import DiscreteActionSpace  # noqa: E402

MARGIN = 1e-3


def _round_checks(pl, batch, beta, stats):
    """Both Huber branches, the greedy-slot margin, and (beta > 0) whether beta changed the greedy slot of some rows."""
    with torch.no_grad():
        qn = pl._Q_target.get_q_value_distribution(batch.next_state, batch.next_available_actions)       # [B, A, N]
        N = qn.shape[-1]
        w = (pl._Q_target.quantiles[1:] - pl._Q_target.quantiles[:-1])
        mean = qn.mean(dim=-1, keepdim=True)
        rho = (mean - beta * (w * torch.square(qn - mean)).sum(dim=-1, keepdim=True)).squeeze(-1)
        mask = batch.next_unavailable_actions_mask
        rho[mask] = -float("inf")
        top = torch.topk(rho, 2, dim=-1).values
        two = (~mask).sum(-1) >= 2
        assert bool((top[two, 0] - top[two, 1] > MARGIN).all()), f"greedy margin below {MARGIN}: {(top[two, 0] - top[two, 1]).min()}"
        g = rho.argmax(-1)
        if beta:
            m0 = mean.squeeze(-1).clone()
            m0[mask] = -float("inf")
            stats["flipped"] += int((m0.argmax(-1) != g).sum())
        T = torch.gather(qn, 1, g.view(-1, 1, 1).expand(-1, 1, N)).view(-1, N) * pl._discount_factor * \
            (1 - batch.terminated.float()).unsqueeze(-1) + batch.reward.unsqueeze(-1)
        theta = pl._Q.get_q_value_distribution(batch.state, batch.action)
        u = (T.unsqueeze(2) - theta.unsqueeze(1)).abs()
        assert bool((u <= 1).any()) and bool((u > 1).any()), "one Huber branch does not occur"


def gen_qrdqn_golden(name, *, obs, n_act, hidden, N, n, batch, rounds, seed, data_seed, beta=None, dynamic=False, p_term=0.1,
                     lr=5e-4, new_lr=None, calls=1, freq=10, tau=0.05, gamma=0.99, learn_batch_calls=0):
    torch.manual_seed(seed)
    random.seed(seed)
    torch.set_num_threads(1)
    full = DiscreteActionSpace(actions=list(torch.arange(n_act).view(-1, 1)))
    pl = QuantileRegressionDeepQLearning(state_dim=obs, action_space=full, hidden_dims=list(hidden), num_quantiles=N, learning_rate=lr,
                                         discount_factor=gamma, training_rounds=rounds, batch_size=batch, target_update_freq=freq,
                                         soft_update_tau=tau, action_representation_module=OneHotActionTensorRepresentationModule(n_act))
    buf = BasicReplayBuffer(n)
    safety = QuantileNetworkMeanVarianceSafetyModule(beta) if beta is not None else None
    agent = PearlAgent(policy_learner=pl, replay_buffer=buf, device_id=-1, safety_module=safety)
    data = make_transitions(n, obs, n_act, seed=data_seed, dynamic=dynamic, p_term=p_term)
    ids = data.get("next_avail_ids", np.tile(np.arange(n_act), (n, 1)))
    cnt = data.get("next_avail_n", np.full(n, n_act))
    for i in range(n):
        nxt = DiscreteActionSpace(actions=[torch.tensor([int(a)]) for a in ids[i, :cnt[i]]]) if dynamic else full
        buf.push(state=torch.from_numpy(data["state"][i]), action=torch.tensor(int(data["action"][i])),
                 reward=float(data["reward"][i]), terminated=bool(data["terminated"][i]), truncated=False,
                 curr_available_actions=full, next_state=torch.from_numpy(data["next_state"][i]), next_available_actions=nxt,
                 max_number_actions=n_act)
    init = flat_params(pl._Q)
    assert np.array_equal(init, flat_params(pl._Q_target))
    idxs = []
    stats = {"flipped": 0}
    orig_sample, orig_learn_batch = buf.sample, pl.learn_batch

    def sample_spy(k):
        pos = {id(t): j for j, t in enumerate(buf.memory)}
        s0 = random.getstate()
        idxs.append([pos[id(t)] for t in random.sample(buf.memory, k)])
        random.setstate(s0)
        return orig_sample(k)

    def learn_batch_spy(b):
        _round_checks(pl, b, beta or 0.0, stats)
        return orig_learn_batch(b)
    buf.sample = sample_spy
    pl.learn_batch = learn_batch_spy
    rs = random.getstate()
    losses, call_lr, q_calls, qt_calls = [], [], [], []
    if learn_batch_calls:
        for _ in range(learn_batch_calls):
            call_lr.append(pl._optimizer.param_groups[0]["lr"])
            losses.append(float(agent.learn_batch(buf.sample(batch))["loss"]))
            q_calls.append(flat_params(pl._Q))
            qt_calls.append(flat_params(pl._Q_target))
        assert pl._training_steps == 0
    else:
        for c in range(calls):
            if c and new_lr is not None:
                pl._optimizer.param_groups[0]["lr"] = new_lr
            call_lr.append(pl._optimizer.param_groups[0]["lr"])
            losses += [float(x) for x in agent.learn()["loss"]]
            q_calls.append(flat_params(pl._Q))
            qt_calls.append(flat_params(pl._Q_target))
    if beta:
        assert stats["flipped"] > 0, "beta never changed the greedy slot"
    params = list(pl._Q.parameters())
    st = pl._optimizer.state
    adam = {k: np.concatenate([st[p][k].numpy().ravel() for p in params]) for k in ("exp_avg", "exp_avg_sq", "max_exp_avg_sq")}
    # max_exp_avg_sq equals exp_avg_sq wherever the second moment never shrank: stored where it differs only (size)
    vmax = adam.pop("max_exp_avg_sq")
    differs = np.flatnonzero(vmax != adam["exp_avg_sq"]).astype(np.int32)
    adam.update(max_exp_avg_sq_idx=differs, max_exp_avg_sq_val=vmax[differs])
    out = dict(seed=seed, obs=obs, n_actions=n_act, hidden=np.asarray(hidden), num_quantiles=N, n=n, batch=batch, rounds=rounds,
               calls=learn_batch_calls or calls, learn_batch=bool(learn_batch_calls), beta=float(beta or 0.0), lr=lr,
               call_lr=np.asarray(call_lr), target_update_freq=freq, tau=tau, gamma=gamma, dynamic=dynamic,
               state=data["state"], next_state=data["next_state"], reward=data["reward"], action=data["action"].astype(np.int32),
               terminated=data["terminated"], next_ids=ids.astype(np.uint8), next_count=cnt.astype(np.int32),
               rng_before=state_words(rs), rng_after=state_words(random.getstate()), idx=np.asarray(idxs, dtype=np.int32),
               loss=np.asarray(losses), init_q=init, q_calls=np.stack(q_calls), qt_calls=np.stack(qt_calls),
               adam_step=float(st[params[0]]["step"]), flipped=stats["flipped"], **{f"adam_{k}": v for k, v in adam.items()})
    path = os.path.join(GOLDEN, f"{name}.npz")
    np.savez_compressed(path, **out)
    print(f"{name}.npz: {os.path.getsize(path) // 1024} KB, loss", losses[:3], "flipped", stats["flipped"])


def gen_first_passing(name, seed, **kw):
    """Random networks put some rows' two best slots within the margin: try seed, seed + 1000, ... until every round
    passes the checks."""
    for k in range(300):
        try:
            return gen_qrdqn_golden(name, seed=seed + 1000 * k, **kw)
        except AssertionError as e:
            print(f"{name}: seed {seed + 1000 * k} rejected ({e})")
    raise RuntimeError(f"{name}: no seed passed the checks")


if __name__ == "__main__":
    gen_first_passing("qrdqn_neutral", 81, obs=4, n_act=2, hidden=(64, 64), N=10, n=300, batch=32, rounds=5, calls=2, freq=3,
                      data_seed=801, p_term=0.15)
    gen_first_passing("qrdqn_variance", 82, obs=6, n_act=6, hidden=(32, 32), N=32, n=300, batch=16, rounds=3, data_seed=802,
                      beta=2.0, dynamic=True, freq=4)
    gen_first_passing("qrdqn_lr", 83, obs=5, n_act=2, hidden=(32, 32), N=16, n=200, batch=24, rounds=3, calls=2, data_seed=803,
                      new_lr=2e-3, freq=3)
    gen_first_passing("qrdqn_batch", 84, obs=6, n_act=3, hidden=(32, 32), N=12, n=240, batch=16, rounds=5, data_seed=804,
                      freq=1, learn_batch_calls=3)
