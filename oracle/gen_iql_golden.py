#!/usr/bin/env python
"""Record tests/golden/iql_*.npz by RUNNING THE REFERENCE's ImplicitQLearning under PearlAgent with a BasicReplayBuffer
(TEST INFRASTRUCTURE; same set-up and stubs as oracle/gen_golden.py, which provides the import path).

    PYTHONDONTWRITEBYTECODE=1 python oracle/gen_iql_golden.py

Four cases:
  iql_discrete    VanillaActorNetwork, one-hot actions, terminal transitions, advantage_clamp small enough to bind on
                  some rows
  iql_continuous  VanillaContinuousActorNetwork on an asymmetric box
  iql_lr          two learn() calls; the learning rates of all three optimizers change in between
  iql_batch       three agent.learn_batch() calls on batches sampled from the buffer (discrete)
Recorded: the transitions, the sampled logical indices of every round (0 = oldest element of the deque), the
torch.randint draws (captured by wrapping torch.randint), torch's CPU RNG state and CPython's `random` state before and
after, per-round losses, the initial and final actor / q1 / q2 / targets / value net, and the value net's AdamW state.
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
from pearl.neural_networks.sequential_decision_making.actor_networks import VanillaContinuousActorNetwork  # noqa: E402
from pearl.pearl_agent import PearlAgent  # noqa: E402
from pearl.policy_learners.sequential_decision_making.implicit_q_learning import ImplicitQLearning  # noqa: E402
from pearl.replay_buffers.basic_replay_buffer import BasicReplayBuffer  # noqa: E402
from pearl.utils.instantiations.spaces.box_action import BoxActionSpace  # noqa: E402
from pearl.utils.instantiations.spaces.discrete_action import DiscreteActionSpace  # noqa: E402


def gen_iql_golden(name, *, obs, hidden, n, batch, rounds, seed, data_seed, n_act=None, low=None, high=None, p_term=0.1,
                   lrs=(3e-4, 5e-4, 4e-4), new_lrs=None, tau=0.05, gamma=0.98, expectile=0.7, temperature=0.5, clamp=100.0,
                   learn_batch_calls=0):
    torch.manual_seed(seed)
    random.seed(seed)
    torch.set_num_threads(1)
    discrete = n_act is not None
    hp = dict(state_dim=obs, actor_hidden_dims=list(hidden), critic_hidden_dims=list(hidden), value_critic_hidden_dims=list(hidden),
              actor_learning_rate=lrs[0], critic_learning_rate=lrs[1], value_critic_learning_rate=lrs[2], critic_soft_update_tau=tau,
              discount_factor=gamma, training_rounds=rounds, batch_size=batch, expectile=expectile,
              temperature_advantage_weighted_regression=temperature, advantage_clamp=clamp)
    rng = np.random.Generator(np.random.PCG64(data_seed))
    q8 = lambda x: (np.rint(x * 256) / 256).astype(np.float32)  # noqa: E731
    st, ns, rw = q8(rng.standard_normal((n, obs))), q8(rng.standard_normal((n, obs))), q8(rng.standard_normal(n))
    term = rng.random(n) < p_term
    if discrete:
        space = DiscreteActionSpace(actions=list(torch.arange(n_act).view(-1, 1)))
        pl = ImplicitQLearning(action_space=space, action_representation_module=OneHotActionTensorRepresentationModule(n_act), **hp)
        ac = rng.integers(0, n_act, size=n).astype(np.int32)
    else:
        low, high = torch.tensor(low, dtype=torch.float32), torch.tensor(high, dtype=torch.float32)
        space = BoxActionSpace(low=low, high=high)
        pl = ImplicitQLearning(action_space=space, actor_network_type=VanillaContinuousActorNetwork, **hp)
        ac = q8(rng.uniform(low.numpy(), high.numpy(), size=(n, low.numel())))
    buf = BasicReplayBuffer(n)
    agent = PearlAgent(policy_learner=pl, replay_buffer=buf, device_id=-1)
    for i in range(n):
        action = torch.tensor(int(ac[i])) if discrete else torch.from_numpy(ac[i])
        buf.push(state=torch.from_numpy(st[i]), action=action, reward=float(rw[i]), terminated=bool(term[i]), truncated=False,
                 curr_available_actions=space, next_state=torch.from_numpy(ns[i]), next_available_actions=space,
                 max_number_actions=n_act if discrete else None)
    nets = lambda: dict(actor=flat_params(pl._actor), q1=flat_params(pl._critic._critic_1), q2=flat_params(pl._critic._critic_2),  # noqa: E731
                        q1t=flat_params(pl._critic_target._critic_1), q2t=flat_params(pl._critic_target._critic_2),
                        value=flat_params(pl._value_network))
    init = nets()
    idxs, bits = [], []
    orig_sample, orig_randint = buf.sample, torch.randint

    def sample_spy(k):
        pos = {id(t): j for j, t in enumerate(buf.memory)}
        s0 = random.getstate()
        idxs.append([pos[id(t)] for t in random.sample(buf.memory, k)])
        random.setstate(s0)
        return orig_sample(k)

    def randint_spy(*a, **k):
        x = orig_randint(*a, **k)
        bits.append(int(x.item()))
        return x
    buf.sample = sample_spy
    torch.randint = randint_spy
    rs, trs = random.getstate(), torch.get_rng_state()
    losses = {"value_loss": [], "actor_loss": [], "critic_loss": []}
    call_lrs = []
    try:
        if learn_batch_calls:
            for _ in range(learn_batch_calls):
                rep = agent.learn_batch(buf.sample(batch))
                for k in losses:
                    losses[k].append(float(rep[k]))
        else:
            for c in range(2 if new_lrs else 1):
                if c:
                    for opt, lr in zip((pl._actor_optimizer, pl._critic_optimizer, pl._value_network_optimizer), new_lrs):
                        opt.param_groups[0]["lr"] = lr
                call_lrs.append([pl._actor_optimizer.param_groups[0]["lr"], pl._critic_optimizer.param_groups[0]["lr"],
                                 pl._value_network_optimizer.param_groups[0]["lr"]])
                rep = agent.learn()
                for k in losses:
                    losses[k] += list(rep[k])
    finally:
        torch.randint = orig_randint
    calls = learn_batch_calls or len(call_lrs)
    assert len(bits) == 2 * (learn_batch_calls or rounds * calls)
    vst = pl._value_network_optimizer.state
    vparams = list(pl._value_network.parameters())
    vstate = {k: np.concatenate([vst[p][k].numpy().ravel() for p in vparams]) for k in ("exp_avg", "exp_avg_sq", "max_exp_avg_sq")}
    out = dict(obs=obs, discrete=discrete, n_actions=n_act or 0, low=np.asarray(low if low is not None else [], np.float32),
               high=np.asarray(high if high is not None else [], np.float32), hidden=np.asarray(hidden), n=n, batch=batch,
               rounds=rounds, calls=calls, learn_batch=bool(learn_batch_calls), lrs=np.asarray(lrs),
               call_lrs=np.asarray(call_lrs).reshape(-1, 3), tau=tau, gamma=gamma, expectile=expectile, temperature=temperature,
               advantage_clamp=clamp, state=st, next_state=ns, reward=rw, action=ac, terminated=term,
               rng_before=state_words(rs), rng_after=state_words(random.getstate()), torch_rng_before=trs.numpy(),
               torch_rng_after=torch.get_rng_state().numpy(), idx=np.asarray(idxs, dtype=np.int32),
               bits=np.asarray(bits, dtype=np.int32).reshape(-1, 2), value_adam_step=float(vst[vparams[0]]["step"]),
               **{k: np.asarray(v) for k, v in losses.items()}, **{f"init_{k}": v for k, v in init.items()},
               **{f"{k}_after": v for k, v in nets().items()}, **{f"value_{k}": v for k, v in vstate.items()})
    np.savez_compressed(os.path.join(GOLDEN, f"{name}.npz"), **out)
    print(f"{name}.npz:", {k: v[:2] for k, v in losses.items()}, "bits", bits[:6])


if __name__ == "__main__":
    gen_iql_golden("iql_discrete", obs=6, n_act=4, hidden=(32, 32), n=300, batch=64, rounds=6, seed=71, data_seed=701, clamp=1.05,
                   temperature=3.0)
    gen_iql_golden("iql_continuous", obs=7, low=[-0.5, -1.0, 0.25], high=[0.5, 2.0, 1.25], hidden=(32, 32), n=260, batch=48, rounds=6,
                   seed=72, data_seed=702, p_term=0.05)
    gen_iql_golden("iql_lr", obs=5, n_act=3, hidden=(32, 32), n=200, batch=48, rounds=4, seed=73, data_seed=703,
                   new_lrs=(1e-3, 2e-4, 7e-4))
    gen_iql_golden("iql_batch", obs=6, n_act=5, hidden=(32, 32), n=240, batch=40, rounds=5, seed=74, data_seed=704, learn_batch_calls=3)
