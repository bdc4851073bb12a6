#!/usr/bin/env python
"""Record tests/golden/rf_*.npz by RUNNING THE REFERENCE's REINFORCE (use_critic=True) under PearlAgent with its
REINFORCEReplayBuffer (TEST INFRASTRUCTURE; same set-up and stubs as oracle/gen_golden.py, which provides the import path).

    PYTHONDONTWRITEBYTECODE=1 python oracle/gen_reinforce_golden.py

Three cases:
  rf_method  REINFORCE_method's shape (obs 4, 2 actions, [64, 64], 8 rounds, batch 64) on a 40-transition buffer: shorter
             than the batch (the batch is clamped to the buffer), two episodes, the newest transition terminated (R has no
             bootstrap term)
  rf_multi   a 300-transition buffer of several episodes, longer than the batch, whose newest transition is NOT terminated:
             a nonzero bootstrap, one R across every episode
  rf_lr      two agent.learn() calls; the agent clears the buffer after each, new transitions are pushed and both learning
             rates change between the calls
Recorded per call: the transitions, R and its bootstrap term, the sampled logical indices of every round (0 = oldest), the
CPython `random` state before and after; per round the losses; the initial and final actor / critic parameters and both
AdamW(amsgrad) states.  The script asserts that the reference's two quirks are what it recorded: every transition holds the
same return tensor, and the first actor loss is B times the per-row form.
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
from pearl.policy_learners.sequential_decision_making.reinforce import REINFORCE, REINFORCEReplayBuffer  # noqa: E402
from pearl.utils.instantiations.spaces.discrete_action import DiscreteActionSpace  # noqa: E402


def _adam(opt, module, key):
    return np.concatenate([opt.state[p][key].detach().numpy().ravel() for p in module.parameters()])


def gen(name, *, obs, n_act, hidden, calls, batch, rounds, seed, data_seed, lrs):
    """calls: [(n, indices of terminated transitions)] per learn() call; lrs: [(actor lr, critic lr)] per call."""
    torch.manual_seed(seed)
    random.seed(seed)
    torch.set_num_threads(1)
    space = DiscreteActionSpace(actions=list(torch.arange(n_act).view(-1, 1)))
    pl = REINFORCE(state_dim=obs, action_space=space, actor_hidden_dims=list(hidden), critic_hidden_dims=list(hidden),
                   use_critic=True, actor_learning_rate=lrs[0][0], critic_learning_rate=lrs[0][1], training_rounds=rounds,
                   batch_size=batch, action_representation_module=OneHotActionTensorRepresentationModule(n_act))
    buf = REINFORCEReplayBuffer(100000)
    agent = PearlAgent(policy_learner=pl, replay_buffer=buf, device_id=-1)
    rng = np.random.Generator(np.random.PCG64(data_seed))
    q8 = lambda x: (np.rint(x * 256) / 256).astype(np.float32)  # noqa: E731
    init_actor, init_critic = flat_params(pl._actor), flat_params(pl._critic)
    out = dict(obs=obs, n_actions=n_act, hidden=np.asarray(hidden), batch=batch, rounds=rounds, calls=len(calls),
               call_n=np.asarray([c[0] for c in calls], dtype=np.int32), call_lr=np.asarray(lrs, dtype=np.float64),
               init_actor=init_actor, init_critic=init_critic)
    cols = {k: [] for k in ("state", "next_state", "reward", "action", "terminated")}
    idxs, rets, boots, al, cl, rng_before, rng_after = [], [], [], [], [], [], []
    orig_sample = buf.sample
    for c, ((n, term_at), (alr, clr)) in enumerate(zip(calls, lrs)):
        pl._actor_optimizer.param_groups[0]["lr"] = alr
        pl._critic_optimizer.param_groups[0]["lr"] = clr
        state = q8(rng.standard_normal((n + 1, obs)))
        reward = q8(rng.standard_normal(n) * 2)
        action = rng.integers(0, n_act, size=n).astype(np.int64)
        term = np.zeros(n, dtype=bool)
        term[list(term_at)] = True
        for i in range(n):
            buf.push(state=torch.from_numpy(state[i]), action=torch.tensor(int(action[i])), reward=float(reward[i]),
                     terminated=bool(term[i]), truncated=False, curr_available_actions=space,
                     next_state=torch.from_numpy(state[i + 1]), next_available_actions=space, max_number_actions=n_act)
        for k, v in (("state", state[:n]), ("next_state", state[1:]), ("reward", reward), ("action", action), ("terminated", term)):
            cols[k].append(v)
        with torch.no_grad():
            boot = (pl._critic(torch.from_numpy(state[n])).detach() * (~torch.tensor([bool(term[-1])]))).numpy().reshape(-1)
        seen = {}

        def sample_spy(k):
            if not seen:        # the agent clears the on-policy buffer after learning: look at the returns now
                ids = {id(t.cum_reward) for t in buf.memory}
                assert len(ids) == 1, "expected every transition to hold the same return tensor"
                seen["R"] = buf.memory[0].cum_reward.detach().numpy().reshape(-1).copy()
            pos = {id(t): j for j, t in enumerate(buf.memory)}
            stt = random.getstate()
            idxs.append([pos[id(t)] for t in random.sample(buf.memory, k)])
            random.setstate(stt)
            b = orig_sample(k)
            assert tuple(b.cum_reward.shape) == (k, 1), b.cum_reward.shape
            return b
        buf.sample = sample_spy
        actor0 = [p.detach().clone() for p in pl._actor.parameters()]
        critic0 = [p.detach().clone() for p in pl._critic.parameters()]
        first = len(idxs)
        rng_before.append(state_words(random.getstate()))
        rep = agent.learn()
        rng_after.append(state_words(random.getstate()))
        assert len(buf) == 0, "PearlAgent clears the on-policy buffer"
        al += list(rep["actor_loss"])
        cl += list(rep["critic_loss"])
        rets.append(seen["R"])
        boots.append(boot)
        # quirk 2: the first round's loss is B times the per-row form sum_j nlp_j (R - v_j)
        from oracle.reinforce_oracle import OracleREINFORCE
        orc = OracleREINFORCE(obs, n_act, hidden, hidden)
        with torch.no_grad():
            for p, q in zip(orc.actor.parameters(), actor0):
                p.copy_(q)
            for p, q in zip(orc.critic.parameters(), critic0):
                p.copy_(q)
            ix = np.asarray(idxs[first])
            s = torch.from_numpy(state[:n][ix])
            pa = torch.softmax(orc.actor(s), -1).gather(1, torch.from_numpy(action[ix]).view(-1, 1)).view(-1)
            per_row = float(torch.sum(-torch.log(pa + 1e-8) * (torch.from_numpy(seen["R"]) - orc.critic(s).view(-1))))
        B = len(ix)
        assert abs(rep["actor_loss"][0] - B * per_row) <= 1e-4 * abs(B * per_row) + 1e-4, (rep["actor_loss"][0], B, per_row)
        # the fold itself, from the recorded bootstrap
        cum = torch.from_numpy(boot.copy())
        for t in range(n - 1, -1, -1):
            cum += torch.tensor(reward[t])
        assert np.array_equal(cum.numpy(), seen["R"]), (cum, seen["R"])
        buf.sample = orig_sample
    out.update(state=np.concatenate(cols["state"]), next_state=np.concatenate(cols["next_state"]),
               reward=np.concatenate(cols["reward"]), action=np.concatenate(cols["action"]).astype(np.int32),
               terminated=np.concatenate(cols["terminated"]), ret=np.concatenate(rets).astype(np.float32),
               bootstrap=np.concatenate(boots).astype(np.float32), idx=np.asarray(idxs, dtype=np.int32),
               rng_before=np.stack(rng_before), rng_after=np.stack(rng_after),
               actor_loss=np.asarray(al), critic_loss=np.asarray(cl), actor_after=flat_params(pl._actor),
               critic_after=flat_params(pl._critic))
    for which, opt, net in (("actor", pl._actor_optimizer, pl._actor), ("critic", pl._critic_optimizer, pl._critic)):
        for key in ("exp_avg", "exp_avg_sq", "max_exp_avg_sq"):
            out[f"{which}_{key}"] = _adam(opt, net, key)
    np.savez_compressed(os.path.join(GOLDEN, f"{name}.npz"), **out)
    print(f"{name}.npz: R", out["ret"], "bootstrap", out["bootstrap"], "actor_loss", al[:2], "critic_loss", cl[:2])


if __name__ == "__main__":
    gen("rf_method", obs=4, n_act=2, hidden=(64, 64), calls=[(40, (19, 39))], batch=64, rounds=8, seed=61, data_seed=601,
        lrs=[(1e-4, 1e-4)])
    gen("rf_multi", obs=6, n_act=3, hidden=(32, 32), calls=[(300, (36, 90, 151, 200, 262))], batch=64, rounds=6, seed=62,
        data_seed=602, lrs=[(3e-4, 1e-3)])
    gen("rf_lr", obs=5, n_act=4, hidden=(32, 32), calls=[(120, (50, 99)), (90, (30,))], batch=48, rounds=4, seed=63,
        data_seed=603, lrs=[(3e-4, 1e-3), (1.5e-4, 5e-4)])
