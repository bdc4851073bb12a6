#!/usr/bin/env python
"""Record tests/golden/rc_{td3,ddpg,zero,lr,td3bc}.npz by RUNNING THE REFERENCE's PearlAgent(TD3 | DDPG | TD3BC,
RCSafetyModuleCostCriticContinuousAction, BasicReplayBuffer) (TEST INFRASTRUCTURE; same set-up and stubs as
oracle/gen_td3bc_golden.py).

    PYTHONDONTWRITEBYTECODE=1 python oracle/gen_rc_safety_golden.py

Every case pushes 220 transitions with costs in [1, 2] on the asymmetric box [-0.5, 0.5] x [-1, 1] x [-0.25, 1.25] and
runs several agent.learn() calls: `rounds` policy rounds on reward - lambda * cost (lambda as the previous call left it),
then one safety-module step on its own sample (cost-critic step and soft update, then the lambda step from the updated
cost critic).
  rc_td3    TD3, constraint 0.05, lr_lambda 0.2, ub 0.4: lambda goes from 0 through interior values to the upper bound
  rc_ddpg   DDPG, lr_lambda 0.5 (the default of the other cases): lambda reaches the upper bound on the second call
  rc_zero   TD3 with a constraint the cost never reaches: lambda stays clamped at 0
  rc_lr     TD3; the cost critic's learning rate changes between calls
  rc_td3bc  TD3BC, the same module settings
Recorded per call: lambda before the call, the cost-critic loss, cq (mean of max(Qc1, Qc2) at (s, actor(s)) with the
updated cost critic, as the reference reads it with .item()), lambda after it, and the cost-critic learning rate; per
sample the logical indices (the policy rounds, then the safety step); every torch.normal draw; the per-round TD3 losses;
the initial and final networks (actor, critics, cost critics and every target) and the final AdamW moments.
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
from pearl.neural_networks.sequential_decision_making.actor_networks import VanillaContinuousActorNetwork  # noqa: E402
from pearl.pearl_agent import PearlAgent  # noqa: E402
from pearl.policy_learners.exploration_modules.common.no_exploration import NoExploration  # noqa: E402
from pearl.policy_learners.sequential_decision_making.ddpg import DeepDeterministicPolicyGradient  # noqa: E402
from pearl.policy_learners.sequential_decision_making.td3 import TD3, TD3BC  # noqa: E402
from pearl.replay_buffers.basic_replay_buffer import BasicReplayBuffer  # noqa: E402
from pearl.safety_modules.reward_constrained_safety_module import RCSafetyModuleCostCriticContinuousAction  # noqa: E402
from pearl.utils.instantiations.spaces.box_action import BoxActionSpace  # noqa: E402


def _moments(opt, params):
    st = [opt.state[p] for p in params]
    return {k: np.concatenate([s[k].detach().numpy().ravel() for s in st]) for k in ("exp_avg", "exp_avg_sq", "max_exp_avg_sq")}


def gen(name, kind, *, calls, seed, data_seed, constraint=0.05, lr_lambda=0.5, ub=0.4, cost_lrs=(1e-2,), cost_gamma=0.5, cost_tau=0.05,
        obs=7, n=220, batch=40, rounds=3, behavior_hidden=(24, 16)):
    torch.manual_seed(seed)
    random.seed(seed)
    torch.set_num_threads(1)
    low, high = torch.tensor([-0.5, -1.0, -0.25]), torch.tensor([0.5, 1.0, 1.25])
    act = int(low.numel())
    space = BoxActionSpace(low=low, high=high)
    hp = dict(actor_tau=0.03, critic_tau=0.05, gamma=0.97)
    lr = (3e-4, 6e-4)
    common = dict(state_dim=obs, action_space=space, actor_hidden_dims=[32, 32], critic_hidden_dims=[32, 32], training_rounds=rounds,
                  batch_size=batch, actor_learning_rate=lr[0], critic_learning_rate=lr[1], actor_soft_update_tau=hp["actor_tau"],
                  critic_soft_update_tau=hp["critic_tau"], discount_factor=hp["gamma"], exploration_module=NoExploration())
    behavior = None
    if kind == "ddpg":
        hp.update(freq=1, noise_std=0.0, noise_clip=0.0)
        pl = DeepDeterministicPolicyGradient(**common)
    else:
        hp.update(freq=2, noise_std=0.2, noise_clip=0.5)
        tkw = dict(actor_update_freq=2, actor_update_noise=0.2, actor_update_noise_clip=0.5, **common)
        if kind == "td3bc":
            behavior = VanillaContinuousActorNetwork(input_dim=obs, hidden_dims=list(behavior_hidden), output_dim=act, action_space=space)
            pl = TD3BC(behavior_policy=behavior, alpha_bc=2.5, **tkw)
        else:
            pl = TD3(**tkw)
    rc = RCSafetyModuleCostCriticContinuousAction(constraint_value=constraint, state_dim=obs, action_space=space,
                                                  critic_hidden_dims=[32, 32], lambda_constraint_ub_value=ub, cost_discount_factor=cost_gamma,
                                                  lr_lambda=lr_lambda, critic_learning_rate=cost_lrs[0], critic_soft_update_tau=cost_tau,
                                                  batch_size=batch)
    buf = BasicReplayBuffer(n)
    agent = PearlAgent(policy_learner=pl, safety_module=rc, replay_buffer=buf, device_id=-1)
    assert pl.safety_module is rc
    rng = np.random.Generator(np.random.PCG64(data_seed))
    q8 = lambda x: (np.rint(x * 256) / 256).astype(np.float32)  # noqa: E731
    st, ns, rw = q8(rng.standard_normal((n, obs))), q8(rng.standard_normal((n, obs))), q8(rng.standard_normal(n))
    ac = q8(rng.uniform(low.numpy(), high.numpy(), size=(n, act)))
    cost = q8(rng.uniform(1.0, 2.0, size=n))
    term = rng.random(n) < 0.08
    for i in range(n):
        buf.push(state=torch.from_numpy(st[i]), action=torch.from_numpy(ac[i]), reward=float(rw[i]), terminated=bool(term[i]),
                 truncated=False, curr_available_actions=space, next_state=torch.from_numpy(ns[i]), next_available_actions=space,
                 cost=float(cost[i]))
    nets = lambda: dict(actor=flat_params(pl._actor), actor_t=flat_params(pl._actor_target), q1=flat_params(pl._critic._critic_1),  # noqa: E731
                        q2=flat_params(pl._critic._critic_2), q1t=flat_params(pl._critic_target._critic_1),
                        q2t=flat_params(pl._critic_target._critic_2), c1=flat_params(rc.cost_critic._critic_1),
                        c2=flat_params(rc.cost_critic._critic_2), c1t=flat_params(rc.target_of_cost_critic._critic_1),
                        c2t=flat_params(rc.target_of_cost_critic._critic_2))
    init = nets()
    if behavior is not None:
        init["behavior"] = flat_params(behavior)
    noises, idxs = [], []
    orig_normal = torch.normal

    def normal_spy(*a, **k):
        x = orig_normal(*a, **k)
        noises.append(x.numpy().copy())
        return x
    orig_sample = buf.sample

    def sample_spy(k):
        pos = {id(t): j for j, t in enumerate(buf.memory)}
        stt = random.getstate()
        idxs.append([pos[id(t)] for t in random.sample(buf.memory, k)])
        random.setstate(stt)
        return orig_sample(k)
    buf.sample = sample_spy
    # cq: the reference's own max / mean / .item() of the last cost-critic evaluation of each learn() (the lambda step's)
    last_q = {}
    orig_q = rc.cost_critic.get_q_values

    def q_spy(*a, **k):
        out = orig_q(*a, **k)
        last_q["q"] = out
        return out
    rc.cost_critic.get_q_values = q_spy
    losses = []
    orig_ccl = rc.cost_critic_learn_batch

    def ccl_spy(*a, **k):
        out = orig_ccl(*a, **k)
        losses.append(out["cost_critic_loss"])
        return out
    rc.cost_critic_learn_batch = ccl_spy
    torch.normal = normal_spy
    rng_before = state_words(random.getstate())
    al, cl, lam_before, lam_after, cqs, call_cost_lr = [], [], [], [], [], []
    for c in range(calls):
        clr = cost_lrs[c % len(cost_lrs)]
        for g in rc.cost_critic_optimizer.param_groups:
            g["lr"] = clr
        call_cost_lr.append(clr)
        lam_before.append(rc.lambda_constraint)
        rep = agent.learn()
        al += list(rep["actor_loss"]); cl += list(rep["critic_loss"])
        q1, q2 = last_q["q"]
        cqs.append(torch.maximum(q1, q2).mean().item())
        lam_after.append(rc.lambda_constraint)
    torch.normal = orig_normal
    assert len(losses) == calls and len(idxs) == calls * (rounds + 1)
    params = list(rc.cost_critic.parameters())
    mom = {f"cost_{k}": v for k, v in _moments(rc.cost_critic_optimizer, params).items()}
    mom.update({f"critic_{k}": v for k, v in _moments(pl._critic_optimizer, list(pl._critic.parameters())).items()})
    mom.update({f"actor_{k}": v for k, v in _moments(pl._actor_optimizer, list(pl._actor.parameters())).items()})
    mom["cost_step"] = np.asarray(int(float(rc.cost_critic_optimizer.state[params[0]]["step"])), dtype=np.int64)
    out = dict(kind=kind, obs=obs, act=act, n=n, batch=batch, rounds=rounds, calls=calls, low=low.numpy(), high=high.numpy(), state=st,
               next_state=ns, reward=rw, action=ac, cost=cost, terminated=term, idx=np.asarray(idxs, dtype=np.int32),
               noise=np.asarray(noises, dtype=np.float32).reshape(len(noises), batch, act) if noises else np.zeros((0, batch, act), np.float32),
               call_lrs=np.asarray([lr] * calls, dtype=np.float64), call_cost_lr=np.asarray(call_cost_lr, dtype=np.float64),
               behavior_hidden=np.asarray(behavior_hidden, dtype=np.int32), rng_before=rng_before, alpha_bc=2.5,
               constraint=constraint, lr_lambda=lr_lambda, ub=ub, cost_gamma=cost_gamma, cost_tau=cost_tau, rc_batch=batch,
               lambda_before=np.asarray(lam_before, dtype=np.float64), lambda_after=np.asarray(lam_after, dtype=np.float64),
               cq=np.asarray(cqs, dtype=np.float64), cost_loss=np.asarray(losses, dtype=np.float64),
               actor_loss=np.asarray(al, dtype=np.float64), critic_loss=np.asarray(cl, dtype=np.float64),
               **{f"init_{k}": v for k, v in init.items()}, **{f"{k}_after": v for k, v in nets().items()}, **mom, **hp)
    np.savez_compressed(os.path.join(GOLDEN, f"{name}.npz"), **out)
    print(f"{name}.npz: lambda", np.round(lam_after, 5).tolist(), "cq", np.round(cqs, 4).tolist())


if __name__ == "__main__":
    gen("rc_td3", "td3", calls=6, seed=91, data_seed=901, lr_lambda=0.2)
    gen("rc_ddpg", "ddpg", calls=5, seed=92, data_seed=902)
    gen("rc_zero", "td3", calls=3, seed=93, data_seed=903, constraint=10.0)
    gen("rc_lr", "td3", calls=4, seed=94, data_seed=904, cost_lrs=(1e-2, 3e-3))
    gen("rc_td3bc", "td3bc", calls=4, seed=95, data_seed=905)
