#!/usr/bin/env python
"""Record tests/golden/sacd_*.npz by RUNNING THE REFERENCE's discrete SoftActorCritic under PearlAgent with a
BasicReplayBuffer (TEST INFRASTRUCTURE; same set-up and stubs as oracle/gen_golden.py, which provides the import path).

    PYTHONDONTWRITEBYTECODE=1 python oracle/gen_sac_discrete_golden.py

Three cases:
  sacd_full     full action space, entropy autotune on, some terminal transitions
  sacd_dynamic  dynamic next-action sets, autotune off, entropy_coef 0.1
  sacd_reset    two learn() calls with agent.reset() between them: the actor's ExponentialLR(0.99) steps once, so the
                second call trains with actor lr * 0.99
Recorded: the transitions, the sampled logical indices of every round (0 = oldest element of the deque), per-round
losses, the initial and final actor / q1 / q2 / targets, log alpha and its Adam state, and the actor lr of each call.
Current action sets are pushed in full (the CUDA replay buffer stores none).
"""
from __future__ import annotations

import os
import random
import sys

import numpy as np

sys.dont_write_bytecode = True
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from oracle.gen_golden import GOLDEN, flat_params  # noqa: E402  (sets up the reference import path and stubs)
from oracle.synth import make_transitions  # noqa: E402

import torch  # noqa: E402
from pearl.action_representation_modules.one_hot_action_representation_module import (  # noqa: E402
    OneHotActionTensorRepresentationModule,
)
from pearl.pearl_agent import PearlAgent  # noqa: E402
from pearl.policy_learners.sequential_decision_making.soft_actor_critic import SoftActorCritic  # noqa: E402
from pearl.replay_buffers.basic_replay_buffer import BasicReplayBuffer  # noqa: E402
from pearl.utils.instantiations.spaces.discrete_action import DiscreteActionSpace  # noqa: E402


def gen_sac_discrete_golden(name, *, obs, n_act, hidden, n, batch, rounds, seed, data_seed, autotune=True, entropy_coef=0.2,
                            dynamic=False, p_term=0.1, actor_lr=3e-4, critic_lr=5e-4, tau=0.05, gamma=0.98, calls=1):
    torch.manual_seed(seed)
    random.seed(seed)
    torch.set_num_threads(1)
    full = DiscreteActionSpace(actions=list(torch.arange(n_act).view(-1, 1)))
    pl = SoftActorCritic(state_dim=obs, action_space=full, actor_hidden_dims=list(hidden), critic_hidden_dims=list(hidden),
                         actor_learning_rate=actor_lr, critic_learning_rate=critic_lr, critic_soft_update_tau=tau,
                         discount_factor=gamma, training_rounds=rounds, batch_size=batch, entropy_coef=entropy_coef,
                         entropy_autotune=autotune, action_representation_module=OneHotActionTensorRepresentationModule(n_act))
    buf = BasicReplayBuffer(n)
    agent = PearlAgent(policy_learner=pl, replay_buffer=buf, device_id=-1)
    data = make_transitions(n, obs, n_act, seed=data_seed, dynamic=dynamic, p_term=p_term)
    ids = data.get("next_avail_ids", np.tile(np.arange(n_act), (n, 1)))
    cnt = data.get("next_avail_n", np.full(n, n_act))
    for i in range(n):
        nxt = DiscreteActionSpace(actions=[torch.tensor([int(a)]) for a in ids[i, :cnt[i]]]) if dynamic else full
        buf.push(state=torch.from_numpy(data["state"][i]), action=torch.tensor(int(data["action"][i])),
                 reward=float(data["reward"][i]), terminated=bool(data["terminated"][i]), truncated=False,
                 curr_available_actions=full, next_state=torch.from_numpy(data["next_state"][i]), next_available_actions=nxt,
                 max_number_actions=n_act)
    init = dict(actor=flat_params(pl._actor), q1=flat_params(pl._critic._critic_1), q2=flat_params(pl._critic._critic_2),
                q1t=flat_params(pl._critic_target._critic_1), q2t=flat_params(pl._critic_target._critic_2))
    idxs = []
    orig_sample = buf.sample

    def sample_spy(k):
        pos = {id(t): j for j, t in enumerate(buf.memory)}
        st = random.getstate()
        idxs.append([pos[id(t)] for t in random.sample(buf.memory, k)])
        random.setstate(st)
        return orig_sample(k)
    buf.sample = sample_spy
    rs = random.getstate()
    al, cl, el, lrs = [], [], [], []
    for c in range(calls):
        if c:
            agent.reset(torch.zeros(obs), full)
        lrs.append(pl._actor_optimizer.param_groups[0]["lr"])
        rep = agent.learn()
        al += list(rep["actor_loss"])
        cl += list(rep["critic_loss"])
        el += [float(x) for x in rep.get("entropy_coef", [])]
    out = dict(obs=obs, n_actions=n_act, hidden=np.asarray(hidden), n=n, batch=batch, rounds=rounds, calls=calls,
               actor_lr=actor_lr, critic_lr=critic_lr, tau=tau, gamma=gamma, autotune=autotune, entropy_coef=entropy_coef,
               call_actor_lr=np.asarray(lrs), state=data["state"], next_state=data["next_state"], reward=data["reward"],
               action=data["action"].astype(np.int32), terminated=data["terminated"], dynamic=dynamic,
               next_ids=ids.astype(np.uint8), next_count=cnt.astype(np.int32),
               rng_before=np.asarray(rs[1], dtype=np.uint64).astype(np.uint32),
               idx=np.asarray(idxs, dtype=np.int32), actor_loss=np.asarray(al), critic_loss=np.asarray(cl),
               entropy_loss=np.asarray(el), actor_after=flat_params(pl._actor), q1_after=flat_params(pl._critic._critic_1),
               q2_after=flat_params(pl._critic._critic_2), q1t_after=flat_params(pl._critic_target._critic_1),
               q2t_after=flat_params(pl._critic_target._critic_2), **{f"init_{k}": v for k, v in init.items()})
    if autotune:
        st = pl._entropy_optimizer.state[pl._log_entropy]
        out.update(log_alpha_after=pl._log_entropy.detach().numpy().copy(), alpha_exp_avg=st["exp_avg"].numpy().copy(),
                   alpha_exp_avg_sq=st["exp_avg_sq"].numpy().copy(), alpha_after=pl._entropy_coef.numpy().reshape(-1).copy())
    np.savez_compressed(os.path.join(GOLDEN, f"{name}.npz"), **out)
    print(f"{name}.npz: actor_loss", al[:2], "critic_loss", cl[:2], "entropy", el[:2])


if __name__ == "__main__":
    gen_sac_discrete_golden("sacd_full", obs=6, n_act=4, hidden=(32, 32), n=300, batch=64, rounds=6, seed=51, data_seed=501)
    gen_sac_discrete_golden("sacd_dynamic", obs=6, n_act=5, hidden=(32, 32), n=300, batch=64, rounds=6, seed=52, data_seed=502,
                            autotune=False, entropy_coef=0.1, dynamic=True)
    gen_sac_discrete_golden("sacd_reset", obs=5, n_act=3, hidden=(32, 32), n=200, batch=48, rounds=4, seed=53, data_seed=503,
                            calls=2)
