#!/usr/bin/env python
"""Record tests/golden/{td3bc_learn,td3bc_batch,td3bc_lr,td3_batch,ddpg_batch}.npz by RUNNING THE REFERENCE's TD3BC / TD3 /
DeepDeterministicPolicyGradient under PearlAgent with a BasicReplayBuffer (TEST INFRASTRUCTURE; same set-up and stubs as
oracle/gen_golden.py, which provides the import path).

    PYTHONDONTWRITEBYTECODE=1 python oracle/gen_td3bc_golden.py

Cases (all on the asymmetric box [-0.5, 0.5] x [-1, 1] x [-0.25, 1.25], so that the behaviour network's raw tanh output
and the actor's scaled action live in different ranges, td3.py:307-309 vs actor_networks.py:472-485):
  td3bc_learn   two PearlAgent.learn() calls of 3 rounds, actor_update_freq 2: the delay phase carries across the calls
  td3bc_batch   three agent.learn_batch() calls at _training_steps 0, then three at 3: the second three update neither
                the actor nor the targets and report the last actor loss again
  td3bc_lr      two learn() calls of 2 rounds; between them the actor and critic learning rates and alpha_bc change.  The
                second call starts at an odd step, so its first round reports the last actor loss of the first call
  td3_batch     TD3.learn_batch, three calls at _training_steps 0, then two at 1
  ddpg_batch    DeepDeterministicPolicyGradient.learn_batch (ActorCriticBase.learn_batch), three calls
Recorded per call: its kind (0 learn, 1 learn_batch), the training-step count before it, the learning rates and alpha_bc
in force; per sample: the logical indices (0 = oldest element of the deque); every torch.normal draw (the target-policy
noise); CPython's `random` state before the first call; per round the losses; the initial and final networks.
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
from pearl.utils.instantiations.spaces.box_action import BoxActionSpace  # noqa: E402


def gen(name, kind, *, calls, seed, data_seed, obs=7, n=220, batch=40, rounds=3, behavior_hidden=(24, 16), alpha_bc=2.5):
    """`calls`: [(kind, training_steps or None, (actor_lr, critic_lr), alpha_bc)], kind "learn" or "batch"; training_steps
    None keeps the learner's count."""
    torch.manual_seed(seed)
    random.seed(seed)
    torch.set_num_threads(1)
    low, high = torch.tensor([-0.5, -1.0, -0.25]), torch.tensor([0.5, 1.0, 1.25])
    act = int(low.numel())
    space = BoxActionSpace(low=low, high=high)
    lrs = calls[0][2]
    hp = dict(actor_tau=0.03, critic_tau=0.05, gamma=0.97)
    common = dict(state_dim=obs, action_space=space, actor_hidden_dims=[32, 32], critic_hidden_dims=[32, 32], training_rounds=rounds,
                  batch_size=batch, actor_learning_rate=lrs[0], critic_learning_rate=lrs[1], actor_soft_update_tau=hp["actor_tau"],
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
            pl = TD3BC(behavior_policy=behavior, alpha_bc=alpha_bc, **tkw)
        else:
            pl = TD3(**tkw)
    buf = BasicReplayBuffer(n)
    agent = PearlAgent(policy_learner=pl, replay_buffer=buf, device_id=-1)
    rng = np.random.Generator(np.random.PCG64(data_seed))
    q8 = lambda x: (np.rint(x * 256) / 256).astype(np.float32)  # noqa: E731
    st, ns, rw = q8(rng.standard_normal((n, obs))), q8(rng.standard_normal((n, obs))), q8(rng.standard_normal(n))
    ac = q8(rng.uniform(low.numpy(), high.numpy(), size=(n, act)))
    term = rng.random(n) < 0.08
    for i in range(n):
        buf.push(state=torch.from_numpy(st[i]), action=torch.from_numpy(ac[i]), reward=float(rw[i]), terminated=bool(term[i]),
                 truncated=False, curr_available_actions=space, next_state=torch.from_numpy(ns[i]), next_available_actions=space)
    nets = lambda: dict(actor=flat_params(pl._actor), actor_t=flat_params(pl._actor_target), q1=flat_params(pl._critic._critic_1),  # noqa: E731
                        q2=flat_params(pl._critic._critic_2), q1t=flat_params(pl._critic_target._critic_1),
                        q2t=flat_params(pl._critic_target._critic_2))
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
    torch.normal = normal_spy
    rng_before = state_words(random.getstate())
    al, cl, kinds, steps, call_lrs, alphas = [], [], [], [], [], []
    for what, step, (alr, clr), alpha in calls:
        for g in pl._actor_optimizer.param_groups:
            g["lr"] = alr
        for g in pl._critic_optimizer.param_groups:
            g["lr"] = clr
        if kind == "td3bc":
            pl.alpha_bc = alpha
        if step is not None:
            pl._training_steps = step
        kinds.append(0 if what == "learn" else 1)
        steps.append(pl._training_steps)
        call_lrs.append((alr, clr))
        alphas.append(alpha)
        if what == "learn":
            rep = agent.learn()
            al += list(rep["actor_loss"]); cl += list(rep["critic_loss"])
        else:
            rep = agent.learn_batch(buf.sample(batch))
            al.append(rep["actor_loss"]); cl.append(rep["critic_loss"])
            assert pl._training_steps == steps[-1]      # learn_batch does not count a step
    torch.normal = orig_normal
    out = dict(kind=kind, obs=obs, act=act, n=n, batch=batch, rounds=rounds, low=low.numpy(), high=high.numpy(), state=st,
               next_state=ns, reward=rw, action=ac, terminated=term, idx=np.asarray(idxs, dtype=np.int32),
               noise=np.asarray(noises, dtype=np.float32).reshape(len(noises), batch, act) if noises else np.zeros((0, batch, act), np.float32),
               call_kind=np.asarray(kinds, dtype=np.int32), call_steps=np.asarray(steps, dtype=np.int64),
               call_lrs=np.asarray(call_lrs, dtype=np.float64), call_alpha=np.asarray(alphas, dtype=np.float64),
               behavior_hidden=np.asarray(behavior_hidden, dtype=np.int32), rng_before=rng_before,
               actor_loss=np.asarray(al, dtype=np.float64), critic_loss=np.asarray(cl, dtype=np.float64),
               **{f"init_{k}": v for k, v in init.items()}, **{f"{k}_after": v for k, v in nets().items()}, **hp)
    np.savez_compressed(os.path.join(GOLDEN, f"{name}.npz"), **out)
    print(f"{name}.npz: actor_loss", np.round(al, 5).tolist(), "critic_loss", np.round(cl[:3], 5).tolist())


if __name__ == "__main__":
    lr = (3e-4, 6e-4)
    gen("td3bc_learn", "td3bc", calls=[("learn", None, lr, 2.5)] * 2, seed=81, data_seed=801)
    gen("td3bc_batch", "td3bc", calls=[("batch", 0, lr, 2.5)] * 3 + [("batch", 3, lr, 2.5)] * 3, seed=82, data_seed=802)
    gen("td3bc_lr", "td3bc", calls=[("learn", None, lr, 2.5), ("learn", None, (1e-3, 2e-4), 1.5)], rounds=2, seed=83, data_seed=803)
    gen("td3_batch", "td3", calls=[("batch", 0, lr, 0.0)] * 3 + [("batch", 1, lr, 0.0)] * 2, seed=84, data_seed=804)
    gen("ddpg_batch", "ddpg", calls=[("batch", None, lr, 0.0)] * 3, seed=85, data_seed=805)
