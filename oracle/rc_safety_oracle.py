"""oracle/rc_safety_oracle.py — CPU restatement of Pearl's reward-constrained safety module with a deterministic
actor-critic policy learner (TEST INFRASTRUCTURE ONLY; eager PyTorch fp32 like the reference), on top of
oracle/td3_oracle.py and oracle/td3bc_oracle.py.

Restated reference sites (paths relative to /root/reference/pearl):
  pearl_agent.py:213-220                                        policy learner first, then the safety module, once per learn()
  policy_learners/sequential_decision_making/actor_critic_base.py:368-383   reward - lambda_constraint * cost in every round
  safety_modules/reward_constrained_safety_module.py:115-216    batch, cost-critic step, soft update, projected lambda step
  utils/functional_utils/learning/critic_utils.py:170-203       twin MSE loss (mse1 + mse2) / 2
The cost critic's next action comes from the ONLINE actor without noise; lambda is updated in Python float64 from
cq = mean(max(Qc1, Qc2)(s, actor(s))) of the UPDATED cost critic, read with .item().  Parity pinned by
tests/golden/rc_*.npz (oracle/gen_rc_safety_golden.py).
"""
from __future__ import annotations

import torch

from .pearl_oracle import _mlp, load_flat
from .td3bc_oracle import OracleTD3, OracleTD3BC


def shaped_reward(reward: torch.Tensor, cost: torch.Tensor, lam: float) -> torch.Tensor:
    """ActorCriticBase.preprocess_batch: a Python float times an fp32 tensor, then a subtraction (two fp32 roundings)."""
    return reward - lam * cost


def lambda_step(lam: float, cq: float, lr_lambda: float, cost_gamma: float, constraint: float, ub: float) -> float:
    """constraint_lambda_update in Python floats (float64), the reference's evaluation order and clamps."""
    out = lam + lr_lambda * (cq * (1 - cost_gamma) - constraint)
    out = max(out, 0.0)
    return min(out, ub)


class OracleCostCritic:
    def __init__(self, obs, act, hidden, *, lr=1e-3, cost_gamma=0.5, tau=0.005, constraint=0.0, lr_lambda=1e-2, ub=20.0, lam=0.0,
                 init=None):
        self.q = [_mlp([obs + act] + list(hidden) + [1]) for _ in range(2)]
        self.qt = [_mlp([obs + act] + list(hidden) + [1]) for _ in range(2)]
        if init is not None:
            for i in range(2):
                load_flat(self.q[i], init[f"c{i + 1}"]); load_flat(self.qt[i], init[f"c{i + 1}t"])
        self.opt = torch.optim.AdamW(list(self.q[0].parameters()) + list(self.q[1].parameters()), lr=lr, amsgrad=True)
        self.cost_gamma, self.tau, self.constraint, self.lr_lambda, self.ub, self.lam = cost_gamma, tau, constraint, lr_lambda, ub, lam

    @staticmethod
    def _qv(net, s, a):
        return net(torch.cat([s, a], dim=-1)).squeeze(-1)

    def learn(self, b, actor_act):
        """One safety-module step on batch `b`; actor_act(s) = the policy's sample_action.  Returns (loss, cq)."""
        s, a, c, s2, term = b["state"], b["action"], b["cost"], b["next_state"], b["terminated"]
        with torch.no_grad():
            a2 = actor_act(s2)
            nq = torch.minimum(self._qv(self.qt[0], s2, a2), self._qv(self.qt[1], s2, a2))
            y = (nq * self.cost_gamma * (1 - term.float())) + c
        mse = torch.nn.MSELoss()
        loss = (mse(self._qv(self.q[0], s, a), y) + mse(self._qv(self.q[1], s, a), y)) / 2.0
        self.opt.zero_grad()
        loss.backward()
        self.opt.step()
        with torch.no_grad():
            for i in range(2):
                for pt, p in zip(self.qt[i].parameters(), self.q[i].parameters()):
                    pt.copy_(self.tau * p + (1.0 - self.tau) * pt)
            act = actor_act(s)
            cq = torch.maximum(self._qv(self.q[0], s, act), self._qv(self.q[1], s, act)).mean().item()
        self.lam = lambda_step(self.lam, cq, self.lr_lambda, self.cost_gamma, self.constraint, self.ub)
        return loss.item(), cq


def oracles_for(fx):
    """(policy oracle, cost-critic oracle) a recording (tests/golden/rc_*.npz) starts from."""
    kind = str(fx["kind"])
    init = {k[5:]: fx[k] for k in fx.files if k.startswith("init_")}
    lrs = fx["call_lrs"][0]
    kw = dict(actor_lr=float(lrs[0]), critic_lr=float(lrs[1]), gamma=float(fx["gamma"]), actor_tau=float(fx["actor_tau"]),
              critic_tau=float(fx["critic_tau"]), actor_update_freq=int(fx["freq"]), noise_clip=float(fx["noise_clip"]), init=init)
    args = (int(fx["obs"]), int(fx["act"]), (32, 32), (32, 32), fx["low"], fx["high"])
    if kind == "td3bc":
        pol = OracleTD3BC(*args, behavior_hidden=tuple(int(x) for x in fx["behavior_hidden"]), alpha_bc=float(fx["alpha_bc"]), **kw)
    else:
        pol = OracleTD3(*args, **kw)
    cc = OracleCostCritic(int(fx["obs"]), int(fx["act"]), (32, 32), lr=float(fx["call_cost_lr"][0]), cost_gamma=float(fx["cost_gamma"]),
                          tau=float(fx["cost_tau"]), constraint=float(fx["constraint"]), lr_lambda=float(fx["lr_lambda"]), ub=float(fx["ub"]),
                          init=init)
    return pol, cc


def agent_learn(pol, cc, rows, rounds, noise=None):
    """PearlAgent.learn(): `rounds` policy rounds on rows[0..rounds) (dicts of tensors with `cost`), shaped with the
    multiplier as it stands, then the safety step on rows[rounds].  noise: [rounds][B][A] or None (DDPG).
    Returns (actor losses, critic losses, cost loss, cq)."""
    al, cl = [], []
    lam = cc.lam
    for r in range(rounds):
        b = dict(rows[r])
        b["reward"] = shaped_reward(b["reward"], b["cost"], lam)
        pol.training_steps += 1
        out = pol.learn_batch(b, None if noise is None else noise[r])
        al.append(out["actor_loss"]); cl.append(out["critic_loss"])
    loss, cq = cc.learn(rows[rounds], lambda s: pol.act(pol.actor, s))
    return al, cl, loss, cq
