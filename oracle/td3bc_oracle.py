"""oracle/td3bc_oracle.py — CPU restatement of Pearl's TD3BC.learn_batch (TEST INFRASTRUCTURE ONLY; eager PyTorch fp32 like the
reference), on top of oracle/td3_oracle.py.

Restated reference sites (paths relative to /root/reference/pearl):
  policy_learners/sequential_decision_making/td3.py:241-318   TD3BC: actor loss mean((a - b)^2) - alpha_bc / mean|q| * mean(q)
  neural_networks/sequential_decision_making/actor_networks.py:448-485  behavior_policy(s) = forward() = the raw tanh output
The behaviour action b is NOT scaled to the box while the actor's a is (sample_action); q is critic 1 only; b and the
weight lambda carry no gradient.  Everything else is TD3 (OracleTD3).  Parity pinned by tests/golden/td3bc_*.npz
(oracle/gen_td3bc_golden.py).
"""
from __future__ import annotations

import torch

from .td3_oracle import OracleTD3, _actor, load_flat


class OracleTD3BC(OracleTD3):
    def __init__(self, obs, act, actor_hidden, critic_hidden, low, high, *, behavior_hidden, alpha_bc=2.5, init=None, **kw):
        super().__init__(obs, act, actor_hidden, critic_hidden, low, high, init=init, **kw)
        self.behavior = _actor(obs, act, behavior_hidden)
        if init is not None and "behavior" in init:
            load_flat(self.behavior, init["behavior"])
        self.alpha_bc = alpha_bc

    def actor_loss(self, s):
        a = self.act(self.actor, s)
        q = self._qv(self.q[0], s, a)
        with torch.no_grad():
            b = self.behavior(s)
        lmbda = self.alpha_bc / q.abs().mean().detach()
        return ((a - b).pow(2)).mean() - lmbda * q.mean()

    def learn_batch(self, b, target_noise=None):
        """OracleTD3.learn_batch with the TD3BC actor loss (the caller advances `training_steps` first when it restates
        PolicyLearner.learn; learn_batch itself does not)."""
        s, a, r, s2, term = b["state"], b["action"], b["reward"], b["next_state"], b["terminated"]
        update_actor = self.freq <= 1 or self.training_steps % self.freq == 0
        if update_actor:
            self.opt_actor.zero_grad()
            loss = self.actor_loss(s)
            loss.backward()
            self.opt_actor.step()
            self.last_actor_loss = loss.item()
        self.opt_critic.zero_grad()
        with torch.no_grad():
            a2 = self.act(self.actor_t, s2)
            if target_noise is not None:
                noise = torch.clamp(target_noise, -self.noise_clip, self.noise_clip) * (self.high - self.low) / 2
                a2 = torch.clamp(a2 + noise, self.low, self.high)
            nq = torch.minimum(self._qv(self.qt[0], s2, a2), self._qv(self.qt[1], s2, a2))
            y = (nq * self.gamma * (1 - term.float())) + r
        mse = torch.nn.MSELoss()
        critic_loss = (mse(self._qv(self.q[0], s, a), y) + mse(self._qv(self.q[1], s, a), y)) / 2.0
        critic_loss.backward()
        self.opt_critic.step()
        if update_actor:
            with torch.no_grad():
                for i in range(2):
                    for pt, p in zip(self.qt[i].parameters(), self.q[i].parameters()):
                        pt.copy_(self.critic_tau * p + (1.0 - self.critic_tau) * pt)
                for pt, p in zip(self.actor_t.parameters(), self.actor.parameters()):
                    pt.copy_(self.actor_tau * p + (1.0 - self.actor_tau) * pt)
        return {"actor_loss": self.last_actor_loss, "critic_loss": critic_loss.item()}


def oracle_for(fx):
    """The oracle a td3bc / td3 / ddpg recording (tests/golden/*_batch.npz, td3bc_*.npz) starts from."""
    kind = str(fx["kind"])
    init = {k[5:]: fx[k] for k in fx.files if k.startswith("init_")}
    lrs = fx["call_lrs"][0]
    kw = dict(actor_lr=float(lrs[0]), critic_lr=float(lrs[1]), gamma=float(fx["gamma"]), actor_tau=float(fx["actor_tau"]),
              critic_tau=float(fx["critic_tau"]), actor_update_freq=int(fx["freq"]), noise_clip=float(fx["noise_clip"]), init=init)
    args = (int(fx["obs"]), int(fx["act"]), (32, 32), (32, 32), fx["low"], fx["high"])
    if kind == "td3bc":
        return OracleTD3BC(*args, behavior_hidden=tuple(int(x) for x in fx["behavior_hidden"]), alpha_bc=float(fx["call_alpha"][0]), **kw)
    return OracleTD3(*args, **kw)


def set_lrs(orc, actor_lr, critic_lr):
    for g in orc.opt_actor.param_groups:
        g["lr"] = actor_lr
    for g in orc.opt_critic.param_groups:
        g["lr"] = critic_lr
