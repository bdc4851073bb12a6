"""oracle/iql_oracle.py — CPU restatement of Implicit Q-Learning's `learn_batch`
(TEST INFRASTRUCTURE ONLY; eager PyTorch fp32 like the reference).

Restated reference sites (paths relative to the Pearl source tree):
  policy_learners/sequential_decision_making/implicit_q_learning.py:159-302  learn_batch, _value_loss, _actor_loss,
      _critic_loss, _expectile_loss
  neural_networks/common/value_networks.py                                   VanillaValueNetwork (mlp_block)
  neural_networks/sequential_decision_making/actor_networks.py               VanillaActorNetwork (softmax),
      VanillaContinuousActorNetwork (tanh, action_scaling)
  utils/functional_utils/learning/critic_utils.py:170-203                    twin_critic_action_value_loss
Per round: value, critic and actor losses from the pre-round parameters (the value and actor losses use the critic TARGET,
the critic target uses V(s') of the pre-step value net), one backward of their sum, the value / actor / critic
AdamW(amsgrad) steps, then the soft update of both critic targets.  The round's two `torch.randint(0, 2, (1,))` draws are
INPUTS (`bits`), so that both sides of a parity test pick the same target critic.  Parity is pinned by
tests/golden/iql_*.npz (oracle/gen_iql_golden.py).
"""
from __future__ import annotations

import torch

from .pearl_oracle import _mlp, flat, load_flat  # noqa: F401


class _DiscreteActor(torch.nn.Module):
    """VanillaActorNetwork: mlp_block with a softmax last activation (same parameter order)."""

    def __init__(self, obs, n_actions, hidden):
        super().__init__()
        self.net = _mlp([obs] + list(hidden) + [n_actions])

    def forward(self, x):
        return torch.softmax(self.net(x), dim=-1)


class _ContinuousActor(torch.nn.Module):
    """VanillaContinuousActorNetwork: mlp_block with a tanh last activation; sample_action scales to [low, high]."""

    def __init__(self, obs, act, hidden, low, high):
        super().__init__()
        self.net = _mlp([obs] + list(hidden) + [act])
        self.low, self.high = low, high

    def forward(self, x):
        return (((self.high - self.low) * (torch.tanh(self.net(x)) + 1.0)) / 2) + self.low


class OracleIQL:
    """Discrete with `n_actions`, continuous with `low` / `high`."""

    def __init__(self, obs, actor_hidden, critic_hidden, value_hidden, *, n_actions=None, low=None, high=None, actor_lr=1e-3,
                 critic_lr=1e-3, value_lr=1e-3, gamma=0.99, tau=0.05, expectile=0.5, temperature=0.5, advantage_clamp=100.0,
                 init=None):
        self.discrete = n_actions is not None
        self.gamma, self.tau, self.expectile, self.temperature, self.clamp = gamma, tau, expectile, temperature, advantage_clamp
        if self.discrete:
            self.A = int(n_actions)
            self.actor = _DiscreteActor(obs, self.A, actor_hidden)
            n_in = obs + self.A
        else:
            low, high = torch.as_tensor(low, dtype=torch.float32), torch.as_tensor(high, dtype=torch.float32)
            self.actor = _ContinuousActor(obs, low.numel(), actor_hidden, low, high)
            n_in = obs + low.numel()
        self.q = [_mlp([n_in] + list(critic_hidden) + [1]) for _ in range(2)]
        self.qt = [_mlp([n_in] + list(critic_hidden) + [1]) for _ in range(2)]
        self.value = _mlp([obs] + list(value_hidden) + [1])
        if init is not None:
            load_flat(self.actor, init["actor"])
            load_flat(self.value, init["value"])
            for i in range(2):
                load_flat(self.q[i], init[f"q{i + 1}"])
                load_flat(self.qt[i], init[f"q{i + 1}t"])
        self.opt_actor = torch.optim.AdamW(self.actor.parameters(), lr=actor_lr, amsgrad=True)
        self.opt_critic = torch.optim.AdamW(list(self.q[0].parameters()) + list(self.q[1].parameters()), lr=critic_lr, amsgrad=True)
        self.opt_value = torch.optim.AdamW(self.value.parameters(), lr=value_lr, amsgrad=True)

    def set_learning_rates(self, actor_lr, critic_lr, value_lr):
        for opt, lr in ((self.opt_actor, actor_lr), (self.opt_critic, critic_lr), (self.opt_value, value_lr)):
            opt.param_groups[0]["lr"] = lr

    def _action_input(self, a):
        return torch.nn.functional.one_hot(a.long(), self.A).float() if self.discrete else a

    @staticmethod
    def _qv(net, s, a):
        return net(torch.cat([s, a], dim=-1)).view(-1)

    def learn_batch(self, b, bits):
        """b: state [B, O], action [B] int (discrete) or [B, act] float, reward [B], next_state [B, O], terminated [B] bool.
        bits: the round's two randint(0, 2) draws (value loss, actor loss)."""
        s, r, s2, term = b["state"], b["reward"], b["next_state"], b["terminated"]
        a = self._action_input(b["action"])
        # ---- value loss (expectile regression towards the picked target critic)
        with torch.no_grad():
            tq = [self._qv(self.qt[i], s, a) for i in range(2)]
        v = self.value(s).view(-1)
        u = tq[int(bits[0])] - v
        value_loss = (torch.where(u > 0, self.expectile, (1 - self.expectile)) * u.pow(2)).mean()
        # ---- critic loss (towards r + gamma V(s') of the pre-step value net)
        with torch.no_grad():
            y = self.value(s2).view(-1) * self.gamma * (1 - term.float()) + r
        mse = torch.nn.MSELoss()
        critic_loss = (mse(self._qv(self.q[0], s, a), y) + mse(self._qv(self.q[1], s, a), y)) / 2.0
        # ---- actor loss (advantage-weighted regression)
        with torch.no_grad():
            adv = torch.clamp(torch.exp((tq[int(bits[1])] - self.value(s).view(-1)) * self.temperature), max=self.clamp)
        if self.discrete:
            p = self.actor(s)
            actor_loss = -(adv * torch.log(torch.gather(p, 1, b["action"].long().view(-1, 1)).view(-1))).mean()
        else:
            actor_loss = (adv * (self.actor(s) - a).pow(2).mean(dim=1)).mean()
        for opt in (self.opt_value, self.opt_actor, self.opt_critic):
            opt.zero_grad()
        (value_loss + critic_loss + actor_loss).backward()
        self.opt_value.step()
        self.opt_actor.step()
        self.opt_critic.step()
        with torch.no_grad():
            for i in range(2):
                for pt, p_ in zip(self.qt[i].parameters(), self.q[i].parameters()):
                    pt.copy_(self.tau * p_ + (1.0 - self.tau) * pt)
        return {"value_loss": value_loss.item(), "actor_loss": actor_loss.item(), "critic_loss": critic_loss.item()}
