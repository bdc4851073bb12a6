"""oracle/sac_discrete_oracle.py — CPU restatement of discrete Soft Actor-Critic's `learn_batch`
(TEST INFRASTRUCTURE ONLY; eager PyTorch fp32 like the reference).

Restated reference sites (paths relative to the Pearl source tree):
  policy_learners/sequential_decision_making/actor_critic_base.py:309-366   actor step, critic step, soft target update
  policy_learners/sequential_decision_making/soft_actor_critic.py           learn_batch (entropy step with
      torch.optim.Adam(lr=critic lr, eps=1e-4)), _actor_loss, _critic_loss, _get_next_state_expected_values, reset
  neural_networks/sequential_decision_making/actor_networks.py              VanillaActorNetwork (MLP + softmax)
  neural_networks/sequential_decision_making/twin_critic.py, q_value_networks.py   get_q_values on state || one-hot
  utils/functional_utils/learning/critic_utils.py                           twin_critic_action_value_loss
Per round, in this order: (1) actor loss on the current critic with the pre-step coefficient, mean over B*A of
pi * (alpha log(pi + 1e-8) - q), AdamW(amsgrad) step; (2) critic target with the UPDATED actor and the critic target:
q~ zeroed on masked next slots, the entropy term summed over all A slots, pi'_k paired with slot k; twin MSE, AdamW step;
(3) soft update of both targets; (4) entropy Adam step with the probabilities cached in (1).  Parity is pinned by
tests/golden/sacd_*.npz (oracle/gen_sac_discrete_golden.py).
"""
from __future__ import annotations

import torch

from .pearl_oracle import _mlp, flat, load_flat  # noqa: F401


class _Actor(torch.nn.Module):
    """VanillaActorNetwork: mlp_block with a softmax last activation (same parameter order)."""

    def __init__(self, obs, n_actions, hidden):
        super().__init__()
        self.net = _mlp([obs] + list(hidden) + [n_actions])

    def forward(self, x):
        return torch.softmax(self.net(x), dim=-1)


class OracleSACDiscrete:
    def __init__(self, obs, n_actions, actor_hidden, critic_hidden, *, actor_lr=1e-4, critic_lr=1e-4, gamma=0.99, tau=0.005,
                 entropy_coef=0.2, autotune=True, target_entropy_scale=0.89, init=None):
        self.obs, self.A, self.gamma, self.tau, self.autotune = obs, n_actions, gamma, tau, autotune
        self.actor = _Actor(obs, n_actions, actor_hidden)
        self.q = [_mlp([obs + n_actions] + list(critic_hidden) + [1]) for _ in range(2)]
        self.qt = [_mlp([obs + n_actions] + list(critic_hidden) + [1]) for _ in range(2)]
        if init is not None:
            load_flat(self.actor, init["actor"])
            for i in range(2):
                load_flat(self.q[i], init[f"q{i + 1}"])
                load_flat(self.qt[i], init[f"q{i + 1}t"])
        self.opt_actor = torch.optim.AdamW(self.actor.parameters(), lr=actor_lr, amsgrad=True)
        self.opt_critic = torch.optim.AdamW(list(self.q[0].parameters()) + list(self.q[1].parameters()), lr=critic_lr, amsgrad=True)
        self.scheduler = torch.optim.lr_scheduler.ExponentialLR(self.opt_actor, gamma=0.99)
        self.log_alpha = torch.nn.Parameter(torch.zeros(1))
        self.opt_alpha = torch.optim.Adam([self.log_alpha], lr=critic_lr, eps=1e-4)
        self.alpha = torch.exp(self.log_alpha).detach() if autotune else torch.tensor(entropy_coef)
        self.target_entropy = -target_entropy_scale * torch.log(1.0 / torch.tensor(n_actions))

    def reset(self):
        """SoftActorCritic.reset: one ExponentialLR(0.99) step of the actor optimizer."""
        self.scheduler.step()

    def _q_all(self, net, s, ids):
        """Q(s, one-hot(ids[b, k])) for every slot: [B, A]."""
        B, A = ids.shape
        onehot = torch.nn.functional.one_hot(ids.long(), self.A).float()            # [B, A, A]
        x = torch.cat([s.unsqueeze(1).expand(B, A, s.shape[1]), onehot], dim=-1)
        return net(x).squeeze(-1)

    def learn_batch(self, b):
        """b: state [B, O], action [B] int, reward [B], next_state [B, O], terminated [B] bool,
        next_ids [B, A] int (slot k holds id_k) and next_mask [B, A] bool (True = unavailable)."""
        s, a, r, s2, term = b["state"], b["action"].long(), b["reward"], b["next_state"], b["terminated"]
        B, A = s.shape[0], self.A
        full = torch.arange(A).expand(B, A)
        # ---- (1) actor step
        q = torch.minimum(self._q_all(self.q[0], s, full), self._q_all(self.q[1], s, full)).detach()
        pi = self.actor(s)
        logp = torch.log(pi + 1e-8)
        actor_loss = (pi * (self.alpha * logp - q)).mean()
        probs_cache, logp_cache = pi.detach(), logp.detach()
        self.opt_actor.zero_grad()
        actor_loss.backward()
        self.opt_actor.step()
        # ---- (2) critic step with the updated actor
        with torch.no_grad():
            nq = torch.minimum(self._q_all(self.qt[0], s2, b["next_ids"]), self._q_all(self.qt[1], s2, b["next_ids"]))
            nq[b["next_mask"]] = 0.0
            pi2 = self.actor(s2)
            v = ((nq - self.alpha * torch.log(pi2 + 1e-8)) * pi2).sum(dim=1)
            y = v * self.gamma * (1 - term.float()) + r
        onehot = torch.nn.functional.one_hot(a, A).float()
        x = torch.cat([s, onehot], dim=-1)
        mse = torch.nn.MSELoss()
        critic_loss = (mse(self.q[0](x).squeeze(-1), y) + mse(self.q[1](x).squeeze(-1), y)) / 2.0
        self.opt_critic.zero_grad()
        critic_loss.backward()
        self.opt_critic.step()
        # ---- (3) soft update
        with torch.no_grad():
            for i in range(2):
                for pt, p in zip(self.qt[i].parameters(), self.q[i].parameters()):
                    pt.copy_(self.tau * p + (1.0 - self.tau) * pt)
        out = {"actor_loss": actor_loss.item(), "critic_loss": critic_loss.item()}
        # ---- (4) entropy step with the actor-step probabilities
        if self.autotune:
            entropy = -(probs_cache * logp_cache).sum(1).mean()
            ent_loss = torch.exp(self.log_alpha) * (entropy - self.target_entropy).detach()
            self.opt_alpha.zero_grad()
            ent_loss.backward()
            self.opt_alpha.step()
            self.alpha = torch.exp(self.log_alpha).detach()
            out["entropy_coef"] = float(ent_loss.detach())
        return out
