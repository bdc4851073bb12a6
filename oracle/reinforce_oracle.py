"""oracle/reinforce_oracle.py — CPU restatement of REINFORCE with a state-value baseline (TEST INFRASTRUCTURE ONLY; eager
PyTorch fp32 like the reference).

Restated reference sites (paths relative to the Pearl source tree):
  policy_learners/sequential_decision_making/reinforce.py:179-208   learn(): the return pass
  policy_learners/sequential_decision_making/reinforce.py:146-167   _actor_loss (use_critic=True), _critic_loss
  policy_learners/sequential_decision_making/actor_critic_base.py:309-366   learn_batch: actor step, then critic step
  neural_networks/sequential_decision_making/actor_networks.py:155-176     get_action_prob (softmax over every action)
  utils/functional_utils/learning/critic_utils.py:139-167                 single_critic_state_value_loss

Both quirks of the reference are kept:
  * the return: cum = critic(s'_newest) * (~terminated_newest), then `cum += reward` for every transition newest -> oldest,
    in place, so every transition holds the SAME final value R (no discount, no episode reset);
  * the actor loss: nlp has shape (B,), cum_reward (B, 1), so `nlp * (cum_reward - v)` is a B x B matrix and the loss is
    sum_i sum_j nlp_j (R - v_j).
Parity is pinned by tests/golden/rf_*.npz (oracle/gen_reinforce_golden.py).
"""
from __future__ import annotations

import torch

from .pearl_oracle import _mlp, flat, load_flat  # noqa: F401


def fold_returns(bootstrap, reward) -> torch.Tensor:
    """The reference's loop from a given bootstrap term: shape (1,) fp32, rewards in time order (0 = oldest)."""
    cum = torch.as_tensor(bootstrap, dtype=torch.float32).reshape(1).clone()
    reward = torch.as_tensor(reward, dtype=torch.float32).reshape(-1)
    for t in range(reward.shape[0] - 1, -1, -1):
        cum += reward[t]
    return cum


def hand_gradients(logits, action, v, R):
    """(dL/dlogits, dL/dv) of the actor loss B sum_j nlp_j (R - v_j) and the critic loss mean((v - R)^2), as the CUDA
    kernel forms them (R: a scalar)."""
    B = logits.shape[0]
    p = torch.softmax(logits, dim=-1)
    pa = p.gather(1, action.long().view(-1, 1)).view(-1)
    g = -((R - v) * B) / (pa + 1e-8)                       # dL/dp_a
    onehot = torch.nn.functional.one_hot(action.long(), logits.shape[1]).to(p.dtype)
    dlogits = p * (onehot * g.view(-1, 1) - (g * pa).view(-1, 1))
    dv = 2.0 * (v - R) / B
    return dlogits, dv


class OracleREINFORCE:
    def __init__(self, obs, n_actions, actor_hidden, critic_hidden, *, actor_lr=1e-4, critic_lr=1e-4, init_actor=None,
                 init_critic=None):
        self.obs, self.A = obs, n_actions
        self.actor = _mlp([obs] + list(actor_hidden) + [n_actions])      # softmax applied in `probs`
        self.critic = _mlp([obs] + list(critic_hidden) + [1])
        if init_actor is not None:
            load_flat(self.actor, init_actor)
        if init_critic is not None:
            load_flat(self.critic, init_critic)
        self.opt_actor = torch.optim.AdamW(self.actor.parameters(), lr=actor_lr, amsgrad=True)
        self.opt_critic = torch.optim.AdamW(self.critic.parameters(), lr=critic_lr, amsgrad=True)

    def set_learning_rates(self, actor_lr, critic_lr):
        self.opt_actor.param_groups[0]["lr"] = actor_lr
        self.opt_critic.param_groups[0]["lr"] = critic_lr

    def bootstrap(self, last_next_state, last_terminated) -> torch.Tensor:
        """critic(next_state of the newest transition).detach() * (~terminated): shape (1,)."""
        s = torch.as_tensor(last_next_state, dtype=torch.float32).reshape(-1)
        term = torch.as_tensor(bool(last_terminated)).reshape(1)
        with torch.no_grad():
            return self.critic(s).detach() * (~term)

    def returns(self, reward, last_next_state, last_terminated) -> torch.Tensor:
        return fold_returns(self.bootstrap(last_next_state, last_terminated), reward)

    def learn_batch(self, state, action, R) -> dict:
        """One ActorCriticBase.learn_batch on rows (state [B, O], action [B] ids) with every row's return R (shape (1,))."""
        B = state.shape[0]
        ret = R.reshape(1, 1).expand(B, 1).clone()                          # batch.cum_reward: (B, 1)
        onehot = torch.nn.functional.one_hot(action.long(), self.A).float()
        pa = torch.sum(torch.softmax(self.actor(state), dim=-1) * onehot, dim=1, keepdim=True).view(-1)
        nlp = -torch.log(pa + 1e-8)
        v = self.critic(state).view(-1)
        actor_loss = torch.sum(nlp * (ret - v.detach()))                      # (B,) * (B, 1): the B x B broadcast
        self.opt_actor.zero_grad()
        actor_loss.backward()
        self.opt_actor.step()
        vs = self.critic(state)
        critic_loss = torch.nn.MSELoss()(vs.reshape_as(ret), ret.detach())
        self.opt_critic.zero_grad()
        critic_loss.backward()
        self.opt_critic.step()
        return {"actor_loss": actor_loss.item(), "critic_loss": critic_loss.item()}

    def adam_state(self, which: str, key: str) -> torch.Tensor:
        opt, net = (self.opt_actor, self.actor) if which == "actor" else (self.opt_critic, self.critic)
        return torch.cat([opt.state[p][key].reshape(-1) for p in net.parameters()])
