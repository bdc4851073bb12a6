"""oracle/dueling_oracle.py — CPU restatement of dueling DQN / DoubleDQN (`network_type=DuelingQValueNetwork`)
(TEST INFRASTRUCTURE ONLY; eager PyTorch fp32 like the reference).

Restated reference sites (paths relative to the Pearl source tree):
  neural_networks/sequential_decision_making/q_value_networks.py:352-510    DuelingQValueNetwork, get_q_values
  policy_learners/sequential_decision_making/deep_td_learning.py:200-360   act, forward (target update first), loss, learn_batch
  policy_learners/sequential_decision_making/deep_q_learning.py:130-167    DQN next-state values
  policy_learners/sequential_decision_making/double_dqn.py:29-57           DoubleDQN next-state values
get_q_values(s, a, curr) = fl(fl(V(s) + Adv(s, a)) - mean Adv(s, .)), the mean over `curr` when given (all its slots,
padding included, the unavailable mask ignored) and over the query actions `a` otherwise.  So:
  forward with current sets:     mean over the A current slots; the taken action's advantage is its own row
  forward without current sets:  mean over the query alone, q = fl(fl(V + Adv) - Adv)
  DQN target:                    query = all A next slots (masked ones with the id they hold), then the masked max
  DoubleDQN target:              the online net over all A next slots picks a*; the target is called with the 2-D query
                                 a*, so V' = fl(fl(V_t + Adv_t(a*)) - Adv_t(a*))
  act:                           query = the available actions, the mean over them
`slot_grad` writes out the gradient of q at the advantage rows (+dq on the taken row, -dq / A on every current slot), held
to torch.autograd by the tests.  Parity with the reference is pinned by tests/golden/duel_*.npz (oracle/gen_dueling_golden.py).
"""
from __future__ import annotations

import torch
import torch.nn.functional as F

from .cql_oracle import one_hot_batch  # noqa: F401
from .pearl_oracle import OracleDQN, _mlp, flat, load_flat  # noqa: F401


class DuelNet(torch.nn.Module):
    """The three MLPs in the reference's parameter order (state, value, advantage; mlp_block each)."""

    def __init__(self, obs, A, hidden) -> None:
        super().__init__()
        h, Fd = list(hidden), hidden[-1]
        self.state_arch = _mlp([obs] + h + [Fd])
        self.value_arch = _mlp([Fd] + h + [1])
        self.advantage_arch = _mlp([Fd + A] + h + [1])


def get_q_values(net, state, action, curr=None):
    """DuelingQValueNetwork.get_q_values, step for step (one-hot actions [B, A] or [B, n, A])."""
    ext = action.unsqueeze(1) if action.dim() == 2 else action
    feat = net.state_arch(state)
    value = net.value_arch(feat)
    nq = ext.shape[1]
    n = nq if curr is None or nq > curr.shape[1] else curr.shape[1]
    ef = torch.repeat_interleave(feat.unsqueeze(1), n, dim=1)
    adv = net.advantage_arch(torch.cat((ef[:, :nq, :], ext), dim=-1)).squeeze(-1)
    if curr is None:
        mean = torch.mean(adv, dim=-1, keepdim=True)
    else:
        mean = torch.mean(net.advantage_arch(torch.cat((ef[:, :curr.shape[1], :], curr), dim=-1)).squeeze(-1), dim=-1, keepdim=True)
    q = value + adv - mean
    return q if action.dim() == 3 else q.squeeze(-1)


def slot_grad(dq, A, query_alone=False):
    """d q_b / d Adv written out for an upstream gradient dq [B]: (taken row [B], current slots [B, A])."""
    if query_alone:
        return torch.zeros_like(dq), torch.zeros(dq.shape[0], A, dtype=dq.dtype)
    return dq.clone(), (-dq / A).view(-1, 1).expand(-1, A).clone()


class OracleDueling(OracleDQN):
    """DeepQLearning / DoubleDQN with a DuelingQValueNetwork.  `learn_batch(b)` takes the batch as preprocess_batch leaves
    it (one_hot_batch); b["curr_available_actions"] None means the batch has no current sets.  The update schedule is
    `self.training_steps` (the caller keeps the reference's count)."""

    def __init__(self, obs, n_actions, hidden, *, init_q=None, init_q_target=None, **kw) -> None:
        super().__init__(obs, n_actions, hidden, **kw)
        self.Q, self.Qt = DuelNet(obs, n_actions, hidden), DuelNet(obs, n_actions, hidden)
        if init_q is not None:
            load_flat(self.Q, init_q)
        load_flat(self.Qt, init_q_target if init_q_target is not None else flat(self.Q))
        self.opt = torch.optim.AdamW(self.Q.parameters(), lr=kw.get("lr", 1e-3), amsgrad=True, weight_decay=kw.get("weight_decay", 0.01))

    def _q_values(self, net, state, action):
        return get_q_values(net, state, action)

    def q_values(self, state, ids, target=False):
        """act's values: the query (and the mean) is the row's id set [n, K]."""
        with torch.no_grad():
            return get_q_values(self.Qt if target else self.Q, state, F.one_hot(torch.as_tensor(ids).long(), self.A).float())

    def learn_batch(self, b) -> float:
        if (self.training_steps + 1) % self.target_update_freq == 0:      # deep_td_learning.py forward: update first
            with torch.no_grad():
                for pt, p in zip(self.Qt.parameters(), self.Q.parameters()):
                    pt.copy_(self.tau * p + (1.0 - self.tau) * pt)
        q = get_q_values(self.Q, b["state"], b["action"], b.get("curr_available_actions"))
        y = self._next_values(b) * self.gamma * (1 - b["terminated"].float()) + b["reward"]
        loss = torch.nn.MSELoss()(q, y)
        self.opt.zero_grad()
        loss.backward()
        self.opt.step()
        return torch.abs(q - y).mean().item()
