"""oracle/multihead_oracle.py — CPU restatement of multi-head DQN / DoubleDQN (`network_type=VanillaQValueMultiHeadNetwork`),
plain or conservative (TEST INFRASTRUCTURE ONLY; eager PyTorch fp32 like the reference).

Restated reference sites (paths relative to the Pearl source tree):
  neural_networks/sequential_decision_making/q_value_networks.py:185-241   VanillaQValueMultiHeadNetwork, get_q_values
  policy_learners/sequential_decision_making/deep_td_learning.py:200-360   act, forward (target update first), loss, learn_batch
  policy_learners/sequential_decision_making/deep_q_learning.py:130-167    DQN next-state values
  policy_learners/sequential_decision_making/double_dqn.py:29-57           DoubleDQN next-state values
  utils/functional_utils/learning/loss_fn_utils.py:17-71                   compute_cql_loss
The network is mlp_block(obs, hidden, A); get_q_values(s, slots) = bmm(one-hot slots, Q(s)), so a slot holding id k reads
Q(s)[k].  Per round: when (training_steps + 1) % target_update_freq == 0 the soft target update with the CURRENT online
parameters; q = Q(s)[a]; y = V gamma (1 - terminated) + r; loss = MSE(q, y) (+ alpha * cql_term when conservative, the
reference's CQL term, cql_oracle.py); one AdamW(amsgrad) step; reported loss mean |q - y|.  `head_grad` writes out the
gradient at the head outputs Q(s_b)[j], held to torch.autograd by the tests.  Parity with the reference is pinned by
tests/golden/mh_*.npz (oracle/gen_multihead_golden.py).
"""
from __future__ import annotations

import torch

from .cql_oracle import cql_grad, cql_term, one_hot_batch  # noqa: F401
from .pearl_oracle import OracleDQN, _mlp, flat, load_flat  # noqa: F401


def get_q_values(net, state, action):
    """VanillaQValueMultiHeadNetwork.get_q_values, step for step (one-hot slots [B, A] or [B, n, A])."""
    ext = action.unsqueeze(1) if action.dim() == 2 else action
    q = torch.bmm(ext, net(state).unsqueeze(-1)).squeeze(-1)
    return q if action.dim() == 3 else q.squeeze(-1)


def head_grad(q_head, action, curr_ids, dq, alpha=None):
    """d loss / d Q(s_b)[j] written out, [B, A]: dq_b at column a_b (dq = 2 (q - y) / B), plus, when `alpha` is given, the
    CQL slot gradients alpha (softmax_k / B - n_k / (B A)) of the current slots c_b[k] (curr_ids [B, A], padding included)
    added on the column of the id each slot holds, slots in ascending order."""
    B, A = q_head.shape
    g = torch.zeros(B, A, dtype=q_head.dtype)
    if alpha is not None:
        cids = torch.as_tensor(curr_ids).long()
        gs = cql_grad(q_head.gather(1, cids), alpha)
        for k in range(A):
            g[torch.arange(B), cids[:, k]] += gs[:, k]
    g[torch.arange(B), torch.as_tensor(action).long()] += dq
    return g


class OracleMultiHead(OracleDQN):
    """DeepQLearning / DoubleDQN with a VanillaQValueMultiHeadNetwork; conservative when `alpha` is not None.
    `learn_batch(b)` takes the batch as preprocess_batch leaves it (one_hot_batch); the update schedule is
    `self.training_steps` (the caller keeps the reference's count)."""

    def __init__(self, obs, n_actions, hidden, *, alpha=None, init_q=None, init_q_target=None, **kw) -> None:
        super().__init__(obs, n_actions, hidden, **kw)
        self.alpha = alpha
        self.Q, self.Qt = _mlp([obs] + list(hidden) + [n_actions]), _mlp([obs] + list(hidden) + [n_actions])
        if init_q is not None:
            load_flat(self.Q, init_q)
        load_flat(self.Qt, init_q_target if init_q_target is not None else flat(self.Q))
        self.opt = torch.optim.AdamW(self.Q.parameters(), lr=kw.get("lr", 1e-3), amsgrad=True, weight_decay=kw.get("weight_decay", 0.01))

    def _q_values(self, net, state, action):
        return get_q_values(net, state, action)

    def q_values(self, state, target=False):
        """Q(s)[a] for every action (what act() ranks over the available ids)."""
        with torch.no_grad():
            return (self.Qt if target else self.Q)(torch.as_tensor(state))

    def learn_batch(self, b) -> float:
        if (self.training_steps + 1) % self.target_update_freq == 0:      # deep_td_learning.py forward: update first
            with torch.no_grad():
                for pt, p in zip(self.Qt.parameters(), self.Q.parameters()):
                    pt.copy_(self.tau * p + (1.0 - self.tau) * pt)
        q = get_q_values(self.Q, b["state"], b["action"])
        y = self._next_values(b) * self.gamma * (1 - b["terminated"].float()) + b["reward"]
        loss = torch.nn.MSELoss()(q, y)
        if self.alpha is not None:
            B = q.shape[0]
            q_all = get_q_values(self.Q, b["state"], b["curr_available_actions"]).view(B, -1)
            loss = self.alpha * cql_term(q_all, b["action"]) + loss
        self.opt.zero_grad()
        loss.backward()
        self.opt.step()
        return torch.abs(q - y).mean().item()
