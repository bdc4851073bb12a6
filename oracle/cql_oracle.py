"""oracle/cql_oracle.py — CPU restatement of conservative DQN / DoubleDQN (`is_conservative=True`)
(TEST INFRASTRUCTURE ONLY; eager PyTorch fp32 like the reference).

Restated reference sites (paths relative to the Pearl source tree):
  policy_learners/sequential_decision_making/deep_td_learning.py:269-360   forward (target update first), loss, learn_batch
  policy_learners/sequential_decision_making/deep_q_learning.py:130-167    DQN next-state values
  policy_learners/sequential_decision_making/double_dqn.py:29-57           DoubleDQN next-state values
  utils/functional_utils/learning/loss_fn_utils.py:17-71                   compute_cql_loss
Per round: when (training_steps + 1) % target_update_freq == 0 the soft target update with the CURRENT online parameters;
q = Q(s, a); y = V gamma (1 - terminated) + r; loss = MSE(q, y) + alpha * cql with

    cql = mean_b logsumexp_k Q(s_b, c_b[k]) - mean(Q_all.gather(1, batch.action.long()))

where batch.action is ALREADY ONE-HOT (preprocess_batch), so the gather reads column 0 in A - 1 places and column 1 in one
place of every row, whatever the taken action; c_b[k] are the current slots padded with action id 0 (the unavailable mask
is ignored, so padded slots count).  One AdamW(amsgrad) step; reported loss mean |q - y|.  `cql_grad` is that term's
gradient on the all-slot values written out, held to torch.autograd by the tests.  Parity with the reference is pinned by
tests/golden/cql_*.npz (oracle/gen_cql_golden.py).
"""
from __future__ import annotations

import torch
import torch.nn.functional as F

from .pearl_oracle import OracleDQN, flat, load_flat  # noqa: F401


def cql_term(q_all, action_one_hot):
    """compute_cql_loss on the current-slot values q_all [B, A] with the batch's one-hot actions [B, A]."""
    return torch.logsumexp(q_all, dim=-1).mean() - q_all.gather(1, action_one_hot.long()).mean()


def cql_grad(q_all, alpha):
    """d(alpha * cql_term) / d q_all written out: alpha (softmax_k / B - [k = 0] (A - 1) / (B A) - [k = 1] / (B A)).  It does
    not depend on the taken action (A >= 2)."""
    B, A = q_all.shape
    n = torch.zeros(A, dtype=q_all.dtype)
    n[0], n[1] = A - 1, 1
    return alpha * (torch.softmax(q_all, dim=-1) / B - n.view(1, A) / (B * A))


class OracleCQL(OracleDQN):
    """DeepQLearning / DoubleDQN with is_conservative=True.  `learn_batch(b)` takes the batch as preprocess_batch leaves
    it: state [B, O], action one-hot [B, A], reward [B], next_state [B, O], terminated [B] bool, curr_available_actions
    one-hot [B, A, A] (padding included), next_available_actions one-hot [B, A, A], next_unavailable_actions_mask [B, A]
    bool; alpha is `self.alpha`, the update schedule `self.training_steps` (the caller keeps the reference's count)."""

    def __init__(self, *args, alpha: float = 2.0, **kw) -> None:
        super().__init__(*args, **kw)
        self.alpha = alpha

    def next_values(self, b):
        return self._next_values(b)

    def learn_batch(self, b) -> float:
        if (self.training_steps + 1) % self.target_update_freq == 0:      # deep_td_learning.py forward: update first
            with torch.no_grad():
                for pt, p in zip(self.Qt.parameters(), self.Q.parameters()):
                    pt.copy_(self.tau * p + (1.0 - self.tau) * pt)
        q = self._q_values(self.Q, b["state"], b["action"])
        y = self._next_values(b) * self.gamma * (1 - b["terminated"].float()) + b["reward"]
        bellman = torch.nn.MSELoss()(q, y)
        B = q.shape[0]
        q_all = self._q_values(self.Q, b["state"], b["curr_available_actions"]).view(B, -1)
        loss = self.alpha * cql_term(q_all, b["action"]) + bellman
        self.opt.zero_grad()
        loss.backward()
        self.opt.step()
        return torch.abs(q - y).mean().item()


def one_hot_batch(A, state, action, reward, next_state, terminated, curr_ids=None, next_ids=None, next_count=None):
    """The batch preprocess_batch hands learn_batch, from ids: curr_ids / next_ids [B, A] padded with 0 (None: every
    action), next_count [B] (slots at and beyond it are unavailable)."""
    B = state.shape[0]
    full = torch.arange(A).view(1, A).expand(B, A)
    curr = full if curr_ids is None else torch.as_tensor(curr_ids).long()
    nxt = full if next_ids is None else torch.as_tensor(next_ids).long()
    cnt = torch.full((B,), A) if next_count is None else torch.as_tensor(next_count).long()
    oh = lambda x: F.one_hot(x, A).float()  # noqa: E731
    return dict(state=torch.as_tensor(state), action=oh(torch.as_tensor(action).long()), reward=torch.as_tensor(reward),
                next_state=torch.as_tensor(next_state), terminated=torch.as_tensor(terminated), curr_available_actions=oh(curr),
                next_available_actions=oh(nxt), next_unavailable_actions_mask=torch.arange(A).view(1, A) >= cnt.view(-1, 1))
