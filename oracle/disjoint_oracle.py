"""Eager-torch restatement of Pearl's disjoint linear bandits (policy_learners/contextual_bandits/disjoint_bandit.py with
LinearBandit arms, disjoint_linear_bandit.py) and of their disjoint explorers (ucb_exploration.py DisjointUCBExploration,
thompson_sampling_exploration.py ThompsonSamplingExplorationLinearDisjoint), on the per-arm Ridge of bandit_oracle.py.
TEST INFRASTRUCTURE: nothing in pearl_b200 imports it.

Routing:
  container   row -> arm `action` (ids outside [0, K) are the reference's AssertionError); an arm without rows learns the
              null batch (one zero row of weight 0), so it still solves and takes its discounting decision, and reports
              (coefs[0], label 0, weight 0); a 3-D state (B, K, f) gives arm k the rows state[:, k]
  linear      row -> arm k when action == k; rows of no arm dropped; an arm without rows is skipped (no solve); x = state,
              or state || space[k] (space[k] = [k]); no discounting
Scores: UCB mu_k + alpha sigma_k in the natural (n, K) layout; Thompson x . theta_k stacked (K, n) and read as (n, K).
"""
from __future__ import annotations

import torch

from oracle.bandit_oracle import Ridge, ones_col


class Disjoint:
    def __init__(self, K: int, d: int, lams, gammas=None, intervals=None, coefs=None, linear: bool = False):
        gammas = gammas if gammas is not None else [1.0] * K
        intervals = intervals if intervals is not None else [0.0] * K
        coefs = coefs if coefs is not None else [None] * K
        self.K, self.d, self.linear = K, d, linear
        self.arms = [Ridge(d, float(lams[k]), float(gammas[k]), float(intervals[k]), coefs[k]) for k in range(K)]

    def rows(self, state: torch.Tensor, k: int, sel: torch.Tensor, act_feat=None) -> torch.Tensor:
        x = state[:, k, :] if state.dim() == 3 else state
        x = x[sel]
        if act_feat is not None:
            x = torch.cat([x, act_feat[k].reshape(1, -1).expand(x.shape[0], -1)], dim=1)
        return x

    def round(self, state, action, reward, weight=None, act_feat=None) -> dict:
        """One learn_batch.  Container: {k: (prediction, label, weight)}; linear: {} (the reference reports nothing)."""
        state = state.float()
        action = action.reshape(action.shape[0], -1)[:, 0]
        reward = reward.float().reshape(-1)
        w = None if weight is None else weight.float().reshape(-1)
        out = {}
        for k, r in enumerate(self.arms):
            sel = action == k
            if int(sel.sum()) == 0:
                if self.linear:
                    continue
                x = torch.zeros(1, self.d - 1)
                out[k] = (r.round(x, torch.zeros(1), torch.zeros(1)), torch.zeros(1, 1), torch.zeros(1, 1))
                continue
            x = self.rows(state, k, sel, act_feat)
            wk = w[sel] if w is not None else torch.ones(int(sel.sum()))
            if self.linear:
                r.interval = 0.0
            p = r.round(x, reward[sel], wk)
            out[k] = (p, reward[sel].reshape(-1, 1), wk.reshape(-1, 1))
        return {} if self.linear else out

    def scores(self, states: torch.Tensor, alpha: float, with_sigma: bool = True, act_feat=None) -> torch.Tensor:
        """DisjointUCBExploration.get_scores (or ensemble_forward's mu): (n, K)."""
        cols = []
        for k, r in enumerate(self.arms):
            x = states if act_feat is None else torch.cat([states, act_feat[k].reshape(1, -1).expand(states.shape[0], -1)], 1)
            x1 = ones_col(x.float())
            mu = x1 @ r.coefs
            if with_sigma:
                s = torch.sqrt(((x1 @ r.inv_A) * x1).sum(-1))
                mu = mu + alpha * torch.where(torch.isnan(s), torch.zeros_like(s), s)
            cols.append(mu)
        return torch.stack(cols, dim=-1)

    def draws(self) -> torch.Tensor:
        """The reference's standard normals: K separate draws of d, in arm order ([K][d])."""
        return torch.stack([torch.empty(self.d).normal_() for _ in range(self.K)])

    def thetas(self, eps: torch.Tensor) -> torch.Tensor:
        """theta_k = coefs_k + U_k^-T eps_k with A_k + lambda_k I = U U^T, the sampler's float64 restatement."""
        out = []
        for k, r in enumerate(self.arms):
            M = (r.A + torch.tensor(r.lam, dtype=torch.float32) * torch.eye(self.d)).double()
            L = torch.linalg.cholesky(torch.flip(M, (0, 1)))
            U = torch.flip(L, (0, 1))
            x = torch.linalg.solve_triangular(U.t(), eps[k].double().reshape(-1, 1), upper=False).reshape(-1)
            out.append((r.coefs.double() + x).float())
        return torch.stack(out)

    def ts_scores(self, states: torch.Tensor, theta: torch.Tensor, act_feat=None) -> torch.Tensor:
        """x1 . theta_k per arm, stacked (K, n) and viewed (n, K), as the reference does."""
        rows = []
        for k in range(self.K):
            x = states if act_feat is None else torch.cat([states, act_feat[k].reshape(1, -1).expand(states.shape[0], -1)], 1)
            rows.append(ones_col(x.float()) @ theta[k])
        return torch.stack(rows).reshape(-1, self.K)
