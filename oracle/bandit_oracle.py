"""Eager-torch restatement of LinearBandit's round and UCB scores (policy_learners/contextual_bandits/linear_bandit.py,
neural_networks/contextual_bandit/linear_regression.py), and the float64 yardstick the long-run tests hold the CUDA ridge
solve to.  TEST INFRASTRUCTURE: nothing in pearl_b200 imports it."""
from __future__ import annotations

import torch


def ones_col(x: torch.Tensor) -> torch.Tensor:
    return torch.cat([torch.ones(x.shape[0], 1, dtype=x.dtype, device=x.device), x], dim=1)


class Ridge:
    """The five buffers and last_sum_weight_when_discounted, fp32 like the reference's."""

    def __init__(self, d: int, lam: float, gamma: float = 1.0, interval: float = 0.0, coefs=None, device="cpu"):
        self.A = torch.zeros(d, d, device=device)
        self.b = torch.zeros(d, device=device)
        self.sum_weight = torch.zeros(1, device=device)
        self.inv_A = torch.zeros(d, d, device=device)
        self.coefs = torch.zeros(d, device=device) if coefs is None else torch.as_tensor(coefs, dtype=torch.float32).clone()
        self.lam, self.gamma, self.interval, self.last = lam, gamma, interval, 0.0

    def solve(self) -> None:
        M = self.A + self.lam * torch.eye(self.A.shape[0], device=self.A.device)
        self.inv_A = torch.linalg.inv(M)
        self.coefs = self.inv_A @ self.b

    def round(self, x: torch.Tensor, y: torch.Tensor, w=None) -> torch.Tensor:
        """LinearBandit.learn_batch on rows x (state || represented action): returns model(x) after the update."""
        x1 = ones_col(x.float())
        w = torch.ones(x.shape[0], device=x.device) if w is None else w.float().reshape(-1)
        dA = x1.t() @ (x1 * w[:, None])
        self.A += (dA + dA.t()) / 2
        self.b += x1.t() @ (y.float().reshape(-1) * w)
        self.sum_weight += w.sum()
        self.solve()
        if self.interval > 0 and self.sum_weight.item() - self.last >= self.interval:
            if self.gamma < 1:
                self.A *= self.gamma
                self.b *= self.gamma
            self.solve()
            self.last = self.sum_weight.item()
        return (x1 @ self.coefs).reshape(-1, 1)


def scores(inv_A: torch.Tensor, coefs: torch.Tensor, x: torch.Tensor, alpha: float, with_sigma: bool = True) -> torch.Tensor:
    """UCBExploration.get_scores over rows x [..., k]: mu + alpha sigma, NaN sigma -> 0 (or mu alone)."""
    x1 = ones_col(x.reshape(-1, x.shape[-1]).float())
    mu = x1 @ coefs
    if not with_sigma:
        return mu.reshape(x.shape[:-1])
    sigma = torch.sqrt(((x1 @ inv_A) * x1).sum(-1))
    sigma = torch.where(torch.isnan(sigma), torch.zeros_like(sigma), sigma)
    return (mu + alpha * sigma).reshape(x.shape[:-1])


def first_max(s: torch.Tensor, mask=None) -> torch.Tensor:
    """get_model_action_index_batch with NO_TIEBREAKING: the first maximum over the available positions."""
    if mask is not None:
        s = torch.where(mask.bool(), s, torch.tensor(-float("inf"), device=s.device))
    return torch.argmax(s, dim=-1)


def features(states: torch.Tensor, act_feat: torch.Tensor) -> torch.Tensor:
    """concatenate_actions_to_state: [n, obs] x [S, a] -> [n, S, obs + a]."""
    n, S = states.shape[0], act_feat.shape[0]
    return torch.cat([states[:, None, :].expand(n, S, -1), act_feat[None].expand(n, S, -1)], dim=-1)


def fp64_yardstick(A: torch.Tensor, b: torch.Tensor, lam: float):
    """inv(A + lambda I) and its product with b in float64, from the fp32 A + lambda I the solve starts from, with the
    2-norm condition number of that matrix."""
    M32 = A.float() + torch.tensor(lam, dtype=torch.float32) * torch.eye(A.shape[0], device=A.device)
    M = M32.double()
    inv = torch.linalg.inv(M)
    return inv, inv @ b.double(), float(torch.linalg.cond(M))
