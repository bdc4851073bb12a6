"""Eager-torch restatement of ThompsonSamplingExplorationLinear (policy_learners/exploration_modules/contextual_bandits/
thompson_sampling_exploration.py) over the ridge of LinearRegression, and its float64 yardstick.  TEST INFRASTRUCTURE:
nothing in pearl_b200 imports it."""
from __future__ import annotations

import torch

from oracle.bandit_oracle import ones_col


def precision(A: torch.Tensor, lam: float) -> torch.Tensor:
    """LinearRegression.A: _A + lambda eye, formed in fp32."""
    return A.float() + lam * torch.eye(A.shape[0], device=A.device)


def sample_theta(A: torch.Tensor, lam: float, coefs: torch.Tensor, eps: torch.Tensor, dtype=torch.float32) -> torch.Tensor:
    """MultivariateNormal(loc=coefs, precision_matrix=A + lambda I).sample() for the standard normals eps it draws:
    M = U U^T with U upper triangular (torch factors the index-reversed M), theta = coefs + U^-T eps.  In float64
    (dtype) from the same fp32 M, this is the yardstick the CUDA sampler is held to."""
    M = precision(A, lam).to(dtype)
    U = torch.flip(torch.linalg.cholesky(torch.flip(M, (-2, -1))), (-2, -1))
    x = torch.linalg.solve_triangular(U.t(), eps.to(dtype).reshape(-1, 1), upper=False).reshape(-1)
    return coefs.to(dtype) + x


def theta_scores(x: torch.Tensor, theta: torch.Tensor) -> torch.Tensor:
    """The default mode's scores over rows x [..., k]: [1, x] . theta."""
    return (ones_col(x.reshape(-1, x.shape[-1]).float()) @ theta.float()).reshape(x.shape[:-1])


def efficient_scores(inv_A: torch.Tensor, coefs: torch.Tensor, x: torch.Tensor, z: torch.Tensor) -> torch.Tensor:
    """enable_efficient_sampling: torch.normal(mean=mu, std=sigma) for the per-score standard normals z it draws, which
    torch evaluates as z * sigma, then + mu.  A NaN sigma raises, as torch.normal does."""
    x1 = ones_col(x.reshape(-1, x.shape[-1]).float())
    mu = x1 @ coefs.float()
    sigma = torch.sqrt(((x1 @ inv_A.float()) * x1).sum(-1))
    if bool(torch.isnan(sigma).any()):
        raise RuntimeError("normal expects all elements of std >= 0.0")
    return z.reshape(-1).float().mul(sigma).add(mu).reshape(x.shape[:-1])
