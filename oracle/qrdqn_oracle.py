"""oracle/qrdqn_oracle.py — CPU restatement of Quantile Regression DQN's `learn_batch`
(TEST INFRASTRUCTURE ONLY; eager PyTorch fp32 like the reference).

Restated reference sites (paths relative to the Pearl source tree):
  policy_learners/sequential_decision_making/quantile_regression_deep_td_learning.py   learn_batch
  policy_learners/sequential_decision_making/quantile_regression_deep_q_learning.py    _get_next_state_quantiles
  neural_networks/sequential_decision_making/q_value_networks.py                       QuantileQValueNetwork
  safety_modules/risk_sensitive_safety_modules.py        RiskNeutralSafetyModule, QuantileNetworkMeanVarianceSafetyModule
  utils/functional_utils/learning/loss_fn_utils.py                                     compute_elementwise_huber_loss
Per round: theta(s, a) of the online net; the target net's quantiles at every next slot; the greedy slot under
mean - beta * variance with masked slots at -inf (first argmax); T = theta'(s', g) * gamma * (1 - terminated) + r; the
pairwise quantile-Huber loss summed over the TARGET index and averaged over (batch, theta index); one AdamW(amsgrad) step;
then the soft target update with the new parameters when `update_target` (the caller evaluates
(training_steps + 1) % target_update_freq == 0).  beta is an input.  `quantile_grad` is the hand-written gradient of the
loss with respect to theta, held to torch.autograd in float64 by the tests.  Parity with the reference is pinned by
tests/golden/qrdqn_*.npz (oracle/gen_qrdqn_golden.py).
"""
from __future__ import annotations

import torch

from .pearl_oracle import _mlp, flat, load_flat  # noqa: F401


def quantile_grid(N: int, dtype=torch.float32):
    """(w, tau_hat): w_j = q[j+1] - q[j] and the midpoints (q[i+1] + q[i]) / 2 of q = arange(N + 1) / N, as the reference
    computes them."""
    q = torch.arange(0, N + 1) / N
    return (q[1:] - q[:-1]).to(dtype), ((q[1:] + q[:-1]) / 2).to(dtype)


def risk_values(quantiles, beta: float):
    """QuantileNetworkMeanVarianceSafetyModule.get_q_values_under_risk_metric on quantiles [..., N]."""
    w, _ = quantile_grid(quantiles.shape[-1], quantiles.dtype)
    mean = quantiles.mean(dim=-1, keepdim=True)
    var = (w * torch.square(quantiles - mean)).sum(dim=-1, keepdim=True)
    return (mean - beta * var).squeeze(-1)


def quantile_loss(theta, target):
    """The reference's quantile Bellman loss of theta [B, N] against target [B, N] (target treated as a constant)."""
    _, tau = quantile_grid(theta.shape[-1], theta.dtype)
    u = target.unsqueeze(2) - theta.unsqueeze(1)                       # u[b, j, i] = T_j - theta_i
    huber = torch.where(torch.abs(u) <= 1.0, 0.5 * u.pow(2), 1.0 * (torch.abs(u) - 0.5))
    with torch.no_grad():
        w = torch.abs(tau.view(1, 1, -1) - (u < 0).to(theta.dtype))
    return (w * huber).sum(dim=1).mean()


def quantile_grad(theta, target):
    """d quantile_loss / d theta written out: -(1 / (B N)) sum_j |tau_i - 1{u < 0}| h'(u), h'(u) = u if |u| <= 1 else
    sign(u)."""
    B, N = theta.shape
    _, tau = quantile_grid(N, theta.dtype)
    u = target.unsqueeze(2) - theta.unsqueeze(1)
    w = torch.abs(tau.view(1, 1, -1) - (u < 0).to(theta.dtype))
    hp = torch.where(torch.abs(u) <= 1.0, u, torch.sign(u))
    return -(w * hp).sum(dim=1) / (B * N)


class OracleQRDQN:
    def __init__(self, obs, n_actions, hidden, num_quantiles, *, lr=5e-4, gamma=0.99, tau=0.05, init=None, init_target=None):
        self.A, self.N, self.gamma, self.tau = int(n_actions), int(num_quantiles), gamma, tau
        self.q = _mlp([obs + self.A] + list(hidden) + [self.N])
        self.qt = _mlp([obs + self.A] + list(hidden) + [self.N])
        if init is not None:
            load_flat(self.q, init)
            load_flat(self.qt, init if init_target is None else init_target)
        else:
            self.qt.load_state_dict(self.q.state_dict())
        self.opt = torch.optim.AdamW(self.q.parameters(), lr=lr, amsgrad=True)

    def set_learning_rate(self, lr):
        self.opt.param_groups[0]["lr"] = lr

    def _quantiles(self, net, s, ids):
        """net(s || one-hot(ids)) for ids [B] -> [B, N] or ids [B, K] -> [B, K, N]."""
        oh = torch.nn.functional.one_hot(ids.long(), self.A).float()
        if ids.dim() == 1:
            return net(torch.cat([s, oh], dim=-1))
        return net(torch.cat([s.unsqueeze(1).expand(-1, ids.shape[1], -1), oh], dim=-1))

    def target(self, b, beta):
        """(T [B, N], greedy slot [B], risk values [B, A] with masked slots at -inf) from the current target net."""
        with torch.no_grad():
            qn = self._quantiles(self.qt, b["next_state"], b["next_ids"])          # [B, A, N]
            rho = risk_values(qn, beta)
            rho[b["next_mask"]] = -float("inf")
            g = torch.argmax(rho, dim=-1)
            sel = torch.gather(qn, 1, g.view(-1, 1, 1).expand(-1, 1, self.N)).view(-1, self.N)
            T = sel * self.gamma * (1 - b["terminated"].float()).unsqueeze(-1) + b["reward"].unsqueeze(-1)
        return T, g, rho

    def learn_batch(self, b, beta, update_target):
        """b: state [B, O], action [B] int, reward [B], next_state [B, O], terminated [B] bool, next_ids [B, A] int (slot k
        holds id_k), next_mask [B, A] bool (True = unavailable).  Returns the reported loss mean |theta - T|."""
        theta = self._quantiles(self.q, b["state"], b["action"])
        T, _, _ = self.target(b, beta)
        loss = quantile_loss(theta, T)
        self.opt.zero_grad()
        loss.backward()
        self.opt.step()
        if update_target:
            with torch.no_grad():
                for pt, p in zip(self.qt.parameters(), self.q.parameters()):
                    pt.copy_(self.tau * p.data + (1.0 - self.tau) * pt.data)
        return torch.abs(theta - T).mean().item()
