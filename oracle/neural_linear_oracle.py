"""Eager-torch restatement of NeuralLinearBandit's round (policy_learners/contextual_bandits/neural_linear_bandit.py
learn_batch over neural_networks/contextual_bandit/neural_linear_regression.py) on a flat parameter vector, for two
hidden layers.  TEST INFRASTRUCTURE: nothing in pearl_b200 imports it."""
from __future__ import annotations

import torch

from oracle.bandit_oracle import Ridge, ones_col


def shapes(f: int, h1: int, h2: int):
    """torch's parameters() order: W1 b1 W2 b2 W3 b3, then linear_layer_e2e.weight."""
    return [(h1, f), (h1,), (h2, h1), (h2,), (h2, h2), (h2,), (1, h2)]


def unflatten(flat: torch.Tensor, f: int, h1: int, h2: int):
    out, off = [], 0
    for s in shapes(f, h1, h2):
        n = int(torch.tensor(s).prod())
        out.append(flat[off:off + n].view(s).clone())
        off += n
    return out


def nn_output(p, x: torch.Tensor, skip: bool) -> torch.Tensor:
    """mlp_block(f, [h1, h2], output_dim=h2): ReLU hidden layers, x + layer(x) where widths agree when skip."""
    h = x
    for i, relu in ((0, True), (2, True), (4, False)):
        z = h @ p[i].t() + p[i + 1]
        z = torch.relu(z) if relu else z
        h = h + z if skip and p[i].shape[0] == p[i].shape[1] else z
    return h


class NeuralLinear:
    """Parameters, torch's AdamW(amsgrad=True) over them and the ridge of oracle/bandit_oracle.py."""

    def __init__(self, flat, f, h1, h2, *, lr, skip=False, e2e=True, loss="mse", sigmoid=False, lam=1.0, gamma=1.0,
                 interval=0.0):
        self.p = [t.requires_grad_() for t in unflatten(torch.as_tensor(flat, dtype=torch.float32), f, h1, h2)]
        self.opt = torch.optim.AdamW(self.p, lr=lr, amsgrad=True)
        self.ridge = Ridge(h2 + 1, lam, gamma, interval)
        self.skip, self.e2e, self.loss, self.sigmoid = skip, e2e, loss, sigmoid

    def round(self, x: torch.Tensor, y: torch.Tensor, w=None):
        """One learn_batch: returns (prediction, loss)."""
        y = y.float().reshape(-1, 1)
        w = torch.ones_like(y) if w is None else w.float().reshape(-1, 1)
        n = nn_output(self.p, x.float(), self.skip)
        mu = n @ self.p[6].t() if self.e2e else (ones_col(n) @ self.ridge.coefs).reshape(-1, 1)
        pred = torch.sigmoid(mu) if self.sigmoid else mu
        if float(w.sum()) == 0:
            loss = torch.tensor(0.0)
        else:
            fn = {"mse": torch.nn.functional.mse_loss, "mae": torch.nn.functional.l1_loss,
                  "cross_entropy": torch.nn.functional.binary_cross_entropy}[self.loss]
            loss = (fn(pred, y, reduction="none") * w).sum() / w.sum()
            self.opt.zero_grad()
            loss.backward()
            self.opt.step()
        self.ridge.round(n.detach(), y, w)
        return pred.detach(), loss.detach()

    def flat(self) -> torch.Tensor:
        return torch.cat([t.detach().reshape(-1) for t in self.p])
