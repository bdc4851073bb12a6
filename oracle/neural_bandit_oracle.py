"""Eager-torch restatement of NeuralBandit's round (policy_learners/contextual_bandits/neural_bandit.py learn_batch over
VanillaValueNetwork with two hidden layers) on a flat parameter vector, and of the SquareCB / FastCB action rule
(exploration_modules/contextual_bandits/squarecb_exploration.py) with the sample taken as torch's one-sample multinomial
takes it.  TEST INFRASTRUCTURE: nothing in pearl_b200 imports it."""
from __future__ import annotations

import torch


def shapes(f: int, h1: int, h2: int):
    """torch's parameters() order: W1 b1 W2 b2 W3 b3."""
    return [(h1, f), (h1,), (h2, h1), (h2,), (1, h2), (1,)]


def unflatten(flat: torch.Tensor, f: int, h1: int, h2: int):
    out, off = [], 0
    for s in shapes(f, h1, h2):
        n = int(torch.tensor(s).prod())
        out.append(flat[off:off + n].view(s).clone())
        off += n
    return out


def value(p, x: torch.Tensor) -> torch.Tensor:
    """VanillaValueNetwork: Linear+ReLU, Linear+ReLU, Linear -> [rows, 1]."""
    h = torch.relu(x @ p[0].t() + p[1])
    h = torch.relu(h @ p[2].t() + p[3])
    return h @ p[4].t() + p[5]


class NeuralBandit:
    """Parameters and torch's AdamW(amsgrad=True) over them."""

    def __init__(self, flat, f, h1, h2, *, lr, loss="mse"):
        self.p = [t.requires_grad_() for t in unflatten(torch.as_tensor(flat, dtype=torch.float32), f, h1, h2)]
        self.opt = torch.optim.AdamW(self.p, lr=lr, amsgrad=True)
        self.loss = loss

    def round(self, x: torch.Tensor, y: torch.Tensor, w=None):
        """One learn_batch: returns (prediction [B, 1], loss).  No short circuit on sum(w) = 0, as the reference."""
        y = y.float().reshape(-1)
        w = torch.ones_like(y) if w is None else w.float().reshape(-1)
        pred = value(self.p, x.float())
        fn = {"mse": torch.nn.functional.mse_loss, "mae": torch.nn.functional.l1_loss}[self.loss]
        loss = (fn(pred.view(y.shape), y, reduction="none") * w).sum() / w.sum()
        self.opt.zero_grad()
        loss.backward()
        self.opt.step()
        return pred.detach(), loss.detach()

    def flat(self) -> torch.Tensor:
        return torch.cat([t.detach().reshape(-1) for t in self.p])


def explore(values: torch.Tensor, *, fastcb: bool, gamma: float, lb: float = 0.0, ub: float = 1.0, clamp: bool = False,
            E: torch.Tensor):
    """SquareCB / FastCB act on one state's fp32 values with the exponential draws E: (p handed to Categorical, its
    normalised probs, the chosen index), in the reference's order of operations."""
    A = values.numel()
    v = values.float().reshape(1, A)
    if clamp or fastcb:
        v = torch.clamp(v, min=lb, max=ub)
    mx, im = torch.max(v, dim=1)
    gaps = mx - v
    if not fastcb:
        p = torch.div(1.0, A + gamma * gaps)
    elif mx <= lb:
        p = torch.ones(gaps.shape) / A
    else:
        p = torch.div(mx - lb, A * (mx - lb) + gamma * gaps)
    p[0, im[0]] = 0.0
    p[0, im[0]] = 1.0 - torch.sum(p)
    p = p[0]
    pn = p / p.sum(-1, keepdim=True)
    return p, pn, int(torch.argmax(pn / E.float()))
