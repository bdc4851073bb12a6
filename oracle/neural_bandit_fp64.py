"""The float64 gradient step of NeuralBandit's round (csrc/neural_bandit.cu), written out by hand rather than through
autograd, so that it can also be evaluated on absolute values: `step(..., absolute=True)` returns, for every value, the
sum of |a||b| over every product that reached it (the scale an fp32 rounding error is measured against).  The network
pieces are neural_linear_fp64.forward's (no skip connections; W3 has one row).  TEST INFRASTRUCTURE: nothing in
pearl_b200 imports it.

Parameters `p` = [W1, b1, W2, b2, W3, b3] (torch's parameters() order).  p = the network's output; the loss
sum(w l) / sum(w) with l = (p - y)^2 or |p - y|, and the gradient in torch's backward forms (2 (p - y), sign(p - y))."""
from __future__ import annotations

import torch

from oracle.neural_linear_fp64 import forward

BLOCKS = ("dW1", "db1", "dW2", "db2", "dW3", "db3")


def step(p, X, y, w, *, loss: str, absolute: bool = False):
    """The gradient of one round: dict of the blocks in BLOCKS, plus `pred`, `loss` and the pre-activations Z1, Z2.
    absolute=True: the scales of the same quantities.  Weights may have either sign; the scale of w / sum(w) then carries
    sum |w| / |sum w|, the factor by which the rounding of sum(w) is magnified."""
    sig = forward(p, X, False)
    m = [(sig["Z1"] > 0).to(X.dtype), (sig["Z2"] > 0).to(X.dtype)]
    fw = forward(p, X, False, True, m) if absolute else sig
    W2, W3 = (p[2].abs(), p[4].abs()) if absolute else (p[2], p[4])
    pr = sig["N"].reshape(-1)
    e = pr - y
    l, g = (e * e, 2 * e) if loss == "mse" else (e.abs(), torch.sign(e))
    if absolute:
        g = 2 * (fw["N"].reshape(-1) + y.abs()) if loss == "mse" else torch.ones_like(g)
        gm = g * w.abs() / w.sum().abs() * (w.abs().sum() / w.sum().abs())
    else:
        gm = g * w / w.sum()
    Xs = X.abs() if absolute else X
    dN = gm[:, None]
    out = dict(pred=fw["N"].reshape(-1), loss=(l * w).sum() / w.sum(), Z1=fw["Z1"], Z2=fw["Z2"])
    out["dW3"], out["db3"] = dN.t() @ fw["H2"], dN.sum(0)
    gZ2 = (dN @ W3) * m[1]
    out["dW2"], out["db2"] = gZ2.t() @ fw["H1"], gZ2.sum(0)
    gZ1 = (gZ2 @ W2) * m[0]
    out["dW1"], out["db1"] = gZ1.t() @ Xs, gZ1.sum(0)
    return out
