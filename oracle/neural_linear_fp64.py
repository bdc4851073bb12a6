"""The float64 gradient step of NeuralLinearBandit's round (csrc/neural_linear.cu), written out by hand rather than
through autograd, so that it can also be evaluated on absolute values: `step(..., absolute=True)` returns, for every
value, the sum of |a||b| over every product that reached it (the scale an fp32 rounding error is measured against).
TEST INFRASTRUCTURE: nothing in pearl_b200 imports it.

Parameters `p` = [W1, b1, W2, b2, W3, b3, we] (torch's parameters() order; we = linear_layer_e2e.weight [1, h2]).
The network is mlp_block(f, [h1, h2], output_dim=h2) with ReLU hidden layers, each layer of equal in / out width wrapped
as x + layer(x) when skip.  mu = nn_output . we (e2e), or coefs[0] + nn_output . coefs[1:]; p = sigmoid(mu) or mu; the
loss sum(w l) / sum(w) with l = mse, l1 or binary cross-entropy (the logs clamped at -100), and the gradient in torch's
backward forms (l1: sign(p - y); bce: (p - y) / max(p (1 - p), 1e-12), times (1 - p) p through the sigmoid)."""
from __future__ import annotations

import torch

BLOCKS = ("dW1", "db1", "dW2", "db2", "dW3", "db3", "dwe")


def forward(p, X, skip: bool, absolute: bool = False, masks=None):
    """nn_output and the intermediates; absolute: |.| everywhere, the ReLU masks taken from `masks` (the signed pass)."""
    W1, b1, W2, b2, W3, b3 = (t.abs() for t in p[:6]) if absolute else p[:6]
    X = X.abs() if absolute else X
    f, h1, h2 = X.shape[1], W1.shape[0], W2.shape[0]
    Z1 = X @ W1.t() + b1
    A1 = Z1 * masks[0] if absolute else torch.relu(Z1)
    H1 = X + A1 if skip and f == h1 else A1
    Z2 = H1 @ W2.t() + b2
    A2 = Z2 * masks[1] if absolute else torch.relu(Z2)
    H2 = H1 + A2 if skip and h1 == h2 else A2
    T3 = H2 @ W3.t() + b3
    N = H2 + T3 if skip else T3
    return dict(Z1=Z1, H1=H1, Z2=Z2, H2=H2, N=N)


def head(N, we, coefs, y, e2e: bool, loss: str, sigmoid: bool):
    """mu, p, the per-row l and dl/dmu (without the weight)."""
    mu = N @ we.reshape(-1) if e2e else coefs[0] + N @ coefs[1:]
    pr = torch.sigmoid(mu) if sigmoid else mu
    e = pr - y
    if loss == "mse":
        l, g = e * e, 2 * e
    elif loss == "mae":
        l, g = e.abs(), torch.sign(e)
    else:
        l = -(y * torch.clamp(torch.log(pr), min=-100) + (1 - y) * torch.clamp(torch.log(1 - pr), min=-100))
        g = e / torch.clamp(pr * (1 - pr), min=1e-12)
    if sigmoid:
        g = g * (1 - pr) * pr
    return mu, pr, l, g


def step(p, X, y, w, coefs, *, e2e: bool, loss: str, sigmoid: bool, skip: bool, absolute: bool = False):
    """The gradient of one round: dict of the blocks in BLOCKS (dwe only with e2e), plus nn_output `N`, `mu`, `pred`,
    `loss` and the pre-activations Z1, Z2.  absolute=True: the scales of the same quantities (see the module docstring)."""
    sig = forward(p, X, skip)
    if absolute:
        m = [(sig["Z1"] > 0).to(X.dtype), (sig["Z2"] > 0).to(X.dtype)]
        fw = forward(p, X, skip, True, m)
    else:
        m, fw = [(sig["Z1"] > 0).to(X.dtype), (sig["Z2"] > 0).to(X.dtype)], sig
    W2, W3 = (p[2].abs(), p[4].abs()) if absolute else (p[2], p[4])
    we = p[6].reshape(-1)
    v = we if e2e else coefs[1:]
    mu, pr, l, g = head(sig["N"], p[6], coefs, y, e2e, loss, sigmoid)
    if absolute:
        # the scale of dl/dmu includes the rounding mu carries in: smu = the scale of mu
        v = v.abs()
        smu = fw["N"] @ v + (0 if e2e else coefs[0].abs())
        if loss == "mse":
            g = 2 * (smu + y.abs())
        elif loss == "mae":
            g = torch.ones_like(g)
        else:
            g = pr.abs() + y.abs() + pr * (1 - pr) * smu
    gm = g * w / w.sum()
    f, h1, h2 = X.shape[1], p[0].shape[0], p[2].shape[0]
    Xs = X.abs() if absolute else X
    dN = gm[:, None] * v[None, :]
    out = dict(N=fw["N"], mu=mu, pred=pr, loss=(l * w).sum() / w.sum(), Z1=fw["Z1"], Z2=fw["Z2"])
    out["dW3"], out["db3"] = dN.t() @ fw["H2"], dN.sum(0)
    gH2 = dN @ W3 + (dN if skip else 0)
    gZ2 = gH2 * m[1]
    out["dW2"], out["db2"] = gZ2.t() @ fw["H1"], gZ2.sum(0)
    gH1 = gZ2 @ W2 + (gH2 if skip and h1 == h2 else 0)
    gZ1 = gH1 * m[0]
    out["dW1"], out["db1"] = gZ1.t() @ Xs, gZ1.sum(0)
    if e2e:
        N = fw["N"]
        out["dwe"] = (gm @ N).reshape(1, -1)
    return out


def flat(grads: dict, e2e: bool) -> torch.Tensor:
    """The blocks in torch's parameters() order (without dwe when not e2e, as torch's AdamW keeps no state for it)."""
    return torch.cat([grads[k].reshape(-1) for k in BLOCKS if k != "dwe" or e2e])
