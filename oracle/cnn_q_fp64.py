"""oracle/cnn_q_fp64.py — one CNN DQN gradient step (csrc/cnnq.cu, oracle/cnn_q_oracle.py) in float64, with an error
scale for every gradient element.  TEST INFRASTRUCTURE ONLY.

The gradient is the backward pass of the Q network's outputs at the taken rows under the head gradient dQ (vanilla:
fl(2 / B)(q_b - y_b) on the one output; multi-head: sum_j 2 / B^2 (q_i - Y_ij) on column a_i, Y_ij as in the oracle).
The scale is the same backward pass applied to |.| of every operand — the network run on |W|, |b| and the pixel values
with each ReLU replaced by the fixed mask of the real forward pass, under the head scale 2 (|q| + |y|) / B (multi-head:
the sum over j of 2 (|q_i| + |Y_ij|) / B^2) — so every gradient element's scale is the sum of |a||b| over the products
that contributed to it.  relu_margin reports the smallest |pre-activation| / its scale, so a test can avoid data where a
last-bit difference could flip a mask."""
from __future__ import annotations

import torch
import torch.nn.functional as F

from .cnn_q_oracle import next_values, unflat


def _forward(spec, ps, x, a, masks=None):
    """The online outputs at the taken rows ([B, 1] vanilla, [B, A] multi-head); masks None: ReLU, recording each layer's
    pre-activations; otherwise each ReLU is the given 0/1 mask (the |.| network)."""
    pre, k = [], 0
    act = (lambda z: (pre.append(z), F.relu(z))[1]) if masks is None else None  # noqa: E731

    def relu(z):
        nonlocal k
        if masks is None:
            return act(z)
        k += 1
        return z * masks[k - 1]
    h = x / 255.0
    for i, (_, _, s, p) in enumerate(spec["conv"]):
        h = relu(F.conv2d(h, ps[2 * i], ps[2 * i + 1], stride=s, padding=p))
    z = h.reshape(x.shape[0], -1)
    if not spec["multi"]:
        z = torch.cat([z, F.one_hot(a, spec["n_actions"]).to(z.dtype)], -1)
    fcp = ps[2 * len(spec["conv"]):]
    n = len(fcp) // 2
    for i in range(n):
        z = F.linear(z, fcp[2 * i], fcp[2 * i + 1])
        if i < n - 1:
            z = relu(z)
    return z, pre


def step(spec, w: torch.Tensor, wt: torch.Tensor, batch: dict, *, double: bool, gamma: float):
    """(gradient, scale, relu margin) of one round's loss at online w / target wt (flat fp32), all float64."""
    w64, wt64 = w.double(), wt.double()
    b64 = {k: (v.double() if v.is_floating_point() else v) for k, v in batch.items()}
    V = next_values(spec, w64, wt64, b64["next_state"], b64["next_ids"], b64["next_count"], double)
    p = w64.clone().requires_grad_(True)
    out, pre = _forward(spec, unflat(spec, p), b64["state"], b64["action"])
    B, A = out.shape[0], spec["n_actions"]
    t, r = b64["terminated"].double(), b64["reward"]
    with torch.no_grad():
        if spec["multi"]:
            q = out.gather(1, b64["action"].view(-1, 1)).squeeze(1)
            Y = V.unsqueeze(1) * gamma * (1 - t.unsqueeze(0)) + r.unsqueeze(0) if double else (V * gamma * (1 - t) + r).unsqueeze(0).expand(B, B)
            gq = (2.0 / (B * B)) * (q.unsqueeze(1) - Y).sum(1)
            sq = (2.0 / (B * B)) * (q.abs().unsqueeze(1) + Y.abs()).sum(1)
            dQ = torch.zeros_like(out).scatter_(1, b64["action"].view(-1, 1), gq.unsqueeze(1))
            sQ = torch.zeros_like(out).scatter_(1, b64["action"].view(-1, 1), sq.unsqueeze(1))
        else:
            y = V * gamma * (1 - t) + r
            q = out.squeeze(1)
            dQ = ((2.0 / B) * (q - y)).unsqueeze(1)
            sQ = ((2.0 / B) * (q.abs() + y.abs())).unsqueeze(1)
    (g,) = torch.autograd.grad(out, p, grad_outputs=dQ)
    masks = [(z > 0).double().detach() for z in pre]
    pa = w64.abs().clone().requires_grad_(True)
    out_a, _ = _forward(spec, unflat(spec, pa), b64["state"], b64["action"], masks)
    (s,) = torch.autograd.grad(out_a, pa, grad_outputs=sQ)
    # the pre-activations' own scales: the |.| network's values before each mask
    with torch.no_grad():
        scales, k = [], 0
        pa2 = unflat(spec, w64.abs())
        h = b64["state"] / 255.0
        for i, (_, _, st, pd) in enumerate(spec["conv"]):
            z = F.conv2d(h, pa2[2 * i], pa2[2 * i + 1], stride=st, padding=pd)
            scales.append(z)
            h = z * masks[k]
            k += 1
        margin = min(float((z0.abs() / zs.clamp_min(1e-300)).min()) for z0, zs in zip(pre[:len(scales)], scales))
    return g.detach(), s.detach(), margin
