"""oracle/sarsa_fp64.py — one DeepSARSA gradient step in float64, with an error scale for every quantity (TEST
INFRASTRUCTURE ONLY).  The step of oracle/dqn_fp64.py with DeepSARSA's target: y_i = Q_target(s'_i, a'_i) gamma
(1 - terminated_i) + r_i at the committed next action a'_i (no max, no available sets).  The same formulas run on |.|
give the error scale of each result (see dqn_fp64.py)."""
from __future__ import annotations

import torch

from .dqn_fp64 import _backward, _forward, unflatten


def sarsa_step(w, wt, batch: dict, obs: int, n_actions: int, gamma: float, hidden=(64, 64)) -> tuple:
    """`batch`: state [B, obs], action [B] ids, reward [B], terminated [B], next_state [B, obs], next_action [B] ids.
    Returns (value, scale): dicts with q, y, mae, loss, grad (flat, torch order) and the blocks of dqn_fp64.BLOCKS."""
    dev = torch.as_tensor(w).device
    f64 = lambda x: torch.as_tensor(x).to(device=dev, dtype=torch.float64)  # noqa: E731
    state, next_state = f64(batch["state"]), f64(batch["next_state"])
    reward, term = f64(batch["reward"]), f64(batch["terminated"])
    eye = torch.eye(n_actions, dtype=torch.float64, device=dev)
    onehot = eye[torch.as_tensor(batch["action"]).long().to(dev)]
    onehot_n = eye[torch.as_tensor(batch["next_action"]).long().to(dev)]
    B = state.shape[0]
    net, net_t = unflatten(f64(w), obs, n_actions, hidden), unflatten(f64(wt), obs, n_actions, hidden)
    absnet, absnet_t = tuple(p.abs() for p in net), tuple(p.abs() for p in net_t)

    z1, h1, z2, h2, q = _forward(net, state, onehot)
    y = _forward(net_t, next_state, onehot_n)[4] * gamma * (1.0 - term) + reward
    m1, m2 = (z1 > 0).to(torch.float64), (z2 > 0).to(torch.float64)
    sz1, sh1, sz2, sh2, sq = _forward(absnet, state.abs(), onehot)
    sy = _forward(absnet_t, next_state.abs(), onehot_n)[4] * gamma * (1.0 - term) + reward.abs()
    dq = (q - y) * (2.0 / B)
    sdq = ((q - y).abs() + sq + sy) * (2.0 / B)
    g = _backward(net, state, onehot, m1, m2, h1, h2, dq)
    sg = _backward(absnet, state.abs(), onehot, m1, m2, sh1, sh2, sdq)

    def pack(d, q, y, mae, loss):
        out = dict(d, q=q, y=y, mae=mae, loss=loss)
        out["grad"] = torch.cat([torch.cat([d["dW1s"], d["dW1a"]], 1).reshape(-1), d["db1"], d["dW2"].reshape(-1),
                                 d["db2"], d["dW3"].reshape(-1), d["db3"]])
        return out

    return (pack(g, q, y, (q - y).abs().mean(), ((q - y) ** 2).mean()),
            pack(sg, sq, sy, (sq + sy).mean(), (2 * (q - y).abs() * (sq + sy)).mean()))
