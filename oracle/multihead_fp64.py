"""oracle/multihead_fp64.py — one multi-head DQN gradient step in float64, with an error scale for every quantity.

TEST INFRASTRUCTURE ONLY (like the rest of oracle/).  The network is VanillaQValueMultiHeadNetwork's mlp_block
obs -> h1 -> h2 -> A in torch parameter order: W1 [h1, obs], b1, W2 [h2, h1], b2, W3 [A, h2], b3 [A].  One step of
DeepQLearning / DoubleDQN.learn_batch, plain or conservative (csrc/multihead.cu, oracle/multihead_oracle.py):

    q_i = Q(s_i)[a_i]
    y_i = max over the available slots k of Q_target(s'_i)[id_ik] * gamma * (1 - terminated_i) + r_i
    DoubleDQN: y_i = Q_target(s'_i)[a*_i] * gamma * (1 - terminated_i) + r_i, a*_i = the id at the first arg-max slot of
          the ONLINE Q(s'_i)[id_ik] over the available slots
    loss = mean (q_i - y_i)^2 [+ alpha cql], and its gradient with respect to the six parameter blocks.

As in dqn_fp64 (whose data builder and comparison the shape test reuses), everything is explicit formulas, so the SAME code
applied to |.| of every operand gives the error scale of each result: the sum of |a||b| over every product that
contributed to it.  The head gradient dQ [B, A] is written out: 2 (q - y) / B at column a_i, plus, when conservative,
alpha (softmax_k / B - n_k / (B A)) of every current slot k added on the column of the id it holds (cql_step explains the
scale of these terms).
"""
from __future__ import annotations

import torch

from .dqn_fp64 import check, make_data  # noqa: F401

BLOCKS = ("dW1", "db1", "dW2", "db2", "dW3", "db3")


def unflatten(flat: torch.Tensor, obs: int, n_actions: int, hidden) -> tuple:
    """(W1, b1, W2, b2, W3, b3) as float64 views of a flat torch-order parameter vector."""
    h1, h2 = hidden
    shapes = [(h1, obs), (h1,), (h2, h1), (h2,), (n_actions, h2), (n_actions,)]
    flat = flat.to(torch.float64)
    out, off = [], 0
    for s in shapes:
        n = 1
        for x in s:
            n *= x
        out.append(flat[off:off + n].view(s))
        off += n
    assert off == flat.numel(), "parameter count does not match the network shape"
    return tuple(out)


def _forward(net, x):
    W1, b1, W2, b2, W3, b3 = net
    z1 = x @ W1.T + b1
    h1 = z1.clamp_min(0)
    z2 = h1 @ W2.T + b2
    h2 = z2.clamp_min(0)
    return z1, h1, z2, h2, h2 @ W3.T + b3


def _slots(head, ids, n):
    """head[i, ids[i, k]] at every slot, -inf at the slots k >= n[i]."""
    v = head.gather(1, ids)
    slot = torch.arange(ids.shape[1], device=v.device).view(1, -1)
    return v.masked_fill(slot >= n.view(-1, 1), float("-inf"))


def _backward(net, x, m1, m2, h1, h2, dQ) -> dict:
    W1, b1, W2, b2, W3, b3 = net
    dz2 = (dQ @ W3) * m2
    dz1 = (dz2 @ W2) * m1
    return dict(dW1=dz1.T @ x, db1=dz1.sum(0), dW2=dz2.T @ h1, db2=dz2.sum(0), dW3=dQ.T @ h2, db3=dQ.sum(0))


def mh_step(w, wt, batch: dict, obs: int, n_actions: int, gamma: float, hidden, double: bool = False, alpha=None,
            curr_ids=None) -> tuple:
    """One step in float64 on the device of `w`.  batch: state [B, obs], action [B] ids, reward [B], terminated [B],
    next_state [B, obs], avail_ids [B, A] (ids of the available next actions first), avail_n [B].  alpha: conservative
    (curr_ids [B, A], padding with id 0 included; None: slot k holds k).  Returns (value, scale): dicts with q, y, z1, z2,
    gap (DoubleDQN: best minus second best available online next value per row, +inf otherwise), mae, grad (flat, torch
    order) and the blocks of BLOCKS."""
    dev = torch.as_tensor(w).device
    f64 = lambda x: torch.as_tensor(x).to(device=dev, dtype=torch.float64)  # noqa: E731
    state, next_state = f64(batch["state"]), f64(batch["next_state"])
    reward, term = f64(batch["reward"]), f64(batch["terminated"])
    action = torch.as_tensor(batch["action"]).long().to(dev).view(-1, 1)
    ids = torch.as_tensor(batch["avail_ids"]).long().to(dev)
    n = torch.as_tensor(batch["avail_n"]).long().to(dev)
    B, A = state.shape[0], n_actions
    net, net_t = unflatten(f64(w), obs, A, hidden), unflatten(f64(wt), obs, A, hidden)
    absnet, absnet_t = tuple(p.abs() for p in net), tuple(p.abs() for p in net_t)
    rows = torch.arange(B, device=dev)

    z1, h1, z2, h2, head = _forward(net, state)
    _, sh1, _, sh2, shead = _forward(absnet, state.abs())
    m1, m2 = (z1 > 0).to(torch.float64), (z2 > 0).to(torch.float64)
    head_t, shead_t = _forward(net_t, next_state)[4], _forward(absnet_t, next_state.abs())[4]
    gap = torch.full((B,), float("inf"), dtype=torch.float64, device=dev)
    if double:
        v = _slots(_forward(net, next_state)[4], ids, n)
        top = torch.topk(v, min(2, A), dim=1).values
        if A > 1:
            gap = torch.where(n >= 2, top[:, 0] - top[:, 1], gap)
        sel = ids[rows, v.max(1)[1]].view(-1, 1)
        V, sV = head_t.gather(1, sel).view(-1), shead_t.gather(1, sel).view(-1)
    else:
        k = _slots(head_t, ids, n).max(1)[1]
        sel = ids[rows, k].view(-1, 1)
        V, sV = head_t.gather(1, sel).view(-1), shead_t.gather(1, sel).view(-1)
    y = V * gamma * (1.0 - term) + reward
    sy = sV * gamma * (1.0 - term) + reward.abs()
    q, sq = head.gather(1, action).view(-1), shead.gather(1, action).view(-1)

    dQ = torch.zeros(B, A, dtype=torch.float64, device=dev)
    sdQ = torch.zeros_like(dQ)
    if alpha is not None:
        curr = (torch.arange(A, device=dev).repeat(B, 1) if curr_ids is None else torch.as_tensor(curr_ids).long().to(dev).view(B, A))
        l, s = head.gather(1, curr), shead.gather(1, curr)
        n_k = torch.zeros(A, dtype=torch.float64, device=dev)
        n_k[0], n_k[1] = A - 1, 1
        p = torch.softmax(l, dim=1)
        dQ.scatter_add_(1, curr, alpha * (p / B - n_k / (B * A)))
        sdQ.scatter_add_(1, curr, alpha * (p * (s + (p * s).sum(1, keepdim=True) + 1.0) / B + n_k / (B * A)))
    dQ[rows, action.view(-1)] += (q - y) * (2.0 / B)
    sdQ[rows, action.view(-1)] += ((q - y).abs() + sq + sy) * (2.0 / B)
    g = _backward(net, state, m1, m2, h1, h2, dQ)
    sg = _backward(absnet, state.abs(), m1, m2, sh1, sh2, sdQ)

    def pack(d, q, y, z1, z2, gap, mae):
        out = dict(d, q=q, y=y, z1=z1, z2=z2, gap=gap, mae=mae)
        out["grad"] = torch.cat([d[k].reshape(-1) for k in BLOCKS])
        return out

    sz1 = state.abs() @ absnet[0].T + absnet[1]
    sz2 = sh1 @ absnet[2].T + absnet[3]
    return pack(g, q, y, z1, z2, gap, (q - y).abs().mean()), pack(sg, sq, sy, sz1, sz2, gap, (sq + sy).mean())


def relu_margin(w, state, obs: int, n_actions: int, hidden) -> torch.Tensor:
    """Per row, the smallest |pre-activation| / scale over both hidden layers of the online net (host tensor)."""
    w = torch.as_tensor(w)
    x = torch.as_tensor(state).to(device=w.device, dtype=torch.float64)
    net = unflatten(w, obs, n_actions, hidden)
    absnet = tuple(p.abs() for p in net)
    z1, _, z2, _, _ = _forward(net, x)
    _, sh1, _, _, _ = _forward(absnet, x.abs())
    sz1 = x.abs() @ absnet[0].T + absnet[1]
    sz2 = sh1 @ absnet[2].T + absnet[3]
    r = torch.cat([z1.abs() / sz1.clamp_min(1e-300), z2.abs() / sz2.clamp_min(1e-300)], 1)
    return r.min(1)[0].cpu()


def next_action_gap(w, next_state, ids, n, obs: int, n_actions: int, hidden) -> torch.Tensor:
    """Per row, DoubleDQN's best minus second-best available online next value over their scale (+inf with fewer than
    two available slots); host tensor."""
    w = torch.as_tensor(w)
    x = torch.as_tensor(next_state).to(device=w.device, dtype=torch.float64)
    ids = torch.as_tensor(ids).long().to(w.device)
    n = torch.as_tensor(n).long().to(w.device)
    if n_actions < 2:
        return torch.full((x.shape[0],), float("inf"), dtype=torch.float64)
    net = unflatten(w, obs, n_actions, hidden)
    v = _slots(_forward(net, x)[4], ids, n)
    sv = _slots(_forward(tuple(p.abs() for p in net), x.abs())[4], ids, n)
    top, slot = v.topk(2, dim=1)
    gap = (top[:, 0] - top[:, 1]) / sv.gather(1, slot).clamp(min=0).sum(1).clamp_min(1e-300)
    return torch.where(n > 1, gap, float("inf")).cpu()
