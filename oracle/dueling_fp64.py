"""oracle/dueling_fp64.py — one dueling DQN gradient step in float64, with an error scale for every quantity.

TEST INFRASTRUCTURE ONLY (like the rest of oracle/).  The network is DuelingQValueNetwork as csrc/dueling.cu runs it:
three MLPs of two Linear+ReLU layers and a Linear head, in the flat torch order of duel_layout:
    state     obs -> sh1 -> sh2 -> F     (no ReLU on the feature f)
    value     F -> vh1 -> vh2 -> 1       V(s)
    advantage F || one-hot(a) -> ah1 -> ah2 -> 1       Adv(s, a)
Q(s, a) = fl(fl(V + Adv(a)) - mean of Adv over a set that depends on the caller (dueling.cu's header,
oracle/dueling_oracle.py):
    online q:          the A current slots (padding, id 0, included); with no current sets, the query alone:
                       q = fl(fl(V + Adv(a)) - Adv(a))
    DQN target:        Q_target over all A next slots (unavailable ones with the id they hold), the masked max
    DoubleDQN target:  a* = the first arg-max over the available slots of the online Q (mean over all A next slots);
                       V' = fl(fl(V_t + Adv_t(a*)) - Adv_t(a*))
y = V' gamma (1 - terminated) + r; loss = mean (q - y)^2; dq = 2 / B (q - y) reaches V as dq, the taken-action
advantage row as +dq and every current slot as -dq / A (both 0 in query-alone mode); the feature gradient is the sum of
the value and advantage paths.

Every formula is written out, as in oracle/dqn_fp64.py, so that the same code on |.| of every operand gives the error
scale.  Each fl(.) the kernel rounds in the dueling combination adds |its value| to the scale, so that fl(fl(V + Adv) -
Adv) != V stays inside C x scale.
"""
from __future__ import annotations

import torch

from oracle.dqn_fp64 import _forward as _vanilla_forward

MLPS = ("S", "V", "A")
BLOCKS = ("dSW1", "dSb1", "dSW2", "dSb2", "dSW3", "dSb3", "dVW1", "dVb1", "dVW2", "dVb2", "dVW3", "dVb3",
          "dAW1f", "dAW1a", "dAb1", "dAW2", "dAb2", "dAW3", "dAb3")


def dims(obs: int, n_actions: int, widths: dict) -> dict:
    """(in, h1, h2, out) of each MLP from the prl_duel_cfg widths (feature_dim, state_h1, ..., adv_h2)."""
    F = widths["feature_dim"]
    return dict(S=(obs, widths["state_h1"], widths["state_h2"], F), V=(F, widths["value_h1"], widths["value_h2"], 1),
                A=(F + n_actions, widths["adv_h1"], widths["adv_h2"], 1))


def widths_of(hidden) -> dict:
    """The widths of Pearl's DuelingQValueNetwork(hidden_dims=hidden): every MLP's hidden layers are `hidden`, F = hidden[-1]."""
    h = list(hidden)
    return dict(feature_dim=h[-1], state_h1=h[0], state_h2=h[1], value_h1=h[0], value_h2=h[1], adv_h1=h[0], adv_h2=h[1])


def layout(obs: int, n_actions: int, widths: dict) -> dict:
    """Block name -> (offset, rows, cols, column offset, row pitch) in the flat vector (element (r, c) of a block is
    flat[offset + r * pitch + col0 + c]), and "P" -> the parameter count."""
    out, o = {}, 0
    for m, (i, h1, h2, k) in dims(obs, n_actions, widths).items():
        for name, rows, cols in (("W1", h1, i), ("b1", 1, h1), ("W2", h2, h1), ("b2", 1, h2), ("W3", k, h2), ("b3", 1, k)):
            if m == "A" and name == "W1":
                F = widths["feature_dim"]
                out["dAW1f"] = (o, rows, F, 0, cols)
                out["dAW1a"] = (o, rows, n_actions, F, cols)
            else:
                out[f"d{m}{name}"] = (o, rows, cols, 0, cols)
            o += rows * cols
    out["P"] = o
    return out


def block_view(flat: torch.Tensor, name: str, obs: int, n_actions: int, widths: dict) -> torch.Tensor:
    off, rows, cols, col0, pitch = layout(obs, n_actions, widths)[name]
    return flat[off:off + rows * pitch].view(rows, pitch)[:, col0:col0 + cols]


def unflatten(flat, obs: int, n_actions: int, widths: dict) -> dict:
    """MLP name -> (W1, b1, W2, b2, W3, b3) as float64 views of a flat torch-order parameter vector."""
    flat = torch.as_tensor(flat).to(torch.float64)
    out, off = {}, 0
    for m, (i, h1, h2, k) in dims(obs, n_actions, widths).items():
        ps = []
        for s in ((h1, i), (h1,), (h2, h1), (h2,), (k, h2), (k,)):
            n = s[0] * (s[1] if len(s) > 1 else 1)
            ps.append(flat[off:off + n].view(s))
            off += n
        out[m] = tuple(ps)
    assert off == flat.numel(), "parameter count does not match the network shape"
    return out


def _abs(net: dict) -> dict:
    return {m: tuple(p.abs() for p in ps) for m, ps in net.items()}


def _mlp_fwd(ps, x):
    W1, b1, W2, b2, W3, b3 = ps
    z1 = x @ W1.T + b1
    h1 = z1.clamp_min(0)
    z2 = h1 @ W2.T + b2
    h2 = z2.clamp_min(0)
    return z1, h1, z2, h2, h2 @ W3.T + b3


def _trunk(net, state):
    """Trunk and value net on the states: dict of every activation, f [n, F] and V [n]."""
    z1, t1, z2, t2, f = _mlp_fwd(net["S"], state)
    y1, v1, y2, v2, V = _mlp_fwd(net["V"], f)
    return dict(z1=z1, t1=t1, z2=z2, t2=t2, f=f, y1=y1, v1=v1, y2=y2, v2=v2, V=V[:, 0])


def _adv(net, f, ids, A):
    """Advantage net at the slot ids [n, K] of every row: (rows of the [n K, .] pass, adv [n, K])."""
    n, K = ids.shape
    onehot = torch.eye(A, dtype=f.dtype, device=f.device)[ids.reshape(-1)]
    fx = f.repeat_interleave(K, dim=0)
    z1, h1, z2, h2, a = _vanilla_forward(net["A"], fx, onehot)   # the one-hot columns follow the feature ones
    return dict(x=fx, onehot=onehot, z1=z1, a1=h1, z2=z2, a2=h2), a.view(n, K)


def _combine(V, sV, adv, sadv, mean, smean):
    """fl(fl(V + adv) - mean) and its scale; every rounded result adds |itself|."""
    s1 = V.unsqueeze(-1) + adv if adv.dim() == 2 else V + adv
    ss1 = (sV.unsqueeze(-1) + sadv if sadv.dim() == 2 else sV + sadv) + s1.abs()
    q = s1 - mean
    return q, ss1 + smean + q.abs()


def _slot_q(net, anet, state, ids, A):
    """Q over the slot ids [n, K] of each row with the mean over the same K slots, and its scale: (q, sq, tr, str, adv,
    sadv)."""
    tr, s_tr = _trunk(net, state), _trunk(anet, state.abs())
    _, adv = _adv(net, tr["f"], ids, A)
    _, sadv = _adv(anet, s_tr["f"], ids, A)
    mean, smean = adv.mean(1, keepdim=True), sadv.mean(1, keepdim=True) + adv.mean(1, keepdim=True).abs()
    q, sq = _combine(tr["V"], s_tr["V"], adv, sadv, mean, smean)
    return q, sq, tr, s_tr, adv, sadv


def q_values(w, state, obs: int, n_actions: int, widths: dict, ids=None) -> tuple:
    """(Q(s_i, ids[i, k]), its error scale) [n, K] with the mean over each row's K ids (None: every action), on the
    device of `w`."""
    w = torch.as_tensor(w)
    dev = w.device
    state = torch.as_tensor(state).to(device=dev, dtype=torch.float64)
    n = state.shape[0]
    ids = torch.arange(n_actions, device=dev).repeat(n, 1) if ids is None else torch.as_tensor(ids).long().to(dev).view(n, -1)
    net = unflatten(w, obs, n_actions, widths)
    q, sq, *_ = _slot_q(net, _abs(net), state, ids, n_actions)
    return q, sq


def _next_q(net, anet, next_state, avail_ids, avail_n, A):
    """Q(s', avail_ids[i, k]) with the mean over all A slots, -inf at slots k >= avail_n[i]; and the scales."""
    q, sq, *_ = _slot_q(net, anet, next_state, avail_ids, A)
    slot = torch.arange(A, device=q.device).view(1, A)
    return q.masked_fill(slot >= avail_n.view(-1, 1), float("-inf")), sq


def next_action_gap(w, next_state, avail_ids, avail_n, obs: int, n_actions: int, widths: dict) -> torch.Tensor:
    """Per row: (top-1 - top-2) of the online dueling Q(s', .) (mean included) over the available slots, over the sum of
    the two values' scales; inf where only one action is available.  As in relu_margin the scale is local: the two heads
    on their exact inputs (sum |w||x| + |b|) and the rounded results of the combination.  Returns a CPU tensor."""
    w = torch.as_tensor(w)
    dev = w.device
    next_state = torch.as_tensor(next_state).to(device=dev, dtype=torch.float64)
    avail_ids = torch.as_tensor(avail_ids).long().to(dev)
    avail_n = torch.as_tensor(avail_n).long().to(dev)
    if n_actions < 2:
        return torch.full((next_state.shape[0],), float("inf"), dtype=torch.float64)
    net = unflatten(w, obs, n_actions, widths)
    n, A = avail_ids.shape
    tr = _trunk(net, next_state)
    ra, adv = _adv(net, tr["f"], avail_ids, n_actions)
    head = lambda ps, h: (h @ ps[4].abs().T + ps[5].abs())[:, 0]  # noqa: E731
    sV, sadv = head(net["V"], tr["v2"]), head(net["A"], ra["a2"]).view(n, A)
    mean = adv.mean(1, keepdim=True)
    s1 = tr["V"].unsqueeze(1) + adv
    q = s1 - mean
    sq = sV.unsqueeze(1) + sadv + s1.abs() + sadv.mean(1, keepdim=True) + mean.abs() + q.abs()
    slot = torch.arange(A, device=dev).view(1, A)
    v = q.masked_fill(slot >= avail_n.view(-1, 1), float("-inf"))
    top, k = v.topk(2, dim=1)
    gap = (top[:, 0] - top[:, 1]) / sq.gather(1, k).sum(1)
    return torch.where(avail_n > 1, gap, float("inf")).cpu()


def _local_ratio(ps, x):
    """|z| / scale of both hidden pre-activations of an MLP on the exact inputs x, the scale of each layer taken from its
    own inputs (sum |w||x| + |b|): [n] per layer, the smallest over the units."""
    W1, b1, W2, b2, _, _ = ps
    z1 = x @ W1.T + b1
    h1 = z1.clamp_min(0)
    z2 = h1 @ W2.T + b2
    r1 = z1.abs() / (x.abs() @ W1.abs().T + b1.abs())
    r2 = z2.abs() / (h1 @ W2.abs().T + b2.abs())
    return torch.minimum(r1.min(1)[0], r2.min(1)[0])


def relu_margin(w, state, slot_ids, obs: int, n_actions: int, widths: dict) -> torch.Tensor:
    """Per row: the smallest |pre-activation| / scale over the trunk, the value net and the advantage net at every slot
    id of slot_ids [B, S] (or [B]).  Unlike dqn_fp64.relu_margin the scale of a layer is taken from its own exact inputs
    (sum |w||x| + |b|), not carried through the network: six layers deep, behind a feature that is a cancelling sum, the
    carried scale is many times the size of the values and would reject almost every row, while the rounding error a
    kernel actually makes in a layer stays a few ulps of that layer's own scale.  Returns a CPU tensor."""
    w = torch.as_tensor(w)
    dev = w.device
    state = torch.as_tensor(state).to(device=dev, dtype=torch.float64)
    ids = torch.as_tensor(slot_ids).long().to(dev)
    ids = ids.view(-1, 1) if ids.dim() == 1 else ids
    B, S = ids.shape
    net = unflatten(w, obs, n_actions, widths)
    tr = _trunk(net, state)
    ra, _ = _adv(net, tr["f"], ids, n_actions)
    row = torch.minimum(_local_ratio(net["S"], state), _local_ratio(net["V"], tr["f"]))
    slot = _local_ratio(net["A"], torch.cat([ra["x"], ra["onehot"]], 1)).view(B, S).min(1)[0]
    return torch.minimum(row, slot).cpu()


def _mlp_bwd(ps, x, m1, m2, h1, h2, dout):
    """Backward of one MLP for the output gradient dout [n, out] with the ReLU masks of the value pass (the |.| pass uses
    them too): the six blocks and dx [n, in]."""
    W1, b1, W2, b2, W3, b3 = ps
    dz2 = (dout @ W3) * m2
    dz1 = (dz2 @ W2) * m1
    return dict(W1=dz1.T @ x, b1=dz1.sum(0), W2=dz2.T @ h1, b2=dz2.sum(0), W3=dout.T @ h2, b3=dout.sum(0)), dz1 @ W1


def _grad(net, state, tr, ra, dq, dslot, masks):
    """Every block of the gradient for dq [B] (reaching V) and the advantage-row gradients dslot [B, S] (rows of ra)."""
    B, S = dslot.shape
    F = tr["f"].shape[1]
    ga, dxa = _mlp_bwd(net["A"], torch.cat([ra["x"], ra["onehot"]], 1), masks["a1"], masks["a2"], ra["a1"], ra["a2"],
                              dslot.reshape(-1, 1))
    df = dxa[:, :F].view(B, S, F).sum(1)
    gv, dxv = _mlp_bwd(net["V"], tr["f"], masks["v1"], masks["v2"], tr["v1"], tr["v2"], dq.view(-1, 1))
    df = df + dxv
    gs, _ = _mlp_bwd(net["S"], state, masks["t1"], masks["t2"], tr["t1"], tr["t2"], df)
    out = {f"dS{k}": v for k, v in gs.items()}
    out.update({f"dV{k}": v for k, v in gv.items()})
    out.update({f"dA{k}": v for k, v in ga.items() if k != "W1"})
    out["dAW1f"], out["dAW1a"] = ga["W1"][:, :F], ga["W1"][:, F:]
    out["df"] = df
    return out


def dueling_step(w, wt, batch: dict, obs: int, n_actions: int, gamma: float, widths: dict, double: bool = False,
                 curr_ids=None, query_alone: bool = False) -> tuple:
    """One dueling DQN step in float64.  `batch` as dqn_step's (avail_ids [B, A] hold the id of EVERY next slot, padding
    included: the target's mean runs over all of them; avail_n [B] how many are available).  curr_ids [B, A]: the current
    sets (None: slot k holds k, as the ring reports); query_alone: the batch has no current sets.  Returns (value, scale):
    dicts with q, y, mae, loss, grad (flat, torch order) and every block of BLOCKS."""
    dev = torch.as_tensor(w).device
    f64 = lambda x: torch.as_tensor(x).to(device=dev, dtype=torch.float64)  # noqa: E731
    state, next_state = f64(batch["state"]), f64(batch["next_state"])
    reward, term = f64(batch["reward"]), f64(batch["terminated"])
    action = torch.as_tensor(batch["action"]).long().to(dev)
    avail_ids = torch.as_tensor(batch["avail_ids"]).long().to(dev)
    avail_n = torch.as_tensor(batch["avail_n"]).long().to(dev)
    B, A = state.shape[0], n_actions
    net, net_t = unflatten(f64(w), obs, A, widths), unflatten(f64(wt), obs, A, widths)
    anet, anet_t = _abs(net), _abs(net_t)

    # online pass: advantage over the A current slots and, as slot A, the taken action
    curr = (torch.arange(A, device=dev).repeat(B, 1) if curr_ids is None
            else torch.as_tensor(curr_ids).long().to(dev).view(B, A))
    cids = torch.cat([curr, action.view(B, 1)], 1)
    tr, s_tr = _trunk(net, state), _trunk(anet, state.abs())
    ra, adv = _adv(net, tr["f"], cids, A)
    sra, sadv = _adv(anet, s_tr["f"], cids, A)
    at, sat = adv[:, A], sadv[:, A]
    if query_alone:
        mean, smean = at, sat
    else:
        mean = adv[:, :A].mean(1)
        smean = sadv[:, :A].mean(1) + mean.abs()
    q, sq = _combine(tr["V"], s_tr["V"], at, sat, mean, smean)

    # target
    if double:
        v, _ = _next_q(net, anet, next_state, avail_ids, avail_n, A)
        slot = v.max(1)[1]
        a_star = avail_ids.gather(1, slot.view(-1, 1))
        tt, s_tt = _trunk(net_t, next_state), _trunk(anet_t, next_state.abs())
        _, ta = _adv(net_t, tt["f"], a_star, A)
        _, sta = _adv(anet_t, s_tt["f"], a_star, A)
        V, sV = _combine(tt["V"], s_tt["V"], ta[:, 0], sta[:, 0], ta[:, 0], sta[:, 0])
    else:
        v, sv = _next_q(net_t, anet_t, next_state, avail_ids, avail_n, A)
        V, slot = v.max(1)
        sV = sv.gather(1, slot.view(-1, 1))[:, 0]
    y = V * gamma * (1.0 - term) + reward
    sy = sV * gamma * (1.0 - term) + reward.abs()

    dq = (q - y) * (2.0 / B)
    sdq = ((q - y).abs() + sq + sy) * (2.0 / B)
    if query_alone:
        dslot, sdslot = torch.zeros(B, A + 1, dtype=torch.float64, device=dev), torch.zeros(B, A + 1, dtype=torch.float64, device=dev)
    else:
        dslot = torch.cat([(-dq / A).view(B, 1).expand(B, A), dq.view(B, 1)], 1)
        sdslot = torch.cat([(sdq / A).view(B, 1).expand(B, A), sdq.view(B, 1)], 1)
    masks = dict(t1=(tr["z1"] > 0).double(), t2=(tr["z2"] > 0).double(), v1=(tr["y1"] > 0).double(),
                 v2=(tr["y2"] > 0).double(), a1=(ra["z1"] > 0).double(), a2=(ra["z2"] > 0).double())
    g = _grad(net, state, tr, ra, dq, dslot, masks)
    sg = _grad(anet, state.abs(), s_tr, sra, sdq, sdslot, masks)

    lay = layout(obs, A, widths)

    def pack(d, q, y, mae):
        out = dict(d, q=q, y=y, mae=mae)
        flat = torch.zeros(lay["P"], dtype=torch.float64, device=dev)
        for name in BLOCKS:
            off, rows, cols, col0, pitch = lay[name]
            flat[off:off + rows * pitch].view(rows, pitch)[:, col0:col0 + cols] = d[name].reshape(rows, cols)
        out["grad"] = flat
        return out

    value = pack(g, q, y, (q - y).abs().mean())
    scale = pack(sg, sq, sy, (sq + sy).mean())
    value["loss"], scale["loss"] = ((q - y) ** 2).mean(), (2 * (q - y).abs() * (sq + sy)).mean()
    return value, scale
