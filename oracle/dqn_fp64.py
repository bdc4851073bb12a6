"""oracle/dqn_fp64.py — one DQN gradient step in float64, with an error scale for every quantity.

TEST INFRASTRUCTURE ONLY (like the rest of oracle/).  The network is the [obs + A] -> h1 -> h2 -> 1 ReLU MLP of
VanillaQValueNetwork in torch parameter order: W1 [h1, obs + A] (state columns, then one-hot action columns), b1,
W2 [h2, h1], b2, W3 [1, h2], b3.  One step of DeepQLearning.learn_batch on a batch:

    q_i = Q(s_i, a_i)
    y_i = max over the available a' of Q_target(s'_i, a') * gamma * (1 - terminated_i) + r_i   (unavailable: -inf;
          `truncated` plays no part, as in the reference)
    DoubleDQN: y_i = Q_target(s'_i, a*_i) * gamma * (1 - terminated_i) + r_i, a*_i = the first arg-max over the
          available slots of the ONLINE Q(s'_i, .)
    loss = mean(w_i (q_i - y_i)^2) (w = 1 without importance weights), and its gradient with respect to the seven
          parameter blocks.

Everything is written as explicit formulas, not autograd, so that the SAME code applied to |.| of every operand gives
the error scale of each result: the sum of |a||b| over every product that contributed to it, carried through the chain
(the natural scale of a rounding error in a chain of dot products).  ReLU is the identity on non-negative values and
the ReLU derivatives are the masks of the value pass, so they need no special case.  The one change is the loss
derivative: |dq_i| becomes w_i (|q_i - y_i| + scale(q_i) + scale(y_i)) 2 / B, so that a row with q ~ y is judged by
the rounding noise of q - y and not by its own tiny value.  The arg-max of DoubleDQN is not continuous: a row whose
top two online values are closer than a kernel's rounding (next_action_gap) has to be left out of a comparison.

cql_step is the same step for the conservative learner (csrc/cql.cu): the online pass over A + 1 slots per row and the
CQL term's slot gradients.  make_data and check are the data builder and the elementwise comparison of the GPU shape
tests.
"""
from __future__ import annotations

import numpy as np
import torch

BLOCKS = ("dW1s", "dW1a", "db1", "dW2", "db2", "dW3", "db3")


def unflatten(flat: torch.Tensor, obs: int, n_actions: int, hidden=(64, 64)) -> tuple:
    """(W1, b1, W2, b2, W3, b3) as float64 views of a flat torch-order parameter vector."""
    h1, h2 = hidden
    D = obs + n_actions
    shapes = [(h1, D), (h1,), (h2, h1), (h2,), (1, h2), (1,)]
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


def _forward(net, state, onehot):
    """Z1, Z2 and Q for rows (state [n, obs], onehot [n, A])."""
    W1, b1, W2, b2, W3, b3 = net
    obs = state.shape[1]
    z1 = state @ W1[:, :obs].T + onehot @ W1[:, obs:].T + b1
    h1 = z1.clamp_min(0)
    z2 = h1 @ W2.T + b2
    h2 = z2.clamp_min(0)
    return z1, h1, z2, h2, h2 @ W3[0] + b3[0]


def _next_q(net, next_state, avail_ids, avail_n):
    """Q(s'_i, avail_ids[i, k]) for every slot k of every row, -inf at the slots k >= avail_n[i]."""
    B, A = avail_ids.shape
    eye = torch.eye(A, dtype=next_state.dtype, device=next_state.device)
    onehot = eye[avail_ids.reshape(-1)]                                        # [B * A, A]
    s = next_state.repeat_interleave(A, dim=0)
    v = _forward(net, s, onehot)[4].view(B, A)
    slot = torch.arange(A, device=v.device).view(1, A)
    return v.masked_fill(slot >= avail_n.view(B, 1), float("-inf"))


def _target(net, next_state, avail_ids, avail_n, gamma, terminated, reward, a_star=None):
    """y per row: the max over the first avail_n[i] entries of avail_ids[i] of Q_target(s'_i, .), then the TD target;
    with `a_star` (DoubleDQN's chosen action id per row) Q_target(s'_i, a_star[i]) instead of the max."""
    if a_star is None:
        v = _next_q(net, next_state, avail_ids, avail_n).max(1)[0]
    else:
        eye = torch.eye(avail_ids.shape[1], dtype=next_state.dtype, device=next_state.device)
        v = _forward(net, next_state, eye[a_star])[4]
    return v * gamma * (1.0 - terminated) + reward


def _double_action(net, next_state, avail_ids, avail_n):
    """DoubleDQN's a*: the action id at the first arg-max slot of the online Q(s', .) over the available slots."""
    slot = _next_q(net, next_state, avail_ids, avail_n).max(1)[1]
    return avail_ids.gather(1, slot.view(-1, 1)).view(-1)


def _backward(net, state, onehot, m1, m2, h1, h2, dq) -> dict:
    W1, b1, W2, b2, W3, b3 = net
    obs = state.shape[1]
    dz2 = dq[:, None] * W3[0][None, :] * m2
    dz1 = (dz2 @ W2) * m1
    return dict(dW1s=dz1.T @ state, dW1a=dz1.T @ onehot, db1=dz1.sum(0), dW2=dz2.T @ h1, db2=dz2.sum(0),
                dW3=(dq @ h2).view(1, -1), db3=dq.sum().view(1))


def dqn_step(w, wt, batch: dict, obs: int, n_actions: int, gamma: float, hidden=(64, 64), double: bool = False,
             weight=None) -> tuple:
    """One DQN step in float64.  `w`, `wt`: flat online / target parameters.  `batch`: state [B, obs], action [B] ids,
    reward [B], terminated [B], next_state [B, obs], avail_ids [B, A] (ids of the available next actions first),
    avail_n [B] (how many are available).  `double`: DoubleDQN's target.  `weight` [B]: importance weights of a
    prioritized draw (dq_i and its scale are multiplied by w_i; mae stays the unweighted mean |q - y|).  Runs on the
    device of `w`.  Returns (value, scale): two dicts with q, y, z1, z2 [B, h], mae (the reported loss, mean |q - y|),
    loss (mean w (q - y)^2), grad (flat, torch order) and the seven blocks of BLOCKS."""
    dev = torch.as_tensor(w).device
    f64 = lambda x: torch.as_tensor(x).to(device=dev, dtype=torch.float64)
    state, next_state = f64(batch["state"]), f64(batch["next_state"])
    reward, term = f64(batch["reward"]), f64(batch["terminated"])
    action = torch.as_tensor(batch["action"]).long().to(dev)
    avail_ids = torch.as_tensor(batch["avail_ids"]).long().to(dev)
    avail_n = torch.as_tensor(batch["avail_n"]).long().to(dev)
    B = state.shape[0]
    onehot = torch.eye(n_actions, dtype=torch.float64, device=dev)[action]
    net, net_t = unflatten(f64(w), obs, n_actions, hidden), unflatten(f64(wt), obs, n_actions, hidden)
    absnet, absnet_t = tuple(p.abs() for p in net), tuple(p.abs() for p in net_t)
    a_star = _double_action(net, next_state, avail_ids, avail_n) if double else None

    z1, h1, z2, h2, q = _forward(net, state, onehot)
    y = _target(net_t, next_state, avail_ids, avail_n, gamma, term, reward, a_star)
    m1, m2 = (z1 > 0).to(torch.float64), (z2 > 0).to(torch.float64)
    sz1, sh1, sz2, sh2, sq = _forward(absnet, state.abs(), onehot)
    sy = _target(absnet_t, next_state.abs(), avail_ids, avail_n, gamma, term, reward.abs(), a_star)

    wgt = torch.ones(B, dtype=torch.float64, device=dev) if weight is None else f64(weight)
    dq = wgt * (q - y) * (2.0 / B)
    sdq = wgt * ((q - y).abs() + sq + sy) * (2.0 / B)
    g = _backward(net, state, onehot, m1, m2, h1, h2, dq)
    sg = _backward(absnet, state.abs(), onehot, m1, m2, sh1, sh2, sdq)

    def pack(d, q, y, z1, z2, mae, loss):
        out = dict(d, q=q, y=y, z1=z1, z2=z2, mae=mae, loss=loss)
        out["grad"] = torch.cat([torch.cat([d["dW1s"], d["dW1a"]], 1).reshape(-1), d["db1"], d["dW2"].reshape(-1),
                                 d["db2"], d["dW3"].reshape(-1), d["db3"]])
        return out

    value = pack(g, q, y, z1, z2, (q - y).abs().mean(), (wgt * (q - y) ** 2).mean())
    scale = pack(sg, sq, sy, sz1, sz2, (sq + sy).mean(), (2 * wgt * (q - y).abs() * (sq + sy)).mean())
    return value, scale


def cql_step(w, wt, batch: dict, obs: int, n_actions: int, gamma: float, alpha: float, hidden=(64, 64),
             double: bool = False, curr_ids=None) -> tuple:
    """One conservative (CQL) DQN step in float64 (csrc/cql.cu, oracle/cql_oracle.py), on the batch of dqn_step.  The
    online pass runs over A + 1 slots per row: the A current slots (curr_ids [B, A], padding with id 0 taking part;
    None: slot k holds k) and, as slot A, the taken action.  y as in dqn_step.  Slot gradients of mean (q - y)^2 +
    alpha cql (the reference's CQL term, whose second part reads columns 0 and 1 of the current-slot values):
        taken slot:     2 / B (q - y)
        current slot k: alpha (softmax_k / B - n_k / (B A)),   n_0 = A - 1, n_1 = 1, n_k = 0 otherwise
    The backward pass runs over the B (A + 1) slot rows: the state columns and b1 see each row's sum over its slots, the
    action columns are scattered by slot id.  The |.| rule does not apply to exp: the scale of a current slot's gradient is
    alpha (p_k (s_k + sum_j p_j s_j + 1) / B + n_k / (B A)) with s the scale of the logits (an error e_j of logit j moves
    p_k by p_k (e_k - sum_j p_j e_j); the trailing p_k / B covers the rounding of expf and of the division).  Returns
    (value, scale) as dqn_step, with q_all [B, A + 1] (the slot values) in place of z1 / z2."""
    dev = torch.as_tensor(w).device
    f64 = lambda x: torch.as_tensor(x).to(device=dev, dtype=torch.float64)  # noqa: E731
    state, next_state = f64(batch["state"]), f64(batch["next_state"])
    reward, term = f64(batch["reward"]), f64(batch["terminated"])
    action = torch.as_tensor(batch["action"]).long().to(dev)
    avail_ids = torch.as_tensor(batch["avail_ids"]).long().to(dev)
    avail_n = torch.as_tensor(batch["avail_n"]).long().to(dev)
    B, A = state.shape[0], n_actions
    curr = (torch.arange(A, device=dev).repeat(B, 1) if curr_ids is None
            else torch.as_tensor(curr_ids).long().to(dev).view(B, A))
    cids = torch.cat([curr, action.view(B, 1)], 1)                                     # [B, A + 1]
    onehot = torch.eye(A, dtype=torch.float64, device=dev)[cids.reshape(-1)]
    xs = state.repeat_interleave(A + 1, dim=0)
    net, net_t = unflatten(f64(w), obs, A, hidden), unflatten(f64(wt), obs, A, hidden)
    absnet, absnet_t = tuple(p.abs() for p in net), tuple(p.abs() for p in net_t)
    a_star = _double_action(net, next_state, avail_ids, avail_n) if double else None

    z1, h1, z2, h2, q_all = _forward(net, xs, onehot)
    m1, m2 = (z1 > 0).to(torch.float64), (z2 > 0).to(torch.float64)
    _, sh1, _, sh2, sq_all = _forward(absnet, xs.abs(), onehot)
    q_all, sq_all = q_all.view(B, A + 1), sq_all.view(B, A + 1)
    q, sq = q_all[:, A], sq_all[:, A]
    y = _target(net_t, next_state, avail_ids, avail_n, gamma, term, reward, a_star)
    sy = _target(absnet_t, next_state.abs(), avail_ids, avail_n, gamma, term, reward.abs(), a_star)

    n_k = torch.zeros(A, dtype=torch.float64, device=dev)
    n_k[0], n_k[1] = A - 1, 1
    p = torch.softmax(q_all[:, :A], dim=1)
    s = sq_all[:, :A]
    dq = torch.cat([alpha * (p / B - n_k / (B * A)), ((q - y) * (2.0 / B)).view(B, 1)], 1)
    sdq = torch.cat([alpha * (p * (s + (p * s).sum(1, keepdim=True) + 1.0) / B + n_k / (B * A)),
                     (((q - y).abs() + sq + sy) * (2.0 / B)).view(B, 1)], 1)
    g = _backward(net, xs, onehot, m1, m2, h1, h2, dq.reshape(-1))
    sg = _backward(absnet, xs.abs(), onehot, m1, m2, sh1, sh2, sdq.reshape(-1))

    def pack(d, q, y, q_all, mae):
        out = dict(d, q=q, y=y, q_all=q_all, mae=mae)
        out["grad"] = torch.cat([torch.cat([d["dW1s"], d["dW1a"]], 1).reshape(-1), d["db1"], d["dW2"].reshape(-1),
                                 d["db2"], d["dW3"].reshape(-1), d["db3"]])
        return out

    return pack(g, q, y, q_all, (q - y).abs().mean()), pack(sg, sq, sy, sq_all, (sq + sy).mean())


def relu_margin(w, state, action, obs: int, n_actions: int, hidden=(64, 64)) -> torch.Tensor:
    """Per row: the smallest |pre-activation| / scale over both hidden layers of the network `w` at (state, action).
    `action`: [B] ids, or a [B, S] matrix of slot ids (a learner whose online pass evaluates S slots per row): then the
    smallest over every slot of the row.  A row whose margin exceeds a kernel's relative rounding error has the same ReLU
    derivatives in the kernel as here.  Runs on the device of `w`; returns a CPU tensor."""
    w = torch.as_tensor(w)
    state = torch.as_tensor(state).to(device=w.device, dtype=torch.float64)
    ids = torch.as_tensor(action).long().to(w.device)
    ids = ids.view(-1, 1) if ids.dim() == 1 else ids
    B, S = ids.shape
    onehot = torch.eye(n_actions, dtype=torch.float64, device=w.device)[ids.reshape(-1)]
    state = state.repeat_interleave(S, dim=0)
    net = unflatten(w, obs, n_actions, hidden)
    z1, _, z2, _, _ = _forward(net, state, onehot)
    s1, _, s2, _, _ = _forward(tuple(p.abs() for p in net), state.abs(), onehot)
    m = torch.minimum((z1.abs() / s1).min(1)[0], (z2.abs() / s2).min(1)[0])
    return m.view(B, S).min(1)[0].cpu()


def next_action_gap(w, next_state, avail_ids, avail_n, obs: int, n_actions: int, hidden=(64, 64)) -> torch.Tensor:
    """Per row: (top-1 - top-2) of the online Q(s', .) of the network `w` over the available slots, over the sum of the
    two values' error scales; inf where only one action is available.  A DoubleDQN row whose gap exceeds a kernel's
    relative rounding error picks the same a* in the kernel as here.  Runs on the device of `w`; returns a CPU tensor."""
    w = torch.as_tensor(w)
    dev = w.device
    next_state = torch.as_tensor(next_state).to(device=dev, dtype=torch.float64)
    avail_ids = torch.as_tensor(avail_ids).long().to(dev)
    avail_n = torch.as_tensor(avail_n).long().to(dev)
    if n_actions < 2:
        return torch.full((next_state.shape[0],), float("inf"), dtype=torch.float64)
    net = unflatten(w, obs, n_actions, hidden)
    v = _next_q(net, next_state, avail_ids, avail_n)
    sv = _next_q(tuple(p.abs() for p in net), next_state.abs(), avail_ids, avail_n)
    top, slot = v.topk(2, dim=1)
    gap = (top[:, 0] - top[:, 1]) / (sv.gather(1, slot).sum(1))
    return torch.where(avail_n > 1, gap, float("inf")).cpu()


def err_over_scale(got, want, scale) -> torch.Tensor:
    """|got - want| / scale elementwise; an element of scale 0 (say a dead hidden unit's gradient) must be exact: 0 if it
    is, inf if not."""
    diff = (torch.as_tensor(got).to(torch.float64) - want).abs()
    return torch.where(scale > 0, diff / scale.clamp_min(1e-300), torch.where(diff > 0, float("inf"), 0.0))


def block_slices(obs: int, n_actions: int, hidden=(64, 64)) -> dict:
    """Where each gradient block lives in the flat torch-order vector: name -> (offset, rows, cols, column offset,
    row pitch) so that element (r, c) of the block is flat[offset + r * pitch + col0 + c]."""
    h1, h2 = hidden
    D = obs + n_actions
    o_b1 = h1 * D
    o_W2 = o_b1 + h1
    o_b2 = o_W2 + h2 * h1
    o_W3 = o_b2 + h2
    o_b3 = o_W3 + h2
    return dict(dW1s=(0, h1, obs, 0, D), dW1a=(0, h1, n_actions, obs, D), db1=(o_b1, 1, h1, 0, h1),
                dW2=(o_W2, h2, h1, 0, h1), db2=(o_b2, 1, h2, 0, h2), dW3=(o_W3, 1, h2, 0, h2), db3=(o_b3, 1, 1, 0, 1))


def block_view(flat: torch.Tensor, name: str, obs: int, n_actions: int, hidden=(64, 64)) -> torch.Tensor:
    """Block `name` of a flat torch-order vector as a [rows, cols] tensor."""
    off, rows, cols, col0, pitch = block_slices(obs, n_actions, hidden)[name]
    return flat[off:off + rows * pitch].view(rows, pitch)[:, col0:col0 + cols]


def make_data(w, obs: int, n_actions: int, B: int, seed: int, dynamic: bool, margin: float, hidden=(64, 64),
              double: bool = False, all_slots: bool = False, margin_fn=None, gap_fn=None) -> dict:
    """2 B + 16 transitions (host tensors, push order) for a shape test of a learner with online parameters `w`:
    about 20 % terminal, some truncated, random actions, full or (`dynamic`) random next-action sets.  A row is kept
    only if every online pre-activation clears `margin` of its scale (relu_margin) and, for DoubleDQN, the online
    next-action gap clears it too (next_action_gap), so a kernel's rounding cannot flip a ReLU derivative or a*.
    `all_slots`: the online pass evaluates every action id as well as the taken one (the A + 1 slots of the conservative
    and dueling learners; any current set drawn from those ids is then covered too), so the margin is taken over the
    [B, A + 1] slot matrix.  `margin_fn(w, state, slot_ids)` / `gap_fn(w, next_state, ids, n)` replace relu_margin /
    next_action_gap for another network (defaults: the VanillaQValueNetwork of `obs`, `n_actions`, `hidden`).
    Candidates are drawn in batches of 3 (2 B + 16) until enough rows are kept; the fp64 filters run on the device of
    `w`."""
    from oracle.synth import make_transitions
    if margin_fn is None:
        margin_fn = lambda w, s, a: relu_margin(w, s, a, obs, n_actions, hidden)  # noqa: E731
    if gap_fn is None:
        gap_fn = lambda w, s, ids, n: next_action_gap(w, s, ids, n, obs, n_actions, hidden)  # noqa: E731
    n = 2 * B + 16
    keys = ("state", "action", "reward", "next_state", "terminated", "truncated", "next_avail_ids", "next_avail_n")
    kept = {k: [] for k in keys}
    have = 0
    for attempt in range(20):
        s = seed + 1000003 * attempt
        d = make_transitions(3 * n, obs, n_actions, seed=s, dynamic=dynamic, p_term=0.2)
        rng = np.random.default_rng(s)
        d["action"] = rng.integers(0, n_actions, 3 * n)
        d["truncated"] = rng.random(3 * n) < 0.1
        if not dynamic:
            d["next_avail_ids"] = np.tile(np.arange(n_actions), (3 * n, 1))
            d["next_avail_n"] = np.full(3 * n, n_actions)
        slots = d["action"]
        if all_slots:
            slots = np.concatenate([np.tile(np.arange(n_actions), (3 * n, 1)), d["action"].reshape(-1, 1)], 1)
        ok = margin_fn(w, d["state"], slots) >= margin
        if double:
            ok &= gap_fn(w, d["next_state"], d["next_avail_ids"], d["next_avail_n"]) >= margin
        keep = np.flatnonzero(ok.numpy())[:n - have]
        for k in keys:
            kept[k].append(d[k][keep])
        have += keep.size
        if have == n:
            break
    assert have == n, "too few rows clear the margin"
    cat = {k: torch.from_numpy(np.concatenate(v)) for k, v in kept.items()}
    return dict(state=cat["state"], action=cat["action"], reward=cat["reward"], next_state=cat["next_state"],
                terminated=cat["terminated"], truncated=cat["truncated"], avail_ids=cat["next_avail_ids"],
                avail_n=cat["next_avail_n"])


def check(what, got, want, scale, worst: dict, bound: float) -> None:
    """|got - want| <= bound * scale elementwise (got: a kernel's values, want / scale: fp64 value and error scale).
    Records the largest err / scale in worst[what]; raises AssertionError naming the first element that exceeds it."""
    want, scale = want.cpu(), scale.cpu()
    got = torch.as_tensor(got).detach().cpu().to(torch.float64).reshape(want.shape)
    r = err_over_scale(got, want, scale)
    m = float(r.max()) if r.numel() else 0.0
    worst[what] = max(worst.get(what, 0.0), m)
    if not m <= bound:
        pos = np.unravel_index(int(r.argmax()), tuple(r.shape)) if r.dim() else ()
        raise AssertionError(f"{what}{tuple(int(i) for i in pos)}: kernel {float(got[pos]):.9e}, fp64 "
                             f"{float(want[pos]):.9e}, |err| = {m:.2e} x scale {float(scale[pos]):.3e} > {bound:g}")


def q_values(w, state, obs: int, n_actions: int, hidden=(64, 64)) -> tuple:
    """(Q(s_i, a), its error scale) for every row and action id, [n, A] each, on the device of `w`."""
    w = torch.as_tensor(w)
    state = torch.as_tensor(state).to(device=w.device, dtype=torch.float64)
    n = state.shape[0]
    ids = torch.arange(n_actions, device=w.device).repeat(n, 1)
    cnt = torch.full((n,), n_actions, device=w.device)
    net = unflatten(w, obs, n_actions, hidden)
    return (_next_q(net, state, ids, cnt), _next_q(tuple(p.abs() for p in net), state.abs(), ids, cnt))
