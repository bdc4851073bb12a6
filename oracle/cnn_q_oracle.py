"""fp32 restatement of one round of the CNN DQN learners (csrc/cnnq.cu; DeepQLearning / DoubleDQN with CNNQValueNetwork or
CNNQValueMultiHeadNetwork), self-contained torch (F.conv2d, autograd, torch.optim.AdamW(amsgrad=True)) on flat parameter
vectors in torch's order.  TEST INFRASTRUCTURE: it does not import the reference.

A network is described by `spec`: dict(input=(C, H, W), conv=[(out, k, stride, pad), ...], hidden=[...], n_actions=A,
multi=bool).  A round follows deep_td_learning.py: target update first (flagged rounds), y = V gamma (1 - term) + r with V
the max over available next slots of the target values (DQN) or the target value at the online first argmax (DoubleDQN),
MSE loss, one AdamW(amsgrad) step; reported mean |q - y|.  Multi-head: the reference's taken-action values are [B, 1]
(and DoubleDQN's next values too), so its MSELoss broadcasts over B x B pairs (loss_and_grad)."""
from __future__ import annotations

import numpy as np
import torch
import torch.nn.functional as F


def conv_shapes(spec):
    C, H, W = spec["input"]
    out = []
    for oc, k, s, p in spec["conv"]:
        Ho, Wo = (H + 2 * p - k) // s + 1, (W + 2 * p - k) // s + 1
        out.append((C, H, W, oc, Ho, Wo))
        C, H, W = oc, Ho, Wo
    return out, C * H * W


def param_shapes(spec):
    """(name, shape) in torch's parameter order: `_model_cnn.{2l}`, then `_model_fc.{i}.0`."""
    convs, feat = conv_shapes(spec)
    out = []
    for i, ((c, _, _, oc, _, _), (_, k, _, _)) in enumerate(zip(convs, spec["conv"])):
        out += [(f"_model_cnn.{2 * i}.weight", (oc, c, k, k)), (f"_model_cnn.{2 * i}.bias", (oc,))]
    A = spec["n_actions"]
    dims = [feat + (0 if spec["multi"] else A)] + list(spec["hidden"]) + [A if spec["multi"] else 1]
    for i in range(len(dims) - 1):
        out += [(f"_model_fc.{i}.0.weight", (dims[i + 1], dims[i])), (f"_model_fc.{i}.0.bias", (dims[i + 1],))]
    return out


def param_count(spec) -> int:
    n = 0
    for _, s in param_shapes(spec):
        k = 1
        for d in s:
            k *= d
        n += k
    return n


def unflat(spec, flat: torch.Tensor) -> list:
    out, off = [], 0
    for _, s in param_shapes(spec):
        k = 1
        for d in s:
            k *= d
        out.append(flat[off:off + k].view(s))
        off += k
    return out


def features(spec, ps, x):
    """The conv trunk on x [N, C, H, W] pixel values: Conv2d + ReLU per layer on x / 255, flattened in (c, h, w) order."""
    h = x / 255.0
    for i, (_, _, s, p) in enumerate(spec["conv"]):
        h = F.relu(F.conv2d(h, ps[2 * i], ps[2 * i + 1], stride=s, padding=p))
    return h.reshape(x.shape[0], -1)


def fc(spec, ps, z):
    fcp = ps[2 * len(spec["conv"]):]
    n = len(fcp) // 2
    for i in range(n):
        z = F.linear(z, fcp[2 * i], fcp[2 * i + 1])
        if i < n - 1:
            z = F.relu(z)
    return z


def q_all(spec, ps, x):
    """Q(s)[a] for every action: [N, A]."""
    f = features(spec, ps, x)
    A = spec["n_actions"]
    if spec["multi"]:
        return fc(spec, ps, f)
    N = f.shape[0]
    eye = torch.eye(A, dtype=f.dtype, device=f.device)
    z = torch.cat([f.unsqueeze(1).expand(N, A, f.shape[1]), eye.unsqueeze(0).expand(N, A, A)], -1).reshape(N * A, -1)
    return fc(spec, ps, z).reshape(N, A)


def q_taken(spec, ps, x, a):
    f = features(spec, ps, x)
    A = spec["n_actions"]
    if spec["multi"]:
        return fc(spec, ps, f).gather(1, a.view(-1, 1)).squeeze(1)
    return fc(spec, ps, torch.cat([f, F.one_hot(a, A).to(f.dtype)], -1)).squeeze(-1)


def next_values(spec, w, wt, next_state, next_ids, next_count, double):
    """V per row: next_ids [B, A] (available slots first), next_count [B]."""
    with torch.no_grad():
        qt = q_all(spec, unflat(spec, wt), next_state).gather(1, next_ids)
        avail = torch.arange(next_ids.shape[1]).unsqueeze(0) < next_count.unsqueeze(1)
        if double:
            qn = q_all(spec, unflat(spec, w), next_state).gather(1, next_ids).masked_fill(~avail, -float("inf"))
            return qt.gather(1, qn.argmax(1, keepdim=True)).squeeze(1)
        return qt.masked_fill(~avail, -float("inf")).max(1).values


def loss_and_grad(spec, w, batch, V, gamma, double):
    """The Bellman loss's gradient with respect to the flat parameters, and the reported loss."""
    p = w.detach().clone().requires_grad_(True)
    ps = unflat(spec, p)
    q = q_taken(spec, ps, batch["state"], batch["action"])
    if spec["multi"]:
        # the reference's taken-action values are [B, 1], and so are DoubleDQN's next values (the target's get_q_values
        # on one action per row): the target is y_j (DQN) or V_i gamma (1 - term_j) + r_j (DoubleDQN), over B x B pairs
        V = V.unsqueeze(1) if double else V
        y = V * gamma * (1 - batch["terminated"].to(V.dtype)) + batch["reward"]
        d = q.unsqueeze(1) - (y if double else y.unsqueeze(0))
    else:
        d = q - (V * gamma * (1 - batch["terminated"].to(V.dtype)) + batch["reward"])
    loss = (d * d).mean()
    (g,) = torch.autograd.grad(loss, p)
    return g, float(d.detach().abs().mean())


def adamw(w, g, m, v, vmax, step, lr, betas=(0.9, 0.999), eps=1e-8, weight_decay=0.01):
    """One torch.optim.AdamW(amsgrad=True) step on the flat vectors; returns the new (w, m, v, vmax, step)."""
    p = torch.nn.Parameter(w.detach().clone())
    opt = torch.optim.AdamW([p], lr=lr, betas=betas, eps=eps, weight_decay=weight_decay, amsgrad=True, foreach=False)
    if step:
        opt.state[p] = dict(step=torch.tensor(float(step)), exp_avg=m.clone(), exp_avg_sq=v.clone(), max_exp_avg_sq=vmax.clone())
    p.grad = g.detach().clone()
    opt.step()
    st = opt.state[p]
    return p.detach(), st["exp_avg"], st["exp_avg_sq"], st["max_exp_avg_sq"], step + 1


def round_step(spec, st: dict, batch: dict, *, double, gamma, tau, lr, update_target, betas=(0.9, 0.999), eps=1e-8,
               weight_decay=0.01):
    """One round on `batch` (state / next_state [B, C, H, W] fp32 pixel values, action [B] ids, reward [B], terminated [B],
    next_ids [B, A], next_count [B]).  st: dict(w, wt, m, v, vmax, step), updated in place; returns the reported loss."""
    if update_target:
        st["wt"] = tau * st["w"] + (1 - tau) * st["wt"]
    V = next_values(spec, st["w"], st["wt"], batch["next_state"], batch["next_ids"], batch["next_count"], double)
    g, rep = loss_and_grad(spec, st["w"], batch, V, gamma, double)
    st["w"], st["m"], st["v"], st["vmax"], st["step"] = adamw(st["w"], g, st["m"], st["v"], st["vmax"], st["step"], lr, betas, eps,
                                                              weight_decay)
    st["grad"] = g
    return rep


# ------------------------------------------------------------------ the recordings (tests/golden/cnnq_*.npz)
def spec_of(fx) -> dict:
    conv = [tuple(int(v) for v in t) for t in zip(fx["channels"], fx["kernels"], fx["strides"], fx["paddings"])]
    return dict(input=tuple(int(v) for v in fx["input"]), conv=conv, hidden=[int(v) for v in fx["fc"]],
                n_actions=int(fx["n_actions"]), multi=bool(fx["multi"]))


def batch_of(fx, idx) -> dict:
    """Rows idx of a recording as fp32 / int64 tensors (pixel values as floats, next slots available first)."""
    g = lambda k: torch.from_numpy(np.asarray(fx[k][idx]))  # noqa: E731
    return dict(state=g("state").float(), next_state=g("next_state").float(), action=g("action").long(), reward=g("reward").float(),
                terminated=g("terminated").bool(), next_ids=g("next_ids").long(), next_count=g("next_count").long())


def replay(fx) -> dict:
    """Every round of a learn recording through round_step: the losses and the nets after every call."""
    spec = spec_of(fx)
    w = torch.from_numpy(fx["init_q"].copy())
    st = dict(w=w, wt=w.clone(), m=torch.zeros_like(w), v=torch.zeros_like(w), vmax=torch.zeros_like(w), step=0)
    R, freq = int(fx["rounds"]), int(fx["target_update_freq"])
    per_call = 1 if bool(fx["learn_batch"]) else R
    steps, losses, q_calls, qt_calls = 0, [], [], []
    for r, idx in enumerate(fx["idx"]):
        if not bool(fx["learn_batch"]):
            steps += 1                        # PolicyLearner.learn counts the round first; learn_batch alone does not
        losses.append(round_step(spec, st, batch_of(fx, idx), double=bool(fx["double"]), gamma=float(fx["gamma"]),
                                 tau=float(fx["tau"]), lr=float(fx["call_lr"][r // per_call]),
                                 update_target=(steps + 1) % freq == 0))
        if (r + 1) % per_call == 0:
            q_calls.append(st["w"].clone())
            qt_calls.append(st["wt"].clone())
    return dict(loss=np.asarray(losses), q_calls=torch.stack(q_calls).numpy(), qt_calls=torch.stack(qt_calls).numpy(), state=st)
