"""oracle/ac_fp64.py — one round of the continuous actor-critic learners in float64, with an error scale for every quantity.

TEST INFRASTRUCTURE ONLY (like the rest of oracle/).  sac_step is one round of csrc/sac.cu (ContinuousSoftActorCritic),
td3_step one round of csrc/td3.cu (TD3, DDPG, TD3BC), each in the order the kernels run it.  The networks are flat
vectors in torch parameters() order:

    SAC actor    W1 [h1, obs], b1, W2 [h2, h1], b2, Wmu [A, h2], bmu, Wsd [A, h2], bsd      (GaussianActorNetwork)
    TD3 actor    W1 [h1, obs], b1, W2 [h2, h1], b2, W3 [A, h2], b3                          (VanillaContinuousActorNetwork)
    behaviour    the TD3 actor layout with its own widths (TD3BC)
    critics      two VanillaQValueNetworks back to back, each W1 [c1, obs + A], b1, W2 [c2, c1], b2, W3 [1, c2], b3

Everything is written as explicit formulas, not autograd, on values of class V that carry (value, scale).  The scale of
a result is the sum of |a||b| over every product that reached it: sums and products act on the scales as the same code
acts on |.| of every operand (s(a + b) = s(a) + s(b), s(ab) = s(a) s(b), s(x W^T) = s(x) |W|^T), so a chain of dot
products has the natural scale of its rounding error.  ReLU keeps the mask of the value pass on the scale as well.

Elementwise functions (tanh, exp, log, 1 - x^2, 1 / x) do not follow the |.| rule: their scale is |f'(x)| times the
scale of the input, plus K_ULP |f(x)|.  The first term carries the error of the input through f; the second is a few ulps
of the value itself (in units of the test's bound, which is at least u = 2^-24 per unit of scale), which covers the
rounding of f in fp32 and CUDA's tanhf / expf / logf, which are not correctly rounded (up to 2 ulp).  A value near a
cancellation (1 - tanh^2 near saturation, the log of it, q - y) thus keeps the scale of the operands it cancelled.

min(q1, q2), the clamps of TD3's target action and |q| are continuous and take the scale of the branch they pick; the
gradient routing of SAC's min (to critic 1 where q1 <= q2, as k_sac_actor_loss) is not, so a row whose |q1 - q2| is
within rounding of 0 has to be left out of a comparison (the shape test redraws it).
"""
from __future__ import annotations

import math

import torch

K_ULP = 4.0
LOG_SQRT_2PI = math.log(math.sqrt(2 * math.pi))


class V:
    """A float64 tensor and its error scale (same shape, non-negative)."""
    __slots__ = ("v", "s")

    def __init__(self, v, s=None):
        self.v = v
        self.s = v.abs() if s is None else s

    @staticmethod
    def lift(x, like):
        if isinstance(x, V):
            return x
        t = torch.as_tensor(x, dtype=torch.float64, device=like.v.device)
        return V(t, t.abs())

    def __add__(self, o):
        o = V.lift(o, self)
        return V(self.v + o.v, self.s + o.s)

    __radd__ = __add__

    def __sub__(self, o):
        o = V.lift(o, self)
        return V(self.v - o.v, self.s + o.s)

    def __rsub__(self, o):
        return V.lift(o, self) - self

    def __neg__(self):
        return V(-self.v, self.s)

    def __mul__(self, o):
        o = V.lift(o, self)
        return V(self.v * o.v, self.s * o.s)

    __rmul__ = __mul__

    def __truediv__(self, o):
        if isinstance(o, V):
            return self * recip(o)
        c = float(o)
        return V(self.v / c, self.s / abs(c))

    def __matmul__(self, o):
        return V(self.v @ o.v, self.s @ o.s)

    def __getitem__(self, i):
        return V(self.v[i], self.s[i])

    @property
    def T(self):
        return V(self.v.T, self.s.T)

    def sum(self, *a, **k):
        return V(self.v.sum(*a, **k), self.s.sum(*a, **k))

    def mean(self, *a, **k):
        return V(self.v.mean(*a, **k), self.s.mean(*a, **k))

    def view(self, *shape):
        return V(self.v.reshape(*shape), self.s.reshape(*shape))


def fn(x: V, f, df) -> V:
    """y = f(x) with scale |f'(x)| s(x) + K_ULP |y| (see the module docstring)."""
    y = f(x.v)
    return V(y, df(x.v, y).abs() * x.s + K_ULP * y.abs())


def tanh(x):
    return fn(x, torch.tanh, lambda x, y: 1 - y * y)


def exp(x):
    return fn(x, torch.exp, lambda x, y: y)


def log(x):
    return fn(x, torch.log, lambda x, y: 1 / x)


def one_minus_sq(x):
    return fn(x, lambda t: 1 - t * t, lambda x, y: 2 * x)


def recip(x):
    return fn(x, lambda t: 1 / t, lambda x, y: y * y)


def relu(z):
    m = (z.v > 0).to(torch.float64)
    return V(z.v * m, z.s * m), m


def masked(x: V, m) -> V:
    return V(x.v * m, x.s * m)


def cat(xs, dim):
    return V(torch.cat([x.v for x in xs], dim), torch.cat([x.s for x in xs], dim))


def minimum(a: V, b: V) -> V:
    first = a.v <= b.v
    return V(torch.where(first, a.v, b.v), torch.where(first, a.s, b.s))


def clamp(x: V, lo: V, hi: V) -> V:
    below, above = x.v < lo.v, x.v > hi.v
    return V(torch.where(below, lo.v, torch.where(above, hi.v, x.v)), torch.where(below, lo.s, torch.where(above, hi.s, x.s)))


def lin(x: V, W: V, b: V) -> V:
    return x @ W.T + b


# ---------------------------------------------------------------------------------------------- layouts
def sac_actor_shapes(obs, A, hidden):
    h1, h2 = hidden
    return dict(W1=(h1, obs), b1=(h1,), W2=(h2, h1), b2=(h2,), Wmu=(A, h2), bmu=(A,), Wsd=(A, h2), bsd=(A,))


def td3_actor_shapes(obs, A, hidden):
    h1, h2 = hidden
    return dict(W1=(h1, obs), b1=(h1,), W2=(h2, h1), b2=(h2,), W3=(A, h2), b3=(A,))


def critic_shapes(obs, A, hidden):
    c1, c2 = hidden
    return dict(W1=(c1, obs + A), b1=(c1,), W2=(c2, c1), b2=(c2,), W3=(1, c2), b3=(1,))


def unflatten(flat, shapes: dict) -> dict:
    """name -> V view of a flat torch-order vector (float64, on the vector's device)."""
    flat = torch.as_tensor(flat).to(torch.float64)
    out, off = {}, 0
    for k, s in shapes.items():
        n = math.prod(s)
        out[k] = V(flat[off:off + n].view(s))
        off += n
    assert off == flat.numel(), "parameter count does not match the network shape"
    return out


def flatten(blocks: dict, shapes: dict) -> V:
    """The blocks of a gradient dict (name -> V) as one flat torch-order V."""
    return cat([blocks[k].view(-1) for k in shapes], 0)


def twin(flat, obs, A, hidden):
    """The two critics of a flat twin vector."""
    flat = torch.as_tensor(flat)
    n = flat.numel() // 2
    return unflatten(flat[:n], critic_shapes(obs, A, hidden)), unflatten(flat[n:], critic_shapes(obs, A, hidden))


# ---------------------------------------------------------------------------------------------- networks
def critic_forward(c: dict, s: V, a: V):
    x = cat([s, a], 1)
    z1 = lin(x, c["W1"], c["b1"])
    h1, m1 = relu(z1)
    z2 = lin(h1, c["W2"], c["b2"])
    h2, m2 = relu(z2)
    q = lin(h2, c["W3"], c["b3"])[:, 0]
    return dict(x=x, z1=z1, h1=h1, m1=m1, z2=z2, h2=h2, m2=m2, q=q)


def critic_backward(c: dict, f: dict, dq: V):
    """Parameter gradient of sum_i dq_i q_i, and the gradient with respect to the critic's input [s || a]."""
    dz2 = masked(dq.view(-1, 1) @ c["W3"], f["m2"])
    dz1 = masked(dz2 @ c["W2"], f["m1"])
    g = dict(W1=dz1.T @ f["x"], b1=dz1.sum(0), W2=dz2.T @ f["h1"], b2=dz2.sum(0), W3=dq.view(1, -1) @ f["h2"],
             b3=dq.sum(0).view(1))
    return g, dz1 @ c["W1"]


def mlp_forward(p: dict, s: V, head: str):
    """The two ReLU layers and the linear head `head` (W3 / Wmu) of an actor."""
    z1 = lin(s, p["W1"], p["b1"])
    h1, m1 = relu(z1)
    z2 = lin(h1, p["W2"], p["b2"])
    h2, m2 = relu(z2)
    return dict(z1=z1, h1=h1, m1=m1, z2=z2, h2=h2, m2=m2, out=lin(h2, p[head], p["b" + head[1:]]))


def mlp_backward(p: dict, f: dict, s: V, dh2: V) -> dict:
    """Gradients of W1 b1 W2 b2 from the gradient at h2 (before its ReLU mask)."""
    dz2 = masked(dh2, f["m2"])
    dz1 = masked(dz2 @ p["W2"], f["m1"])
    return dict(W1=dz1.T @ s, b1=dz1.sum(0), W2=dz2.T @ f["h1"], b2=dz2.sum(0))


def _box(low, high, like):
    lo, hi = V.lift(low, like), V.lift(high, like)
    return lo, hi, (hi - lo) / 2


def sac_sample(actor: dict, s: V, eps: V, low, high) -> dict:
    """GaussianActorNetwork.sample_action with the rsample noise given (k_sac_sample)."""
    f = mlp_forward(actor, s, "Wmu")
    mean, z = f["out"], lin(f["h2"], actor["Wsd"], actor["bsd"])
    tz = tanh(z)
    log_std = (tz + 1.0) * 3.5 - 5.0
    sd = exp(log_std)
    u = mean + sd * eps
    na = tanh(u)
    lo, hi, bound = _box(low, high, s)
    action = (hi - lo) * (na + 1.0) / 2 + lo
    diff = u - mean
    omn = one_minus_sq(na)
    arg = bound * omn + 1e-6
    t = -(diff * diff) * recip(sd * sd * 2.0) - log_std - LOG_SQRT_2PI - log(arg)
    return dict(f, mean=mean, z=z, tz=tz, log_std=log_std, sd=sd, u=u, na=na, omn=omn, arg=arg, action=action,
                logp=t.sum(1))


def _adamw1(w, g, lr, beta1=0.9, beta2=0.999, eps=1e-8, weight_decay=0.01):
    """The first AdamW(amsgrad) step from zero state, in float64."""
    m, v = (1 - beta1) * g, (1 - beta2) * g * g
    return w * (1 - lr * weight_decay) - lr / (1 - beta1) * m / ((v / (1 - beta2)).sqrt() + eps)


def _f64(x, dev):
    return torch.as_tensor(x).to(device=dev, dtype=torch.float64)


def _batch(batch, dev):
    s, a, r, s2 = (V(_f64(batch[k], dev)) for k in ("state", "action", "reward", "next_state"))
    term = _f64(batch["terminated"], dev)
    return s, a, r, s2, term


def _critic_step(critics, s, a, y, B, obs):
    """Twin MSE (mse1 + mse2) / 2 with dq_i = (q_i - y) / B: gradients of both critics (flat), q, the loss."""
    grads, qs, loss = [], [], None
    for c in critics:
        f = critic_forward(c, s, a)
        e = f["q"] - y
        g, _ = critic_backward(c, f, e / B)
        grads.append(g)
        qs.append(f["q"])
        sq = (e * e).sum(0)
        loss = sq if loss is None else loss + sq
    return grads, qs, loss / (2 * B), f


def _pack(prefix, g: dict, out_v: dict, out_s: dict):
    for k, x in g.items():
        out_v[prefix + k], out_s[prefix + k] = x.v, x.s


def _split(d: dict):
    return {k: x.v for k, x in d.items()}, {k: x.s for k, x in d.items()}


def sac_step(actor, critics, critic_targets, actor_after, log_alpha, batch: dict, noise, low, high, *, obs, A,
             actor_hidden, critic_hidden, gamma, alpha=None, autotune=True, lr_entropy=1e-3) -> tuple:
    """One round of csrc/sac.cu in float64.  `actor`, `critics` (twin flat vector), `critic_targets`: parameters before the
    round; `actor_after`: the actor after this round's actor step (the kernel's own fp32 vector; the critic step samples
    the next action with it); `log_alpha`: the entropy parameter before the round; `alpha`: the coefficient the round uses
    (exp(log_alpha) with autotune, else the fixed coefficient); `noise` [2, B, A]: the rsample draws of the actor step and
    of the critic step.  Returns (value, scale) dicts with the actor gradient blocks a.W1 .. a.bsd, the critics' q1.W1 ..
    q2.b3, `actor_grad` / `critic_grad` (flat, torch order), `actor_loss`, `critic_loss`, `q_pi` [2, B] (both critics at
    (s, pi(s))), `q` [2, B] (at (s, a)), `y`, `logp`, `logp2`, `u` (the actor step's pre-tanh sample), and with autotune
    `entropy_loss`, `log_alpha_grad` and `log_alpha_new` (one AdamW step from zero state at lr_entropy)."""
    dev = torch.as_tensor(actor).device
    s, a, r, s2, term = _batch(batch, dev)
    B = s.v.shape[0]
    nz = _f64(noise, dev)
    ash = sac_actor_shapes(obs, A, actor_hidden)
    p, p_after = unflatten(actor, ash), unflatten(actor_after, ash)
    q_nets, t_nets = twin(critics, obs, A, critic_hidden), twin(critic_targets, obs, A, critic_hidden)
    la = float(log_alpha)
    al = V.lift(math.exp(la) if alpha is None else float(alpha), s)
    # ---- actor step
    smp = sac_sample(p, s, V(nz[0]), low, high)
    fs = [critic_forward(c, s, smp["action"]) for c in q_nets]
    q1, q2 = fs[0]["q"], fs[1]["q"]
    actor_loss = (al * smp["logp"] - minimum(q1, q2)).mean(0)
    first = (q1.v <= q2.v).to(torch.float64)
    da = None
    for c, f, w in zip(q_nets, fs, (first, 1 - first)):
        _, dx = critic_backward(c, f, V(-w / B))
        da = dx[:, obs:] if da is None else da + dx[:, obs:]
    lo, hi, bound = _box(low, high, s)
    al_b = al / B
    n = smp["na"]
    dna = da * bound + al_b * (bound * n * 2.0) * recip(smp["arg"])
    du = dna * smp["omn"]
    dlogstd = du * smp["sd"] * V(nz[0]) - al_b
    dz = dlogstd * 3.5 * one_minus_sq(smp["tz"])
    ga = dict(Wmu=du.T @ smp["h2"], bmu=du.sum(0), Wsd=dz.T @ smp["h2"], bsd=dz.sum(0))
    ga.update(mlp_backward(p, smp, s, du @ p["Wmu"] + dz @ p["Wsd"]))
    ga = {k: ga[k] for k in ash}
    # ---- critic step, the next action from the UPDATED actor
    smp2 = sac_sample(p_after, s2, V(nz[1]), low, high)
    qt = [critic_forward(c, s2, smp2["action"])["q"] for c in t_nets]
    y = (minimum(qt[0], qt[1]) - al * smp2["logp"]) * gamma * V(1 - term) + r
    gc, qs, critic_loss, _ = _critic_step(q_nets, s, a, y, B, obs)
    cs = critic_shapes(obs, A, critic_hidden)
    value, scale = {}, {}
    _pack("a.", ga, value, scale)
    _pack("q1.", gc[0], value, scale)
    _pack("q2.", gc[1], value, scale)
    flat_a, flat_c = flatten(ga, ash), cat([flatten(gc[0], cs), flatten(gc[1], cs)], 0)
    extra = dict(actor_grad=flat_a, critic_grad=flat_c, actor_loss=actor_loss, critic_loss=critic_loss,
                 q_pi=V(torch.stack([q1.v, q2.v]), torch.stack([q1.s, q2.s])),
                 q=V(torch.stack([qs[0].v, qs[1].v]), torch.stack([qs[0].s, qs[1].s])), y=y, logp=smp["logp"],
                 logp2=smp2["logp"], u=smp["u"])
    if autotune:
        ea = exp(V.lift(la, s))
        ent = -(ea * (smp["logp"] - float(A)).mean(0))
        extra.update(entropy_loss=ent, log_alpha_grad=ent)
    ev, es = _split(extra)
    value.update(ev)
    scale.update(es)
    if autotune:
        value["log_alpha_new"] = _adamw1(torch.tensor(la, dtype=torch.float64), value["log_alpha_grad"], lr_entropy)
    return value, scale


def td3_act(p: dict, s: V, low, high):
    f = mlp_forward(p, s, "W3")
    na = tanh(f["out"])
    lo, hi, _ = _box(low, high, s)
    return dict(f, na=na, action=(hi - lo) * (na + 1.0) / 2 + lo)


def td3_step(actor, critics, actor_target, critic_targets, batch: dict, low, high, *, obs, A, actor_hidden, critic_hidden,
             gamma, kind="td3", update_actor=True, noise=None, noise_clip=0.5, behavior=None, behavior_hidden=None,
             alpha_bc=2.5) -> tuple:
    """One round of csrc/td3.cu in float64.  `kind`: "td3", "ddpg" or "td3bc" (with `behavior`, its flat parameters, and
    `behavior_hidden`); `update_actor`: the round runs the actor step; `noise` [B, A]: the target-policy draws (None:
    DDPG, no noise).  The target uses the actor target before the round.  Returns (value, scale) dicts with the actor
    gradient blocks a.W1 .. a.b3 (update rounds), the critics' q1.W1 .. q2.b3, `actor_grad` / `critic_grad` (flat, torch
    order), `actor_loss` (update rounds), `critic_loss`, `q_pi` [B] (critic 1 at (s, pi(s))), `pre` (the actor's
    pre-tanh output at s), `q` [2, B], `y`, `target_action` and, for TD3BC, `lambda`."""
    dev = torch.as_tensor(actor).device
    s, a, r, s2, term = _batch(batch, dev)
    B = s.v.shape[0]
    ash = td3_actor_shapes(obs, A, actor_hidden)
    q_nets, t_nets = twin(critics, obs, A, critic_hidden), twin(critic_targets, obs, A, critic_hidden)
    lo, hi, bound = _box(low, high, s)
    value, scale = {}, {}
    extra = {}
    if update_actor:
        p = unflatten(actor, ash)
        fa = td3_act(p, s, low, high)
        f1 = critic_forward(q_nets[0], s, fa["action"])
        q1 = f1["q"]
        if kind == "td3bc":
            bnet = unflatten(behavior, td3_actor_shapes(obs, A, behavior_hidden))
            b = tanh(mlp_forward(bnet, s, "W3")["out"])
            lam = V.lift(alpha_bc, s) * recip(V(q1.v.abs(), q1.s).mean(0))
            d = fa["action"] - b
            extra["actor_loss"] = (d * d).mean() - lam * q1.mean(0)
            extra["lambda"] = lam
            dq = V(-lam.v.expand(B) / B, lam.s.expand(B) / B)
        else:
            extra["actor_loss"] = -q1.mean(0)
            dq = V(torch.full((B,), -1.0 / B, dtype=torch.float64, device=dev))
        _, dx = critic_backward(q_nets[0], f1, dq)
        g = dx[:, obs:]
        if kind == "td3bc":
            g = g + d * (2.0 / (B * A))
        dpre = g * bound * one_minus_sq(fa["na"])
        ga = dict(W3=dpre.T @ fa["h2"], b3=dpre.sum(0))
        ga.update(mlp_backward(p, fa, s, dpre @ p["W3"]))
        ga = {k: ga[k] for k in ash}
        _pack("a.", ga, value, scale)
        extra.update(actor_grad=flatten(ga, ash), q_pi=q1, pre=fa["out"])
    ft = td3_act(unflatten(actor_target, ash), s2, low, high)
    at = ft["action"]
    if noise is not None:
        nz = V(_f64(noise, dev))
        nz = clamp(nz, V.lift(-noise_clip, s), V.lift(noise_clip, s)) * (hi - lo) / 2
        at = clamp(at + nz, lo.view(1, -1), hi.view(1, -1))
    qt = [critic_forward(c, s2, at)["q"] for c in t_nets]
    y = minimum(qt[0], qt[1]) * gamma * V(1 - term) + r
    gc, qs, critic_loss, _ = _critic_step(q_nets, s, a, y, B, obs)
    cs = critic_shapes(obs, A, critic_hidden)
    _pack("q1.", gc[0], value, scale)
    _pack("q2.", gc[1], value, scale)
    extra.update(critic_grad=cat([flatten(gc[0], cs), flatten(gc[1], cs)], 0), critic_loss=critic_loss,
                 q=V(torch.stack([qs[0].v, qs[1].v]), torch.stack([qs[0].s, qs[1].s])), y=y, target_action=at)
    ev, es = _split(extra)
    value.update(ev)
    scale.update(es)
    return value, scale


# ---------------------------------------------------------------------------------------------- data filters
def relu_margin_of(*forwards) -> torch.Tensor:
    """Per row: the smallest |pre-activation| / scale over the hidden layers of the given forward dicts."""
    m = None
    for f in forwards:
        for k in ("z1", "z2"):
            z = f[k]
            r = (z.v.abs() / z.s.clamp_min(1e-300)).min(1)[0]
            m = r if m is None else torch.minimum(m, r)
    return m
