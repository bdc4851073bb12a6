"""oracle/ac_fp64.py (the float64 round of the continuous actor-critic learners, written as explicit formulas) against
torch autograd in float64 on the restatements of the reference (oracle/sac_oracle.py, td3_oracle.py, td3bc_oracle.py,
cast to float64): every gradient block, the losses, the TD target and SAC's log-probs and entropy gradient, at a handful
of small shapes with asymmetric per-dimension boxes, for SAC (autotune on and off), TD3, DDPG and TD3BC.  Also checks
that every scale covers its value (scale >= |value|), the property the GPU shape tests' bound rests on.  CPU only."""
import math

import pytest
import torch

from oracle import ac_fp64
from oracle.sac_oracle import OracleSAC
from oracle.td3_oracle import OracleTD3
from oracle.td3bc_oracle import OracleTD3BC

# (obs, A, actor hidden, critic hidden, behaviour hidden, B)
SHAPES = [
    (1, 1, (1, 1), (1, 1), (1, 1), 1),
    (3, 2, (5, 3), (4, 6), (2, 7), 7),
    (5, 6, (8, 8), (7, 9), (6, 4), 16),
    (4, 33, (9, 5), (6, 10), (3, 3), 5),
]
GAMMA = 0.97


def _ids(c):
    return "obs{}-A{}-a{}x{}-c{}x{}-B{}".format(c[0], c[1], *c[2], *c[3], c[5])


def _box(A, g):
    lo = -torch.rand(A, generator=g, dtype=torch.float64) * 2
    hi = lo + 0.1 + torch.rand(A, generator=g, dtype=torch.float64) * 4
    return lo.float().double(), hi.float().double()     # the oracles hold the box in float32


def _vec(n, g, scale=0.5):
    return (torch.rand(n, generator=g, dtype=torch.float64) * 2 - 1) * scale


def _load64(module, vec):
    off = 0
    with torch.no_grad():
        for p in module.parameters():
            p.copy_(vec[off:off + p.numel()].view_as(p))
            off += p.numel()
    assert off == vec.numel()


def _grad(module):
    return torch.cat([p.grad.reshape(-1) for p in module.parameters()])


def _nparams(module):
    return sum(p.numel() for p in module.parameters())


def _batch(obs, A, B, lo, hi, g):
    return dict(state=torch.randn(B, obs, generator=g, dtype=torch.float64),
                action=lo + (hi - lo) * torch.rand(B, A, generator=g, dtype=torch.float64),
                reward=torch.randn(B, generator=g, dtype=torch.float64),
                next_state=torch.randn(B, obs, generator=g, dtype=torch.float64),
                terminated=(torch.rand(B, generator=g) < 0.3).to(torch.float64))


def _close(name, got, want):
    want = torch.as_tensor(want, dtype=torch.float64).reshape(-1)
    got = torch.as_tensor(got, dtype=torch.float64).reshape(-1)
    tol = 1e-10 * (1 + want.abs().max())
    assert float((got - want).abs().max()) <= tol, f"{name}: max |diff| {float((got - want).abs().max()):.3e}"


def _covers(val, sc):
    for k, v in val.items():
        if k in sc:
            v, s = torch.as_tensor(v), torch.as_tensor(sc[k])
            assert bool((s >= v.abs() * (1 - 1e-12)).all()), f"scale of {k} below its value"


def _double(orc, nets):
    for n in nets:
        n.double()
    orc.low, orc.high = orc.low.double(), orc.high.double()


@pytest.mark.parametrize("autotune", [True, False])
@pytest.mark.parametrize("shape", SHAPES, ids=_ids)
def test_sac_step_matches_autograd(shape, autotune):
    obs, A, ah, ch, _, B = shape
    g = torch.Generator().manual_seed(obs * 131 + A * 7 + B)
    lo, hi = _box(A, g)
    orc = OracleSAC(obs, A, ah, ch, lo.float(), hi.float(), autotune=autotune, entropy_coef=0.3)
    _double(orc, [orc.actor] + orc.q + orc.qt)
    orc.bound = (orc.high - orc.low) / 2
    pa, pc = _nparams(orc.actor), _nparams(orc.q[0])
    actor, after = _vec(pa, g), None
    after = actor + 1e-2 * _vec(pa, g)
    crit, targ = _vec(2 * pc, g), _vec(2 * pc, g)
    _load64(orc.actor, actor)
    for i in range(2):
        _load64(orc.q[i], crit[i * pc:(i + 1) * pc])
        _load64(orc.qt[i], targ[i * pc:(i + 1) * pc])
    log_alpha = -0.4
    alpha = math.exp(log_alpha) if autotune else 0.3
    orc.alpha = torch.tensor(alpha, dtype=torch.float64)
    b = _batch(obs, A, B, lo, hi, g)
    noise = torch.randn(2, B, A, generator=g, dtype=torch.float64)

    val, sc = ac_fp64.sac_step(actor, crit, targ, after, log_alpha, b, noise, lo, hi, obs=obs, A=A, actor_hidden=ah,
                               critic_hidden=ch, gamma=GAMMA, alpha=alpha, autotune=autotune)
    # actor step through autograd
    s = b["state"]
    act, logp = orc.sample_action(s, noise[0])
    q = torch.minimum(orc._qv(orc.q[0], s, act), orc._qv(orc.q[1], s, act)).unsqueeze(-1)
    loss = (orc.alpha * logp - q).mean()
    loss.backward()
    _close("actor_grad", val["actor_grad"], _grad(orc.actor))
    _close("actor_loss", val["actor_loss"], loss.detach())
    _close("logp", val["logp"], logp.detach())
    # critic step with the updated actor
    _load64(orc.actor, after)
    for n in orc.q:
        n.zero_grad()
    with torch.no_grad():
        a2, logp2 = orc.sample_action(b["next_state"], noise[1])
        nq = torch.minimum(orc._qv(orc.qt[0], b["next_state"], a2), orc._qv(orc.qt[1], b["next_state"], a2)).unsqueeze(-1)
        y = ((nq - orc.alpha * logp2).view(-1) * GAMMA * (1 - b["terminated"])) + b["reward"]
    mse = torch.nn.MSELoss()
    closs = (mse(orc._qv(orc.q[0], s, b["action"]), y) + mse(orc._qv(orc.q[1], s, b["action"]), y)) / 2.0
    closs.backward()
    _close("critic_grad", val["critic_grad"], torch.cat([_grad(orc.q[0]), _grad(orc.q[1])]))
    _close("critic_loss", val["critic_loss"], closs.detach())
    _close("y", val["y"], y)
    _close("logp2", val["logp2"], logp2)
    for k in ac_fp64.sac_actor_shapes(obs, A, ah):
        assert val["a." + k].shape == ac_fp64.sac_actor_shapes(obs, A, ah)[k]
    if autotune:
        la = torch.tensor([log_alpha], dtype=torch.float64, requires_grad=True)
        ent = (-torch.exp(la) * (logp.detach() - A)).mean()
        ent.backward()
        _close("entropy_loss", val["entropy_loss"], ent.detach())
        _close("log_alpha_grad", val["log_alpha_grad"], la.grad)
    _covers(val, sc)


@pytest.mark.parametrize("kind", ["td3", "ddpg", "td3bc"])
@pytest.mark.parametrize("shape", SHAPES, ids=_ids)
def test_td3_step_matches_autograd(shape, kind):
    obs, A, ah, ch, bh, B = shape
    g = torch.Generator().manual_seed(obs * 17 + A * 3 + B + len(kind))
    lo, hi = _box(A, g)
    clip = 0.4
    if kind == "td3bc":
        orc = OracleTD3BC(obs, A, ah, ch, lo.float(), hi.float(), behavior_hidden=bh, alpha_bc=1.7, noise_clip=clip)
        _double(orc, [orc.actor, orc.actor_t, orc.behavior] + orc.q + orc.qt)
    else:
        orc = OracleTD3(obs, A, ah, ch, lo.float(), hi.float(), noise_clip=clip)
        _double(orc, [orc.actor, orc.actor_t] + orc.q + orc.qt)
    pa, pc = _nparams(orc.actor), _nparams(orc.q[0])
    actor, actor_t = _vec(pa, g, 0.8), _vec(pa, g, 0.8)
    crit, targ = _vec(2 * pc, g), _vec(2 * pc, g)
    _load64(orc.actor, actor)
    _load64(orc.actor_t, actor_t)
    for i in range(2):
        _load64(orc.q[i], crit[i * pc:(i + 1) * pc])
        _load64(orc.qt[i], targ[i * pc:(i + 1) * pc])
    behavior = None
    if kind == "td3bc":
        behavior = _vec(_nparams(orc.behavior), g, 0.8)
        _load64(orc.behavior, behavior)
    b = _batch(obs, A, B, lo, hi, g)
    noise = None if kind == "ddpg" else 0.6 * torch.randn(B, A, generator=g, dtype=torch.float64)
    if noise is not None:
        noise[0, 0] = -3 * clip          # one entry past the clip, pushing the target action to the box
    for update in (True, False):
        val, sc = ac_fp64.td3_step(actor, crit, actor_t, targ, b, lo, hi, obs=obs, A=A, actor_hidden=ah, critic_hidden=ch,
                                   gamma=GAMMA, kind=kind, update_actor=update, noise=noise, noise_clip=clip,
                                   behavior=behavior, behavior_hidden=bh, alpha_bc=1.7)
        s = b["state"]
        if update:
            orc.actor.zero_grad()
            for n in orc.q:
                n.zero_grad()
            loss = orc.actor_loss(s) if kind == "td3bc" else -orc._qv(orc.q[0], s, orc.act(orc.actor, s)).mean()
            loss.backward()
            _close("actor_grad", val["actor_grad"], _grad(orc.actor))
            _close("actor_loss", val["actor_loss"], loss.detach())
        else:
            assert "actor_grad" not in val and "actor_loss" not in val
        for n in orc.q:
            n.zero_grad()
        with torch.no_grad():
            a2 = orc.act(orc.actor_t, b["next_state"])
            if noise is not None:
                a2 = torch.clamp(a2 + torch.clamp(noise, -clip, clip) * (orc.high - orc.low) / 2, orc.low, orc.high)
            nq = torch.minimum(orc._qv(orc.qt[0], b["next_state"], a2), orc._qv(orc.qt[1], b["next_state"], a2))
            y = nq * GAMMA * (1 - b["terminated"]) + b["reward"]
        mse = torch.nn.MSELoss()
        closs = (mse(orc._qv(orc.q[0], s, b["action"]), y) + mse(orc._qv(orc.q[1], s, b["action"]), y)) / 2.0
        closs.backward()
        _close("critic_grad", val["critic_grad"], torch.cat([_grad(orc.q[0]), _grad(orc.q[1])]))
        _close("critic_loss", val["critic_loss"], closs.detach())
        _close("y", val["y"], y)
        _close("target_action", val["target_action"], a2)
        _covers(val, sc)
