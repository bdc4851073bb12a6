"""The reward-constrained safety module on the CPU: the restatement (oracle/rc_safety_oracle.py) against the recordings of
the reference's PearlAgent(TD3 | DDPG | TD3BC, RCSafetyModuleCostCriticContinuousAction) (tests/golden/rc_*.npz,
oracle/gen_rc_safety_golden.py), the float64 lambda recursion and the fp32 reward shaping bit for bit, the host arithmetic
of the cost column and of the cost-critic handle, and the plugin's refusals with stand-in modules."""
import os
import types

import numpy as np
import pytest
import torch

from conftest import GOLDEN
from oracle.pearl_oracle import flat
from oracle.rc_safety_oracle import agent_learn, lambda_step, oracles_for, shaped_reward

CASES = ["rc_td3", "rc_ddpg", "rc_zero", "rc_lr", "rc_td3bc"]


def _rows(fx, ix):
    t = torch.from_numpy
    ix = ix.astype(np.int64)
    return dict(state=t(fx["state"][ix]), action=t(fx["action"][ix]), reward=t(fx["reward"][ix]), next_state=t(fx["next_state"][ix]),
                terminated=t(fx["terminated"][ix]), cost=t(fx["cost"][ix]))


def replay(fx):
    pol, cc = oracles_for(fx)
    R = int(fx["rounds"])
    noise = torch.from_numpy(fx["noise"]) if len(fx["noise"]) else None
    out = dict(actor_loss=[], critic_loss=[], cost_loss=[], cq=[], lam=[])
    for c in range(int(fx["calls"])):
        for g in cc.opt.param_groups:
            g["lr"] = float(fx["call_cost_lr"][c])
        rows = [_rows(fx, fx["idx"][c * (R + 1) + r]) for r in range(R + 1)]
        al, cl, loss, cq = agent_learn(pol, cc, rows, R, None if noise is None else noise[c * R:(c + 1) * R])
        out["actor_loss"] += al; out["critic_loss"] += cl
        out["cost_loss"].append(loss); out["cq"].append(cq); out["lam"].append(cc.lam)
    return pol, cc, out


@pytest.mark.parametrize("case", CASES)
def test_oracle_reproduces_the_reference_recording(case):
    fx = np.load(os.path.join(GOLDEN, f"{case}.npz"))
    pol, cc, out = replay(fx)
    tol = dict(rtol=5e-6, atol=1e-7)
    np.testing.assert_allclose(out["actor_loss"], fx["actor_loss"], **tol)
    np.testing.assert_allclose(out["critic_loss"], fx["critic_loss"], **tol)
    np.testing.assert_allclose(out["cost_loss"], fx["cost_loss"], **tol)
    np.testing.assert_allclose(out["cq"], fx["cq"], **tol)
    np.testing.assert_allclose(out["lam"], fx["lambda_after"], **tol)
    nets = dict(actor=pol.actor, actor_t=pol.actor_t, q1=pol.q[0], q2=pol.q[1], q1t=pol.qt[0], q2t=pol.qt[1], c1=cc.q[0], c2=cc.q[1],
                c1t=cc.qt[0], c2t=cc.qt[1])
    for name, net in nets.items():
        np.testing.assert_allclose(flat(net).numpy(), fx[f"{name}_after"], err_msg=name, **tol)


@pytest.mark.parametrize("case", CASES)
def test_lambda_recursion_is_exact_given_the_recorded_cq(case):
    fx = np.load(os.path.join(GOLDEN, f"{case}.npz"))
    lam = 0.0
    for c in range(int(fx["calls"])):
        assert lam == fx["lambda_before"][c]
        lam = lambda_step(lam, float(fx["cq"][c]), float(fx["lr_lambda"]), float(fx["cost_gamma"]), float(fx["constraint"]), float(fx["ub"]))
        assert lam == fx["lambda_after"][c], (c, lam, fx["lambda_after"][c])


def test_recordings_cover_zero_interior_and_upper_bound():
    fx = np.load(os.path.join(GOLDEN, "rc_td3.npz"))
    lam, ub = fx["lambda_after"], float(fx["ub"])
    assert fx["lambda_before"][0] == 0.0
    assert ((lam > 0) & (lam < ub)).sum() >= 2 and (lam == ub).any()
    assert (np.load(os.path.join(GOLDEN, "rc_zero.npz"))["lambda_after"] == 0.0).all()
    lr = np.load(os.path.join(GOLDEN, "rc_lr.npz"))["call_cost_lr"]
    assert len(set(lr.tolist())) == 2


def test_shaped_reward_is_two_fp32_roundings():
    """reward - lambda * cost in torch fp32 is fp32(r - fp32(fp32(lambda) * c)): what k_td3_gather computes (no FMA, the
    Python float rounded to fp32 once)."""
    g = np.random.default_rng(7)
    r = g.standard_normal(4096).astype(np.float32)
    c = g.uniform(0.0, 3.0, 4096).astype(np.float32)
    lams = [0.1, 0.21621233, 1 / 3, 0.4, 19.7, 1e-3 + 2 ** -40, float(np.float64(0.3) + 2 ** -30)]
    differs = False
    for lam in lams:
        got = shaped_reward(torch.from_numpy(r), torch.from_numpy(c), lam).numpy()
        want = r - np.float32(np.float32(lam) * c)
        assert got.dtype == np.float32
        assert np.array_equal(got.view(np.uint32), want.view(np.uint32)), lam
        fused = (r.astype(np.float64) - lam * c.astype(np.float64)).astype(np.float32)   # one rounding, lambda in float64
        differs |= not np.array_equal(fused, want)
    assert differs      # the data tell the two evaluations apart


def _lib():
    from pearl_b200 import _lib as L
    return L, L.load()


def _layout(L, lib, flags, obs, act, n_act, cap=64):
    import ctypes as C
    d = L.BufDesc(cap, obs, act, n_act, flags)
    lay = L.BufLayout()
    assert lib.prl_buf_layout_of(C.byref(d), C.byref(lay)) == 0
    off = C.c_int32(-7)
    rc = lib.prl_buf_cost_offset(C.byref(d), C.byref(off))
    return lay, rc, off.value


def test_cost_column_moves_no_offset():
    L, lib = _lib()
    fields = ["record_words", "off_state", "off_next_state", "off_action", "off_reward", "off_flags", "off_avail", "act_words", "storage_bytes"]
    n = 0
    for obs, act, n_act in [(1, 1, 1), (4, 1, 2), (7, 3, 5), (17, 6, 9), (8, 1, 255), (33, 12, 16)]:
        kinds = [(L.PRL_BUF_CONTINUOUS, act, 0)] + [(L.PRL_BUF_DISCRETE | x, 1, n_act) for x in
                                                    (0, L.PRL_BUF_DYNAMIC_ACTIONS, L.PRL_BUF_NEXT_ACTION,
                                                     L.PRL_BUF_DYNAMIC_ACTIONS | L.PRL_BUF_NEXT_ACTION)]
        for flags, a, na in kinds:
            plain, rc0, _ = _layout(L, lib, flags, obs, a, na)
            with_cost, rc1, off = _layout(L, lib, flags | L.PRL_BUF_COST, obs, a, na)
            assert rc0 == L.PRL_EINVAL and rc1 == 0
            for f in fields[1:-1]:
                assert getattr(plain, f) == getattr(with_cost, f), (flags, f)
            dyn = (na + 3) // 4 if flags & L.PRL_BUF_DYNAMIC_ACTIONS else 0
            assert off == plain.off_avail + dyn
            assert with_cost.record_words == (off + 1 + 3) // 4 * 4 and with_cost.record_words >= plain.record_words
            assert with_cost.storage_bytes == 64 * with_cost.record_words * 4
            n += 1
    assert n == 30


def _rc_cfg(L, **kw):
    d = dict(obs_dim=17, act_dim=6, actor_h1=256, actor_h2=256, critic_h1=256, critic_h2=256, max_batch=256, critic_lr=1e-3,
             beta1=0.9, beta2=0.999, eps=1e-8, weight_decay=0.01, cost_gamma=0.5, tau=0.005)
    d.update(kw)
    return L.RcsafetyCfg(**d)


def test_rcsafety_param_count_and_workspace_host_arithmetic():
    import ctypes as C
    L, lib = _lib()
    up = lambda b: (b + 255) // 256 * 256  # noqa: E731
    for O, A, H1, H2, C1, C2, B in [(17, 6, 256, 256, 256, 256, 256), (7, 3, 32, 32, 32, 32, 40), (5, 1, 8, 24, 16, 12, 3)]:
        cfg = _rc_cfg(L, obs_dim=O, act_dim=A, actor_h1=H1, actor_h2=H2, critic_h1=C1, critic_h2=C2, max_batch=B)
        pc = C1 * (O + A) + C1 + C2 * C1 + C2 + C2 + 1
        assert lib.prl_rcsafety_param_count(C.byref(cfg)) == pc
        pa = H1 * O + H1 + H2 * H1 + H2 + A * H2 + A
        floats = [B * O, B * A, B, B * O, B, pa, B * H1, B * H2, B * A, B * A, 2 * B * C1, 2 * B * C2, 2 * B, 2 * B, 2 * B, 2 * B * C2,
                  2 * B * C1, B, 2 * pc]
        tail = 8 + (8 + 3 * 8 + 4 * 8 + 8) + 4    # AdamW scalars | call block (slots + step) | round counter
        want = sum(up(4 * f) for f in floats) + up(4 * B) + up(4 * B) + up(tail)
        assert lib.prl_rcsafety_workspace_bytes(C.byref(cfg)) == want
    assert lib.prl_rcsafety_param_count(C.byref(_rc_cfg(L, critic_h1=0))) == -1
    assert lib.prl_rcsafety_workspace_bytes(C.byref(_rc_cfg(L, max_batch=0))) == -1
    assert C.sizeof(L.RcsafetyStep) == 3 * 8 + 4 * 8 + 8


def _named(cls_name, base=torch.nn.Module):
    return type(cls_name, (base,), {})


def _twin(dims, name="TwinCritic", inner="VanillaQValueNetwork"):
    from oracle.pearl_oracle import _mlp
    t = _named(name)()
    for k in ("_critic_1", "_critic_2"):
        net = _mlp(dims)
        net.__class__ = type(inner, (torch.nn.Sequential,), {})
        setattr(t, k, net)
    return t


def _module(**over):
    m = types.SimpleNamespace(use_twin_critic=True, cost_critic=_twin([10, 32, 16, 1]), target_of_cost_critic=_twin([10, 32, 16, 1]),
                              state_dim=7, action_dim=3)
    for k, v in over.items():
        setattr(m, k, v)
    return m


def test_plugin_checks_and_refusals():
    import pearl_b200.rc_safety as rc
    if not rc.HAVE_REFERENCE_RC:
        assert rc.B200RCSafetyModuleCostCriticContinuousAction is rc.B200RCSafetyModule
    else:   # pragma: no cover - with Pearl installed
        from pearl.safety_modules.reward_constrained_safety_module import RCSafetyModuleCostCriticContinuousAction
        assert issubclass(rc.B200RCSafetyModuleCostCriticContinuousAction, RCSafetyModuleCostCriticContinuousAction)
    assert rc._check_reference_module(_module()) == [32, 16]
    refused = {
        "use_twin_critic=False": dict(use_twin_critic=False),
        "single critic": dict(cost_critic=_twin([10, 32, 16, 1], name="VanillaQValueNetwork")),
        "other critic network": dict(cost_critic=_twin([10, 32, 16, 1], inner="VanillaQValueMultiHeadNetwork")),
        "three hidden layers": dict(cost_critic=_twin([10, 32, 16, 8, 1])),
        "other dimensions": dict(state_dim=8),
    }
    for what, over in refused.items():
        with pytest.raises(NotImplementedError):
            rc._check_reference_module(_module(**over))
        print("refused:", what)
    rc._check_policy_learner(types.SimpleNamespace(_history_summarization_module=_named("IdentityHistorySummarizationModule")()))
    with pytest.raises(NotImplementedError):
        rc._check_policy_learner(types.SimpleNamespace(_history_summarization_module=_named("LSTMHistorySummarizationModule")()))
    for other in (object(), types.SimpleNamespace(_b200=object(), _ensure_core=lambda: None)):
        with pytest.raises(NotImplementedError):
            rc._td3_core(other)


def test_policy_plugins_refuse_or_forward_the_multiplier():
    """Plugins without cost shaping (SAC, discrete SAC, PPO, IQL, REINFORCE) refuse a safety module with a multiplier;
    TD3 / DDPG / TD3BC hand it to the CUDA learner on every learn()."""
    from pearl_b200.actor_critic import _B200ActorCriticMixin

    class Buf:
        def __len__(self):
            return 5

    class Core:
        lambda_constraint = "unset"

        def learn(self, buf):
            return {}

    def plugin(shaping, lam):
        cls = type("Plugin", (_B200ActorCriticMixin,), dict(_cost_shaping=shaping, _optimizer_triples=lambda self, core: [],
                                                             _core_steps=lambda self, core: ()))
        p = cls.__new__(cls)
        p._training_rounds, p._batch_size, p._training_steps = 1, 4, 0
        p.safety_module = types.SimpleNamespace(lambda_constraint=lam) if lam is not None else None
        p._core = Core()
        p._ensure_core = lambda: p._core
        return p
    with pytest.raises(NotImplementedError, match="reward-constrained"):
        plugin(False, 0.25).learn(Buf())
    p = plugin(False, None)
    p.learn(Buf())
    assert p._core.lambda_constraint == "unset"
    p = plugin(True, 0.25)
    p.learn(Buf())
    assert p._core.lambda_constraint == 0.25
    p = plugin(True, None)
    p.learn(Buf())
    assert p._core.lambda_constraint is None
