"""One round of B200DisjointBanditContainer / B200DisjointLinearBandit against float64, arm by arm, across the supported
shape class: K 1..1024 arms, d 2..128, batches 1..65536 (many 256-row chunks, arms spanning several statistic chunks),
skewed routings (every row to one arm, most arms empty, one row per arm), 3-D state, DisjointLinearBandit's dropped
rows.  A, b and sum_weight elementwise against float64 sums with test_gpu_bandit_shapes.py's bound; inv_A and coefs
within its yardstick bound 4 d (2^-24 + cond 2^-53) normwise, for every arm; the per-arm Thompson sampler within
test_gpu_ts_sample_shapes.py's bound 2 u32 |theta64| + 8 d u64 cond |x64|."""
from __future__ import annotations

import os
import sys

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import bandit_oracle as bo  # noqa: E402
from oracle import ts_oracle  # noqa: E402

pytestmark = pytest.mark.gpu

DEV = "cuda:0"
U32, U64 = 2.0 ** -24, 2.0 ** -53


class Space:
    def __init__(self, n):
        self.n = n
        self.actions = [torch.tensor([i]) for i in range(n)]


def routing(kind, B, K, g):
    if kind == "random":
        return torch.randint(0, K, (B,), generator=g)
    if kind == "one_arm":
        return torch.full((B,), K // 2, dtype=torch.long)
    if kind == "few_arms":                     # most arms empty
        return torch.randint(0, min(K, 3), (B,), generator=g) * max(K // 3, 1)
    if kind == "one_per_arm":
        return torch.randperm(K, generator=g)[:B]
    raise ValueError(kind)


def check_arm(m, x, y, w, lam, what):
    """m's buffers after one round from zero on rows x (state [|| action]), against float64."""
    d = x.shape[1] + 1
    x1 = bo.ones_col(x.double())
    wd, yd = w.double(), y.double()
    A64, b64 = x1.t() @ (x1 * wd[:, None]), x1.t() @ (yd * wd)
    sA = x1.abs().t() @ (x1.abs() * wd[:, None])
    assert ((m._A.cpu().double() - A64).abs() <= 1e-4 * sA + 1e-6).all(), f"{what}: A"
    assert ((m._b.cpu().double() - b64).abs() <= 1e-4 * (x1.abs().t() @ (yd.abs() * wd)) + 1e-6).all(), f"{what}: b"
    assert abs(float(m._sum_weight) - float(wd.sum())) <= 1e-4 * float(wd.sum()) + 1e-6, f"{what}: sum_weight"
    inv64, coefs64, cond = bo.fp64_yardstick(m._A.cpu(), m._b.cpu(), lam)
    bound = 4 * d * (U32 + cond * U64)
    e_inv = float((m._inv_A.cpu().double() - inv64).norm()) / float(inv64.norm())
    e_c = float((m._coefs.cpu().double() - coefs64).norm()) / max(float(coefs64.norm()), 1e-30)
    assert e_inv <= bound and e_c <= bound, f"{what}: cond {cond:.3g}, inv {e_inv:.3g}, coefs {e_c:.3g}, bound {bound:.3g}"


CASES = [  # K, feature width (d - 1), batch, routing
    (1, 1, 1, "random"), (1, 127, 65536, "random"), (7, 16, 1000, "random"), (26, 16, 4096, "random"),
    (300, 31, 20000, "few_arms"), (128, 127, 4096, "random"), (1024, 7, 65536, "random"), (1024, 127, 1024, "one_per_arm"),
    (64, 127, 65536, "one_arm"), (513, 40, 3000, "random"),
]


@pytest.mark.parametrize("K,f,B,kind", CASES)
def test_container_round_against_float64(K, f, B, kind):
    import pearl_b200 as P
    from pearl_b200._compat import _RefLinearBandit
    torch.cuda.set_device(0)
    g = torch.Generator().manual_seed(K * 131 + f * 7 + B)
    lams = (0.5 + torch.rand(K, generator=g)).tolist()
    arms = [_RefLinearBandit(feature_dim=f, l2_reg_lambda=lams[k]) for k in range(K)]
    dc = P.B200DisjointBanditContainer(feature_dim=f, arm_bandits=arms, exploration_module=P.DisjointUCBExploration(1.0),
                                       batch_size=B)
    arm = routing(kind, B, K, g)
    three_d = K <= 26 and B <= 4096                          # arm k reads state[:, k]
    state = torch.randn(B, K, f, generator=g) if three_d else torch.randn(B, f, generator=g)
    y, w = torch.randn(B, generator=g), torch.rand(B, generator=g) * 2
    rep = dc.learn_batch(P.TransitionBatch(state=state.to(DEV), action=arm.reshape(B, 1).to(DEV), reward=y.to(DEV),
                                           weight=w.to(DEV)))
    for k in range(K):
        sel = arm == k
        if int(sel.sum()) == 0:
            # the null batch: zeros added, the solve still runs on lambda I
            assert float(dc.models[k]._A.abs().max()) == 0.0 and rep[f"arm_{k}_weight"].shape == (1, 1)
            assert torch.allclose(dc.models[k]._inv_A.cpu(), torch.eye(f + 1) / lams[k])
            continue
        x = (state[:, k, :] if three_d else state)[sel]
        check_arm(dc.models[k], x, y[sel], w[sel], lams[k], f"K={K} f={f} B={B} {kind} arm {k}")
        assert rep[f"arm_{k}_prediction"].shape == (int(sel.sum()), 1)
        assert torch.equal(rep[f"arm_{k}_label"].cpu().reshape(-1), y[sel])   # partition order = batch order per arm


@pytest.mark.parametrize("K,B,sfo", [(3, 65536, False), (1024, 65536, True), (200, 777, False)])
def test_disjoint_linear_round_against_float64(K, B, sfo):
    import pearl_b200 as P
    torch.cuda.set_device(0)
    g = torch.Generator().manual_seed(K + B)
    obs = 20
    f = obs if sfo else obs + 1
    lb = P.B200DisjointLinearBandit(feature_dim=f, action_space=Space(K), exploration_module=P.DisjointUCBExploration(1.0),
                                    l2_reg_lambda=0.7, state_features_only=sfo, batch_size=B)
    a = torch.randint(-2, K + 3, (B,), generator=g)            # some rows match no arm and are dropped
    state, y = torch.randn(B, obs, generator=g), torch.randn(B, generator=g)
    lb.learn_batch(P.TransitionBatch(state=state.to(DEV), action=a.reshape(B, 1).to(DEV), reward=y.to(DEV)))
    for k in range(K):
        sel = a == k
        m = lb._linear_regressions[k]
        if int(sel.sum()) == 0:
            assert float(m._inv_A.abs().max()) == 0.0          # skipped: never solved
            continue
        x = state[sel] if sfo else torch.cat([state[sel], torch.full((int(sel.sum()), 1), float(k))], 1)
        check_arm(m, x, y[sel], torch.ones(int(sel.sum())), 0.7, f"K={K} B={B} arm {k}")


@pytest.mark.parametrize("K,f", [(1, 1), (16, 33), (128, 127), (1024, 15)])
def test_per_arm_sampler_against_float64(K, f):
    import pearl_b200 as P
    from pearl_b200._compat import _RefLinearBandit
    torch.cuda.set_device(0)
    g = torch.Generator().manual_seed(K * 17 + f)
    d = f + 1
    lams = (0.5 + torch.rand(K, generator=g)).tolist()
    arms = [_RefLinearBandit(feature_dim=f, l2_reg_lambda=lams[k]) for k in range(K)]
    dc = P.B200DisjointBanditContainer(feature_dim=f, arm_bandits=arms, exploration_module=P.DisjointUCBExploration(1.0),
                                       batch_size=8 * K)
    B = 8 * K + 4 * d
    x = torch.randn(B, f, generator=g) * torch.logspace(0, 1.5, f)      # spread the spectrum: cond up to ~1e3..1e4
    arm = torch.arange(B) % K
    dc.learn_batch(P.TransitionBatch(state=x.to(DEV), action=arm.reshape(B, 1).to(DEV), reward=torch.randn(B, generator=g).to(DEV)))
    rg = dc._dj
    eps = torch.randn(K, d, generator=g)
    theta = torch.empty(K, d, device=DEV)
    status = torch.full((K,), 7, dtype=torch.int32, device=DEV)
    p = P._lib.ptr
    e = eps.to(DEV)
    P._lib.check(rg.lib.prl_dcb_ts_sample(rg.handle, p(e), p(theta), p(status), None))
    assert int(status.abs().max()) == 0
    for k in range(K):
        m = dc.models[k]
        A, c = m._A.cpu(), m._coefs.cpu()
        t64 = ts_oracle.sample_theta(A, lams[k], c, eps[k], torch.float64)
        kappa = float(torch.linalg.cond(ts_oracle.precision(A, lams[k]).double()))
        x64 = t64 - c.double()
        err = float((theta[k].cpu().double() - t64).abs().max())
        bound = 2 * U32 * float(t64.abs().max()) + 8 * d * U64 * kappa * float(x64.abs().max())
        assert err <= bound, f"K={K} d={d} arm {k}: cond {kappa:.3g}, err {err:.3g}, bound {bound:.3g}"
