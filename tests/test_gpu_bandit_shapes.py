"""The CUDA ridge solve (csrc/bandit.cu, k_cb_solve) across its supported widths d = 2..128 and batches 1..65536, against
the float64 inverse of the GPU's own fp32 A + lambda I (oracle/bandit_oracle.py fp64_yardstick).

Bound: the yardstick inverts the same fp32 matrix the kernel starts from, so the only differences are the kernel's own
arithmetic and its output rounding.  Gauss-Jordan elimination with partial pivoting in fp64 on d columns is accurate to
about d cond 2^-53 normwise, and rounding the result to fp32 adds 2^-24 per element.  So inv_A and coefs are held to
4 d (2^-24 + cond 2^-53) of the largest magnitude of the fp64 result.  A solve carried out in fp32 would be off by about
cond 2^-24, which this bound rejects once cond exceeds a few hundred (the 1.4M-row run reaches cond > 1e4).  A, b and sum_weight are sums
and are held elementwise to 1e-4 of the fp64 sums of the same rows (with an absolute floor for cancelling entries)."""
from __future__ import annotations

import os
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import bandit_oracle as bo  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def check_solve(lb, lam):
    inv64, coefs64, cond = bo.fp64_yardstick(lb.model._A.cpu(), lb.model._b.cpu(), lam)
    d = inv64.shape[0]
    bound = 4 * d * (2.0 ** -24 + cond * 2.0 ** -53)
    e_inv = (lb.model._inv_A.cpu().double() - inv64).abs().max().item() / inv64.abs().max().item()
    e_c = (lb.model._coefs.cpu().double() - coefs64).abs().max().item() / max(coefs64.abs().max().item(), 1e-30)
    assert e_inv <= bound and e_c <= bound, f"d={d} cond={cond:.3g}: inv err {e_inv:.3g}, coefs err {e_c:.3g}, bound {bound:.3g}"
    return cond


@pytest.mark.parametrize("k,B", [(1, 1), (1, 65536), (7, 300), (16, 128), (26, 4096), (63, 1000), (100, 257), (127, 65536),
                                 (127, 1)])
def test_ridge_solve_against_fp64(k, B):
    import pearl_b200 as P
    torch.cuda.set_device(0)
    g = torch.Generator(device=DEV).manual_seed(k * 7919 + B)
    lam = 0.5
    lb = P.B200LinearBandit(feature_dim=k, l2_reg_lambda=lam, batch_size=B).to(DEV)
    x = torch.randn(B, k, device=DEV, generator=g)
    y = torch.randn(B, device=DEV, generator=g)
    w = torch.rand(B, device=DEV, generator=g) * 2
    lb.learn_batch(P.TransitionBatch(state=x[:, : k // 2], action=x[:, k // 2:], reward=y, weight=w))
    x1 = bo.ones_col(x.double())
    A64 = x1.t() @ (x1 * w.double()[:, None])
    b64 = x1.t() @ (y.double() * w.double())
    scale = (x1.abs().t() @ (x1.abs() * w.double()[:, None]))
    assert ((lb.model._A.double() - A64).abs() <= 1e-4 * scale + 1e-6).all()
    assert ((lb.model._b.double() - b64).abs() <= 1e-4 * (x1.abs().t() @ (y.double().abs() * w.double())) + 1e-6).all()
    assert abs(lb.model._sum_weight.item() - w.double().sum().item()) <= 1e-4 * w.double().sum().item()
    check_solve(lb, lam)


def test_a_million_rows_one_hot_with_intercept():
    """The CB benchmark's regime: obs 16 with one-hot codes of 10 actions (the intercept column is the sum of the code
    columns, so cond grows with the rows absorbed), 1.3M rows in learn() rounds of 128 rows."""
    import pearl_b200 as P
    torch.cuda.set_device(0)
    g = torch.Generator().manual_seed(11)
    n, A = 20000, 10
    s = torch.randn(n, 16, generator=g)
    a = torch.randint(0, A, (n,), generator=g)
    r = s[:, 0] + 0.1 * a + 0.1 * torch.randn(n, generator=g)
    buf = P.B200ReplayBuffer(n, rng="device")
    buf.push_batch(s, a, r, None, torch.ones(n, dtype=torch.bool), torch.zeros(n, dtype=torch.bool), max_number_actions=A)
    buf.seed(1)
    lb = P.B200LinearBandit(feature_dim=16 + A, exploration_module=P.UCBExploration(1.0), training_rounds=1000, batch_size=128,
                            action_representation_module=P.OneHotActionTensorRepresentationModule(A))
    for _ in range(11):
        lb.learn(buf)
    assert lb.model._sum_weight.item() == 11 * 1000 * 128
    cond = check_solve(lb, 1.0)
    assert cond > 1e4, "the run is meant to reach the ill-conditioned regime"


def test_learners_of_different_widths_share_the_process():
    """The solve kernel's shared-memory limit belongs to the kernel: creating a narrow learner after a wide one must not
    lower it under the wide one's launches."""
    import pearl_b200 as P
    torch.cuda.set_device(0)
    g = torch.Generator().manual_seed(3)
    wide = P.B200LinearBandit(feature_dim=127, batch_size=64).to(DEV)
    narrow = P.B200LinearBandit(feature_dim=21, batch_size=64).to(DEV)

    def step(lb, k):
        x = torch.randn(64, k, generator=g).to(DEV)
        lb.learn_batch(P.TransitionBatch(state=x[:, :k - 1], action=x[:, k - 1:], reward=torch.randn(64, generator=g).to(DEV)))

    step(wide, 127)
    step(narrow, 21)
    for lb, k in ((wide, 127), (narrow, 21), (wide, 127)):
        lb.use_cuda_graph = False
        step(lb, k)
        lb.use_cuda_graph = True
        step(lb, k)
    torch.cuda.synchronize()
    check_solve(wide, 1.0)
    check_solve(narrow, 1.0)
