"""The Thompson sampler (prl_cb_ts_sample, ridge.cuh's k_cb_ts_sample) alone against float64, across its whole supported
width d = 1 .. 128 and conditioning from 1 to about 1e6, with a normwise bound.

Bound.  The kernel forms M = A + lambda I in fp32 (as the reference does) and everything after in fp64; the yardstick is
theta64 = coefs + U64^-T eps from the same fp32 M in float64 (oracle/ts_oracle.sample_theta).  Cholesky and the
triangular solve are backward stable: the computed x = U^-T eps is the exact solution for a perturbation of M of relative
size c d u64, so |x - x64| <= c d u64 cond(M) |x64| with a small c (4 is ample).  The result is then rounded once to fp32,
which adds at most u32 |theta64|.  So the test asserts
    |theta - theta64|_inf <= 2 u32 |theta64|_inf + 8 d u64 cond(M) |x64|_inf,
and prints the measured error against the bound for every shape."""
from __future__ import annotations

import os
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import ts_oracle  # noqa: E402

pytestmark = pytest.mark.gpu

U32, U64 = 2.0 ** -24, 2.0 ** -53
LAM = 0.5


def spd(d, cond, g):
    """A symmetric fp32 A such that A + LAM I has eigenvalues spread from 1 to cond (log-spaced)."""
    q, _ = torch.linalg.qr(torch.randn(d, d, generator=g, dtype=torch.float64))
    ev = torch.logspace(0, np.log10(cond), d, dtype=torch.float64) if d > 1 else torch.ones(1, dtype=torch.float64)
    M = (q * ev) @ q.t()
    M = (M + M.t()) / 2 - LAM * torch.eye(d, dtype=torch.float64)
    A = M.float()
    return (A + A.t()) / 2


@pytest.mark.parametrize("d", [1, 2, 17, 64, 127, 128])
@pytest.mark.parametrize("cond", [1.0, 1e2, 1e4, 1e6])
def test_sampler_against_float64(d, cond):
    import pearl_b200 as P
    if d == 1 and cond != 1.0:
        pytest.skip("a 1 x 1 matrix has condition number 1")
    lib = P._lib.init(0)
    g = torch.Generator().manual_seed(1000 * d + int(np.log10(cond)))
    A = spd(d, cond, g)
    coefs = torch.randn(d, generator=g)
    eps = torch.randn(d, generator=g)
    dev = [t.to("cuda:0") for t in (A, coefs, eps)]
    theta = torch.empty(d, device="cuda:0")
    status = torch.full((1,), 7, dtype=torch.int32, device="cuda:0")
    p = P._lib.ptr
    P._lib.check(lib.prl_cb_ts_sample(d, LAM, p(dev[0]), p(dev[1]), p(dev[2]), p(theta), p(status), None))
    assert int(status.item()) == 0
    t64 = ts_oracle.sample_theta(A, LAM, coefs, eps, torch.float64)
    M = ts_oracle.precision(A, LAM).double()
    kappa = float(torch.linalg.cond(M))
    x64 = t64 - coefs.double()
    err = float((theta.cpu().double() - t64).abs().max())
    bound = 2 * U32 * float(t64.abs().max()) + 8 * d * U64 * kappa * float(x64.abs().max())
    print(f"d={d:3d} cond={kappa:9.3g}: |theta - theta64| = {err:.3e}, bound {bound:.3e} ({err / bound:.2f} of it)")
    assert err <= bound


def test_sampler_flags_an_indefinite_matrix_and_recovers():
    import pearl_b200 as P
    lib = P._lib.init(0)
    p = P._lib.ptr
    d = 33
    theta = torch.full((d,), 5.0, device="cuda:0")
    status = torch.empty(1, dtype=torch.int32, device="cuda:0")
    coefs, eps = torch.zeros(d, device="cuda:0"), torch.ones(d, device="cuda:0")
    A = torch.eye(d, device="cuda:0")
    A[3, 3] = -2.0                                    # one negative eigenvalue of A + 0.5 I
    P._lib.check(lib.prl_cb_ts_sample(d, LAM, p(A), p(coefs), p(eps), p(theta), p(status), None))
    assert int(status.item()) == 1 and bool((theta == 5.0).all())
    A[3, 3] = float("nan")
    P._lib.check(lib.prl_cb_ts_sample(d, LAM, p(A), p(coefs), p(eps), p(theta), p(status), None))
    assert int(status.item()) == 1
    A[3, 3] = 1.0
    P._lib.check(lib.prl_cb_ts_sample(d, LAM, p(A), p(coefs), p(eps), p(theta), p(status), None))
    assert int(status.item()) == 0
    assert torch.allclose(theta, torch.full((d,), 1 / 1.5 ** 0.5, device="cuda:0"))
    assert lib.prl_cb_ts_sample(129, LAM, p(A), p(coefs), p(eps), p(theta), p(status), None) != 0
