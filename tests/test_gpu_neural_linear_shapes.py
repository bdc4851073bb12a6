"""B200NeuralLinearBandit (csrc/neural_linear.cu) across its shape space against the float64 step of
oracle/neural_linear_fp64.py: one learn_batch round per case under contraction engines 0 (SIMT tiles), 1 (the library
default: wgmma from 4096 output rows on) and 2 (wgmma always).  Every gradient block is read back from exp_avg / (1 -
beta1) (the first AdamW step from zero state stores (1 - beta1) g) and held within C x scale elementwise, scale = the
sum of |a||b| over every product that reached the value (neural_linear_fp64.step(absolute=True)); the loss is held to
1e-4.  The ridge statistics A and b are held against the fp64 network output within C x their scale, and
inv_A and coefs against bandit_oracle.fp64_yardstick of the GPU's own fp32 A + lambda I within 4 d (2^-24 + cond 2^-53)
normwise, as test_gpu_bandit_shapes.py does.

The grid reaches: input widths 1 to 257 (odd ones, so unaligned rows on the wgmma operands), h1 1 to 640, h2 1 to 127
(h2 = 1: mlp2_backward's k_head_bwd branch; with skip connections the residual chain instead), batches 1 to 65536 (the
single-CTA k_nl_loss and the k_nl_grad grid at their largest), all three losses, both e2e settings (e2e: the M = 1
weight-gradient contraction) and both skip settings, with every residual combination (first layer f == h1, middle
h1 == h2, last always).

Data: inputs, labels and weights on a 1/256 grid; a row is kept only if every pre-activation of both hidden layers
clears MARGIN of its scale (a ReLU must not flip between fp32 and fp64) and, for MAE, |p - y| clears it too.  The fp64
step runs on the GPU.

Bound: |kernel - fp64| <= max(C, 4 u sqrt(B)) x scale, u = 2^-24.  Every block of this learner is a sum over the B batch
rows (the per-row head gradient reaches every weight), and the fp32 accumulators of the SIMT and wgmma tiles make a
random-walk error that grows with that length.  Measured on an H100 80GB HBM3 (700 W power limit), largest err / scale:
5.2e-6 (dW3 at f 16, [16, 16], B 4097, all residual, engine 2, 3xTF32), 1.0e-6 at B 5000 on engine 2, 4.6e-9 at B 128 on
engine 0; C = 1e-5 and 4 u sqrt(4097) = 1.5e-5 leave about three times that.  A wrong index, mask or missing term is off
by O(1) of the scale.
"""
from __future__ import annotations

import os
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import bandit_oracle as bo  # noqa: E402
from oracle import neural_linear_fp64 as f64  # noqa: E402

pytestmark = pytest.mark.gpu

DEV = "cuda:0"
C = 1e-5
MARGIN = 4e-6         # ReLU / l1 margin of the accepted rows, relative to the value's scale (well above the error)
U = 2.0 ** -24
ENGINES = (0, 1, 2)
BETA1 = np.float32(1.0 - 0.9)      # k_adamw's (float)(1 - beta1)

# (f, h1, h2, B, loss, e2e, skip)
CASES = [
    (1, 1, 1, 1, "mse", True, False),          # smallest; h2 = 1 (k_head_bwd)
    (21, 64, 16, 128, "mse", True, False),     # the CB benchmark network
    (257, 640, 127, 65536, "cross_entropy", False, False),   # every maximum
    (16, 16, 16, 4097, "mae", True, True),     # all three residual layers, ragged row tile
    (33, 127, 127, 300, "mse", False, True),   # middle and last residual
    (127, 256, 127, 256, "cross_entropy", True, True),       # the wide shape
    (5, 3, 1, 7, "mae", False, True),          # h2 = 1 with a residual last layer
    (64, 64, 9, 5000, "mae", True, True),      # first and last residual, engine 1 on wgmma
]


def data(f, h1, h2, B, loss, e2e, skip, seed):
    g = torch.Generator().manual_seed(seed)
    grid = lambda t: torch.round(t * 256) / 256  # noqa: E731
    sh = [(h1, f), (h1,), (h2, h1), (h2,), (h2, h2), (h2,), (1, h2)]
    fan = [f, f, h1, h1, h2, h2, h2]
    p32 = [grid((torch.rand(s, generator=g) * 2 - 1) / fan[i] ** 0.5) for i, s in enumerate(sh)]
    coefs = grid(torch.randn(h2 + 1, generator=g) * 0.5)
    n = 2 * B + 64
    X = grid(torch.randn(n, f, generator=g))
    y = grid(torch.rand(n, generator=g)) if loss == "cross_entropy" else grid(torch.randn(n, generator=g))
    w = grid(torch.rand(n, generator=g) * 1.75 + 0.25)
    p = [t.double().to(DEV) for t in p32]
    Xd, yd, wd, cd = X.double().to(DEV), y.double().to(DEV), w.double().to(DEV), coefs.double().to(DEV)
    s, a = f64.forward(p, Xd, skip), f64.forward(p, Xd, skip, True, [torch.ones(1, device=DEV)] * 2)
    ok = ((s["Z1"].abs() > MARGIN * a["Z1"]).all(1) & (s["Z2"].abs() > MARGIN * a["Z2"]).all(1))
    if loss == "mae":
        _, pr, _, _ = f64.head(s["N"], p[6], cd, yd, e2e, loss, False)
        ok &= (pr - yd).abs() > MARGIN * (1 + yd.abs())
    keep = torch.nonzero(ok).reshape(-1)[:B].cpu()
    assert keep.numel() == B, "too few rows clear the margin"
    return p32, coefs, X[keep], y[keep], w[keep]


def run(case, engine, seed=0):
    import pearl_b200 as P
    from pearl_b200 import _lib
    f, h1, h2, B, loss, e2e, skip = case
    p32, coefs, X, y, w = data(*case, seed)
    lib = _lib.load()
    old = lib.prl_get_contraction_engine()
    _lib.check(lib.prl_set_contraction_engine(engine))
    try:
        nl = P.B200NeuralLinearBandit(feature_dim=f, hidden_dims=[h1, h2], batch_size=B, learning_rate=1e-3, loss_type=loss,
                                      output_activation_name="sigmoid" if loss == "cross_entropy" else "linear",
                                      use_skip_connections=skip, nn_e2e=e2e).to(DEV)
        with torch.no_grad():
            for q, t in zip(nl.model.parameters(), p32):
                q.copy_(t)
            nl.model._linear_regression_layer._coefs.copy_(coefs)
        rep = nl.learn_batch(P.TransitionBatch(state=X.to(DEV), action=torch.zeros(B, 0, device=DEV), reward=y.to(DEV),
                                               weight=w.to(DEV)))
        torch.cuda.synchronize()
    finally:
        _lib.check(lib.prl_set_contraction_engine(old))
    return nl, rep, (p32, coefs, X, y, w)


@pytest.mark.parametrize("engine", ENGINES)
@pytest.mark.parametrize("case", CASES, ids=lambda c: "f{}_h{}x{}_B{}_{}_{}_{}".format(
    c[0], c[1], c[2], c[3], c[4], "e2e" if c[5] else "ridge", "skip" if c[6] else "plain"))
def test_one_round_against_fp64(case, engine):
    f, h1, h2, B, loss, e2e, skip = case
    nl, rep, (p32, coefs, X, y, w) = run(case, engine)
    p = [t.double().to(DEV) for t in p32]
    args = (p, X.double().to(DEV), y.double().to(DEV), w.double().to(DEV), coefs.double().to(DEV))
    kw = dict(e2e=e2e, loss=loss, sigmoid=loss == "cross_entropy", skip=skip)
    want, scale = f64.step(*args, **kw), f64.step(*args, **kw, absolute=True)
    st = nl.optimizer.state
    params = list(nl.model.parameters())
    worst = {}
    for k, q in zip(f64.BLOCKS, params):
        if k == "dwe" and not e2e:
            assert q not in st
            continue
        got = st[q]["exp_avg"].double().reshape(-1) / float(BETA1)
        err = (got - want[k].reshape(-1)).abs()
        bound = max(C, 4 * U * B ** 0.5) * scale[k].reshape(-1) + 1e-30
        worst[k] = float((err / bound).max())
        assert bool((err <= bound).all()), f"{k}: {int((err > bound).sum())} elements beyond C x scale (worst {worst[k]:.3g})"
    print("   ", case, "engine", engine, {k: f"{v:.2e}" for k, v in worst.items()})
    np.testing.assert_allclose(float(rep["loss"]), float(want["loss"]), rtol=1e-4, atol=1e-6)
    # the ridge on the network's output
    N = want["N"]
    x1 = bo.ones_col(N)
    a1 = bo.ones_col(scale["N"])
    wd = args[3]
    A64, As = x1.t() @ (x1 * wd[:, None]), a1.t() @ (a1 * wd[:, None])
    b64, bs = x1.t() @ (args[2] * wd), a1.t() @ (args[2].abs() * wd)
    lin = nl.model._linear_regression_layer
    cb = max(C, 4 * U * B ** 0.5)
    assert bool(((lin._A.double() - A64).abs() <= cb * As).all()), "A"
    assert bool(((lin._b.double() - b64).abs() <= cb * bs).all()), "b"
    inv64, coefs64, cond = bo.fp64_yardstick(lin._A.cpu(), lin._b.cpu(), 1.0)
    bound = 4 * (h2 + 1) * (2.0 ** -24 + cond * 2.0 ** -53)
    assert float((lin._inv_A.cpu().double() - inv64).abs().max()) <= bound * float(inv64.abs().max())
    assert float((lin._coefs.cpu().double() - coefs64).abs().max()) <= bound * float(coefs64.abs().max())
