"""B200NeuralBandit (csrc/neural_bandit.cu) across its shape space against the float64 step of oracle/neural_bandit_fp64.py:
one learn_batch round per case under contraction engines 0 (SIMT tiles), 1 (the library default: wgmma from 4096 output
rows on) and 2 (wgmma always).  Every gradient block is read back from exp_avg / (1 - beta1) (the first AdamW step from
zero state stores (1 - beta1) g) and held within the bound below elementwise, scale = the sum of |a||b| over every product
that reached the value (neural_bandit_fp64.step(absolute=True)); the loss is held to 1e-4.

The grid reaches: input widths 1 to 257 (odd ones, so unaligned rows on the wgmma operands), split into state and action
columns or state alone, h1 and h2 from 1 to 640, batches 1 to 65536 (the single-CTA head at its largest), both losses,
and weights of both signs.

Data: inputs, labels and weights on a 1/256 grid; a row is kept only if every pre-activation of both hidden layers clears
MARGIN of its scale (a ReLU must not flip between fp32 and fp64) and, for MAE, |p - y| clears it too.  The fp64 step runs
on the GPU.

Bound: |kernel - fp64| <= max(C, 4 u sqrt(B)) x scale, u = 2^-24: every block is a sum over the B batch rows, and the
fp32 accumulators make a random-walk error that grows with that length.  Measured on an H100 80GB HBM3 (700 W power
limit), the largest err / bound over the grid is 0.12 (db3 at f 15, [33, 1], B 4097, engine 2, 3xTF32); engines 0 and 1
stay below 5e-3.  C = 1e-5 thus leaves about eight times the worst case.  A wrong index, mask or missing term is off by
O(1) of the scale.
"""
from __future__ import annotations

import os
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import neural_bandit_fp64 as f64  # noqa: E402
from oracle import neural_linear_fp64 as nl64  # noqa: E402

pytestmark = pytest.mark.gpu

DEV = "cuda:0"
C = 1e-5
MARGIN = 4e-6
U = 2.0 ** -24
ENGINES = (0, 1, 2)
BETA1 = np.float32(1.0 - 0.9)      # k_adamw's (float)(1 - beta1)

# (obs, act_dim, h1, h2, B, loss)
CASES = [
    (1, 0, 1, 1, 1, "mse"),             # smallest
    (16, 5, 64, 16, 128, "mse"),        # the CB benchmark network, binary action code
    (200, 57, 640, 300, 65536, "mae"),  # every maximum
    (9, 6, 33, 1, 4097, "mae"),         # h2 = 1, ragged row tile
    (127, 0, 255, 129, 300, "mse"),     # odd widths, state only
    (3, 2, 500, 7, 5000, "mse"),        # wide h1, engine 1 on wgmma
    (1, 256, 17, 640, 77, "mae"),       # action columns only past one state column
]


def data(obs, act_dim, h1, h2, B, loss, seed):
    f = obs + act_dim
    g = torch.Generator().manual_seed(seed)
    grid = lambda t: torch.round(t * 256) / 256  # noqa: E731
    sh = [(h1, f), (h1,), (h2, h1), (h2,), (1, h2), (1,)]
    fan = [f, f, h1, h1, h2, h2]
    p32 = [grid((torch.rand(s, generator=g) * 2 - 1) / fan[i] ** 0.5) for i, s in enumerate(sh)]
    n = 2 * B + 64
    X = grid(torch.randn(n, f, generator=g))
    y = grid(torch.randn(n, generator=g))
    w = grid((torch.rand(n, generator=g) * 1.75 + 0.25) * torch.where(torch.rand(n, generator=g) < 0.2, -1.0, 1.0))
    p = [t.double().to(DEV) for t in p32]
    Xd, yd = X.double().to(DEV), y.double().to(DEV)
    s, a = nl64.forward(p, Xd, False), nl64.forward(p, Xd, False, True, [torch.ones(1, device=DEV)] * 2)
    ok = ((s["Z1"].abs() > MARGIN * a["Z1"]).all(1) & (s["Z2"].abs() > MARGIN * a["Z2"]).all(1))
    if loss == "mae":
        ok &= (s["N"].reshape(-1) - yd).abs() > MARGIN * (a["N"].reshape(-1) + yd.abs() + 1)
    keep = torch.nonzero(ok).reshape(-1)[:B].cpu()
    assert keep.numel() == B, "too few rows clear the margin"
    w = w[keep]
    if float(w.sum()) < 0.25 * float(w.abs().sum()):
        w = w.abs()           # keep sum(w) away from 0
    return p32, X[keep], y[keep], w


def run(case, engine, seed=0):
    import pearl_b200 as P
    from pearl_b200 import _lib
    obs, act_dim, h1, h2, B, loss = case
    p32, X, y, w = data(*case, seed)
    lib = _lib.load()
    old = lib.prl_get_contraction_engine()
    _lib.check(lib.prl_set_contraction_engine(engine))
    try:
        nb = P.B200NeuralBandit(feature_dim=obs + act_dim, hidden_dims=[h1, h2], exploration_module=P.NoExploration(),
                                batch_size=B, learning_rate=1e-3, loss_type=loss, state_features_only=act_dim == 0).to(DEV)
        with torch.no_grad():
            for q, t in zip(nb.model.parameters(), p32):
                q.copy_(t)
        rep = nb.learn_batch(P.TransitionBatch(state=X[:, :obs].to(DEV), action=X[:, obs:].to(DEV), reward=y.to(DEV),
                                               weight=w.to(DEV)))
        torch.cuda.synchronize()
    finally:
        _lib.check(lib.prl_set_contraction_engine(old))
    return nb, rep, (p32, X, y, w)


@pytest.mark.parametrize("engine", ENGINES)
@pytest.mark.parametrize("case", CASES, ids=lambda c: "s{}_a{}_h{}x{}_B{}_{}".format(*c))
def test_one_round_against_fp64(case, engine):
    obs, act_dim, h1, h2, B, loss = case
    nb, rep, (p32, X, y, w) = run(case, engine)
    p = [t.double().to(DEV) for t in p32]
    args = (p, X.double().to(DEV), y.double().to(DEV), w.double().to(DEV))
    want, scale = f64.step(*args, loss=loss), f64.step(*args, loss=loss, absolute=True)
    st = nb.optimizer.state
    worst = {}
    for k, q in zip(f64.BLOCKS, nb.model.parameters()):
        got = st[q]["exp_avg"].double().reshape(-1) / float(BETA1)
        err = (got - want[k].reshape(-1)).abs()
        bound = max(C, 4 * U * B ** 0.5) * scale[k].reshape(-1) + 1e-30
        worst[k] = float((err / bound).max())
        assert bool((err <= bound).all()), f"{k}: {int((err > bound).sum())} elements beyond the bound (worst {worst[k]:.3g})"
    print("   ", case, "engine", engine, {k: f"{v:.2e}" for k, v in worst.items()})
    np.testing.assert_allclose(float(rep["loss"]), float(want["loss"]), rtol=1e-4, atol=1e-6)
    pr = rep["prediction"].double().reshape(-1)
    assert bool(((pr - want["pred"]).abs() <= max(C, 4 * U) * (scale["pred"] + 1e-30)).all()), "prediction"
