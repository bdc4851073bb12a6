"""The CNN DQN learner (csrc/cnnq.cu) across its shape space against float64 gradients (oracle/cnn_q_fp64.py).

One learn_batch step from zero AdamW moments leaves exp_avg = fl(fl(1 - beta1) g), so the kernel's fp32 gradient g is
recovered from the first moment, and held elementwise to the float64 gradient of the same batch:

    |g_kernel - g_fp64| <= (C + R * U / 32) * scale,    U = 2^-24

where scale is the sum of |a||b| over every product that contributed (cnn_q_fp64.step) and R the longest contraction of
the step (B OH OW rows for the first conv layer's weight gradient).  Data whose ReLU pre-activations lie within MARGIN of
their scale are redrawn, since a last-bit difference could flip a mask.  The largest err / scale of each case is printed.

The grid covers 1x1 kernels and kernels wider than their stride, paddings 0-2, a 1x1 final feature map, 1 and 4 input
channels, 0 / 1 / 2 hidden FC layers, A from 1 to 255, batch 1 to 1024, DQN and DoubleDQN, both networks, under the SIMT
(0) and tensor-core (2) contraction engines.
"""
import numpy as np
import pytest
import torch

from oracle import cnn_q_fp64, cnn_q_oracle as orc

pytestmark = pytest.mark.gpu

C = 2e-6
U = 2.0 ** -24
MARGIN = 3e-7
OMB1 = float(np.float32(1.0 - 0.9))

# (input, conv layers (out, k, stride, pad), hidden, A, B, multi, double)
GRID = [
    ((1, 8, 8), [(4, 1, 1, 0)], [], 1, 1, False, False),
    ((4, 12, 12), [(8, 5, 2, 2), (8, 3, 1, 1)], [16], 3, 16, True, True),
    ((1, 9, 9), [(6, 3, 3, 0), (5, 3, 1, 0)], [32, 8], 255, 8, True, False),
    ((4, 20, 20), [(8, 4, 2, 1), (16, 3, 1, 0), (16, 8, 1, 0)], [7], 6, 32, False, True),
    ((2, 16, 16), [(4, 6, 2, 2), (8, 1, 1, 0)], [16, 16], 255, 4, False, False),
    ((4, 36, 36), [(16, 8, 4, 0), (32, 4, 2, 0), (32, 3, 1, 0)], [64], 6, 64, False, True),
    ((4, 36, 36), [(16, 8, 4, 0), (32, 4, 2, 0), (32, 3, 1, 0)], [64], 6, 64, True, False),
    ((1, 12, 12), [(4, 3, 2, 1)], [8], 4, 1024, True, True),
]
IDS = [f"in{'x'.join(map(str, g[0]))}-L{len(g[1])}-fc{len(g[2])}-A{g[3]}-B{g[4]}-{'mh' if g[5] else 'v'}-{'ddqn' if g[6] else 'dqn'}"
       for g in GRID]


def _data(spec, B, seed):
    rng = np.random.Generator(np.random.PCG64(seed))
    A = spec["n_actions"]
    ids, cnt = np.zeros((B, A), np.int64), np.zeros(B, np.int64)
    for i in range(B):
        m = int(rng.integers(1, A + 1))
        ids[i, :m] = np.sort(rng.choice(A, size=m, replace=False))
        cnt[i] = m
    shape = (B,) + tuple(spec["input"])
    return dict(state=torch.from_numpy(rng.integers(0, 256, shape).astype(np.float32)),
                next_state=torch.from_numpy(rng.integers(0, 256, shape).astype(np.float32)),
                action=torch.from_numpy(rng.integers(0, A, B)), reward=torch.from_numpy(rng.standard_normal(B).astype(np.float32)),
                terminated=torch.from_numpy(rng.random(B) < 0.2), next_ids=torch.from_numpy(ids), next_count=torch.from_numpy(cnt))


@pytest.mark.parametrize("engine", [0, 2])
@pytest.mark.parametrize("inp,conv,hidden,A,B,multi,double", GRID, ids=IDS)
def test_cnn_q_gradient_against_fp64(inp, conv, hidden, A, B, multi, double, engine):
    import pearl_b200
    from pearl_b200 import _lib
    from test_cnn_q import _learner
    spec = dict(input=inp, conv=conv, hidden=hidden, n_actions=A, multi=multi)
    torch.manual_seed(B + A)
    pl = _learner(spec, double, learning_rate=1e-3, training_rounds=1, batch_size=B, target_update_freq=1000)
    w = pl.flat_parameters.cpu().clone()
    wt = w + 0.01 * torch.randn(w.shape, generator=torch.Generator().manual_seed(1)) * w.abs().mean()
    pl.flat_target_parameters.copy_(wt.cuda())
    for seed in range(20):
        d = _data(spec, B, seed)
        g64, scale, margin = cnn_q_fp64.step(spec, w, wt, d, double=double, gamma=0.99)
        if margin > MARGIN:
            break
    else:
        pytest.fail("no data with ReLU margins above MARGIN")
    lib = _lib.init(0)
    prev = lib.prl_get_contraction_engine()
    _lib.check(lib.prl_set_contraction_engine(engine))
    try:
        batch = pearl_b200.TransitionBatch(state=d["state"], action=d["action"], reward=d["reward"], terminated=d["terminated"],
                                           next_state=d["next_state"],
                                           next_available_actions=d["next_ids"],
                                           next_unavailable_actions_mask=torch.arange(A).unsqueeze(0) >= d["next_count"].unsqueeze(1))
        pl.learn_batch(batch)
    finally:
        lib.prl_set_contraction_engine(prev)
    g = pl.adam_state()["exp_avg"].cpu().double() / OMB1
    R = max([B] + [B * h * w for h, w in _out_hw(spec)])
    err = (g - g64).abs()
    ratio = float((err / scale.clamp_min(1e-300)).max())
    print(f"    max err / scale {ratio:.3e}, bound {C + R * U / 32:.3e} (R = {R})")
    bad = err > (C + R * U / 32) * scale + 1e-30
    assert not bool(bad.any()), f"{int(bad.sum())} of {g.numel()} gradient elements outside the bound (worst ratio {ratio:.3e})"


def _out_hw(spec):
    convs, _ = orc.conv_shapes(spec)
    return [(c[4], c[5]) for c in convs]
