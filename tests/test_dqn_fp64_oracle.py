"""The float64 DQN step of oracle/dqn_fp64.py (the yardstick of tests/test_gpu_dqn_tc_shapes.py) against torch.autograd
in float64 on OracleDQN's network: forward values and all seven gradient blocks to 1e-12 of their error scale, which in
turn must bound every value.  CPU only."""
import numpy as np
import pytest
import torch

from oracle.dqn_fp64 import BLOCKS, block_view, dqn_step, err_over_scale
from oracle.pearl_oracle import OracleDQN, flat


@pytest.mark.parametrize("obs,A,B,dynamic", [(8, 1, 32, False), (24, 4, 48, True), (40, 16, 64, True)])
def test_fp64_step_matches_autograd(obs, A, B, dynamic):
    torch.manual_seed(obs * 100 + A)
    orc = OracleDQN(obs, A, (64, 64), batch_size=B)
    with torch.no_grad():
        for p in orc.Qt.parameters():
            p.add_(0.05 * torch.randn(p.shape))
    Q, Qt = orc.Q.double(), orc.Qt.double()
    rng = np.random.default_rng(obs + A)
    state = torch.from_numpy(rng.standard_normal((B, obs)))
    next_state = torch.from_numpy(rng.standard_normal((B, obs)))
    reward = torch.from_numpy(rng.standard_normal(B))
    term = torch.from_numpy(rng.random(B) < 0.2)
    action = torch.from_numpy(rng.integers(0, A, B))
    ids = np.tile(np.arange(A), (B, 1))
    cnt = np.full(B, A)
    if dynamic:
        for i in range(B):
            cnt[i] = rng.integers(1, A + 1)
            ids[i, :cnt[i]] = np.sort(rng.choice(A, cnt[i], replace=False))
            ids[i, cnt[i]:] = 0
    batch = dict(state=state, action=action, reward=reward, terminated=term, next_state=next_state,
                 avail_ids=torch.from_numpy(ids), avail_n=torch.from_numpy(cnt))

    # autograd on the reference network: the padded one-hot action list and the unavailable mask of the reference
    eye = torch.eye(A, dtype=torch.float64)
    q = orc._q_values(Q, state, eye[action])
    with torch.no_grad():
        v = orc._q_values(Qt, next_state, eye[torch.from_numpy(ids)])
        v[torch.arange(A).view(1, A) >= torch.from_numpy(cnt).view(B, 1)] = -float("inf")
        y = v.max(1)[0] * orc.gamma * (1 - term.double()) + reward
    loss = torch.nn.MSELoss()(q, y)
    Q.zero_grad()
    loss.backward()
    want_grad = torch.cat([p.grad.reshape(-1) for p in Q.parameters()])

    val, sc = dqn_step(flat(Q), flat(Qt), batch, obs, A, orc.gamma)
    for name, got, want in (("q", val["q"], q.detach()), ("y", val["y"], y), ("loss", val["loss"], loss.detach()),
                            ("grad", val["grad"], want_grad)):
        s = sc[name] if name != "loss" else sc["mae"]
        err = float(err_over_scale(got, want, s).max())
        print(f"    {name}: max err / scale {err:.2e}")
        assert err <= 1e-12, name
    # the scale bounds every value (|sum a b| <= sum |a||b|), and the blocks tile the flat gradient
    for name in ("q", "y", "z1", "z2", "grad") + BLOCKS:
        assert bool((val[name].abs() <= sc[name] * (1 + 1e-12)).all()), name
    for name in BLOCKS:
        assert torch.equal(block_view(val["grad"], name, obs, A), val[name].reshape(block_view(val["grad"], name, obs, A).shape))
