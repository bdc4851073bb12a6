"""The float64 DQN step of oracle/dqn_fp64.py (the yardstick of the GPU shape tests of both DQN kernels) against
torch.autograd in float64 on OracleDQN's network and its own target rule (DQN or DoubleDQN, optionally importance-weighted
rows): forward values and all seven gradient blocks to 1e-12 of their error scale, which in turn must bound every value.
Hidden sizes include ones that are not multiples of 4 or 64.  CPU only."""
import numpy as np
import pytest
import torch

from oracle.dqn_fp64 import BLOCKS, block_view, dqn_step, err_over_scale, next_action_gap
from oracle.pearl_oracle import OracleDQN, flat


@pytest.mark.parametrize("obs,A,B,dynamic", [(8, 1, 32, False), (24, 4, 48, True), (40, 16, 64, True)])
def test_fp64_step_matches_autograd(obs, A, B, dynamic):
    _compare_with_autograd(obs, A, B, dynamic, (64, 64), double=False, weighted=False)


CASES = [  # obs, A, B, dynamic next-action sets, hidden, DoubleDQN, importance weights
    (24, 7, 48, True, (64, 64), True, False),
    (16, 5, 40, False, (64, 64), True, True),
    (12, 6, 32, True, (65, 33), False, True),
    (9, 3, 24, True, (129, 257), True, True),
    (3, 2, 16, False, (5, 3), False, False),
    (5, 17, 20, True, (5, 3), True, False),
]


@pytest.mark.parametrize("obs,A,B,dynamic,hidden,double,weighted", CASES,
                         ids=[f"obs{c[0]}-A{c[1]}-B{c[2]}-{'dyn' if c[3] else 'full'}-h{c[4][0]}x{c[4][1]}"
                              f"{'-double' if c[5] else ''}{'-weighted' if c[6] else ''}" for c in CASES])
def test_fp64_double_weighted_and_odd_hidden_match_autograd(obs, A, B, dynamic, hidden, double, weighted):
    _compare_with_autograd(obs, A, B, dynamic, hidden, double, weighted)


def _compare_with_autograd(obs, A, B, dynamic, hidden, double, weighted):
    torch.manual_seed(obs * 100 + A)
    orc = OracleDQN(obs, A, hidden, batch_size=B, double=double)
    with torch.no_grad():
        for p in orc.Qt.parameters():
            p.add_(0.05 * torch.randn(p.shape))
    orc.Q, orc.Qt = orc.Q.double(), orc.Qt.double()
    Q, Qt = orc.Q, orc.Qt
    rng = np.random.default_rng(obs + A)
    state = torch.from_numpy(rng.standard_normal((B, obs)))
    next_state = torch.from_numpy(rng.standard_normal((B, obs)))
    reward = torch.from_numpy(rng.standard_normal(B))
    term = torch.from_numpy(rng.random(B) < 0.2)
    action = torch.from_numpy(rng.integers(0, A, B))
    weight = torch.from_numpy(rng.uniform(0.1, 1.0, B)) if weighted else None
    ids = np.tile(np.arange(A), (B, 1))
    cnt = np.full(B, A)
    if dynamic:
        for i in range(B):
            cnt[i] = rng.integers(1, A + 1)
            ids[i, :cnt[i]] = rng.permutation(rng.choice(A, cnt[i], replace=False))
            ids[i, cnt[i]:] = 0
    batch = dict(state=state, action=action, reward=reward, terminated=term, next_state=next_state,
                 avail_ids=torch.from_numpy(ids), avail_n=torch.from_numpy(cnt))

    # autograd on the reference network, with OracleDQN's own bootstrap rule (padded one-hot action list, unavailable mask)
    eye = torch.eye(A, dtype=torch.float64)
    q = orc._q_values(Q, state, eye[action])
    mask = torch.arange(A).view(1, A) >= torch.from_numpy(cnt).view(B, 1)
    y = orc._next_values(dict(next_state=next_state, next_available_actions=eye[torch.from_numpy(ids)],
                              next_unavailable_actions_mask=mask)) * orc.gamma * (1 - term.double()) + reward
    loss = (weight * (q - y) ** 2).mean() if weighted else torch.nn.MSELoss()(q, y)
    Q.zero_grad()
    loss.backward()
    want_grad = torch.cat([p.grad.reshape(-1) for p in Q.parameters()])

    val, sc = dqn_step(flat(Q), flat(Qt), batch, obs, A, orc.gamma, hidden=hidden, double=double, weight=weight)
    for name, got, want in (("q", val["q"], q.detach()), ("y", val["y"], y), ("loss", val["loss"], loss.detach()),
                            ("mae", val["mae"], (q - y).abs().mean().detach()), ("grad", val["grad"], want_grad)):
        s = sc[name] if name != "loss" else sc["mae"]
        err = float(err_over_scale(got, want, s).max())
        print(f"    {name}: max err / scale {err:.2e}")
        assert err <= 1e-12, name
    # the scale bounds every value (|sum a b| <= sum |a||b|), and the blocks tile the flat gradient
    for name in ("q", "y", "z1", "z2", "grad") + BLOCKS:
        assert bool((val[name].abs() <= sc[name] * (1 + 1e-12)).all()), name
    for name in BLOCKS:
        got = block_view(val["grad"], name, obs, A, hidden)
        assert torch.equal(got, val[name].reshape(got.shape))
    if double:
        # the gap is inf exactly where one action is available and positive elsewhere
        gap = next_action_gap(flat(Q), next_state, ids, cnt, obs, A, hidden)
        assert bool((torch.isinf(gap) == torch.from_numpy(cnt == 1)).all()) and bool((gap > 0).all())
