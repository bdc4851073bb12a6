"""The float64 DQN step of oracle/dqn_fp64.py (the yardstick of the GPU shape tests of both DQN kernels) against
torch.autograd in float64 on OracleDQN's network and its own target rule (DQN or DoubleDQN, optionally importance-weighted
rows): forward values and all seven gradient blocks to 1e-12 of their error scale, which in turn must bound every value.
Hidden sizes include ones that are not multiples of 4 or 64.  The same for the conservative step (cql_step, on
OracleCQL's CQL term, and equal to the DQN step at alpha 0) and the dueling step (oracle/dueling_fp64.py, through the
reference's get_q_values on networks whose three MLPs have independent widths).  CPU only."""
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


# ---------------------------------------------------------------------------------------------- conservative (CQL)
def _random_batch(rng, obs, A, B, dynamic):
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
            ids[i, :cnt[i]] = rng.permutation(rng.choice(A, cnt[i], replace=False))
            ids[i, cnt[i]:] = 0
    return dict(state=state, action=action, reward=reward, terminated=term, next_state=next_state,
                avail_ids=torch.from_numpy(ids), avail_n=torch.from_numpy(cnt))


def _partial_sets(rng, A, B):
    """Current sets of 1..A distinct ids in random order, padded with id 0."""
    curr = np.zeros((B, A), np.int64)
    for i in range(B):
        m = int(rng.integers(1, A + 1))
        curr[i, :m] = rng.permutation(rng.choice(A, m, replace=False))
    return curr


def _check_values_and_scales(pairs, val, sc, names):
    for name, got, want, s in pairs:
        err = float(err_over_scale(got, want, s).max())
        print(f"    {name}: max err / scale {err:.2e}")
        assert err <= 1e-12, name
    for name in names:
        assert bool((val[name].abs() <= sc[name] * (1 + 1e-12)).all()), f"scale does not bound {name}"


CQL_CASES = [  # obs, A, B, dynamic next sets, hidden, DoubleDQN, partial current sets
    (8, 2, 16, False, (64, 64), False, False),
    (6, 3, 24, True, (5, 3), True, True),
    (10, 17, 20, True, (65, 33), False, True),
    (5, 17, 12, True, (129, 7), True, False),
    (3, 4, 32, False, (1, 1), True, True),
]


@pytest.mark.parametrize("obs,A,B,dynamic,hidden,double,partial", CQL_CASES,
                         ids=[f"obs{c[0]}-A{c[1]}-B{c[2]}-{'dyn' if c[3] else 'full'}-h{c[4][0]}x{c[4][1]}"
                              f"{'-double' if c[5] else ''}{'-partial' if c[6] else ''}" for c in CQL_CASES])
def test_fp64_cql_step_matches_autograd(obs, A, B, dynamic, hidden, double, partial):
    """cql_step against autograd on OracleCQL's network with its own CQL term and target rule: q, y, the slot values,
    mae and every gradient element to 1e-12 of their scale, which must bound every value."""
    from oracle.cql_oracle import OracleCQL, cql_term
    from oracle.dqn_fp64 import cql_step
    torch.manual_seed(obs * 100 + A)
    alpha = 1.7
    orc = OracleCQL(obs, A, hidden, batch_size=B, double=double, alpha=alpha)
    with torch.no_grad():
        for p in orc.Qt.parameters():
            p.add_(0.05 * torch.randn(p.shape))
    orc.Q, orc.Qt = orc.Q.double(), orc.Qt.double()
    rng = np.random.default_rng(obs + 7 * A)
    batch = _random_batch(rng, obs, A, B, dynamic)
    curr = _partial_sets(rng, A, B) if partial else None
    eye = torch.eye(A, dtype=torch.float64)
    mask = torch.arange(A).view(1, A) >= batch["avail_n"].view(B, 1)
    oh_action = eye[batch["action"]]
    q = orc._q_values(orc.Q, batch["state"], oh_action)
    y = orc._next_values(dict(next_state=batch["next_state"], next_available_actions=eye[batch["avail_ids"]],
                              next_unavailable_actions_mask=mask)) * orc.gamma * (1 - batch["terminated"].double()) \
        + batch["reward"]
    cur_ids = torch.arange(A).repeat(B, 1) if curr is None else torch.from_numpy(curr)
    q_all = orc._q_values(orc.Q, batch["state"], eye[cur_ids]).view(B, A)
    loss = torch.nn.MSELoss()(q, y) + alpha * cql_term(q_all, oh_action)
    orc.Q.zero_grad()
    loss.backward()
    want_grad = torch.cat([p.grad.reshape(-1) for p in orc.Q.parameters()])

    val, sc = cql_step(flat(orc.Q), flat(orc.Qt), batch, obs, A, orc.gamma, alpha, hidden=hidden, double=double,
                       curr_ids=curr)
    _check_values_and_scales(
        [("q", val["q"], q.detach(), sc["q"]), ("y", val["y"], y, sc["y"]),
         ("q_all", val["q_all"][:, :A], q_all.detach(), sc["q_all"][:, :A]),
         ("mae", val["mae"], (q - y).abs().mean().detach(), sc["mae"]), ("grad", val["grad"], want_grad, sc["grad"])],
        val, sc, ("q", "y", "q_all", "grad") + BLOCKS)
    for name in BLOCKS:
        got = block_view(val["grad"], name, obs, A, hidden)
        assert torch.equal(got, val[name].reshape(got.shape))


@pytest.mark.parametrize("double", [False, True])
def test_fp64_cql_step_with_alpha_zero_is_the_dqn_step(double):
    from oracle.dqn_fp64 import cql_step
    obs, A, B, hidden = 7, 5, 24, (33, 17)
    torch.manual_seed(3)
    orc = OracleDQN(obs, A, hidden, batch_size=B, double=double)
    w, wt = flat(orc.Q).double(), flat(orc.Qt).double() + 0.05 * torch.randn(flat(orc.Qt).numel(), dtype=torch.float64)
    batch = _random_batch(np.random.default_rng(5), obs, A, B, True)
    v0, s0 = dqn_step(w, wt, batch, obs, A, 0.99, hidden=hidden, double=double)
    v1, s1 = cql_step(w, wt, batch, obs, A, 0.99, 0.0, hidden=hidden, double=double)
    for name in ("q", "y", "mae", "grad"):
        assert float(err_over_scale(v1[name], v0[name], s0[name]).max()) <= 1e-12, name


# ---------------------------------------------------------------------------------------------- dueling
DUEL_CASES = [  # obs, A, B, dynamic next sets, widths (F, sh1, sh2, vh1, vh2, ah1, ah2), DoubleDQN, current sets
    (8, 1, 16, False, (64, 64, 64, 64, 64, 64, 64), False, "full"),
    (6, 2, 24, True, (3, 5, 3, 5, 3, 5, 3), True, "partial"),
    (4, 3, 20, True, (7, 9, 5, 6, 4, 11, 3), False, "none"),
    (5, 17, 12, True, (33, 65, 33, 17, 9, 65, 31), True, "partial"),
    (3, 17, 16, False, (1, 1, 1, 1, 1, 1, 1), True, "none"),
    (9, 4, 32, True, (13, 129, 7, 3, 5, 9, 257), True, "full"),
]
_WKEYS = ("feature_dim", "state_h1", "state_h2", "value_h1", "value_h2", "adv_h1", "adv_h2")


class _DuelNet(torch.nn.Module):
    """DuelingQValueNetwork's three MLPs with independent widths (oracle.dueling_oracle.DuelNet ties them to one list)."""

    def __init__(self, obs, A, w):
        super().__init__()
        from oracle.pearl_oracle import _mlp
        self.state_arch = _mlp([obs, w["state_h1"], w["state_h2"], w["feature_dim"]])
        self.value_arch = _mlp([w["feature_dim"], w["value_h1"], w["value_h2"], 1])
        self.advantage_arch = _mlp([w["feature_dim"] + A, w["adv_h1"], w["adv_h2"], 1])


@pytest.mark.parametrize("obs,A,B,dynamic,wl,double,curr", DUEL_CASES,
                         ids=[f"obs{c[0]}-A{c[1]}-B{c[2]}-{'dyn' if c[3] else 'full'}-F{c[4][0]}"
                              f"{'-double' if c[5] else ''}-curr_{c[6]}" for c in DUEL_CASES])
def test_fp64_dueling_step_matches_autograd(obs, A, B, dynamic, wl, double, curr):
    """dueling_step against autograd through the reference's get_q_values on a dueling network (independent widths),
    with its own target rules (DQN: masked max over all next slots; DoubleDQN: online a*, then the query-alone target):
    q, y, mae and every gradient element to 1e-12 of their scale, which must bound every value; every block tiles the
    flat gradient."""
    from oracle.dueling_fp64 import BLOCKS as DB, block_view as dbv, dueling_step, layout, next_action_gap as dgap
    from oracle.dueling_oracle import get_q_values
    widths = dict(zip(_WKEYS, wl))
    torch.manual_seed(obs * 100 + A)
    Q, Qt = _DuelNet(obs, A, widths).double(), _DuelNet(obs, A, widths).double()
    with torch.no_grad():
        for p, pt in zip(Q.parameters(), Qt.parameters()):
            pt.copy_(p + 0.05 * torch.randn(p.shape, dtype=torch.float64))
    rng = np.random.default_rng(obs + 11 * A)
    batch = _random_batch(rng, obs, A, B, dynamic)
    cur = _partial_sets(rng, A, B) if curr == "partial" else None
    eye = torch.eye(A, dtype=torch.float64)
    mask = torch.arange(A).view(1, A) >= batch["avail_n"].view(B, 1)
    nxt = eye[batch["avail_ids"]]
    cur_oh = None if curr == "none" else eye[torch.arange(A).repeat(B, 1) if cur is None else torch.from_numpy(cur)]
    q = get_q_values(Q, batch["state"], eye[batch["action"]], cur_oh)
    with torch.no_grad():
        if double:
            v = get_q_values(Q, batch["next_state"], nxt)
            v[mask] = -float("inf")
            chosen = nxt[torch.arange(B), v.max(1)[1]]
            V = get_q_values(Qt, batch["next_state"], chosen)
        else:
            v = get_q_values(Qt, batch["next_state"], nxt)
            v[mask] = -float("inf")
            V = v.max(1)[0]
    y = V * 0.99 * (1 - batch["terminated"].double()) + batch["reward"]
    loss = torch.nn.MSELoss()(q, y)
    Q.zero_grad()
    loss.backward()
    want_grad = torch.cat([p.grad.reshape(-1) for p in Q.parameters()])
    assert want_grad.numel() == layout(obs, A, widths)["P"]

    val, sc = dueling_step(flat(Q), flat(Qt), batch, obs, A, 0.99, widths, double=double, curr_ids=cur,
                           query_alone=curr == "none")
    _check_values_and_scales(
        [("q", val["q"], q.detach(), sc["q"]), ("y", val["y"], y, sc["y"]), ("loss", val["loss"], loss.detach(), sc["loss"]),
         ("mae", val["mae"], (q - y).abs().mean().detach(), sc["mae"]), ("grad", val["grad"], want_grad, sc["grad"])],
        val, sc, ("q", "y", "grad") + DB)
    for name in DB:
        got = dbv(val["grad"], name, obs, A, widths)
        assert torch.equal(got, val[name].reshape(got.shape)), name
    if curr == "none":      # query-alone: q does not depend on the advantage net
        for name in DB:
            if name.startswith("dA"):
                assert not bool(val[name].any()) and not bool(sc[name].any()), name
    if double:
        gap = dgap(flat(Q), batch["next_state"], batch["avail_ids"], batch["avail_n"], obs, A, widths)
        assert bool((torch.isinf(gap) == (batch["avail_n"] == 1)).all()) and bool((gap >= 0).all())


def test_fp64_dueling_q_values_and_margin():
    """dueling q_values over caller id sets against get_q_values (the mean over each row's set), and the margin is the
    smallest over the trunk, the value net and every advantage slot of the row."""
    from oracle.dueling_fp64 import q_values as dq, relu_margin as dm
    from oracle.dueling_oracle import get_q_values
    obs, A, n = 5, 6, 9
    widths = dict(zip(_WKEYS, (7, 9, 5, 6, 4, 11, 3)))
    torch.manual_seed(1)
    Q = _DuelNet(obs, A, widths).double()
    rng = np.random.default_rng(2)
    s = torch.from_numpy(rng.standard_normal((n, obs)))
    eye = torch.eye(A, dtype=torch.float64)
    for ids in (None, torch.from_numpy(np.stack([rng.permutation(A)[:3] for _ in range(n)]))):
        got, scale = dq(flat(Q), s, obs, A, widths, ids)
        full = torch.arange(A).repeat(n, 1) if ids is None else ids
        with torch.no_grad():
            want = get_q_values(Q, s, eye[full])
        assert float(err_over_scale(got, want, scale).max()) <= 1e-12
        assert bool((got.abs() <= scale).all())
    slots = torch.from_numpy(rng.integers(0, A, (n, 4)))
    m = dm(flat(Q), s, slots, obs, A, widths)
    per_slot = torch.stack([dm(flat(Q), s, slots[:, k], obs, A, widths) for k in range(4)], 1)
    assert torch.equal(m, per_slot.min(1)[0])
