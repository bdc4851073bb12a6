"""The cooperative fp32 DQN learner (k_dqn_learn, pearl_b200/csrc/dqn.cu; engine="simt") across its shape space against
the float64 step of oracle/dqn_fp64.py: DQN and DoubleDQN, full and dynamic next-action sets, prioritized steps,
learn_batch with arbitrary masks, q_values / act, several rounds in one launch, and the edge of what its shared-memory
plan can hold.

This learner runs every engine="auto" DQN, every DoubleDQN, every prioritized step and every learn_batch.  Its tiling
has many branches, and the grid below is a covering design (not a full product) chosen so that each branch runs in at
least one case.  `tiling` restates make_plan / choose_tiling; `branches` names what a case reaches, and
test_grid_reaches_every_branch fails if the case list stops reaching one of them:

| branch                 | in dqn.cu                                              | reached when                          |
|------------------------|--------------------------------------------------------|---------------------------------------|
| k_panels               | second / third K panel of cta_linear (k0 += KCMAX)     | obs, H1 or H2 > 128                   |
| ragged_n_panel         | ragged last N panel after a full one (nc < NC)         | H1 or H2 > 64, not a multiple of 64   |
| scalar_panel           | unaligned scalar panel loads (!vec_ok)                 | obs + A, H1 or H1 (obs + A + 1) % 4   |
| vector_panel           | 16-byte cp.async panel loads                           | all of those multiples of 4           |
| k_split                | K-slice split + fixed-order reduction (KS > 1)         | a row block of <= 32 rows             |
| k_unsplit              | one K slice (KS == 1)                                  | a row block of >= 33 rows             |
| head_tail              | cta_head loop over j >= 256                            | H2 > 256                              |
| target_chunks          | target rows in several chunks (all_actions_q)          | rows * A > mch                        |
| r_doubled              | choose_tiling doubles R                                | B > 4 (SMs - 1)                       |
| mch_halved             | choose_tiling halves mch to fit                        | large network / many actions          |
| all_ctas               | G = every SM but one                                   | B = R (SMs - 1)                       |
| one_cta                | G = 1 with a forced R >= B                             |                                       |
| short_last_cta         | the last CTA's remainder rows                          | B % R != 0                            |
| double_dqn             | arg-max -> action id -> target evaluation              | DoubleDQN                             |
| double_dqn_dynamic_ids | ... with the id read from the record's action list     | DoubleDQN, dynamic sets               |
| importance_weight      | dq *= w, out_td -> priorities                          | test_prioritized_step (PER_GRID)      |
| pack_mask              | mask compaction in k_pack_batch                        | test_learn_batch_and_q_values         |

Data as in the tensor-core shape test (oracle.dqn_fp64.make_data): the target network is perturbed away from the
online one, about 20 % of the rows are terminal and some truncated, the buffer holds about 2 B rows, and a row is kept
only if every online pre-activation clears MARGIN of its scale and, for DoubleDQN, the online next-action gap clears it
too.  Dynamic sets list the available ids in random order.  The fp64 yardstick runs on the GPU.

C is set from the largest max |err| / scale over the whole grid, both update frequencies and every block, measured on
an H100 SXM (80 GB HBM3, 700 W power limit): 1.16e-7 (y at obs 3, A 16, hidden [1, 1], B 8384, DoubleDQN, dynamic
sets; the other blocks: dW1s 4.4e-8, dW1a 4.3e-8, q 4.3e-8, db3 4.1e-8, dW2 3.9e-8, db1 2.9e-8, loss 2.6e-8, db2 2.4e-8,
dW3 1.2e-8).  C = 4e-7 is under four times that.  On that card the edge of the plan is a first hidden layer of 76
units at 255 actions (obs 8, H2 64, batch 256) and a batch of 8384 rows for a [64, 64] network (obs 8, 4 actions); the
whole file ran in about 35 s there.
"""
import random
from collections import namedtuple

import numpy as np
import pytest
import torch

from _tol import close, close_params

pytestmark = pytest.mark.gpu

C = 4e-7              # elementwise bound |kernel - fp64| <= C * scale (measured maximum 1.16e-7, see above)
MARGIN = 5e-6         # ReLU and next-action-gap margin of the accepted rows (must stay well above C)
GAMMA = 0.99
BLOCKS = ("dW1s", "dW1a", "db1", "dW2", "db2", "dW3", "db3")

# ---------------------------------------------------------------------------------------------- restated plan
NT, NC, KCMAX, MB, MAX_CTAS = 256, 64, 128, 64, 148
STATIC_SMEM = 5024    # k_dqn_learn's static shared memory (the sampler CTA's MT19937 state; ptxas -v), not for the plan
STAGE_FLOATS, RED_FLOATS = KCMAX * (NC + 4), NT * 16
Tiling = namedtuple("Tiling", "R G mch mch0 bytes")


def _r4(x):
    return (x + 3) // 4 * 4


def record_words(obs, A, dynamic):
    """prl_buf_layout_of: state | next_state (each padded to 4 words) | action | reward | flags | [action ids]."""
    return _r4(2 * _r4(obs) + 3 + ((A + 3) // 4 if dynamic else 0))


def plan_floats(obs, A, H1, H2, R, W, mch):
    """make_plan(...).total."""
    H1p, H2p = _r4(H1), _r4(H2)
    return (2 * R * W + 5 * R * H1p + 2 * R * H2p + mch * (H1p + H2p) + 2 * A * H1p + _r4(R * A) + _r4(9 * R)
            + STAGE_FLOATS + RED_FLOATS + _r4(2 * (R + 1) + 16))


def tiling(obs, A, H1, H2, W, B, rows_per_cta, sms, smem):
    """choose_tiling: Tiling(R, G, mch, mch before fitting, bytes), or None when the plan does not fit."""
    max_ctas = min(sms, MAX_CTAS) - 1
    R = rows_per_cta
    if R <= 0:
        R = 4
        while -(-B // R) > max_ctas:
            R *= 2
    assert -(-B // R) <= max_ctas and R <= NT, "outside choose_tiling's row limits"
    mch = 64
    while mch > 4 and mch // 2 >= R * A:
        mch //= 2
    mch0 = mch
    while True:
        b = 4 * plan_floats(obs, A, H1, H2, R, W, mch)
        if b <= smem:
            return Tiling(R, -(-B // R), mch, mch0, b)
        if mch <= 4:
            return None
        mch //= 2


def _props():
    """(SM count, bytes of dynamic shared memory a k_dqn_learn launch may use)."""
    p = torch.cuda.get_device_properties(torch.cuda.current_device())
    return p.multi_processor_count, p.shared_memory_per_block_optin - STATIC_SMEM


# ---------------------------------------------------------------------------------------------- the grid
Case = namedtuple("Case", "obs A H1 H2 B R double dynamic")
# B: "S4" = 4 (SMs - 1), "S4+1", "S64" = 64 (SMs - 1), the largest batch of R 64; H1 "max": the largest that fits
GRID = [
    Case(1, 1, 1, 1, 1, 0, False, False),
    Case(3, 2, 5, 3, 2, 0, True, True),
    Case(3, 3, 5, 3, 5, 1, False, True),
    Case(8, 16, 64, 64, 5, 3, True, False),
    Case(8, 4, 64, 64, "S64", 0, False, False),
    Case(3, 16, 1, 1, "S64", 0, True, True),
    Case(8, 17, 64, 64, 4096, 64, True, True),
    Case(1, 2, 65, 63, 4096, 64, False, True),
    Case(127, 17, 65, 63, "S4", 0, False, True),
    Case(128, 16, 128, 128, "S4+1", 0, True, False),
    Case(129, 16, 129, 257, 1024, 0, False, True),
    Case(257, 3, 300, 300, "S4", 0, True, True),
    Case(257, 3, 512, 512, "S4", 0, False, False),
    Case(8, 255, "max", 64, "S4", 0, True, True),
    Case(1, 255, "max", 128, 1024, 0, False, False),
    Case(3, 64, "max", 128, 1024, 0, False, True),
    Case(127, 64, "max", 64, 5, 1, True, False),
    Case(127, 64, 128, 128, 2, 0, True, False),
    Case(129, 2, 65, 63, 1024, 0, True, True),
    Case(8, 2, 65, 63, 5, 64, True, False),
    Case(128, 1, 512, 512, 5, 0, True, False),
    Case(257, 17, 129, 257, "S4+1", 0, True, True),
    Case(3, 1, 64, 64, 4096, 0, False, False),
    Case(127, 255, 5, 3, 1024, 0, False, True),
    Case(129, 255, 5, 3, 5, 1, True, True),
    Case(8, 64, 5, 3, 1024, 64, False, True),
    Case(1, 16, 128, 128, 5, 3, False, False),
    Case(257, 2, 65, 63, 1, 0, False, True),
    Case(128, 3, 300, 300, "S4+1", 0, False, True),
    Case(1, 17, 512, 512, 2, 3, True, False),
    Case(129, 16, 300, 300, 1, 0, False, False),
    Case(257, 1, 64, 64, "S4+1", 0, False, False),
    Case(127, 3, 129, 257, 1024, 0, True, False),
]


def _cid(c):
    return (f"obs{c.obs}-A{c.A}-h{c.H1}x{c.H2}-B{c.B}-R{c.R or 'auto'}-{'ddqn' if c.double else 'dqn'}-"
            f"{'dyn' if c.dynamic else 'full'}")


GRID_IDS = [_cid(c) for c in GRID]
PER_GRID = [c for c in GRID if isinstance(c.B, int) and c.B <= 1024 and c.A in (2, 16, 17, 64, 255)
            and c.H1 != 1][:10]
BATCH_GRID = [GRID[i] for i in (2, 3, 10, 11, 14, 23, 27)]
LAUNCH_GRID = [GRID[i] for i in (6, 9, 10, 11, 12, 13, 18, 32)]
TRAJ_GRID = [GRID[i] for i in (6, 12, 18)]


def resolve(c):
    """The case with its batch and "max" hidden size made concrete for this device, and its predicted tiling."""
    sms, smem = _props()
    S = min(sms, MAX_CTAS) - 1
    B = {"S4": 4 * S, "S4+1": 4 * S + 1, "S64": 64 * S}.get(c.B, c.B)
    W = record_words(c.obs, c.A, c.dynamic)
    H1 = c.H1
    if H1 == "max":
        H1 = 1
        while tiling(c.obs, c.A, H1 + 1, c.H2, W, B, c.R, sms, smem) is not None:
            H1 += 1
    c = c._replace(B=B, H1=H1)
    return c, tiling(c.obs, c.A, c.H1, c.H2, W, B, c.R, sms, smem)


def branches(c, t, max_ctas):
    """Names of the table's branches that the resolved case `c` with tiling `t` reaches."""
    out = set()
    D = c.obs + c.A
    if max(c.obs, c.H1, c.H2) > KCMAX:
        out.add("k_panels")
    if any(h > NC and h % NC for h in (c.H1, c.H2)):
        out.add("ragged_n_panel")
    out.add("scalar_panel" if D % 4 or c.H1 % 4 or c.H1 * (D + 1) % 4 else "vector_panel")
    rows = {min(t.R, c.B), c.B - (t.G - 1) * t.R}          # rows of the first and of the last CTA
    ms = set(rows)
    for rv in rows:                                        # target chunk sizes of all_actions_q
        ms |= {min(t.mch, rv * c.A - c0) for c0 in range(0, rv * c.A, t.mch)}
    blocks = {min(MB, m - m0) for m in ms for m0 in range(0, m, MB)}
    if min(blocks) <= 32:
        out.add("k_split")
    if max(blocks) >= 33:
        out.add("k_unsplit")
    if c.H2 > 256:
        out.add("head_tail")
    if min(t.R, c.B) * c.A > t.mch:
        out.add("target_chunks")
    if c.R <= 0 and t.R > 4:
        out.add("r_doubled")
    if t.mch < t.mch0:
        out.add("mch_halved")
    if t.G == max_ctas:
        out.add("all_ctas")
    if t.G == 1 and c.R >= c.B:
        out.add("one_cta")
    if c.B % t.R:
        out.add("short_last_cta")
    if c.double:
        out.add("double_dqn")
        if c.dynamic:
            out.add("double_dqn_dynamic_ids")
    return out


ALL_BRANCHES = {line.split("|")[1].strip() for line in __doc__.splitlines()
                if line.startswith("| ") and not line.startswith("| branch")}


# ---------------------------------------------------------------------------------------------- helpers
class _Space:
    def __init__(self, n):
        self.n = n
        self.actions = [torch.tensor([i]) for i in range(n)]

    @property
    def actions_batch(self):
        return torch.stack(self.actions)


def _seed(c, extra=0):
    return (c.obs * 7919 + c.A * 104729 + (c.H1 if isinstance(c.H1, int) else 0) * 31 + c.H2 * 17
            + int(c.double) * 5 + int(c.dynamic) * 3 + extra) % (2 ** 31)


def _learner(c, seed, *, freq=1000, tau=0.3, rounds=1, per_call=32, B=None):
    import pearl_b200
    torch.manual_seed(seed)
    cls = pearl_b200.B200DoubleDQN if c.double else pearl_b200.B200DeepQLearning
    learner = cls(state_dim=c.obs, action_space=_Space(c.A), hidden_dims=[c.H1, c.H2], learning_rate=1e-3,
                  discount_factor=GAMMA, training_rounds=rounds, batch_size=c.B if B is None else B,
                  target_update_freq=freq, soft_update_tau=tau, max_rounds_per_call=per_call, rows_per_cta=c.R,
                  engine="simt", action_representation_module=pearl_b200.OneHotActionTensorRepresentationModule(c.A))
    learner = learner.to("cuda")
    with torch.no_grad():
        for p in learner._Q_target.parameters():
            p.add_(0.05 * torch.randn(p.shape, device=p.device))
    return learner


def _data(learner, c, seed):
    from oracle.dqn_fp64 import make_data
    d = make_data(learner.flat_parameters.detach().clone(), c.obs, c.A, c.B, seed, c.dynamic, MARGIN,
                  hidden=(c.H1, c.H2), double=c.double)
    if c.dynamic:   # the available ids in random order (the slot order is not the id order)
        rng = np.random.default_rng(seed + 1)
        ids = d["avail_ids"].numpy().copy()
        for i, k in enumerate(d["avail_n"].numpy()):
            ids[i, :k] = rng.permutation(ids[i, :k])
        d["avail_ids"] = torch.from_numpy(ids)
    return d


def _push(buf, data, c):
    kw = {}
    if c.dynamic:
        kw = dict(next_available_ids=data["avail_ids"].to(torch.uint8), next_available_count=data["avail_n"].to(torch.int32))
    buf.push_batch(data["state"], data["action"].to(torch.int32), data["reward"], data["next_state"],
                   data["terminated"], data["truncated"], max_number_actions=c.A, **kw)
    return buf


def _buffer(data, c, seed, rng="device"):
    import pearl_b200
    buf = _push(pearl_b200.B200ReplayBuffer(data["state"].shape[0], rng=rng, dynamic_action_space=c.dynamic), data, c)
    buf.seed(seed)
    return buf


def _check_step(c, learner, w0, wt, batch, q, y, loss, weight=None, tag=""):
    """q, y, the loss and the seven gradient blocks (from exp_avg after one step from zero moments) within C x scale
    of the fp64 step; exp_avg_sq, max_exp_avg_sq and the parameters equal AdamW applied in fp64 to that gradient."""
    from oracle.dqn_fp64 import block_view, check, dqn_step
    hp = learner._adam_hparams()
    dev = w0.device
    val, sc = dqn_step(w0.double(), wt.double().to(dev), batch, c.obs, c.A, GAMMA, hidden=(c.H1, c.H2),
                       double=c.double, weight=weight)
    worst = {}
    if q is not None:
        check("q", q, val["q"], sc["q"], worst, C)
        check("y", y, val["y"], sc["y"], worst, C)
    check("loss", torch.tensor(loss), val["mae"], sc["mae"], worst, C)
    st = learner.adam_state()
    assert st["step"] == 1
    m, v, vmax = st["exp_avg"], st["exp_avg_sq"], st["max_exp_avg_sq"]
    g = m / torch.tensor(1.0 - hp["beta1"], dtype=torch.float32, device=m.device)
    h = (c.H1, c.H2)
    for name in BLOCKS:
        gb = block_view(g, name, c.obs, c.A, h)
        check(name, gb, val[name].reshape(gb.shape), sc[name].reshape(gb.shape), worst, C)
    print(f"    MAXERR {_cid(c)}{tag} " + " ".join(f"{k}={e:.2e}" for k, e in worst.items()))
    g64, m64, w64 = g.double(), m.double(), w0.double()
    v_want = (1.0 - hp["beta2"]) * g64 * g64
    assert float(((v.double() - v_want).abs() - 1e-6 * v_want).max()) <= 0, "exp_avg_sq"
    assert torch.equal(vmax, v), "max_exp_avg_sq after the first step"
    bc1, bc2 = 1.0 - hp["beta1"], 1.0 - hp["beta2"]
    w_want = w64 * (1.0 - hp["lr"] * hp["weight_decay"]) - hp["lr"] / bc1 * m64 / ((vmax.double() / bc2).sqrt() + hp["eps"])
    err = (learner.flat_parameters.double() - w_want).abs() - (3e-7 * w64.abs() + 1e-5 * hp["lr"])
    assert float(err.max()) <= 0, f"AdamW update of parameter {int(err.argmax())}"
    return val, sc


def _one_step(c, t, freq, seed):
    """One learn() of the resolved case `c`: launch geometry as predicted, soft update as scheduled, step vs fp64."""
    learner = _learner(c, seed, freq=freq)
    data = _data(learner, c, seed)
    buf = _buffer(data, c, seed)
    w0, wt0 = learner.flat_parameters.clone(), learner.flat_target_parameters.clone()
    rep = learner.learn(buf, trace=True)
    info = learner.launch_info()
    assert (info["rows_per_cta"], info["ctas"]) == (t.R, t.G), f"launch {info}, restated plan {t}"
    wt = learner.flat_target_parameters
    if freq == 2:   # (training_steps + 1) % freq == 0 at the first step: tau w + (1 - tau) w_target, in fp32
        want_t = 0.3 * w0.double() + 0.7 * wt0.double()
        scale_t = 0.3 * w0.double().abs() + 0.7 * wt0.double().abs()
        assert float(((wt.double() - want_t).abs() - 2.0 ** -21 * scale_t).max()) <= 0, "soft target update"
    else:
        assert torch.equal(wt, wt0), "the target moved without a scheduled update"
    idx = rep["idx"][0].long().cpu()
    batch = {k: v[idx] for k, v in data.items()}
    _check_step(c, learner, w0, wt, batch, rep["q"][0], rep["y"][0], rep["loss"][0], tag=f" freq={freq}")


# ---------------------------------------------------------------------------------------------- coverage
def test_grid_reaches_every_branch():
    """Every grid case fits the restated plan, and together the cases reach every branch of the table above; the
    prioritized and learn_batch subsets have the shapes they are meant to have."""
    sms, _ = _props()
    max_ctas = min(sms, MAX_CTAS) - 1
    reached = {}
    for c in GRID:
        rc, t = resolve(c)
        assert t is not None, f"{_cid(c)} does not fit the restated plan"
        for b in branches(rc, t, max_ctas):
            reached.setdefault(b, []).append(_cid(c))
    reached["importance_weight"] = [_cid(c) for c in PER_GRID]
    reached["pack_mask"] = [_cid(c) for c in BATCH_GRID]
    for b in sorted(ALL_BRANCHES):
        print(f"    {b}: {len(reached.get(b, []))} cases, e.g. {reached.get(b, ['-'])[0]}")
    assert not ALL_BRANCHES - set(reached), f"branches no case reaches: {sorted(ALL_BRANCHES - set(reached))}"
    assert len(ALL_BRANCHES) == 17
    # every value of each axis appears
    res = [resolve(c)[0] for c in GRID]
    S = max_ctas
    assert {1, 3, 8, 127, 128, 129, 257} <= {c.obs for c in res}
    assert {1, 2, 3, 16, 17, 64, 255} <= {c.A for c in res}
    assert {(1, 1), (5, 3), (64, 64), (65, 63), (128, 128), (129, 257), (300, 300), (512, 512)} <= {(c.H1, c.H2) for c in res}
    assert {1, 2, 5, 4 * S, 4 * S + 1, 1024, 4096, 64 * S} <= {c.B for c in res}
    assert {1, 3, 64} <= {c.R for c in res}
    assert {(d, y) for d in (False, True) for y in (False, True)} <= {(c.double, c.dynamic) for c in res}
    # pairs that must meet in one case
    assert any(c.obs > 128 and c.H1 > 64 for c in res)
    assert any(c.H2 > 256 and c.H1 > 128 for c in res)
    assert {64, 255} <= {c.A for c in GRID if c.H1 == "max"}
    assert any(c.B >= 4096 and t.R == 64 for c, t in map(resolve, GRID))
    assert len(PER_GRID) >= 8 and all(c.B <= 1024 for c in PER_GRID)
    assert any(c.A == 255 for c in PER_GRID) and any((c.H1, c.H2) == (129, 257) for c in PER_GRID)
    assert len(BATCH_GRID) >= 6 and any(c.A == 255 for c in BATCH_GRID) and any(c.obs == 257 for c in BATCH_GRID)


# ---------------------------------------------------------------------------------------------- a. one step
@pytest.mark.parametrize("case", GRID, ids=GRID_IDS)
def test_one_step_gradient_matches_fp64(case):
    """One gradient step, without (freq 1000) and with (freq 2) a soft update before it."""
    c, t = resolve(case)
    for freq in (1000, 2):
        _one_step(c, t, freq, _seed(case, freq))


# ---------------------------------------------------------------------------------------------- b. prioritized step
@pytest.mark.parametrize("case", PER_GRID, ids=[_cid(c) for c in PER_GRID])
def test_prioritized_step(case):
    """A step of prl_dqn_learn_per: the importance-weighted fp64 step with the draw's weights, and the priorities the
    kernel wrote at the sampled slots, (|q - y| + eps)^alpha of its own q and y, against PerOracle.priority_of and,
    through the propagated tolerance, against the fp64 |q - y|."""
    import pearl_b200
    from oracle.per_oracle import PerOracle
    c, t = resolve(case)
    seed = _seed(case, 7)
    learner = _learner(c, seed)
    data = _data(learner, c, seed)
    n = data["state"].shape[0]
    buf = _push(pearl_b200.B200PrioritizedReplayBuffer(n, seed=seed, dynamic_action_space=c.dynamic), data, c)
    td = torch.from_numpy(np.random.default_rng(seed).exponential(size=n)).float()   # unequal priorities: weights < 1
    for i0 in range(0, n, 1024):
        buf.update_priorities(torch.arange(i0, min(n, i0 + 1024)), td[i0:i0 + 1024])
    w0, wt0 = learner.flat_parameters.clone(), learner.flat_target_parameters.clone()
    rep = learner.learn(buf, trace=True)
    info = learner.launch_info()
    assert info["rows_per_cta"] == t.R and info["ctas"] == t.G
    slots, weight = rep["slots"][0].long().cpu(), rep["weight"][0]
    assert float(weight.max()) <= 1.0 and float(weight.min()) > 0 and float(weight.min()) < 1.0
    batch = {k: v[slots] for k, v in data.items()}
    val, sc = _check_step(c, learner, w0, wt0, batch, rep["q"][0], rep["y"][0], rep["loss"][0], weight=weight.double())
    orc = PerOracle(n, buf.alpha, buf.beta, buf.eps)
    q, y = rep["q"][0].cpu().numpy(), rep["y"][0].cpu().numpy()
    leaves = buf.sum_tree.cpu().numpy()[orc.C2 + slots.numpy()]
    want = orc.priority_of(q - y)
    # CUDA's powf is not correctly rounded (documented bound: 4 ulp), numpy's float32 power is
    ulp = np.abs(leaves.view(np.int32).astype(np.int64) - want.view(np.int32).astype(np.int64))
    print(f"    PRIORITY leaves {leaves.size}: bit-exact {int((ulp == 0).sum())}, max ulp {int(ulp.max())}")
    assert int(ulp.max()) <= 4, "leaf priorities differ from (|q - y| + eps)^alpha of the kernel's q, y"
    # against fp64: |q - y| is within C (scale(q) + scale(y)) of its fp64 value
    td64 = (val["q"] - val["y"]).abs().cpu().numpy()
    tol = C * (sc["q"] + sc["y"]).cpu().numpy()
    a, e = float(buf.alpha), float(buf.eps)
    lo, hi = np.maximum(td64 - tol, 0) + e, td64 + tol + e
    assert np.all(leaves >= lo ** a * (1 - 1e-6)) and np.all(leaves <= hi ** a * (1 + 1e-6)), "priorities vs fp64 |q - y|"


# ---------------------------------------------------------------------------------------------- c. learn_batch, q_values
@pytest.mark.parametrize("case", BATCH_GRID, ids=[_cid(c) for c in BATCH_GRID])
def test_learn_batch_and_q_values(case):
    """learn_batch with random non-prefix unavailable masks over permuted next_available_actions ids equals the fp64
    step on the compacted sets; q_values for 1, 3, 5 and 1000 rows equals the fp64 forward; act(exploit=True) picks
    the fp64 arg-max on rows whose arg-max gap clears MARGIN."""
    from oracle.dqn_fp64 import check, next_action_gap, q_values
    from pearl_b200._compat import TransitionBatch
    c, t = resolve(case._replace(dynamic=True))    # learn_batch packs records with the dynamic layout
    seed = _seed(case, 11)
    learner = _learner(c, seed)
    cd = c._replace(dynamic=False)
    data = _data(learner, cd, seed)
    n, A, B = data["state"].shape[0], c.A, c.B
    rng = np.random.default_rng(seed)
    perm = np.stack([rng.permutation(A) for _ in range(n)])
    mask = rng.random((n, A)) < 0.4
    mask[np.arange(n), rng.integers(0, A, n)] = False             # at least one action kept per row
    cnt = (~mask).sum(1)
    comp = np.zeros((n, A), dtype=np.int64)
    for i in range(n):
        comp[i, :cnt[i]] = perm[i][~mask[i]]
    keep = np.arange(n)
    if c.double:
        w = learner.flat_parameters.detach().clone()
        keep = np.flatnonzero((next_action_gap(w, data["next_state"], comp, cnt, c.obs, A, (c.H1, c.H2)) >= MARGIN).numpy())
    keep = keep[:B]
    assert keep.size == B, "too few rows clear the next-action gap"
    batch = {k: v[keep] for k, v in data.items()}
    batch["avail_ids"], batch["avail_n"] = torch.from_numpy(comp[keep]), torch.from_numpy(cnt[keep])
    tb = TransitionBatch(state=batch["state"], action=batch["action"], reward=batch["reward"],
                         next_state=batch["next_state"], terminated=batch["terminated"], truncated=batch["truncated"],
                         next_available_actions=torch.from_numpy(perm[keep]).float().unsqueeze(-1),
                         next_unavailable_actions_mask=torch.from_numpy(mask[keep]))
    w0, wt0 = learner.flat_parameters.clone(), learner.flat_target_parameters.clone()
    rep = learner.learn_batch(tb)
    info = learner.launch_info()
    assert info["rows_per_cta"] == t.R and info["ctas"] == t.G and info["launches"] == 2
    assert torch.equal(learner.flat_target_parameters, wt0)
    _check_step(c, learner, w0, wt0, batch, None, None, rep["loss"], tag=" learn_batch")

    w1 = learner.flat_parameters.clone()
    srng = np.random.default_rng(seed + 2)
    for nrows in (1, 3, 5, 1000):
        s = torch.from_numpy(np.rint(srng.standard_normal((nrows, c.obs)) * 256) / 256).float()
        for target, w in ((False, w1), (True, wt0)):
            want, scale = q_values(w.double(), s, c.obs, A, (c.H1, c.H2))
            check(f"q_values[{nrows}, target={target}]", learner.q_values(s, target=target), want, scale, {}, C)
    s = torch.from_numpy(np.rint(srng.standard_normal((40, c.obs)) * 256) / 256).float()
    want, _ = q_values(w1.double(), s, c.obs, A, (c.H1, c.H2))
    gap = next_action_gap(w1.double(), s, np.tile(np.arange(A), (40, 1)), np.full(40, A), c.obs, A, (c.H1, c.H2))
    for i in np.flatnonzero((gap >= MARGIN).numpy())[:8]:
        got = int(learner.act(s[i], _Space(A), exploit=True))
        assert got == int(want[i].argmax()), f"act row {i}"


# ---------------------------------------------------------------------------------------------- d. rounds in a launch
@pytest.mark.parametrize("case", LAUNCH_GRID, ids=[_cid(c) for c in LAUNCH_GRID])
def test_rounds_in_one_launch_match_one_round_calls(case):
    """7 rounds in one launch vs 7 one-round calls (soft updates every 3 rounds): the look-ahead soft update of phase B,
    the double-buffered records of consecutive rounds and the shared memory zeroed once per launch must give the same
    arithmetic as separate launches: losses, parameters, target parameters and AdamW moments bit-identical."""
    c, _ = resolve(case)
    seed = _seed(case, 13)
    out = []
    for per_call in (7, 1):
        learner = _learner(c, seed, freq=3, tau=0.5, rounds=7, per_call=per_call)
        buf = _buffer(_data(learner, c, seed), c, seed)
        rep = learner.learn(buf)
        st = learner.adam_state()
        out.append((rep["loss"], learner.flat_parameters.clone(), learner.flat_target_parameters.clone(),
                    st["exp_avg"].clone(), st["exp_avg_sq"].clone(), st["max_exp_avg_sq"].clone()))
    a, b = out
    assert a[0] == b[0], "losses"
    for what, x, y in zip(("params", "target params", "exp_avg", "exp_avg_sq", "max_exp_avg_sq"), a[1:], b[1:]):
        assert torch.equal(x, y), f"{what}: {int((x != y).sum())} elements differ"


# ---------------------------------------------------------------------------------------------- e. short trajectory
@pytest.mark.parametrize("case", TRAJ_GRID, ids=[_cid(c) for c in TRAJ_GRID])
def test_short_trajectory_against_oracle(case):
    """20 rounds on the learner's own sampled indices, replayed by the fp32 CPU oracle (soft updates every 5 rounds)."""
    from oracle.pearl_oracle import OracleDQN, flat
    c, _ = resolve(case)
    rounds, seed = 20, _seed(case, 17)
    learner = _learner(c, seed, freq=5, tau=0.5, rounds=rounds)
    data = _data(learner, c, seed)
    buf = _buffer(data, c, seed)
    orc = OracleDQN(c.obs, c.A, (c.H1, c.H2), lr=1e-3, gamma=GAMMA, batch_size=c.B, target_update_freq=5, tau=0.5,
                    double=c.double, init_q=flat(learner._Q).cpu(), init_q_target=flat(learner._Q_target).cpu())
    rep = learner.learn(buf, trace=True)
    idx = rep["idx"].long().cpu()
    eye = torch.eye(c.A)
    slot = torch.arange(c.A).view(1, c.A)
    losses = []
    for r in range(rounds):
        b = {k: v[idx[r]] for k, v in data.items()}
        orc.training_steps += 1
        losses.append(orc.learn_batch(dict(
            state=b["state"], action=eye[b["action"]], reward=b["reward"], terminated=b["terminated"],
            next_state=b["next_state"], next_available_actions=eye[b["avail_ids"]],
            next_unavailable_actions_mask=slot >= b["avail_n"].view(-1, 1))))
    tag = _cid(c)
    close(np.asarray(rep["loss"]), np.asarray(losses), f"{tag} loss")
    close_params(learner.flat_parameters.cpu().numpy(), flat(orc.Q).numpy(), f"{tag} params", 1e-3, rounds)
    close_params(learner.flat_target_parameters.cpu().numpy(), flat(orc.Qt).numpy(), f"{tag} target", 1e-3, rounds)


# ---------------------------------------------------------------------------------------------- f. support boundary
def _boundary_pairs():
    """(inside, outside) case pairs at the edge of the plan: H1 at 255 actions, and the batch across the point where R
    doubles beyond what fits."""
    sms, smem = _props()
    S = min(sms, MAX_CTAS) - 1
    obs, A, H2, B = 8, 255, 64, 256
    W = record_words(obs, A, False)
    H1 = 1
    while tiling(obs, A, H1 + 1, H2, W, B, 0, sms, smem) is not None:
        H1 += 1
    pairs = [(Case(obs, A, H1, H2, B, 0, False, False), Case(obs, A, H1 + 1, H2, B, 0, False, False))]
    W = record_words(8, 4, False)
    Bmax = 64 * S
    assert tiling(8, 4, 64, 64, W, Bmax, 0, sms, smem) is not None and tiling(8, 4, 64, 64, W, Bmax + 1, 0, sms, smem) is None
    pairs.append((Case(8, 4, 64, 64, Bmax, 0, True, False), Case(8, 4, 64, 64, Bmax + 1, 0, True, False)))
    return pairs


def test_support_boundary():
    """Just inside the plan a case runs and passes the one-step check; just outside, learn() raises RuntimeError
    ("does not fit shared memory") and leaves parameters, target, AdamW state, the step count and the buffer's
    sampler (rng="device" and rng="python") untouched, without consuming Python's `random` state.  Prints the limits:
    the largest first hidden layer at 255 actions and the largest batch of a [64, 64] network."""
    sms, smem = _props()
    for inside, outside in _boundary_pairs():
        print(f"    LIMIT {torch.cuda.get_device_name()} ({sms} SMs, {smem} B opt-in shared memory): "
              f"inside {_cid(inside)}, outside {_cid(outside)}")
        c, t = resolve(inside)
        _one_step(c, t, 1000, _seed(inside, 19))
        for rng_mode in ("device", "python"):
            c = outside
            seed = _seed(c, 23)
            learner = _learner(c, seed)
            buf = _buffer(_data(learner, c, seed), c, seed, rng=rng_mode)
            if rng_mode == "python":
                random.seed(seed)
                buf.set_rng_state(random.getstate()[1])
            learner.flat_parameters
            before = [learner.flat_parameters.clone(), learner.flat_target_parameters.clone()] + [
                learner.adam_state()[k].clone() for k in ("exp_avg", "exp_avg_sq", "max_exp_avg_sq")]
            rng0, py0 = buf.get_rng_state(), random.getstate()
            with pytest.raises(RuntimeError, match="does not fit shared memory"):
                learner.learn(buf)
            torch.cuda.synchronize()
            after = [learner.flat_parameters, learner.flat_target_parameters] + [
                learner.adam_state()[k] for k in ("exp_avg", "exp_avg_sq", "max_exp_avg_sq")]
            for what, x, y in zip(("params", "target", "exp_avg", "exp_avg_sq", "max_exp_avg_sq"), before, after):
                assert torch.equal(x, y), f"{_cid(c)} {rng_mode}: {what} changed"
            assert learner._training_steps == 0 and learner.adam_state()["step"] == 0
            assert np.array_equal(buf.get_rng_state(), rng0), f"{rng_mode}: the sampler ran"
            assert random.getstate() == py0, "Python's random state was consumed"
