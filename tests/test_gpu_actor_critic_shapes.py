"""The continuous actor-critic learners — SAC (pearl_b200/csrc/sac.cu) and TD3, DDPG and TD3BC (pearl_b200/csrc/td3.cu) —
across their shape space against the float64 rounds of oracle/ac_fp64.py (sac_step, td3_step).  One round from zero
AdamW state per case, under contraction engines 0, 1 and 2: every gradient block of the actor and of both critics, read
back from exp_avg / (1 - beta1), within the bound below elementwise (scale = the sum of |a||b| over every product that
reached the value); the AdamW moments and parameters against AdamW applied in fp64 to that gradient; the critic target's
soft update fused into AdamW and TD3's actor-target update (bitwise, in fp32); the reported losses; and for SAC the
log-alpha gradient, the new log-alpha and alpha after the entropy step.  SAC runs through learn() from the ring (the
sampled rows from trace, the rsample noise given); TD3, DDPG and TD3BC through learn() and learn_batch() with the target
noise given.  test_td3_round_without_actor_update runs two TD3 rounds at actor_update_freq 2 and checks the second one,
which must leave the actor, its moments and both targets untouched, report the previous actor loss and still step the
critics.

`products` restates the contractions of sac.cu::round and td3.cu::round_variant and `kernel_of` the dispatch of
GemmLauncher::run and gemm_tc_launch; test_grid_reaches_every_branch fails if the case list stops reaching one of these:

| branch                | reached when                                                                            |
|-----------------------|-----------------------------------------------------------------------------------------|
| simt_64x64_fwd        | a forward product on the 64x64 SIMT tiles (>= 96 output tiles over the stacked nets)    |
| simt_64x64_bwd_x      | a backward-data product there                                                           |
| simt_64x64_bwd_w      | a backward-weight product there                                                         |
| simt_32_ks4_fwd       | a forward product on the 32x32 tiles with four K slices (Kc > 64)                       |
| simt_32_ks4_bwd_x     | a backward-data product there                                                           |
| simt_32_ks4_bwd_w     | a backward-weight product there                                                         |
| simt_32_ks1_fwd       | a forward product on the 32x32 tiles with one K slice (Kc <= 64)                        |
| simt_32_ks1_bwd_x     | a backward-data product there                                                           |
| simt_32_ks1_bwd_w     | a backward-weight product there                                                         |
| tc_tn64               | a wgmma product with No > 32                                                            |
| tc_tn32               | a wgmma product with No <= 32                                                           |
| tc_edge_chunk         | a wgmma product with Kc % 32 != 0                                                       |
| tc_scalar_loads       | a wgmma operand read along its rows whose pitch or base is not 16-byte aligned          |
| tc_ragged_rows        | a wgmma product with Mo % 128 != 0                                                      |
| tc_two_source         | the state || action operand of a critic's first layer on wgmma                          |
| tc_nets2              | a twin-critic product (blockIdx.z = critic) on wgmma                                    |
| tc_accumulate_mask    | SAC's dh2 += dz W_sd (masked by h2 > 0) on wgmma                                        |
| simt_accumulate_mask  | the same product on the SIMT tiles                                                      |
| mixed_round           | engine 1: a forward product on wgmma and another product of the round on SIMT          |
| wide_action           | A > 32: the gather's lane loop runs more than once, the head kernels' e % A wraps later  |
| one_row               | B = 1                                                                                   |
| autotune_on           | SAC with the entropy autotune                                                           |
| autotune_off          | SAC with a fixed entropy coefficient                                                    |
| clip_and_box          | TD3 / TD3BC target noise past the clip and target actions clamped to the box            |
| td3_non_update_round  | a TD3 round without the actor update (test_td3_round_without_actor_update)              |
| learn_batch           | TD3 / DDPG / TD3BC through learn_batch                                                  |

The RS form of the wgmma kernel (gemm_ts_launch) is not in the table: it runs only under the engines 164 / 132, which
prl_set_contraction_engine refuses, so no learner shape reaches it (`rs_form` restates that check; test_gpu_contraction
tests the form on its own).

Data.  States, actions, rewards and next states on a 1/256 grid, actions inside asymmetric per-dimension boxes
([-1, 1], [0, 5], [-0.1, 2] in turn), about 20 % terminal rows, about 2 B rows in the ring so that a draw is a strict
subset, and networks from the learners' own initialisation (SAC's mean and log-std heads scaled by 1/4) with the
targets perturbed away from the online nets.  A
row (SAC: a row and its rsample noise at that batch position) is redrawn when a ReLU pre-activation of a pass that is
differentiated lies within MARGIN of its scale — the actor at s, both online critics at (s, pi(s)) (TD3: critic 1) and
at (s, a) — and for SAC when |q1 - q2| at (s, pi(s)) does (k_sac_actor_loss routes the gradient by q1 <= q2), or when
the actor's pre-tanh value at s leaves |u| <= 4 (near saturation 1 - tanh^2 cancels in fp32, which is the formula's own
behaviour, not a kernel defect; test_saturated_actor_stays_finite keeps one such case).  The passes that run forward
only (the next-state actor, the target critics, the behaviour net) are continuous in their ReLUs: a flip there moves a
value by at most the margin, which the bound absorbs.  The fp64 rounds run on the GPU.

Bound.  |kernel - fp64| <= max(C, 4 u sqrt(B)) x scale, u = 2^-24, for every gradient block and loss (each is a sum
over the B rows, and the fp32 accumulators make a random-walk error that grows with that length).  Measured on an H100
80GB HBM3 (700 W power limit) over the whole grid, every engine and the two-round cases: the largest err / scale is
2.9e-6 (TD3BC a.b3 at obs 257, B 65536, engine 2), inside its 4 u sqrt(B) = 6.1e-5; where the floor C binds (4 u sqrt(B)
below the error) the largest is 4.8e-7 (TD3 q1.W3 at obs 1, A 1, B 1, engine 2; DDPG q2.W1 3.8e-7 at B 2).  C = 1e-6 is
about twice that.  A wrong index, box bound, mask or a missing product term is off by O(1e-3) to O(1) of the scale.
The whole file ran in about 30 s on that card.
"""
import math
import types
from collections import namedtuple

import numpy as np
import pytest
import torch

from oracle import ac_fp64

pytestmark = pytest.mark.gpu

C = 1e-6              # elementwise floor of the bound (measured maximum 4.8e-7 where it binds, see above)
U = 2.0 ** -24
MARGIN = 2e-7
GAMMA, TAU, ACTOR_TAU = 0.97, 0.3, 0.2
LR = 1e-3
CLIP = 1.0
ENGINES = (0, 1, 2)
BETA1 = np.float32(1.0 - 0.9)      # k_adamw's (float)(1 - beta1)
BOXES = ((-1.0, 1.0), (0.0, 5.0), (-0.1, 2.0))

# kind: sac / td3 / ddpg / td3bc; ah, ch, bh: actor, critic, behaviour widths; entry: learn / batch; tune: SAC autotune
Case = namedtuple("Case", "kind obs A ah ch bh B entry tune")
GRID = [
    Case("sac", 1, 1, (1, 1), (1, 1), None, 1, "learn", True),
    Case("sac", 3, 2, (3, 5), (5, 3), None, 2, "learn", False),
    Case("sac", 17, 6, (256, 256), (256, 256), None, 256, "learn", True),
    Case("sac", 31, 33, (65, 63), (63, 65), None, 255, "learn", False),
    Case("sac", 257, 17, (64, 32), (129, 257), None, 257, "learn", True),
    Case("sac", 376, 17, (640, 640), (640, 640), None, 1000, "learn", True),
    Case("sac", 128, 6, (32, 16), (64, 64), None, 4096, "learn", False),
    Case("sac", 3, 2, (5, 3), (3, 5), None, 16384, "learn", True),
    Case("td3", 1, 1, (1, 1), (1, 1), None, 1, "learn", None),
    Case("td3", 17, 6, (65, 63), (256, 256), None, 256, "batch", None),
    Case("td3", 31, 33, (3, 5), (5, 3), None, 31, "learn", None),
    Case("td3", 257, 2, (128, 64), (64, 128), None, 4096, "batch", None),
    Case("td3", 376, 17, (256, 256), (640, 640), None, 1000, "learn", None),
    Case("ddpg", 3, 64, (64, 64), (65, 63), None, 257, "learn", None),
    Case("ddpg", 128, 1, (640, 640), (1, 1), None, 2, "batch", None),
    Case("ddpg", 31, 6, (16, 16), (32, 32), None, 16384, "learn", None),
    Case("td3bc", 17, 6, (256, 256), (256, 256), (64, 128), 256, "batch", None),
    Case("td3bc", 1, 33, (3, 5), (5, 3), (7, 2), 1, "learn", None),
    Case("td3bc", 128, 64, (65, 63), (129, 33), (31, 17), 4096, "batch", None),
    Case("td3bc", 257, 2, (1, 1), (16, 16), (64, 128), 65536, "batch", None),
]


def _cid(c):
    bh = f"-b{c.bh[0]}x{c.bh[1]}" if c.bh else ""
    tune = "" if c.tune is None else ("-tune" if c.tune else "-fixed")
    return f"{c.kind}-obs{c.obs}-A{c.A}-a{c.ah[0]}x{c.ah[1]}-c{c.ch[0]}x{c.ch[1]}{bh}-B{c.B}-{c.entry}{tune}"


GRID_IDS = [_cid(c) for c in GRID]
NON_UPDATE_GRID = [Case("td3", 31, 33, (65, 63), (63, 65), None, 255, "learn", None),
                   Case("td3", 3, 2, (3, 5), (5, 3), None, 4096, "learn", None)]


# ---------------------------------------------------------------------------------------------- restated dispatch
# one contraction: op, Mo, No, Kc, nets, and the (row pitch, float offset) of every operand the wgmma loader reads along
# its rows (gemm_tc.cu's XO operands: both of a forward, dy of a backward-data), tags: two_source / accumulate_mask
Prod = namedtuple("Prod", "op Mo No Kc nets xo tags")


def _fwd(M, N, K, x, w, nets=1, tags=()):
    return Prod("fwd", M, N, K, nets, tuple(x) + tuple(w), tuple(tags))


def _bwd_x(M, N, Kx, dy, nets=1, tags=()):
    return Prod("bwd_x", M, Kx, N, nets, tuple(dy), tuple(tags))


def _bwd_w(M, N, K, nets=1, tags=()):
    return Prod("bwd_w", N, K + 1, M, nets, (), tuple(tags))


def products(c):
    """Every contraction of one round of case `c` (sac.cu::round / td3.cu::round_variant with the actor update)."""
    O, A, B = c.obs, c.A, c.B
    H1, H2 = c.ah
    C1, C2 = c.ch
    D = O + A
    Pc = C1 * D + C1 + C2 * C1 + C2 + C2 + 1
    cW2, cW3 = C1 * D + C1, C1 * D + C1 + C2 * C1 + C2
    aW2 = H1 * O + H1
    aW3 = aW2 + H2 * H1 + H2
    aWsd = aW3 + A * H2 + A

    def crit(nets):
        zs = range(nets)
        x = [(O, 0), (A, -O)]                     # S || Act: Act read with the split subtracted from its base
        w1 = [(D, z * Pc) for z in zs]
        return [_fwd(B, C1, D, x, w1, nets, ("two_source",)),
                _fwd(B, C2, C1, [(C1, z * B * C1) for z in zs], [(C1, cW2 + z * Pc) for z in zs], nets),
                _fwd(B, 1, C2, [(C2, z * B * C2) for z in zs], [(C2, cW3 + z * Pc) for z in zs], nets)]

    def actor_fwd(heads):
        out = [_fwd(B, H1, O, [(O, 0)], [(O, 0)]), _fwd(B, H2, H1, [(H1, 0)], [(H1, aW2)])]
        for off in heads:
            out.append(_fwd(B, A, H2, [(H2, 0)], [(H2, off)]))
        return out

    def crit_bwd(nets):
        zs = range(nets)
        return [_bwd_w(B, 1, C2, nets), _bwd_w(B, C2, C1, nets), _bwd_x(B, C2, C1, [(C2, z * B * C2) for z in zs], nets),
                _bwd_w(B, C1, D, nets, ("two_source",))]

    out = []
    if c.kind == "sac":
        out += actor_fwd((aW3, aWsd))
        out += crit(2)
        out += [_bwd_x(B, C2, C1, [(C2, z * B * C2) for z in range(2)], 2), _bwd_x(B, C1, A, [(C1, z * B * C1) for z in range(2)], 2)]
        out += [_bwd_w(B, A, H2), _bwd_w(B, A, H2), _bwd_x(B, A, H2, [(A, 0)]),
                _bwd_x(B, A, H2, [(A, 0)], 1, ("accumulate_mask",)), _bwd_w(B, H2, H1), _bwd_x(B, H2, H1, [(H2, 0)]),
                _bwd_w(B, H1, O)]
        out += actor_fwd((aW3, aWsd)) + crit(2) + crit(2) + crit_bwd(2)
        return out
    out += actor_fwd((aW3,)) + crit(1)
    if c.kind == "td3bc":
        K1, K2 = c.bh
        bW2 = K1 * O + K1
        out += [_fwd(B, K1, O, [(O, 0)], [(O, 0)]), _fwd(B, K2, K1, [(K1, 0)], [(K1, bW2)]),
                _fwd(B, A, K2, [(K2, 0)], [(K2, bW2 + K2 * K1 + K2)])]
    out += [_bwd_x(B, C2, C1, [(C2, 0)], 1), _bwd_x(B, C1, A, [(C1, 0)], 1)]
    out += [_bwd_w(B, A, H2), _bwd_x(B, A, H2, [(A, 0)]), _bwd_w(B, H2, H1), _bwd_x(B, H2, H1, [(H2, 0)]), _bwd_w(B, H1, O)]
    out += actor_fwd((aW3,)) + crit(2) + crit(2) + crit_bwd(2)
    return out


def kernel_of(p, engine):
    """gemm_tc_launch, then GemmLauncher::run: "tc64" / "tc32" or "simt_64x64" / "simt_32_ks4" / "simt_32_ks1"."""
    ao, bo = p.op != "bwd_w", p.op == "fwd"
    if engine != 0 and not (engine == 1 and p.Mo < 4096) and not (not ao and bo):
        return "tc64" if p.No > 32 else "tc32"
    if -(-p.Mo // 64) * -(-p.No // 64) * p.nets >= 96:
        return "simt_64x64"
    return "simt_32_ks4" if p.Kc > 64 else "simt_32_ks1"


def rs_form(engine):
    """gemm_ts_launch accepts a product only under engine 164 / 132 (the learners' GemmLauncher uses the library engine)."""
    return engine in (164, 132)


def branches(c, engine):
    """Names of the table's branches that one round of case `c` under `engine` reaches."""
    out = set()
    kinds = set()
    for p in products(c):
        k = kernel_of(p, engine)
        kinds.add("tc" if k.startswith("tc") else "simt")
        if k.startswith("simt"):
            out.add(f"{k}_{p.op}")
            if "accumulate_mask" in p.tags:
                out.add("simt_accumulate_mask")
            continue
        out.add("tc_tn64" if k == "tc64" else "tc_tn32")
        if p.Kc % 32:
            out.add("tc_edge_chunk")
        if any(ld % 4 or o % 4 for ld, o in p.xo):
            out.add("tc_scalar_loads")
        if p.Mo % 128:
            out.add("tc_ragged_rows")
        if "two_source" in p.tags:
            out.add("tc_two_source")
        if p.nets == 2:
            out.add("tc_nets2")
        if "accumulate_mask" in p.tags:
            out.add("tc_accumulate_mask")
    if engine == 1 and kinds == {"tc", "simt"}:
        out.add("mixed_round")
    if c.A > 32:
        out.add("wide_action")
    if c.B == 1:
        out.add("one_row")
    if c.kind == "sac":
        out.add("autotune_on" if c.tune else "autotune_off")
    if c.kind in ("td3", "td3bc"):
        out.add("clip_and_box")
    if c.entry == "batch":
        out.add("learn_batch")
    return out


ALL_BRANCHES = {line.split("|")[1].strip() for line in __doc__.splitlines()
                if line.startswith("| ") and not line.startswith("| branch")}


# ---------------------------------------------------------------------------------------------- helpers
class _Engine:
    """prl_set_contraction_engine for the duration of a with-block; the previous engine is restored in any case."""

    def __init__(self, engine):
        from pearl_b200 import _lib
        self.lib, self.engine = _lib.load(), engine

    def __enter__(self):
        from pearl_b200 import _lib
        self.prev = self.lib.prl_get_contraction_engine()
        _lib.check(self.lib.prl_set_contraction_engine(self.engine))

    def __exit__(self, *exc):
        from pearl_b200 import _lib
        _lib.check(self.lib.prl_set_contraction_engine(self.prev))


def _seed(c, extra=0):
    return (c.obs * 7919 + c.A * 104729 + sum(c.ah) * 31 + sum(c.ch) * 17 + (sum(c.bh) * 13 if c.bh else 0) + c.B * 3
            + len(c.kind) * 99991 + extra) % (2 ** 31)


def _box(A):
    lo = np.array([BOXES[d % 3][0] for d in range(A)], np.float32)
    hi = np.array([BOXES[d % 3][1] for d in range(A)], np.float32)
    return lo, hi


def _learner(c, seed, freq=None):
    from pearl_b200 import sac, td3
    lo, hi = _box(c.A)
    common = dict(state_dim=c.obs, actor_hidden_dims=list(c.ah), critic_hidden_dims=list(c.ch), actor_learning_rate=LR,
                  critic_learning_rate=LR, critic_soft_update_tau=TAU, discount_factor=GAMMA, training_rounds=1,
                  batch_size=c.B, low=lo, high=hi, device="cuda", seed=seed)
    if c.kind == "sac":
        pl = sac.B200ContinuousSoftActorCritic(entropy_coef=0.3, entropy_autotune=c.tune, **common)
        H1, H2 = c.ah
        with torch.no_grad():             # smaller mean / log-std heads: pre-tanh samples mostly inside |u| <= 4
            pl.actor_params[H1 * c.obs + H1 + H2 * H1 + H2:] *= 0.25
        if c.tune:                        # a coefficient away from 1: log alpha = -0.5
            pl._log_entropy[0] = -0.5
            pl._entropy_coef.copy_(torch.exp(pl._log_entropy[:1]))
    elif c.kind == "ddpg":
        pl = td3.B200DeepDeterministicPolicyGradient(actor_soft_update_tau=ACTOR_TAU, **common)
    else:
        kw = dict(actor_update_freq=2 if freq is None else freq, actor_update_noise=0.4, actor_update_noise_clip=CLIP,
                  actor_soft_update_tau=ACTOR_TAU)
        if c.kind == "td3bc":
            pl = td3.B200TD3BC(behavior_hidden_dims=list(c.bh), alpha_bc=1.7, **kw, **common)
        else:
            pl = td3.B200TD3(**kw, **common)
    g = torch.Generator(device="cuda").manual_seed(seed + 1)
    with torch.no_grad():
        pl.critic_target_params.add_(0.05 * torch.randn(pl.critic_target_params.shape, device="cuda", generator=g))
        if c.kind != "sac":
            pl.actor_target_params.add_(0.05 * torch.randn(pl.actor_target_params.shape, device="cuda", generator=g))
        if c.kind == "td3bc":
            K1, K2 = c.bh
            fan = [c.obs] * (K1 * c.obs + K1) + [K1] * (K2 * K1 + K2) + [K2] * (c.A * K2 + c.A)
            bound = torch.tensor(fan, dtype=torch.float32, device="cuda").rsqrt()
            pl.behavior_params.copy_((torch.rand(bound.shape, device="cuda", generator=g) * 2 - 1) * bound)
    return pl


def _q8(x):
    return torch.round(x * 256) / 256


def _rows(c, n, seed):
    """n candidate transitions (CPU float32)."""
    g = torch.Generator().manual_seed(seed)
    lo, hi = (torch.from_numpy(x) for x in _box(c.A))
    return dict(state=_q8(torch.randn(n, c.obs, generator=g)), next_state=_q8(torch.randn(n, c.obs, generator=g)),
                action=_q8(lo + (hi - lo) * torch.rand(n, c.A, generator=g)).clamp(lo, hi),
                reward=_q8(torch.randn(n, generator=g)), terminated=torch.rand(n, generator=g) < 0.2)


def _nets(c, pl):
    """The learner's parameters as V dicts (float64, on the GPU)."""
    sh = (ac_fp64.sac_actor_shapes if c.kind == "sac" else ac_fp64.td3_actor_shapes)(c.obs, c.A, c.ah)
    actor = ac_fp64.unflatten(pl.actor_params.double(), sh)
    q = ac_fp64.twin(pl.critic_params.double(), c.obs, c.A, c.ch)
    return actor, q


def _row_margin(c, pl, d):
    """Per row (CPU): the smallest pre-activation margin over the differentiated passes that do not depend on noise, and
    for TD3 also |pre| <= 4 (as a margin of -1 when violated)."""
    V = ac_fp64.V
    actor, q = _nets(c, pl)
    s, a = V(d["state"].double().cuda()), V(d["action"].double().cuda())
    fs = [ac_fp64.critic_forward(n, s, a) for n in q]
    if c.kind == "sac":        # and a mean that leaves room for |u| <= 4
        fa = ac_fp64.mlp_forward(actor, s, "Wmu")
        m = ac_fp64.relu_margin_of(fa, *fs)
        return torch.where(fa["out"].v.abs().amax(1) <= 3, m, torch.full_like(m, -1.0)).cpu()
    lo, hi = _box(c.A)
    fa = ac_fp64.td3_act(actor, s, lo.astype(np.float64), hi.astype(np.float64))
    f1 = ac_fp64.critic_forward(q[0], s, fa["action"])
    m = ac_fp64.relu_margin_of(fa, *fs, f1)
    m = torch.where(fa["out"].v.abs().amax(1) <= 4, m, torch.full_like(m, -1.0))
    return m.cpu()


def _pool(c, pl, n, seed):
    """n rows that clear the row filter, drawn in batches of 3 n."""
    kept, have = [], 0
    for attempt in range(20):
        d = _rows(c, 3 * n, seed + 1000003 * attempt)
        ok = torch.nonzero(_row_margin(c, pl, d) >= MARGIN).reshape(-1)[:n - have]
        kept.append({k: v[ok] for k, v in d.items()})
        have += ok.numel()
        if have == n:
            break
    assert have == n, "too few rows clear the margin"
    return {k: torch.cat([x[k] for x in kept]) for k in kept[0]}


def _sac_noise(c, pl, batch, seed):
    """[2, B, A] rsample draws; the actor step's draw at a batch position is redrawn until both critics at (s, pi(s)) clear
    the ReLU margin, |q1 - q2| clears it too and the pre-tanh sample stays within |u| <= 4."""
    V = ac_fp64.V
    g = torch.Generator().manual_seed(seed)
    B, A = c.B, c.A
    noise = torch.randn(2, B, A, generator=g)
    actor, q = _nets(c, pl)
    s = V(batch["state"].double().cuda())
    lo, hi = (x.astype(np.float64) for x in _box(A))
    todo = torch.ones(B, dtype=torch.bool)
    for _ in range(200):
        smp = ac_fp64.sac_sample(actor, s, V(noise[0].double().cuda()), lo, hi)
        fs = [ac_fp64.critic_forward(n, s, smp["action"]) for n in q]
        q1, q2 = fs[0]["q"], fs[1]["q"]
        ok = ac_fp64.relu_margin_of(*fs) >= MARGIN
        ok &= (q1.v - q2.v).abs() >= MARGIN * (q1.s + q2.s)
        ok &= smp["u"].v.abs().amax(1) <= 4
        todo = ~ok.cpu()
        if not todo.any():
            return noise
        noise[0][todo] = torch.randn(int(todo.sum()), A, generator=g)
    raise AssertionError("too few noise draws clear the margin")


def _buffer(pool, seed):
    from pearl_b200 import B200ReplayBuffer
    n = pool["state"].shape[0]
    buf = B200ReplayBuffer(n, rng="device")
    buf.is_action_continuous = True
    buf.push_batch(pool["state"], pool["action"], pool["reward"], pool["next_state"], pool["terminated"],
                   torch.zeros(n, dtype=torch.bool))
    buf.seed(seed)
    return buf


def _bound(B):
    return max(C, 4 * U * math.sqrt(B))


def _check(what, got, want, scale, worst, bound):
    from oracle.dqn_fp64 import check
    check(what, got, want, scale, worst, bound)


def _grad_of(m):
    return m.double() / float(BETA1)


def _check_adamw(what, w0, w, st, g, step=1):
    """exp_avg_sq, max_exp_avg_sq and the parameters after the first AdamW(amsgrad) step equal AdamW applied in fp64 to the
    kernel's gradient g (recovered from exp_avg)."""
    m, v, vmax = (x.double() for x in st)
    v_want = 0.001 * g * g
    assert float(((v - v_want).abs() - 1e-6 * v_want - 2.0 ** -126).max()) <= 0, f"{what} exp_avg_sq"
    assert torch.equal(st[2], st[1]), f"{what} max_exp_avg_sq after the first step"
    w64 = w0.double()
    w_want = w64 * (1.0 - LR * 0.01) - LR / 0.1 * m / ((vmax / 0.001).sqrt() + 1e-8)
    err = (w.double() - w_want).abs() - (3e-7 * w64.abs() + 1e-5 * LR)
    assert float(err.max()) <= 0, f"{what}: AdamW update of parameter {int(err.argmax())}"


def _soft_f32(tau, w, t):
    """k_adamw's / k_td3_soft_update's fp32 soft update: fl(fl(tau w) + fl((1 - tau) t)), tau and 1 - tau from double."""
    a, b = torch.tensor(tau, dtype=torch.float32), torch.tensor(1.0 - tau, dtype=torch.float32)
    return (a.to(w.device) * w) + (b.to(w.device) * t)


def _blocks(val, prefix, pl_state, shapes, B, worst, tag, sc):
    """Every gradient block under `prefix` of a flat kernel gradient against the fp64 value."""
    off = 0
    for k, shp in shapes.items():
        n = math.prod(shp)
        name = prefix + k
        _check(f"{name}{tag}", pl_state[off:off + n].reshape(shp), val[name], sc[name], worst, _bound(B))
        off += n
    assert off == pl_state.numel()


def _run_case(c, engine, worst):
    """One round of case `c` under `engine`; every check of the module docstring."""
    seed = _seed(c)
    pl = _learner(c, seed)
    B, A = c.B, c.A
    lo, hi = (x.astype(np.float64) for x in _box(A))
    n = 2 * B + 16 if c.entry == "learn" else B
    pool = _pool(c, pl, n, seed)
    nz = None
    if c.entry == "learn":
        buf = _buffer(pool, seed)
        logical, _ = buf.sample_indices(B, 1)
        buf.seed(seed)
        idx = logical[0].long().cpu()
        batch = {k: v[idx] for k, v in pool.items()}
    else:
        batch = pool
    if c.kind == "sac":
        nz = _sac_noise(c, pl, batch, seed + 5)
    elif c.kind != "ddpg":
        g = torch.Generator().manual_seed(seed + 7)
        nz = 0.8 * torch.randn(B, A, generator=g)
        at, _ = _nets(c, types.SimpleNamespace(actor_params=pl.actor_target_params, critic_params=pl.critic_params))
        na = ac_fp64.td3_act(at, ac_fp64.V(batch["next_state"][:1].double().cuda()), lo, hi)["na"].v
        nz[0, 0] = 3 * CLIP * (1.0 if float(na[0, 0]) >= 0 else -1.0)   # past the clip, towards the box it then meets
    actor0, critic0, ct0 = pl.actor_params.clone(), pl.critic_params.clone(), pl.critic_target_params.clone()
    at0 = None if c.kind == "sac" else pl.actor_target_params.clone()
    tag = f" [{_cid(c)} engine {engine}]"
    if c.kind == "sac":
        la0, alpha0 = float(pl._log_entropy[0]), float(pl._entropy_coef[0])
        trace = {}
        rep = pl.learn(buf, noise=nz.unsqueeze(0), trace=trace)
        assert torch.equal(trace["idx"][0].long(), idx), "the learner drew other rows than sample_indices"
        val, sc = ac_fp64.sac_step(actor0.double(), critic0.double(), ct0.double(), pl.actor_params.double(), la0, batch,
                                   nz, lo, hi, obs=c.obs, A=A, actor_hidden=c.ah, critic_hidden=c.ch, gamma=GAMMA,
                                   alpha=alpha0, autotune=c.tune, lr_entropy=LR)
        actor_loss, critic_loss = rep["actor_loss"][0], rep["critic_loss"][0]
    else:
        pl._training_steps = 1 if c.entry == "learn" else 0      # an update round (learn counts the round first)
        if c.entry == "learn":
            trace = {}
            rep = pl.learn(buf, noise=None if nz is None else nz.unsqueeze(0), trace=trace)
            assert torch.equal(trace["idx"][0].long(), idx), "the learner drew other rows than sample_indices"
            actor_loss, critic_loss = rep["actor_loss"][0], rep["critic_loss"][0]
        else:
            tb = types.SimpleNamespace(**batch)
            rep = pl.learn_batch(tb, noise=nz)
            actor_loss, critic_loss = rep["actor_loss"], rep["critic_loss"]
        val, sc = ac_fp64.td3_step(actor0.double(), critic0.double(), at0.double(), ct0.double(), batch, lo, hi, obs=c.obs,
                                   A=A, actor_hidden=c.ah, critic_hidden=c.ch, gamma=GAMMA, kind=c.kind,
                                   update_actor=True, noise=nz, noise_clip=CLIP,
                                   behavior=pl.behavior_params.double() if c.kind == "td3bc" else None,
                                   behavior_hidden=c.bh, alpha_bc=1.7)
        if nz is not None:        # the clip and the box are active
            assert bool((nz.abs() > CLIP).any())
            ta = val["target_action"].cpu()
            assert bool(((ta == torch.from_numpy(lo)) | (ta == torch.from_numpy(hi))).any()), "no target action on the box"
    torch.cuda.synchronize()
    ash = (ac_fp64.sac_actor_shapes if c.kind == "sac" else ac_fp64.td3_actor_shapes)(c.obs, A, c.ah)
    csh = ac_fp64.critic_shapes(c.obs, A, c.ch)
    ga, gc = _grad_of(pl._actor_state[0]), _grad_of(pl._critic_state[0])
    _blocks(val, "a.", ga, ash, B, worst, tag, sc)
    pc = gc.numel() // 2
    _blocks(val, "q1.", gc[:pc], csh, B, worst, tag, sc)
    _blocks(val, "q2.", gc[pc:], csh, B, worst, tag, sc)
    _check(f"actor_loss{tag}", torch.tensor(actor_loss), val["actor_loss"], sc["actor_loss"], worst, _bound(B))
    _check(f"critic_loss{tag}", torch.tensor(critic_loss), val["critic_loss"], sc["critic_loss"], worst, _bound(B))
    _check_adamw("actor" + tag, actor0, pl.actor_params, pl._actor_state, ga)
    _check_adamw("critic" + tag, critic0, pl.critic_params, pl._critic_state, gc)
    assert torch.equal(pl.critic_target_params, _soft_f32(TAU, pl.critic_params, ct0)), "critic target soft update" + tag
    if c.kind != "sac":
        assert torch.equal(pl.actor_target_params, _soft_f32(ACTOR_TAU, pl.actor_params, at0)), "actor target update" + tag
    if c.kind == "sac" and c.tune:
        _check(f"entropy_loss{tag}", torch.tensor(rep["entropy_coef"][0]), val["entropy_loss"], sc["entropy_loss"], worst,
               _bound(B))
        g = _grad_of(pl._log_entropy[1:2])
        _check(f"log_alpha_grad{tag}", g, val["log_alpha_grad"].reshape(1), sc["log_alpha_grad"].reshape(1), worst,
               _bound(B))
        _check_adamw("log_alpha" + tag, torch.tensor([la0], device="cuda"), pl._log_entropy[0:1],
                     [pl._log_entropy[i:i + 1] for i in (1, 2, 3)], g)
        la = float(pl._log_entropy[0])
        assert abs(float(pl._entropy_coef[0]) - math.exp(la)) <= 4 * U * math.exp(la), "alpha = exp(log_alpha)" + tag
    elif c.kind == "sac":
        assert "entropy_coef" not in rep and float(pl._entropy_coef[0]) == np.float32(0.3), "fixed coefficient" + tag
        assert torch.equal(pl._log_entropy, torch.tensor([0.0, 0, 0, 0], device="cuda"))
    return pl


# ---------------------------------------------------------------------------------------------- coverage
def test_grid_reaches_every_branch():
    """Together the cases (under the three engines) and the TD3 two-round cases reach every branch of the table, the RS
    form stays out of reach of every engine a learner can run under, and every value of each axis appears."""
    reached = {}
    for c in GRID:
        for e in ENGINES:
            assert not rs_form(e)
            for b in branches(c, e):
                reached.setdefault(b, []).append(f"{_cid(c)} engine {e}")
    reached["td3_non_update_round"] = [_cid(c) for c in NON_UPDATE_GRID]
    for b in sorted(ALL_BRANCHES):
        print(f"    {b}: {len(reached.get(b, []))} runs, e.g. {reached.get(b, ['-'])[0]}")
    assert not ALL_BRANCHES - set(reached), f"branches no case reaches: {sorted(ALL_BRANCHES - set(reached))}"
    assert len(ALL_BRANCHES) == 26
    assert {1, 3, 17, 31, 128, 257, 376} <= {c.obs for c in GRID}
    assert {1, 2, 6, 17, 33, 64} <= {c.A for c in GRID}
    assert {1, 2, 31, 255, 256, 257, 1000, 4096, 16384, 65536} <= {c.B for c in GRID}
    widths = {c.ah for c in GRID} | {c.ch for c in GRID}
    assert {(1, 1), (3, 5), (65, 63), (640, 640)} <= widths
    assert any(c.ah != c.ch for c in GRID)
    assert all(c.bh != c.ah for c in GRID if c.kind == "td3bc")
    for kind in ("sac", "td3", "ddpg", "td3bc"):
        assert any(c.kind == kind for c in GRID)
    for kind in ("td3", "ddpg", "td3bc"):
        assert {c.entry for c in GRID if c.kind == kind} == {"learn", "batch"}


# ---------------------------------------------------------------------------------------------- one round
@pytest.mark.parametrize("case", GRID, ids=GRID_IDS)
def test_one_round_matches_fp64(case):
    """One round from zero AdamW state under contraction engines 0, 1 and 2 (see the module docstring)."""
    worst = {}
    for engine in ENGINES:
        with _Engine(engine):
            pl = _run_case(case, engine, worst)
            del pl
    top = sorted(worst.items(), key=lambda kv: -kv[1])[:4]
    print(f"    MAXERR {_cid(case)} " + " ".join(f"{k}={e:.3e}" for k, e in top))


@pytest.mark.parametrize("case", NON_UPDATE_GRID, ids=[_cid(c) for c in NON_UPDATE_GRID])
def test_td3_round_without_actor_update(case):
    """Two TD3 rounds in one learn() at actor_update_freq 2, the first with the actor update and the second without, next
    to a one-round learner of the same seed: the second round leaves the actor, its moments, the actor target and the
    critic target as the first round left them, reports the first round's actor loss again (k_td3_repeat_actor_loss),
    and steps the critics with the gradient of the fp64 round on its rows."""
    c = case
    seed = _seed(c, 17)
    B, A = c.B, c.A
    lo, hi = (x.astype(np.float64) for x in _box(A))
    worst = {}
    for engine in ENGINES:
        with _Engine(engine):
            one, two = _learner(c, seed), _learner(c, seed)
            pool = _pool(c, one, 2 * B + 16, seed)
            g = torch.Generator().manual_seed(seed + 7)
            nz = 0.4 * torch.randn(2, B, A, generator=g)
            reps = []
            for pl, rounds in ((one, 1), (two, 2)):
                buf = _buffer(pool, seed)
                pl._training_rounds, pl._training_steps = rounds, 1       # round 0 updates the actor, round 1 does not
                trace = {}
                reps.append((pl.learn(buf, noise=nz[:rounds], trace=trace), trace["idx"]))
            (r1, i1), (r2, i2) = reps
            assert torch.equal(i1[0], i2[0])
            assert r2["actor_loss"][1] == r2["actor_loss"][0] == r1["actor_loss"][0], "repeated actor loss"
            assert torch.equal(two.actor_params, one.actor_params), "the actor moved in a round without its update"
            for x, y in zip(two._actor_state, one._actor_state):
                assert torch.equal(x, y), "the actor's moments moved in a round without its update"
            assert torch.equal(two.actor_target_params, one.actor_target_params), "actor target"
            assert torch.equal(two.critic_target_params, one.critic_target_params), "critic target"
            assert not torch.equal(two.critic_params, one.critic_params), "the critics were not stepped"
            steps = (int(two._lib.prl_td3_actor_adam_step(two._handle)), int(two._lib.prl_td3_critic_adam_step(two._handle)))
            assert steps == (1, 2), steps
            batch = {k: v[i2[1].long()] for k, v in pool.items()}
            val, sc = ac_fp64.td3_step(one.actor_params.double(), one.critic_params.double(), one.actor_target_params.double(),
                                       one.critic_target_params.double(), batch, lo, hi, obs=c.obs, A=A, actor_hidden=c.ah,
                                       critic_hidden=c.ch, gamma=GAMMA, kind="td3", update_actor=False, noise=nz[1],
                                       noise_clip=CLIP)
            m1, m2 = one._critic_state[0].double(), two._critic_state[0].double()
            g = (m2 - m1) / float(BETA1) + m1          # m2 = fma(0.1, g - m1, m1)
            slack = 16 * U * (m1.abs() + m2.abs()) / float(BETA1)
            csh = ac_fp64.critic_shapes(c.obs, A, c.ch)
            pc = g.numel() // 2
            for z, prefix in ((0, "q1."), (1, "q2.")):
                off = 0
                for k, shp in csh.items():
                    nel = math.prod(shp)
                    sl = slice(z * pc + off, z * pc + off + nel)
                    got = g[sl].reshape(shp).cpu()
                    want, scale = val[prefix + k].cpu(), sc[prefix + k].cpu()
                    err = (got - want).abs() - slack[sl].reshape(shp).cpu()
                    r = err.clamp_min(0) / scale.clamp_min(1e-300)
                    worst[prefix + k] = max(worst.get(prefix + k, 0.0), float(r.max()))
                    assert float(r.max()) <= _bound(B), f"{prefix}{k} engine {engine}: {float(r.max()):.3e}"
                    off += nel
            _check(f"critic_loss engine {engine}", torch.tensor(r2["critic_loss"][1]), val["critic_loss"], sc["critic_loss"],
                   worst, _bound(B))
            del one, two
    print(f"    MAXERR {_cid(c)} non-update " + " ".join(f"{k}={e:.3e}" for k, e in worst.items()))


def test_saturated_actor_stays_finite():
    """A SAC actor driven into saturation (pre-tanh samples of |u| > 10, where 1 - tanh^2 cancels in fp32): the round
    stays finite and agrees with the fp32 restatement of the reference (oracle/sac_oracle.py) on the losses."""
    from oracle.sac_oracle import OracleSAC
    c = Case("sac", 17, 6, (64, 64), (64, 64), None, 256, "learn", True)
    seed = _seed(c, 23)
    pl = _learner(c, seed)
    lo, hi = _box(c.A)
    with torch.no_grad():
        sh = ac_fp64.sac_actor_shapes(c.obs, c.A, c.ah)
        off = sum(math.prod(s) for k, s in sh.items() if k in ("W1", "b1", "W2", "b2", "Wmu"))
        pl.actor_params[off:off + c.A] = 12.0              # bmu: the mean far past the tanh knee
        pl.critic_target_params.copy_(pl.critic_params)
    pool = _rows(c, 2 * c.B + 16, seed)
    buf = _buffer(pool, seed)
    g = torch.Generator().manual_seed(seed)
    nz = torch.randn(1, 2, c.B, c.A, generator=g)
    a0, q0 = pl.actor_params.cpu().clone(), pl.critic_params.cpu().clone()
    trace = {}
    rep = pl.learn(buf, noise=nz, trace=trace)
    for t in (pl.actor_params, pl.critic_params, pl.critic_target_params, pl._log_entropy, pl._entropy_coef):
        assert bool(torch.isfinite(t).all())
    orc = OracleSAC(c.obs, c.A, c.ah, c.ch, lo, hi, actor_lr=LR, critic_lr=LR, gamma=GAMMA, tau=TAU, autotune=True)
    pc = q0.numel() // 2
    orc.actor.load_state_dict(orc.actor.state_dict())
    from oracle.pearl_oracle import load_flat
    load_flat(orc.actor, a0)
    for i in range(2):
        load_flat(orc.q[i], q0[i * pc:(i + 1) * pc])
        load_flat(orc.qt[i], q0[i * pc:(i + 1) * pc])
    with torch.no_grad():
        orc.log_alpha.fill_(-0.5)
    orc.alpha = torch.exp(orc.log_alpha).detach()
    idx = trace["idx"][0].long()
    out = orc.learn_batch({k: v[idx] for k, v in pool.items()}, nz[0, 0], nz[0, 1])
    for k, got in (("actor_loss", rep["actor_loss"][0]), ("critic_loss", rep["critic_loss"][0])):
        assert math.isfinite(got)
        assert abs(got - out[k]) <= 1e-4 * abs(out[k]) + 1e-5, (k, got, out[k])
