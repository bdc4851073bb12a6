"""The conservative (CQL, pearl_b200/csrc/cql.cu) and dueling (pearl_b200/csrc/dueling.cu) DQN learners across their
shape space against the float64 steps of oracle/dqn_fp64.py (cql_step) and oracle/dueling_fp64.py (dueling_step): every
gradient block of one round, read back from exp_avg / (1 - beta1), within C x scale elementwise (scale = the sum of
|a||b| over every product that reached the value), the AdamW moments and parameters against AdamW applied in fp64 to
that gradient, the target (untouched, or the fp32 soft update that precedes the step), learn_batch with partial padded
current sets and non-prefix next masks, and q_values.

Both learners run their contractions through gemm.cuh's GemmLauncher: SIMT tiles, or the wgmma tiles of gemm_tc.cu
(3xTF32), which contraction engine 1 (the library default) selects from 4096 output rows on and engine 2 always.  Both
are exercised per case under engines 0, 1 and 2.  `products` restates the contractions of cql_round / duel_round and
`branches` the dispatch of GemmLauncher::run and gemm_tc_launch; test_grid_reaches_every_branch fails if the case list
stops reaching one of these:

| branch                | reached when                                                                          |
|-----------------------|---------------------------------------------------------------------------------------|
| simt_64x64_fwd        | a forward product on the 64x64 SIMT tiles (>= 96 output tiles)                        |
| simt_64x64_bwd_x      | a backward-data product there                                                         |
| simt_64x64_bwd_w      | a backward-weight product there                                                       |
| simt_32_ks4_fwd       | a forward product on the 32x32 tiles with four K slices (Kc > 64)                     |
| simt_32_ks4_bwd_x     | a backward-data product there                                                         |
| simt_32_ks4_bwd_w     | a backward-weight product there                                                       |
| simt_32_ks1_fwd       | a forward product on the 32x32 tiles with one K slice (Kc <= 64)                      |
| simt_32_ks1_bwd_x     | a backward-data product there                                                         |
| simt_32_ks1_bwd_w     | a backward-weight product there                                                       |
| tc_tn64               | a wgmma product with No > 32                                                          |
| tc_tn32               | a wgmma product with No <= 32 (the scalar heads)                                      |
| tc_edge_chunk         | a wgmma product with Kc % 32 != 0                                                     |
| tc_scalar_loads       | a wgmma operand read along its rows whose pitch or base is not 16-byte aligned (!vec1) |
| tc_ragged_rows        | a wgmma product with Mo % 128 != 0                                                    |
| mixed_round           | engine 1: the online pass on wgmma, the next-slot pass on SIMT                        |
| slot_loop             | A > 32: the warp loops of the target kernels, slot_mean and the load kernels          |
| byte_ids_high         | A = 255 with dynamic next sets (ids >= 128 read from the ring)                        |
| a_min                 | CQL A = 2 (n_0 = n_1 = 1); dueling A = 1                                              |
| padded_current_sets   | learn_batch with partial current sets padded with id 0                                |
| query_alone           | dueling learn_batch without current sets                                              |
| flagged_update        | target_update_freq = 1: the soft update precedes the step and y uses the new target   |
| double                | DoubleDQN                                                                             |
| dynamic               | dynamic next-action sets in the ring                                                  |
| one_row               | B = 1                                                                                 |
| independent_widths    | dueling: trunk, value and advantage widths and F all differ, F odd                    |

Data as in the DQN shape tests (oracle.dqn_fp64.make_data): inputs on a 1/256 grid, the target network perturbed away
from the online one, about 20 % terminal rows, about 2 B rows in the buffer, and a row is kept only if every online
pre-activation at EVERY one of its A + 1 slots (dueling: and of the trunk and value net) clears MARGIN of its scale and,
for DoubleDQN, the online next-action gap (dueling: with the advantage mean) clears it too.  The fp64 steps run on the GPU.

C is set from the largest err / scale over the whole grid, every engine, both update frequencies and every block,
measured on an H100 80GB HBM3 (700 W power limit): 1.52e-7 (dueling dVW1 at obs 1, A 1, hidden [1, 1], B 1, engine 2;
CQL: dW1s 1.30e-7 at obs 3, A 3, hidden [5, 3], B 2, DoubleDQN, engine 2).  C = 4e-7 is under three times that.

Length-aware bound.  The blocks whose sums run over the B (A + 1) slot rows (every CQL block; the dueling advantage
blocks and, through the feature gradient, the trunk blocks) grow with that length instead of staying O(u).  Measured on
the same card: 6.9e-6 (CQL db2 at A 255, B 256: 65536 rows), 6.0e-6 (CQL dW2 at A 64, B 255: 16575 rows), 3.7e-6 (CQL
dW1a at A 17, B 4096: 73728 rows; dW1s 6.4e-7 and db1 4.2e-7 there and at A 255, summed per row over the slots and then
over the B rows), 4.3e-7 at 4335 rows.  The CQL term puts a same-sign gradient alpha p_k / B on every current slot, so these sums
do not cancel: their value is as large as their scale, and the fp32 accumulators (one serial sum per output in
k_fold_w1a_grad and per thread in the SIMT and wgmma tiles) make a random-walk error of about u sqrt(n) of the scale.
Those blocks are held to max(C, 2 u sqrt(B (A + 1))), u = 2^-24, twice that size; a pairwise or split-K reduction in
those kernels would bring them back to O(u).  The whole file ran in about 35 s on that card.
"""
import ctypes
from collections import namedtuple

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

C = 4e-7              # elementwise bound |kernel - fp64| <= C * scale (measured maximum 1.52e-7, see above)
U = 2.0 ** -24
# the blocks whose sums run over the B (A + 1) slot rows (directly, or through k_slot_rowsum and then the B rows)
SLOT_ROW_BLOCKS = {"dW1s", "dW1a", "db1", "dW2", "db2", "dW3", "db3", "dSW1", "dSb1", "dSW2", "dSb2", "dSW3", "dSb3",
                   "dAW1f", "dAW1a", "dAb1", "dAW2", "dAb2", "dAW3", "dAb3"}
MARGIN = 1e-6         # ReLU and next-action-gap margin of the accepted rows (must stay well above C)
GAMMA, TAU, ALPHA = 0.99, 0.3, 1.5
ENGINES = (0, 1, 2)

# ---------------------------------------------------------------------------------------------- the grid
# W (dueling only): (F, state_h1, state_h2, value_h1, value_h2, adv_h1, adv_h2); None: every MLP [H1, H2], F = H2
Case = namedtuple("Case", "kind obs A H1 H2 B double dynamic W")
CQL_GRID = [
    Case("cql", 1, 2, 1, 1, 1, False, False, None),
    Case("cql", 3, 3, 5, 3, 2, True, True, None),
    Case("cql", 127, 16, 64, 64, 255, False, True, None),
    Case("cql", 128, 17, 65, 63, 256, True, False, None),
    Case("cql", 257, 33, 129, 257, 5, False, True, None),
    Case("cql", 3, 255, 5, 3, 256, True, True, None),
    Case("cql", 1, 64, 129, 257, 255, False, False, None),
    Case("cql", 128, 2, 512, 512, 1024, True, True, None),
    Case("cql", 257, 3, 300, 300, 1024, False, True, None),
    Case("cql", 3, 17, 1, 1, 4096, True, True, None),
    Case("cql", 127, 64, 65, 63, 2, True, False, None),
    Case("cql", 127, 3, 640, 640, 64, True, False, None),
]
DUEL_GRID = [
    Case("duel", 1, 1, 1, 1, 1, False, False, None),
    Case("duel", 3, 3, 5, 3, 2, True, True, None),
    Case("duel", 127, 16, 64, 64, 255, False, True, None),
    Case("duel", 128, 17, 65, 63, 256, True, False, None),
    Case("duel", 257, 33, 129, 257, 5, False, True, None),
    Case("duel", 3, 255, 5, 3, 256, False, True, None),
    Case("duel", 1, 64, 129, 257, 255, False, False, None),
    Case("duel", 128, 1, 512, 512, 1024, True, False, None),
    Case("duel", 257, 3, 300, 300, 1024, False, True, None),
    Case("duel", 3, 3, 0, 0, 4096, True, True, (33, 65, 7, 129, 5, 63, 257)),
    Case("duel", 127, 64, 0, 0, 2, True, False, (7, 3, 5, 300, 2, 17, 9)),
    Case("duel", 127, 3, 640, 640, 64, True, False, None),
]
GRID = CQL_GRID + DUEL_GRID


def _cid(c):
    h = f"h{c.H1}x{c.H2}" if c.W is None else "w" + "-".join(map(str, c.W))
    return (f"{c.kind}-obs{c.obs}-A{c.A}-{h}-B{c.B}-{'ddqn' if c.double else 'dqn'}-"
            f"{'dyn' if c.dynamic else 'full'}")


GRID_IDS = [_cid(c) for c in GRID]
BATCH_GRID = [GRID[i] for i in (0, 1, 3, 5, 8, 12, 13, 14, 17, 21)]
Q_GRID = [GRID[i] for i in (0, 4, 6, 12, 16, 21)]


def widths(c) -> dict:
    """The prl_duel_cfg widths of a dueling case."""
    from oracle.dueling_fp64 import widths_of
    if c.W is None:
        return widths_of((c.H1, c.H2))
    return dict(zip(("feature_dim", "state_h1", "state_h2", "value_h1", "value_h2", "adv_h1", "adv_h2"), c.W))


# ---------------------------------------------------------------------------------------------- restated dispatch
# one contraction: op, output rows Mo, output columns No, contraction length Kc, and the (row pitch, float offset) of every
# operand the wgmma loader reads along its rows (gemm_tc.cu's XO operands: both of a forward, dy of a backward-data)
Prod = namedtuple("Prod", "op Mo No Kc pass_ xo")


def _fwd(M, N, K, x_ld, w_ld, w_off, pass_):
    return Prod("fwd", M, N, K, pass_, ((x_ld, 0), (w_ld, w_off)))


def _bwd_x(M, N, Kx, pass_):
    return Prod("bwd_x", M, Kx, N, pass_, ((N, 0),))


def _bwd_w(M, N, K, pass_):
    return Prod("bwd_w", N, K + 1, M, pass_, ())


def products(c):
    """Every contraction of one round of case `c` (cql_round / duel_round), in launch order."""
    O, A, B = c.obs, c.A, c.B
    BA, BA1 = B * A, B * (A + 1)
    out = []
    if c.kind == "cql":
        H1, H2, D = c.H1, c.H2, O + A
        oW2 = H1 * D + H1
        oW3 = oW2 + H2 * H1 + H2

        def pass_(M, name):
            return [_fwd(B, H1, O, O, D, 0, name), _fwd(M, H2, H1, H1, H1, oW2, name), _fwd(M, 1, H2, H2, H2, oW3, name)]
        out += pass_(BA1, "online")
        for _ in range(2 if c.double else 1):
            out += pass_(BA, "next")
        out += [_bwd_w(BA1, 1, H2, "bwd"), _bwd_w(BA1, H2, H1, "bwd"), _bwd_x(BA1, H2, H1, "bwd"), _bwd_w(B, H1, O, "bwd")]
        return out
    from oracle.dueling_fp64 import layout
    w = widths(c)
    F, sh1, sh2, vh1, vh2, ah1, ah2 = (w[k] for k in ("feature_dim", "state_h1", "state_h2", "value_h1", "value_h2",
                                                        "adv_h1", "adv_h2"))
    lay = layout(O, A, w)
    off = lambda name: lay[name][0]  # noqa: E731

    def duel_fwd(K, name):
        m = B
        return [_fwd(m, sh1, O, O, O, off("dSW1"), name), _fwd(m, sh2, sh1, sh1, sh1, off("dSW2"), name),
                _fwd(m, F, sh2, sh2, sh2, off("dSW3"), name), _fwd(m, vh1, F, F, F, off("dVW1"), name),
                _fwd(m, vh2, vh1, vh1, vh1, off("dVW2"), name), _fwd(m, 1, vh2, vh2, vh2, off("dVW3"), name),
                _fwd(m, ah1, F, F, F + A, off("dAW1f"), name), _fwd(m * K, ah2, ah1, ah1, ah1, off("dAW2"), name),
                _fwd(m * K, 1, ah2, ah2, ah2, off("dAW3"), name)]
    out += duel_fwd(A + 1, "online")
    for _ in range(2 if c.double else 1):
        out += duel_fwd(A, "next")
    out += [_bwd_w(BA1, 1, ah2, "bwd"), _bwd_w(BA1, ah2, ah1, "bwd"), _bwd_x(BA1, ah2, ah1, "bwd"), _bwd_w(B, ah1, F, "bwd"),
            _bwd_x(B, ah1, F, "bwd"),
            _bwd_w(B, 1, vh2, "bwd"), _bwd_w(B, vh2, vh1, "bwd"), _bwd_x(B, vh2, vh1, "bwd"), _bwd_w(B, vh1, F, "bwd"),
            _bwd_x(B, vh1, F, "bwd"),
            _bwd_w(B, F, sh2, "bwd"), _bwd_x(B, F, sh2, "bwd"), _bwd_w(B, sh2, sh1, "bwd"), _bwd_x(B, sh2, sh1, "bwd"),
            _bwd_w(B, sh1, O, "bwd")]
    return out


def kernel_of(p, engine):
    """gemm_tc_launch, then GemmLauncher::run: "tc64" / "tc32" or "simt_64x64" / "simt_32_ks4" / "simt_32_ks1"."""
    ao, bo = p.op != "bwd_w", p.op == "fwd"
    if engine != 0 and not (engine == 1 and p.Mo < 4096) and not (not ao and bo):
        return "tc64" if p.No > 32 else "tc32"
    if -(-p.Mo // 64) * -(-p.No // 64) >= 96:
        return "simt_64x64"
    return "simt_32_ks4" if p.Kc > 64 else "simt_32_ks1"


def branches(c, engine):
    """Names of the table's branches that one learn() of case `c` under `engine` reaches."""
    out = set()
    slot_rows = {"online": c.B * (c.A + 1), "next": c.B * c.A}
    on_tc = {"online": False, "next": False}          # a slot-expanded forward product of the pass runs on wgmma
    for p in products(c):
        k = kernel_of(p, engine)
        if k.startswith("simt"):
            out.add(f"{k}_{p.op}")
            continue
        if p.op == "fwd" and p.Mo == slot_rows[p.pass_]:
            on_tc[p.pass_] = True
        out.add("tc_tn64" if k == "tc64" else "tc_tn32")
        if p.Kc % 32:
            out.add("tc_edge_chunk")
        if any(ld % 4 or o % 4 for ld, o in p.xo):
            out.add("tc_scalar_loads")
        if p.Mo % 128:
            out.add("tc_ragged_rows")
    if engine == 1 and on_tc["online"] and not on_tc["next"]:
        out.add("mixed_round")
    if c.A > 32:
        out.add("slot_loop")
    if c.A == 255 and c.dynamic:
        out.add("byte_ids_high")
    if c.A == (2 if c.kind == "cql" else 1):
        out.add("a_min")
    if c.double:
        out.add("double")
    if c.dynamic:
        out.add("dynamic")
    if c.B == 1:
        out.add("one_row")
    if c.W is not None and len(set(c.W)) == 7 and c.W[0] % 2:
        out.add("independent_widths")
    return out


ALL_BRANCHES = {line.split("|")[1].strip() for line in __doc__.splitlines()
                if line.startswith("| ") and not line.startswith("| branch")}
BATCH_BRANCHES = {"padded_current_sets", "query_alone"}


# ---------------------------------------------------------------------------------------------- helpers
class _Space:
    def __init__(self, n):
        self.n = n
        self.actions = [torch.tensor([i]) for i in range(n)]
        self.actions_batch = torch.arange(n).view(n, 1)


def _seed(c, extra=0):
    return (c.obs * 7919 + c.A * 104729 + c.H1 * 31 + c.H2 * 17 + int(c.double) * 5 + int(c.dynamic) * 3
            + (sum(c.W) * 13 if c.W else 0) + (1 if c.kind == "duel" else 0) * 99991 + extra) % (2 ** 31)


def _learner(c, seed, *, freq=1000, B=None):
    import pearl_b200
    torch.manual_seed(seed)
    cls = pearl_b200.B200DoubleDQN if c.double else pearl_b200.B200DeepQLearning
    kw = dict(state_dim=c.obs, action_space=_Space(c.A), learning_rate=1e-3, discount_factor=GAMMA, training_rounds=1,
              batch_size=c.B if B is None else B, target_update_freq=freq, soft_update_tau=TAU,
              action_representation_module=pearl_b200.OneHotActionTensorRepresentationModule(c.A))
    if c.kind == "cql":
        pl = cls(hidden_dims=[c.H1, c.H2], is_conservative=True, conservative_alpha=ALPHA, **kw)
    elif c.W is None:
        pl = cls(hidden_dims=[c.H1, c.H2], network_type=pearl_b200.DuelingQValueNetwork, **kw)
    else:
        w = widths(c)
        net = pearl_b200.DuelingQValueNetwork(
            state_dim=c.obs, action_dim=c.A, hidden_dims=[w["state_h1"], w["feature_dim"]], output_dim=1,
            state_hidden_dims=[w["state_h1"], w["state_h2"]], value_hidden_dims=[w["value_h1"], w["value_h2"]],
            advantage_hidden_dims=[w["adv_h1"], w["adv_h2"]])
        pl = cls(hidden_dims=[w["state_h1"], w["feature_dim"]], network_instance=net, **kw)
    pl = pl.to("cuda")
    with torch.no_grad():
        for p in pl._Q_target.parameters():
            p.add_(0.05 * torch.randn(p.shape, device=p.device))
    return pl


def _fns(c):
    """(margin_fn, gap_fn) of make_data for the case's network."""
    if c.kind == "cql":
        return None, None
    from oracle import dueling_fp64 as d
    w = widths(c)
    return (lambda w_, s, a: d.relu_margin(w_, s, a, c.obs, c.A, w),
            lambda w_, s, ids, n: d.next_action_gap(w_, s, ids, n, c.obs, c.A, w))


def _data(pl, c, seed, dynamic=None):
    from oracle.dqn_fp64 import make_data
    dynamic = c.dynamic if dynamic is None else dynamic
    mf, gf = _fns(c)
    d = make_data(pl.flat_parameters.detach().clone(), c.obs, c.A, c.B, seed, dynamic, MARGIN,
                  hidden=(c.H1, c.H2), double=c.double, all_slots=True, margin_fn=mf, gap_fn=gf)
    if dynamic:   # the available ids in random order (the slot order is not the id order)
        rng = np.random.default_rng(seed + 1)
        ids = d["avail_ids"].numpy().copy()
        for i, k in enumerate(d["avail_n"].numpy()):
            ids[i, :k] = rng.permutation(ids[i, :k])
        d["avail_ids"] = torch.from_numpy(ids)
    return d


def _buffer(data, c, seed):
    import pearl_b200
    buf = pearl_b200.B200ReplayBuffer(data["state"].shape[0], rng="device", dynamic_action_space=c.dynamic)
    kw = {}
    if c.dynamic:
        kw = dict(next_available_ids=data["avail_ids"].to(torch.uint8), next_available_count=data["avail_n"].to(torch.int32))
    buf.push_batch(data["state"], data["action"].to(torch.int32), data["reward"], data["next_state"],
                   data["terminated"], data["truncated"], max_number_actions=c.A, **kw)
    buf.seed(seed)
    return buf


def _bound(c, block=None):
    """C, or for a block summed over the B (A + 1) slot rows the length-aware bound of the module docstring."""
    return max(C, 2 * U * (c.B * (c.A + 1)) ** 0.5) if block in SLOT_ROW_BLOCKS else C


def _step(c, w0, wt, batch, curr_ids=None, query_alone=False):
    from oracle import dueling_fp64
    from oracle.dqn_fp64 import cql_step
    dev = w0.device
    if c.kind == "cql":
        return cql_step(w0.double(), wt.double().to(dev), batch, c.obs, c.A, GAMMA, ALPHA, hidden=(c.H1, c.H2),
                        double=c.double, curr_ids=curr_ids)
    return dueling_fp64.dueling_step(w0.double(), wt.double().to(dev), batch, c.obs, c.A, GAMMA, widths(c),
                                     double=c.double, curr_ids=curr_ids, query_alone=query_alone)


def _blocks(c):
    from oracle import dqn_fp64, dueling_fp64
    if c.kind == "cql":
        return dqn_fp64.BLOCKS, lambda g, n: dqn_fp64.block_view(g, n, c.obs, c.A, (c.H1, c.H2))
    return dueling_fp64.BLOCKS, lambda g, n: dueling_fp64.block_view(g, n, c.obs, c.A, widths(c))


def _check_step(c, pl, w0, wt, batch, loss, tag, curr_ids=None, query_alone=False):
    """The loss and every gradient block (from exp_avg after one step from zero moments) within C x scale of the fp64
    step; exp_avg_sq, max_exp_avg_sq and the parameters equal AdamW applied in fp64 to that gradient."""
    from oracle.dqn_fp64 import check
    hp = pl._adam_hparams()
    val, sc = _step(c, w0, wt, batch, curr_ids, query_alone)
    worst = {}
    bound = _bound(c)
    check("loss", torch.tensor(loss), val["mae"], sc["mae"], worst, bound)
    st = pl.adam_state()
    assert st["step"] == 1
    m, v, vmax = st["exp_avg"], st["exp_avg_sq"], st["max_exp_avg_sq"]
    g = m / torch.tensor(1.0 - hp["beta1"], dtype=torch.float32, device=m.device)
    names, view = _blocks(c)
    for name in names:
        gb = view(g, name)
        check(name, gb, val[name].reshape(gb.shape), sc[name].reshape(gb.shape), worst, _bound(c, name))
    print(f"    MAXERR {_cid(c)}{tag} " + " ".join(f"{k}={e:.2e}" for k, e in worst.items()))
    g64, m64, w64 = g.double(), m.double(), w0.double()
    v_want = (1.0 - hp["beta2"]) * g64 * g64
    # g * g of a cancelled gradient element (say the dueling advantage net at A = 1) can be a subnormal float
    assert float(((v.double() - v_want).abs() - 1e-6 * v_want - 2.0 ** -126).max()) <= 0, "exp_avg_sq"
    assert torch.equal(vmax, v), "max_exp_avg_sq after the first step"
    bc1, bc2 = 1.0 - hp["beta1"], 1.0 - hp["beta2"]
    w_want = w64 * (1.0 - hp["lr"] * hp["weight_decay"]) - hp["lr"] / bc1 * m64 / ((vmax.double() / bc2).sqrt() + hp["eps"])
    err = (pl.flat_parameters.double() - w_want).abs() - (3e-7 * w64.abs() + 1e-5 * hp["lr"])
    assert float(err.max()) <= 0, f"AdamW update of parameter {int(err.argmax())}"
    return worst


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


def _soft_update_f32(w, t):
    """k_soft_update_flagged in fp32: fl(fl(tau w) + fl((1 - tau) t)), tau and 1 - tau rounded from double."""
    tau, omtau = torch.tensor(TAU, dtype=torch.float32), torch.tensor(1.0 - TAU, dtype=torch.float32)
    return (tau.to(w.device) * w) + (omtau.to(w.device) * t)


# ---------------------------------------------------------------------------------------------- coverage
def test_grid_reaches_every_branch():
    """Together the cases (under the three engines) and the learn_batch subset reach every branch of the table above,
    and every value of each axis appears."""
    reached = {}
    for c in GRID:
        for e in ENGINES:
            for b in branches(c, e):
                reached.setdefault(b, []).append(f"{_cid(c)} engine {e}")
    reached["flagged_update"] = [_cid(c) for c in GRID]                          # every case runs freq 1
    reached["padded_current_sets"] = [_cid(c) for c in BATCH_GRID]
    reached["query_alone"] = [_cid(c) for c in BATCH_GRID if c.kind == "duel"]
    for b in sorted(ALL_BRANCHES):
        print(f"    {b}: {len(reached.get(b, []))} runs, e.g. {reached.get(b, ['-'])[0]}")
    assert not ALL_BRANCHES - set(reached), f"branches no case reaches: {sorted(ALL_BRANCHES - set(reached))}"
    assert len(ALL_BRANCHES) == 25
    for kind, grid in (("cql", CQL_GRID), ("duel", DUEL_GRID)):
        k_reached = set()
        for c in grid:
            for e in ENGINES:
                k_reached |= branches(c, e)
        missing = ALL_BRANCHES - BATCH_BRANCHES - {"flagged_update"} - k_reached - ({"independent_widths"} if kind == "cql" else set())
        assert not missing, f"{kind}: {sorted(missing)}"
        assert {1, 3, 127, 128, 257} <= {c.obs for c in grid}
        assert ({2} if kind == "cql" else {1}) | {3, 16, 17, 33, 64, 255} <= {c.A for c in grid}
        assert {(1, 1), (5, 3), (64, 64), (65, 63), (129, 257), (300, 300), (512, 512)} <= {(c.H1, c.H2) for c in grid}
        assert {1, 2, 5, 255, 256, 1024, 4096} <= {c.B for c in grid}
        assert {(d, y) for d in (False, True) for y in (False, True)} <= {(c.double, c.dynamic) for c in grid}
    assert any(c.kind == "cql" and c.A == 2 for c in BATCH_GRID) and any(c.kind == "duel" and c.A == 1 for c in BATCH_GRID)
    for c in GRID:   # the largest slot-expanded array of the grid stays a few hundred MB
        rows = c.B * (c.A + 1)
        width = max(c.H1, c.H2) if c.W is None else max(c.W)
        assert rows * width * 4 <= 300 * 2 ** 20, _cid(c)


# ---------------------------------------------------------------------------------------------- a. one learn()
@pytest.mark.parametrize("case", GRID, ids=GRID_IDS)
def test_one_round_gradient_matches_fp64(case):
    """One learn() from a ring, without (freq 1000) and with (freq 1) the soft update before the step, under
    contraction engines 0, 1 and 2: loss, every gradient block, the AdamW moments and parameters, and the target."""
    c = case
    data = {}
    for engine in ENGINES:
        with _Engine(engine):
            for freq in (1000, 1):
                seed = _seed(c, freq)
                pl = _learner(c, seed, freq=freq)       # the same initial networks under every engine
                if freq not in data:
                    data[freq] = _data(pl, c, seed)
                buf = _buffer(data[freq], c, seed)
                w0, wt0 = pl.flat_parameters.clone(), pl.flat_target_parameters.clone()
                rep = pl.learn(buf, trace=True)
                wt = pl.flat_target_parameters
                if freq == 1:    # the update precedes the step, with the parameters before it
                    assert torch.equal(wt, _soft_update_f32(w0, wt0)), "soft target update"
                else:
                    assert torch.equal(wt, wt0), "the target moved without a scheduled update"
                idx = rep["idx"][0].long().cpu()
                batch = {k: v[idx] for k, v in data[freq].items()}
                _check_step(c, pl, w0, wt.clone(), batch, rep["loss"][0], f" engine={engine} freq={freq}")
                del pl, buf


# ---------------------------------------------------------------------------------------------- b. learn_batch
def _learn_batch_data(pl, c, seed):
    """B rows of the case with partial current sets padded with id 0, and next sets given as a random permutation of
    every id with a random non-prefix unavailable mask (at least one available per row).  Returns (rows, current ids,
    permuted ids, mask, ids compacted with the available ones first, available count)."""
    d = _data(pl, c, seed, dynamic=False)
    n, A, B = d["state"].shape[0], c.A, c.B
    rng = np.random.default_rng(seed)
    perm = np.stack([rng.permutation(A) for _ in range(n)])
    mask = rng.random((n, A)) < 0.4
    mask[np.arange(n), rng.integers(0, A, n)] = False
    comp = np.stack([np.concatenate([perm[i][~mask[i]], perm[i][mask[i]]]) for i in range(n)])
    cnt = (~mask).sum(1)
    curr = np.zeros((n, A), np.int64)
    for i in range(n):
        m = int(rng.integers(1, A + 1))
        curr[i, :m] = rng.permutation(rng.choice(A, m, replace=False))
    keep = np.arange(n)
    if c.double:
        _, gap_fn = _fns(c)
        w = pl.flat_parameters.detach().clone()
        if gap_fn is None:
            from oracle.dqn_fp64 import next_action_gap
            gap = next_action_gap(w, d["next_state"], comp, cnt, c.obs, A, (c.H1, c.H2))
        else:
            gap = gap_fn(w, d["next_state"], comp, cnt)
        keep = np.flatnonzero((gap >= MARGIN).numpy())
    keep = keep[:B]
    assert keep.size == B, "too few rows clear the next-action gap"
    return {k: v[keep] for k, v in d.items()}, curr[keep], perm[keep], mask[keep], comp[keep], cnt[keep]


@pytest.mark.parametrize("case", BATCH_GRID, ids=[_cid(c) for c in BATCH_GRID])
def test_learn_batch_matches_fp64(case):
    """learn_batch with partial padded current sets (raw ids and one-hot), non-prefix next masks over permuted ids,
    and for dueling no current sets (the query-alone mean), under engines 1 and 2: the fp64 step on the same rows."""
    import pearl_b200
    c = case
    seed = _seed(c, 11)
    A = c.A
    modes = [("ids", True), ("one_hot", True)] + ([("ids", False)] if c.kind == "duel" else [])
    for engine in (1, 2):
        with _Engine(engine):
            for form, with_curr in modes:
                if form == "one_hot" and A == 1:
                    continue   # a one-hot column of width 1 reads as the id 1
                pl = _learner(c, seed)
                rows, curr, perm, mask, comp, cnt = _learn_batch_data(pl, c, seed)
                eye = torch.eye(A)
                t = torch.from_numpy
                if form == "ids":
                    act, cur, nxt = rows["action"].view(-1, 1), t(curr).float().unsqueeze(-1), t(perm).float().unsqueeze(-1)
                else:
                    act, cur, nxt = eye[rows["action"]], eye[t(curr)], eye[t(perm)]
                tb = pearl_b200.TransitionBatch(state=rows["state"], action=act, reward=rows["reward"],
                                                next_state=rows["next_state"], terminated=rows["terminated"],
                                                curr_available_actions=cur if with_curr else None,
                                                next_available_actions=nxt, next_unavailable_actions_mask=t(mask))
                w0, wt0 = pl.flat_parameters.clone(), pl.flat_target_parameters.clone()
                rep = pl.learn_batch(tb)
                assert torch.equal(pl.flat_target_parameters, wt0)
                batch = dict(rows, avail_ids=t(comp), avail_n=t(cnt))
                _check_step(c, pl, w0, wt0, batch, rep["loss"], f" learn_batch engine={engine} {form} "
                            f"{'curr' if with_curr else 'no-curr'}", curr_ids=curr if with_curr else None,
                            query_alone=not with_curr)
                del pl


# ---------------------------------------------------------------------------------------------- c. q_values
@pytest.mark.parametrize("case", Q_GRID, ids=[_cid(c) for c in Q_GRID])
def test_q_values_match_fp64(case):
    """q_values for 1, 3, 5 and 1000 rows, online and target, against fp64; for dueling also over caller id sets
    (the advantage mean over each row's set)."""
    from oracle import dueling_fp64
    from oracle.dqn_fp64 import check, q_values
    from pearl_b200 import dueling
    c = case
    seed = _seed(c, 13)
    pl = _learner(c, seed, B=min(c.B, 256))
    pl.learn_batch(pearl_batch(c, seed))            # the chunks run through a bound workspace (max_batch rows)
    w, wt = pl.flat_parameters.clone(), pl.flat_target_parameters.clone()
    rng = np.random.default_rng(seed + 2)
    worst = {}
    for nrows in (1, 3, 5, 1000):
        s = torch.from_numpy(np.rint(rng.standard_normal((nrows, c.obs)) * 256) / 256).float()
        for target, p in ((False, w), (True, wt)):
            if c.kind == "cql":
                want, scale = q_values(p.double(), s, c.obs, c.A, (c.H1, c.H2))
                check(f"q_values[{nrows}, target={target}]", pl.q_values(s, target=target), want, scale, worst, C)
                continue
            want, scale = dueling_fp64.q_values(p.double(), s, c.obs, c.A, widths(c))
            check(f"q_values[{nrows}, target={target}]", pl.q_values(s, target=target), want, scale, worst, C)
            K = min(c.A + 1, 3)
            ids = torch.from_numpy(rng.integers(0, c.A, (nrows, K)))
            want, scale = dueling_fp64.q_values(p.double(), s, c.obs, c.A, widths(c), ids)
            got = dueling.q_values(pl, s, target, ids)
            check(f"q_values[{nrows}, ids K={K}, target={target}]", got, want, scale, worst, C)
    print(f"    MAXERR {_cid(c)} q_values " + " ".join(f"{k}={e:.2e}" for k, e in worst.items()))


def pearl_batch(c, seed):
    """A small learn_batch input of the case (every action current, every next action available)."""
    import pearl_b200
    rng = np.random.default_rng(seed)
    B = min(c.B, 256)
    q8 = lambda x: torch.from_numpy(np.rint(x * 256) / 256).float()  # noqa: E731
    return pearl_b200.TransitionBatch(state=q8(rng.standard_normal((B, c.obs))),
                                      action=torch.from_numpy(rng.integers(0, c.A, (B, 1))),
                                      reward=q8(rng.standard_normal(B)), next_state=q8(rng.standard_normal((B, c.obs))),
                                      terminated=torch.from_numpy(rng.random(B) < 0.2))


# ---------------------------------------------------------------------------------------------- d. size limit
@pytest.mark.parametrize("kind", ["cql", "duel"])
def test_bind_refuses_shapes_past_32_bit_offsets(kind):
    """batch 8192, 255 actions and a slot-expanded width of 1024 put 2^31 elements in one activation array (about 32 GB
    of workspace): binding such a learner raises ValueError naming the limit before anything is allocated or launched,
    and leaves no handle; one row less passes the same check (param_count / workspace_bytes), without allocating."""
    import pearl_b200
    from pearl_b200 import _lib
    A, B = 255, 8192
    c = Case(kind, 4, A, 1024, 1024, B, False, False, None)
    pl = _learner(c, 1)
    torch.cuda.synchronize()
    before = torch.cuda.memory_allocated()
    with pytest.raises(ValueError, match="2\\^31"):
        pl._bind(B)
    torch.cuda.synchronize()
    assert torch.cuda.memory_allocated() == before, "the refused bind allocated device memory"
    assert not pl._handle.value
    hp = pl._adam_hparams()
    mod = pearl_b200.cql if kind == "cql" else pearl_b200.dueling
    lib = _lib.load()
    for batch, ok in ((B - 1, True), (B, False)):
        cfg = mod.make_cfg(pl, hp, batch)
        ws = (lib.prl_cql_workspace_bytes if kind == "cql" else lib.prl_duel_workspace_bytes)(ctypes.byref(cfg))
        assert (ws > 0) == ok, (batch, _lib.last_error())
