"""The multi-head DQN learner (csrc/multihead.cu) across its shape space against float64 gradients (oracle/multihead_fp64.py).

One learn_batch step from zero AdamW moments leaves exp_avg = fl(fl(1 - beta1) g), so the kernel's fp32 gradient g is
recovered from the first moment to within 2^-24 relative, and held elementwise to the float64 gradient of the same batch:

    |g_kernel - g_fp64| <= (C + B * U / 32) * scale,    U = 2^-24

where scale is the sum of |a||b| over every product that contributed (the float64 code applied to |.| of every operand).
C = 4e-7 covers the fp32 rounding of the chain of dot products (a few units of U) and the recovery (U).  The second term
covers the weight-gradient contractions over the B rows: their rounding error grows with B, slowly under the SIMT tiles
(about sqrt(B) U) and linearly, at a small rate, under the tensor-core tiles, whose fp32 accumulation over long
contraction axes loses more than round-to-nearest would.  Largest err / scale seen on an H100 80GB HBM3 (700 W) over this
grid: 2.2e-7 up to batch 512; 6.2e-7 at batch 1000 (engine 2); 2.2e-6 at batch 4096 (engine 2); 2.0e-6 (engine 0) and
3.7e-5 (engine 2) at batch 65536, where B U / 32 = 1.2e-4.
Rows whose ReLU pre-activations, or DoubleDQN's best two next values, lie within MARGIN of their scale are not drawn
(dqn_fp64.make_data), since a last-bit difference could flip them.

The grid covers A from 1 to 255, hidden widths from (1, 1) to (512, 512), batch from 1 to 65536, DQN, DoubleDQN and the
conservative variants with partial current sets that repeat the padding id, under the SIMT (0) and tensor-core (2)
contraction engines; the configured maxima themselves are checked on the host (a batch past the 32-bit limit is refused).
"""
import numpy as np
import pytest
import torch

from oracle.multihead_fp64 import check, make_data, mh_step, next_action_gap, relu_margin

pytestmark = pytest.mark.gpu

C = 4e-7
U = 2.0 ** -24
MARGIN = 1e-6
OMB1 = float(np.float32(1.0 - 0.9))

# (obs, A, (h1, h2), B, double, alpha, dynamic)
GRID = [
    (3, 1, (1, 1), 1, False, None, False),
    (4, 1, (64, 64), 128, True, None, False),
    (4, 2, (64, 64), 128, False, 2.0, False),
    (9, 255, (32, 48), 64, True, None, True),
    (5, 255, (16, 16), 32, True, 8.0, True),
    (128, 16, (256, 256), 256, False, 2.0, True),
    (128, 16, (256, 256), 256, True, None, True),
    (33, 7, (512, 512), 512, True, 0.5, True),
    (6, 3, (1, 7), 1000, False, None, False),
    (17, 5, (512, 512), 64, False, 4.0, False),
    (2, 2, (1, 1), 65536, False, None, False),
    (12, 33, (17, 129), 4096, True, 1.0, False),
]
IDS = [f"obs{o}-A{a}-h{h[0]}x{h[1]}-B{b}-{'ddqn' if d else 'dqn'}{'-cql' if al is not None else ''}{'-dyn' if dy else ''}"
       for o, a, h, b, d, al, dy in GRID]


def _space(A):
    class Space:
        n = A
        actions = [torch.tensor([i]) for i in range(A)]
        actions_batch = torch.arange(A).view(A, 1)
    return Space()


def _curr_ids(B, A, seed):
    """Partial current sets padded with id 0: slot k < m holds a sorted subset, the rest repeat 0."""
    rng = np.random.default_rng(seed)
    ids = np.zeros((B, A), np.int64)
    for i in range(B):
        m = int(rng.integers(1, A + 1))
        ids[i, :m] = np.sort(rng.choice(A, size=m, replace=False))
    return ids


@pytest.mark.parametrize("engine", [0, 2])
@pytest.mark.parametrize("case", GRID, ids=IDS)
def test_one_step_gradient_matches_fp64(case, engine):
    import pearl_b200
    from pearl_b200 import TransitionBatch, _lib
    obs, A, hidden, B, double, alpha, dynamic = case
    torch.manual_seed(B + A)
    cls = pearl_b200.B200DoubleDQN if double else pearl_b200.B200DeepQLearning
    cons = dict(is_conservative=True, conservative_alpha=alpha) if alpha is not None else {}
    pl = cls(state_dim=obs, action_space=_space(A), hidden_dims=list(hidden), batch_size=B, target_update_freq=1000,
             network_type=pearl_b200.VanillaQValueMultiHeadNetwork,
             action_representation_module=pearl_b200.OneHotActionTensorRepresentationModule(A), **cons).to("cuda:0")
    with torch.no_grad():                                  # a target that differs from the online net
        for p in pl._Q_target.parameters():
            p.mul_(0.9)
    w0 = torch.cat([p.detach().reshape(-1) for p in pl._Q.parameters()]).cuda()
    wt = torch.cat([p.detach().reshape(-1) for p in pl._Q_target.parameters()]).cuda()
    d = make_data(w0, obs, A, B, seed=7 * B + A, dynamic=dynamic, margin=MARGIN, hidden=hidden, double=double,
                  margin_fn=lambda w, s, a: relu_margin(w, s, obs, A, hidden),
                  gap_fn=lambda w, s, ids, n: next_action_gap(w, s, ids, n, obs, A, hidden))
    d = {k: v[:B] for k, v in d.items()}
    curr = _curr_ids(B, A, B) if alpha is not None else None
    mask = torch.arange(A).view(1, A) >= d["avail_n"].view(-1, 1)
    batch = TransitionBatch(state=d["state"], action=d["action"].view(-1, 1), reward=d["reward"], next_state=d["next_state"],
                            terminated=d["terminated"], next_available_actions=d["avail_ids"].view(B, A, 1).float(),
                            next_unavailable_actions_mask=mask,
                            curr_available_actions=None if curr is None else torch.from_numpy(curr).view(B, A, 1).float())
    lib = _lib.load()
    prev = lib.prl_get_contraction_engine()
    _lib.check(lib.prl_set_contraction_engine(engine))
    try:
        rep = pl.learn_batch(batch)
    finally:
        _lib.check(lib.prl_set_contraction_engine(prev))
    got = pl.adam_state()["exp_avg"].double() / OMB1
    value, scale = mh_step(w0, wt, d, obs, A, 0.99, hidden, double=double, alpha=alpha, curr_ids=curr)
    worst, bound = {}, C + B * U / 32
    check("grad", got, value["grad"], scale["grad"], worst, bound)
    check("loss", torch.tensor(rep["loss"]), value["mae"], scale["mae"], worst, bound)
    print(f"    max err / scale: {worst} (bound {bound:.2e})")

