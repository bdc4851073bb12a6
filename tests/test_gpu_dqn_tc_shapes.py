"""The tensor-core DQN learner (k_dqn_tc, pearl_b200/csrc/dqn_tc.cu) over its whole supported shape class: hidden
[64, 64], obs in {8, 16, ..., 128} (multiples of 8), n_actions in {1, 2, 4, 8, 16}, batch 128 or 256, DQN.

The yardstick is the float64 step of oracle/dqn_fp64.py.  After ONE AdamW step from zero moments exp_avg = fl(0.1 g), so
exp_avg / 0.1f returns every gradient element to within an ulp, and the seven gradient blocks (dW1s, dW1a, db1, dW2,
db2, dW3, db3) are compared element by element with their fp64 values, within C times their error scale (sum of |a||b|
over the chain, see the oracle).  The data of every case is built so that such a check is sharp:

- the target network is perturbed away from the online one (a phase that reads the wrong network shows);
- about 20 % of the rows are terminal and some are truncated (truncation must not matter);
- a row enters the buffer only if every pre-activation of the online network is at least MARGIN of its scale away from
  zero, so a 3xTF32 rounding cannot flip a ReLU derivative (the target net needs no filter: ReLU and max are continuous);
- the buffer holds about 2 B rows, so a batch is a strict subset, gathered by the traced indices;
- half of the shapes (chosen deterministically) store a dynamic next-action set per row.

C is set from the largest max |err| / scale over the whole grid, both update frequencies and every block, measured on
an H100 SXM (80 GB HBM3, 700 W power limit): 5.25e-8 (dW1a at obs 8, A 16, B 128; the other blocks: dW2 3.5e-8, y
2.2e-8, q 1.8e-8, db2 1.4e-8, dW1s 1.1e-8, db1 6e-9, loss 3.4e-9, db3 2.1e-9, dW3 5.4e-10).  C = 2e-7 is under four times
that, and a single weight-gradient product issued without its lo terms (1xTF32) already misses it by more than 50x.  The
whole file ran in about a minute on that machine.
"""
import numpy as np
import pytest
import torch

from _tol import close, close_params

pytestmark = pytest.mark.gpu

OBS = (8, 16, 24, 32, 40, 56, 64, 72, 80, 96, 120, 128)
ACTS = (1, 2, 4, 8, 16)
BATCHES = (128, 256)
GRID = [(o, a, b) for o in OBS for a in ACTS for b in BATCHES]
GRID_IDS = [f"obs{o}-A{a}-B{b}" for o, a, b in GRID]
C = 2e-7              # elementwise bound |kernel - fp64| <= C * scale (measured maximum 5.25e-8, see above)
MARGIN = 2e-5         # ReLU margin of the accepted rows (must stay well above C)
GAMMA = 0.99
BLOCKS = ("dW1s", "dW1a", "db1", "dW2", "db2", "dW3", "db3")


class _Space:
    def __init__(self, n):
        self.n = n
        self.actions = [torch.tensor([i]) for i in range(n)]

    @property
    def actions_batch(self):
        return torch.stack(self.actions)


def _seed(obs, A, B):
    return obs * 1000 + A * 10 + B // 128


def _dynamic(obs, A, B):
    return (OBS.index(obs) + ACTS.index(A) + BATCHES.index(B)) % 2 == 1


def _learner(obs, A, B, seed, *, freq=1000, tau=0.5, rounds=1, per_call=4096, cls=None, hidden=(64, 64)):
    """A tensor-core learner whose target network differs from the online one."""
    import pearl_b200
    torch.manual_seed(seed)
    cls = cls or pearl_b200.B200DeepQLearning
    learner = cls(state_dim=obs, action_space=_Space(A), hidden_dims=list(hidden), learning_rate=1e-3,
                  discount_factor=GAMMA, training_rounds=rounds, batch_size=B, target_update_freq=freq,
                  soft_update_tau=tau, max_rounds_per_call=per_call, engine="tc",
                  action_representation_module=pearl_b200.OneHotActionTensorRepresentationModule(A)).to("cuda")
    with torch.no_grad():
        for p in learner._Q_target.parameters():
            p.add_(0.05 * torch.randn(p.shape, device=p.device))
    return learner


def _data(learner, obs, A, B, seed, dynamic):
    """About 2 B transitions whose online pre-activations all clear MARGIN (host tensors, push order)."""
    from oracle.dqn_fp64 import make_data
    from oracle.pearl_oracle import flat
    return make_data(flat(learner._Q).cpu(), obs, A, B, seed, dynamic, MARGIN)


def _buffer(data, A, seed, dynamic, dynamic_layout=None):
    import pearl_b200
    n = data["state"].shape[0]
    buf = pearl_b200.B200ReplayBuffer(n, rng="device", dynamic_action_space=dynamic if dynamic_layout is None else dynamic_layout)
    kw = {}
    if dynamic:
        kw = dict(next_available_ids=data["avail_ids"].to(torch.uint8), next_available_count=data["avail_n"].to(torch.int32))
    buf.push_batch(data["state"], data["action"].to(torch.int32), data["reward"], data["next_state"], data["terminated"],
                   data["truncated"], max_number_actions=A, **kw)
    buf.seed(seed)
    return buf


def _setup(obs, A, B, **kw):
    seed = _seed(obs, A, B) + kw.pop("seed_offset", 0)
    dynamic = _dynamic(obs, A, B)
    learner = _learner(obs, A, B, seed, **kw)
    data = _data(learner, obs, A, B, seed, dynamic)
    return learner, _buffer(data, A, seed, dynamic), data


def _check(what, got, want, scale, worst):
    from oracle.dqn_fp64 import check
    check(what, got, want, scale, worst, C)


# --------------------------------------------------------------------------- a. one-step gradient, whole class
@pytest.mark.parametrize("obs,A,B", GRID, ids=GRID_IDS)
def test_one_step_gradient_matches_fp64(obs, A, B):
    """One gradient step: q, y, the reported loss, and every element of the seven gradient blocks (recovered from
    exp_avg) within C x scale of fp64; exp_avg_sq, max_exp_avg_sq and the updated parameters equal AdamW applied in
    fp64 to the recovered gradient.  target_update_freq 2 puts a soft update before the step (its result is checked
    too), 1000 none."""
    from oracle.dqn_fp64 import block_view, dqn_step
    for freq in (1000, 2):
        learner, buf, data = _setup(obs, A, B, freq=freq, tau=0.3, seed_offset=freq)
        hp = learner._adam_hparams()
        w0, wt0 = learner.flat_parameters.clone(), learner.flat_target_parameters.clone()
        rep = learner.learn(buf, trace=True)
        wt = learner.flat_target_parameters.double().cpu()
        if freq == 2:   # (training_steps + 1) % freq == 0 at the first step: tau w + (1 - tau) w_target, in fp32
            want_t = 0.3 * w0.double().cpu() + 0.7 * wt0.double().cpu()
            scale_t = 0.3 * w0.double().abs().cpu() + 0.7 * wt0.double().abs().cpu()
            assert float(((wt - want_t).abs() - 2.0 ** -21 * scale_t).max()) <= 0, "soft target update"
        else:
            assert torch.equal(learner.flat_target_parameters, wt0), "the target moved without a scheduled update"
        idx = rep["idx"][0].long().cpu()
        batch = {k: v[idx] for k, v in data.items()}
        val, sc = dqn_step(w0.cpu(), wt, batch, obs, A, GAMMA)
        worst = {}
        _check("q", rep["q"][0], val["q"], sc["q"], worst)
        _check("y", rep["y"][0], val["y"], sc["y"], worst)
        _check("loss", torch.tensor(rep["loss"][0]), val["mae"], sc["mae"], worst)

        st = learner.adam_state()
        assert st["step"] == 1
        m, v, vmax = st["exp_avg"], st["exp_avg_sq"], st["max_exp_avg_sq"]
        g = (m / torch.tensor(1.0 - hp["beta1"], dtype=torch.float32, device=m.device)).cpu()
        for name in BLOCKS:
            _check(name, block_view(g, name, obs, A), val[name].reshape(block_view(g, name, obs, A).shape),
                   sc[name].reshape(block_view(g, name, obs, A).shape), worst)
        print(f"    MAXERR obs={obs} A={A} B={B} freq={freq} " + " ".join(f"{k}={e:.2e}" for k, e in worst.items()))

        # AdamW in fp64 on the recovered gradient (first step: bias corrections 1 - beta^1)
        g64, m64, w64 = g.double(), m.double().cpu(), w0.double().cpu()
        v_want = (1.0 - hp["beta2"]) * g64 * g64
        assert float(((v.double().cpu() - v_want).abs() - 1e-6 * v_want).max()) <= 0, "exp_avg_sq"
        assert torch.equal(vmax, v), "max_exp_avg_sq after the first step"
        bc1, bc2 = 1.0 - hp["beta1"], 1.0 - hp["beta2"]
        w_want = w64 * (1.0 - hp["lr"] * hp["weight_decay"]) - hp["lr"] / bc1 * m64 / (
            (vmax.double().cpu() / bc2).sqrt() + hp["eps"])
        err = (learner.flat_parameters.double().cpu() - w_want).abs() - (3e-7 * w64.abs() + 1e-5 * hp["lr"])
        assert float(err.max()) <= 0, f"AdamW update of parameter {int(err.argmax())}"


# --------------------------------------------------------------------------- b. tile coherence, whole class
@pytest.mark.parametrize("obs,A,B", GRID, ids=GRID_IDS)
def test_tiles_coherent_within_a_launch(obs, A, B):
    """7 rounds in one launch vs 7 one-round calls: inside a launch the operand-layout weight tiles come from AdamW's
    tile writes (or the rebuild after the scalar sweep when obs + A is not a multiple of 4) and the tile-order soft
    update; at a call boundary they are rebuilt from the flat vectors.  Same arithmetic either way, so losses,
    parameters, target parameters and the AdamW moments must be bit-identical.  Soft updates (freq 3, tau 0.5) land
    inside both."""
    out = []
    for per_call in (7, 1):
        learner, buf, _ = _setup(obs, A, B, freq=3, tau=0.5, rounds=7, per_call=per_call)
        rep = learner.learn(buf)
        st = learner.adam_state()
        out.append((rep["loss"], learner.flat_parameters.clone(), learner.flat_target_parameters.clone(),
                    st["exp_avg"].clone(), st["exp_avg_sq"].clone(), st["max_exp_avg_sq"].clone()))
    a, b = out
    assert a[0] == b[0], "losses"
    for what, x, y in zip(("params", "target params", "exp_avg", "exp_avg_sq", "max_exp_avg_sq"), a[1:], b[1:]):
        assert torch.equal(x, y), f"{what}: {int((x != y).sum())} elements differ"


# --------------------------------------------------------------------------- c. short trajectory vs the fp32 oracle
@pytest.mark.parametrize("obs,A,B", [(8, 1, 128), (16, 2, 256), (80, 4, 128)])
def test_short_trajectory_against_oracle(obs, A, B):
    """20 rounds on the learner's own sampled indices, replayed by the fp32 CPU oracle (soft updates every 5 rounds)."""
    from oracle.pearl_oracle import OracleDQN, flat
    rounds = 20
    learner, buf, data = _setup(obs, A, B, freq=5, tau=0.5, rounds=rounds)
    orc = OracleDQN(obs, A, (64, 64), lr=1e-3, gamma=GAMMA, batch_size=B, target_update_freq=5, tau=0.5,
                    init_q=flat(learner._Q).cpu(), init_q_target=flat(learner._Q_target).cpu())
    rep = learner.learn(buf, trace=True)
    idx = rep["idx"].long().cpu()
    eye = torch.eye(A)
    losses = []
    for r in range(rounds):
        b = {k: v[idx[r]] for k, v in data.items()}
        orc.training_steps += 1
        slot = torch.arange(A).view(1, A)
        losses.append(orc.learn_batch(dict(
            state=b["state"], action=eye[b["action"]], reward=b["reward"], terminated=b["terminated"],
            next_state=b["next_state"], next_available_actions=eye[b["avail_ids"]],
            next_unavailable_actions_mask=slot >= b["avail_n"].view(B, 1))))
    close(np.asarray(rep["loss"]), np.asarray(losses), f"obs{obs} A{A} loss")
    close_params(learner.flat_parameters.cpu().numpy(), flat(orc.Q).numpy(), f"obs{obs} A{A} params", 1e-3, rounds)
    close_params(learner.flat_target_parameters.cpu().numpy(), flat(orc.Qt).numpy(), f"obs{obs} A{A} target", 1e-3, rounds)


# --------------------------------------------------------------------------- d. heterogeneous group
def _hetero_group(lr_detour):
    import pearl_b200
    obs, A, B, rounds, pre = 56, 8, 128, 6, (0, 1, 3, 5)
    runs = {}
    for mode in ("group", "solo"):
        learners, bufs = [], []
        for i, k in enumerate(pre):
            seed = 9100 + i
            learner = _learner(obs, A, B, seed, freq=3, tau=0.5, rounds=max(k, 1))
            dynamic = i % 2 == 1
            data = _data(learner, obs, A, B, seed, dynamic)
            buf = _buffer(data, A, seed, dynamic, dynamic_layout=True)   # one record layout per group
            if lr_detour and i == 2:
                learner._optimizer.param_groups[0]["lr"] = 3e-3
            if k:
                learner.learn(buf)
            if lr_detour and i == 2:
                learner._optimizer.param_groups[0]["lr"] = 1e-3
            learner._training_rounds = rounds
            learners.append(learner)
            bufs.append(buf)
        if mode == "group":
            reps = pearl_b200.B200LearnerGroup(learners, bufs).learn()
        else:
            reps = [l.learn(b) for l, b in zip(learners, bufs)]
        runs[mode] = (learners, bufs, reps)
    for i, k in enumerate(pre):
        lg, ls = runs["group"][0][i], runs["solo"][0][i]
        assert lg._training_steps == ls._training_steps == k + rounds
        assert np.array_equal(runs["group"][1][i].get_rng_state(), runs["solo"][1][i].get_rng_state())
        assert runs["group"][2][i]["loss"] == runs["solo"][2][i]["loss"], f"learner {i}: losses"
        assert torch.equal(lg.flat_parameters, ls.flat_parameters), f"learner {i}: params"
        assert torch.equal(lg.flat_target_parameters, ls.flat_target_parameters), f"learner {i}: target params"
        sg, ss = lg.adam_state(), ls.adam_state()
        assert sg["step"] == ss["step"] == k + rounds
        for key in ("exp_avg", "exp_avg_sq", "max_exp_avg_sq"):
            assert torch.equal(sg[key], ss[key]), f"learner {i}: {key}"


def test_group_of_learners_at_different_steps_is_bit_identical_to_solo_runs():
    """Four learners pre-trained by 0, 1, 3 and 5 rounds (each its own AdamW scalars and soft-update phase, freq 3),
    restricted and full next-action sets, in one B200LearnerGroup.learn() vs each trained alone (a group of one)."""
    _hetero_group(lr_detour=False)


def test_group_after_a_learning_rate_detour_is_bit_identical_to_solo_runs():
    """As above, with one learner pre-trained at another learning rate that was then restored."""
    _hetero_group(lr_detour=True)


# --------------------------------------------------------------------------- e. eligibility boundary
def test_tc_eligibility_boundary():
    """prl_dqn_tc_supported is 1 on the whole class and 0 just outside it; outside, engine="tc" learn() and
    B200LearnerGroup.learn() raise NotImplementedError instead of running anything else."""
    import pearl_b200
    for obs in OBS:
        for A in ACTS:
            learner = _learner(obs, A, 128, 1)
            learner.flat_parameters   # binds the learner
            for B in BATCHES:
                assert learner._libh.prl_dqn_tc_supported(learner._handle, B) == 1, (obs, A, B)
    outside = [dict(obs=4), dict(obs=36), dict(obs=136), dict(A=3), dict(A=32), dict(B=64), dict(B=192),
               dict(hidden=(64, 32)), dict(cls=pearl_b200.B200DoubleDQN)]
    for case in outside:
        obs, A, B = case.get("obs", 16), case.get("A", 4), case.get("B", 128)
        kw = {k: case[k] for k in ("hidden", "cls") if k in case}
        learner = _learner(obs, A, B, 2, **kw)
        learner.flat_parameters
        assert learner._libh.prl_dqn_tc_supported(learner._handle, B) == 0, case
        data = _data(learner, obs, A, B, 2, False) if "hidden" not in case else None
        if data is None:   # the margin filter assumes [64, 64]; any rows will do here
            from oracle.synth import make_transitions
            d = make_transitions(2 * B, obs, A, seed=2)
            data = {k: torch.from_numpy(d[k]) for k in ("state", "action", "reward", "next_state", "terminated", "truncated")}
        buf = _buffer(data, A, 2, False)
        w0 = learner.flat_parameters.clone()
        with pytest.raises(NotImplementedError):
            learner.learn(buf)
        with pytest.raises(NotImplementedError):
            pearl_b200.B200LearnerGroup([learner], [buf]).learn()
        assert torch.equal(learner.flat_parameters, w0) and learner._training_steps == 0, case


# --------------------------------------------------------------------------- f. sharded replay buffer
def test_tc_learner_rejects_a_sharded_buffer():
    """A shard of a multi-GPU buffer samples global slots in [0, capacity * world): the tensor-core learner, which
    indexes its local records with them, refuses such a buffer (ValueError) before launching anything."""
    import pearl_b200
    obs, A, B = 16, 4, 128
    learner = _learner(obs, A, B, 5)
    data = _data(learner, obs, A, B, 5, False)
    sharded = pearl_b200.B200ReplayBuffer(data["state"].shape[0], rng="device")
    sharded.push_batch_sharded(0, 2, data["state"], data["action"].to(torch.int32), data["reward"], data["next_state"],
                               data["terminated"], data["truncated"], max_number_actions=A)
    sharded.seed(5)
    other = _learner(obs, A, B, 6)
    plain = _buffer(_data(other, obs, A, B, 6, False), A, 6, False)
    rng0 = sharded.get_rng_state()
    w0, w1 = learner.flat_parameters.clone(), other.flat_parameters.clone()
    with pytest.raises(ValueError, match="shard"):
        learner.learn(sharded)
    with pytest.raises(ValueError, match="shard"):
        pearl_b200.B200LearnerGroup([other, learner], [plain, sharded]).learn()
    torch.cuda.synchronize()
    assert np.array_equal(sharded.get_rng_state(), rng0), "the sampler ran"
    assert torch.equal(learner.flat_parameters, w0) and torch.equal(other.flat_parameters, w1), "a learner ran"
    assert learner.adam_state()["step"] == 0 and other.adam_state()["step"] == 0
