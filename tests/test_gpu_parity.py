"""GPU parity tests (H100): the CUDA path, called through the C ABI via the
pearl_b200 plugins, against (a) golden fixtures recorded from the reference,
(b) the CPU oracle on the same seeded inputs, (c) size-independent properties
at BASELINE.json's full sizes.

Tolerances: indices / gathered transitions bit-exact; Q-values, Bellman targets,
losses, parameters and AdamW state within 1e-4 relative fp32 (north_star) — the
assertions below use rtol=1e-4 with a small atol for values near zero, and
print the achieved maxima.
"""
import glob
import json
import os
import random

import numpy as np
import pytest
import torch

from conftest import GOLDEN

pytestmark = pytest.mark.gpu

KAT = json.load(open(os.path.join(GOLDEN, "random_sample_kat.json")))["cases"]
CASES = sorted(os.path.basename(p)[:-4] for pat in ("dqn_*.npz", "ddqn_*.npz") for p in glob.glob(os.path.join(GOLDEN, pat)))
RTOL = 1e-4


def _imports():
    import pearl_b200
    from oracle import c_oracle
    from oracle.pearl_oracle import OracleDQN
    from oracle.synth import from_fixture, make_transitions
    return pearl_b200, c_oracle, OracleDQN, from_fixture, make_transitions


class _Space:  # minimal DiscreteActionSpace stand-in for the constructor / act()
    def __init__(self, n):
        self.n = n
        self.actions = [torch.tensor([i]) for i in range(n)]

    @property
    def actions_batch(self):
        return torch.stack(self.actions)


def relerr(got, want, atol):
    got, want = np.asarray(got, dtype=np.float64), np.asarray(want, dtype=np.float64)
    return float(np.max(np.abs(got - want) / (np.abs(want) + atol / RTOL)))


def assert_close(got, want, what, atol=1e-6):
    e = relerr(got, want, atol)
    print(f"    {what}: max rel err {e:.3e}")
    np.testing.assert_allclose(np.asarray(got), np.asarray(want), rtol=RTOL, atol=atol, err_msg=what)


def assert_close_adamw(got, want, what, lr, rounds, atol=1e-6, max_outliers=4):
    """Elementwise 1e-4 relative like assert_close, with an explicit, counted and bounded outlier list.  AdamW moves an
    element by lr * m / (sqrt(v) + eps): where a gradient is zero to within fp32 summation noise (|g| ~ eps = 1e-8)
    the step depends on that noise, so two correct summation orders can differ there by a fraction of lr per round.
    At most `max_outliers` such elements are tolerated, each within 5 % of lr * rounds; they are printed."""
    got, want = np.asarray(got, dtype=np.float64), np.asarray(want, dtype=np.float64)
    diff = np.abs(got - want)
    bad = np.flatnonzero(diff > atol + RTOL * np.abs(want))
    print(f"    {what}: max rel err {relerr(got, want, atol):.3e}; AdamW eps-sensitive outliers: "
          f"{[(int(i), float(got[i]), float(want[i])) for i in bad]}")
    assert bad.size <= max_outliers, f"{what}: {bad.size} elements outside 1e-4 (allowed outliers: {max_outliers})"
    if bad.size:
        assert diff[bad].max() <= 0.05 * lr * rounds, f"{what}: outlier off by {diff[bad].max():.3e} > 5% of lr * rounds"


def filled_buffer(n, obs=1, n_act=2, capacity=None, rng="device"):
    pearl_b200 = _imports()[0]
    buf = pearl_b200.B200ReplayBuffer(capacity or n, rng=rng)
    dev = buf.device
    chunk = 1 << 18
    for s in range(0, n, chunk):
        m = min(chunk, n - s)
        buf.push_batch(torch.zeros((m, obs), device=dev), torch.zeros(m, dtype=torch.int32, device=dev),
                       torch.arange(s, s + m, device=dev, dtype=torch.float32), torch.zeros((m, obs), device=dev),
                       torch.zeros(m, dtype=torch.bool, device=dev), torch.zeros(m, dtype=torch.bool, device=dev),
                       max_number_actions=n_act)
    return buf


# --------------------------------------------------------------------------- sampler
@pytest.mark.parametrize("case", KAT, ids=lambda c: f"seed{c['seed']}_n{c['n']}_k{c['k']}")
def test_sampler_matches_cpython_known_answers(case):
    buf = filled_buffer(case["n"])
    buf.seed(case["seed"])
    st0 = buf.get_rng_state()
    assert int(np.bitwise_xor.reduce(st0[:624])) == case["state_before_xor"]
    logical, slot = buf.sample_indices(case["k"], rounds=case["reps"])
    assert logical.cpu().tolist() == case["samples"]
    assert torch.equal(logical, slot)  # ring not wrapped: slot == logical
    st1 = buf.get_rng_state()
    assert int(st1[624]) == case["state_after_index"]
    assert int(np.bitwise_xor.reduce(st1[:624])) == case["state_after_xor"]


def test_sampler_full_size_against_c_oracle_and_python_handoff():
    """cfg2 buffer size (1e6, k=256), many rounds, vs the C restatement; and the
    rng='python' mode continues / hands back the global `random` state."""
    _, c_oracle, *_ = _imports()
    n, k, rounds = 1_000_000, 256, 200
    buf = filled_buffer(n, rng="python")
    random.seed(2024)
    mt = c_oracle.MT(state=np.asarray(random.getstate()[1], dtype=np.uint64).astype(np.uint32))
    logical, _ = buf.sample_indices(k, rounds=rounds)
    want = np.stack([mt.sample(n, k) for _ in range(rounds)])
    got = logical.cpu().numpy()
    assert np.array_equal(got, want)
    assert all(len(set(r.tolist())) == k for r in got)
    assert np.array_equal(np.asarray(random.getstate()[1], dtype=np.uint64).astype(np.uint32), mt.st)
    # the next draw of the host interpreter continues the same stream
    assert random.getrandbits(32) == mt.getrandbits32()


def test_sample_too_large_raises_value_error():
    buf = filled_buffer(10)
    with pytest.raises(ValueError):
        buf.sample(11)


# --------------------------------------------------------------------------- ring + gather
def test_ring_wraps_fifo_and_gather_is_bit_exact():
    pearl_b200, _, _, _, make_transitions = _imports()
    cap, n, obs, A = 37, 100, 7, 3
    d = make_transitions(n, obs, A, seed=9)
    buf = pearl_b200.B200ReplayBuffer(cap, rng="device")
    # mixed single pushes (host), host batches and device batches
    for i in range(5):
        buf.push(torch.from_numpy(d["state"][i]), torch.tensor([int(d["action"][i])]), float(d["reward"][i]),
                 bool(d["terminated"][i]), bool(d["truncated"][i]), curr_available_actions=_Space(A),
                 next_state=torch.from_numpy(d["next_state"][i]), next_available_actions=_Space(A),
                 max_number_actions=A)
    t = lambda k, s, e, dev="cpu": torch.from_numpy(d[k][s:e]).to(dev)
    buf.push_batch(t("state", 5, 60), t("action", 5, 60), t("reward", 5, 60), t("next_state", 5, 60),
                   t("terminated", 5, 60), t("truncated", 5, 60))
    buf.push_batch(t("state", 60, n, "cuda"), t("action", 60, n, "cuda"), t("reward", 60, n, "cuda"),
                   t("next_state", 60, n, "cuda"), t("terminated", 60, n, "cuda"), t("truncated", 60, n, "cuda"))
    assert len(buf) == cap
    buf.seed(5)
    b = buf.sample(cap)  # k == n: every stored element exactly once (test_trajectories_in_replay_buffer.py)
    logical = np.arange(n - cap, n)
    # identify rows through the state (unique with probability 1)
    pos = {d["state"][j].tobytes(): j for j in logical}
    rows = [pos[s.tobytes()] for s in b.state.cpu().numpy()]
    assert sorted(rows) == logical.tolist()
    rows = np.asarray(rows)
    assert np.array_equal(b.next_state.cpu().numpy(), d["next_state"][rows])
    assert np.array_equal(b.reward.cpu().numpy(), d["reward"][rows])
    assert np.array_equal(b.action.cpu().numpy().reshape(-1), d["action"][rows])
    assert np.array_equal(b.terminated.cpu().numpy(), d["terminated"][rows])
    assert b.terminated.dtype == torch.bool and b.truncated.dtype == torch.bool
    assert b.action.dtype == torch.int64 and b.action.shape == (cap, 1)
    assert b.next_available_actions.shape == (cap, A, 1) and b.next_unavailable_actions_mask.shape == (cap, A)
    assert not b.next_unavailable_actions_mask.any()
    buf.clear()
    assert len(buf) == 0


# --------------------------------------------------------------------------- learner vs golden
def build_from_fixture(name, rows_per_cta=0):
    pearl_b200, _, _, from_fixture, _ = _imports()
    fx = np.load(os.path.join(GOLDEN, name + ".npz"))
    cfg = json.loads(bytes(fx["config"]).decode())
    data = from_fixture(fx)
    A = cfg["n_act"]
    buf = pearl_b200.B200ReplayBuffer(cfg["capacity"], rng="python")
    n = cfg["n_push"]
    kw = {}
    if cfg["dynamic"]:
        kw = dict(next_available_ids=torch.from_numpy(data["next_avail_ids"].astype(np.uint8)),
                  next_available_count=torch.from_numpy(data["next_avail_n"].astype(np.int32)))
    buf.push_batch(torch.from_numpy(data["state"]), torch.from_numpy(data["action"]), torch.from_numpy(data["reward"]),
                   torch.from_numpy(data["next_state"]), torch.from_numpy(data["terminated"]),
                   torch.from_numpy(data["truncated"]), max_number_actions=A, **kw)
    cls = pearl_b200.B200DoubleDQN if cfg["double"] else pearl_b200.B200DeepQLearning
    learner = cls(state_dim=cfg["obs"], action_space=_Space(A), hidden_dims=cfg["hidden"],
                  learning_rate=cfg["lr"], discount_factor=cfg["gamma"], training_rounds=cfg["rounds"],
                  batch_size=cfg["batch"], target_update_freq=cfg["target_update_freq"],
                  soft_update_tau=cfg["tau"],
                  action_representation_module=pearl_b200.OneHotActionTensorRepresentationModule(A),
                  rows_per_cta=rows_per_cta)
    learner.to("cuda")
    from oracle.pearl_oracle import load_flat
    load_flat(learner._Q, fx["init_q"])
    load_flat(learner._Q_target, fx["init_q_target"])
    return fx, cfg, data, buf, learner


@pytest.mark.parametrize("name", CASES)
def test_learn_matches_reference_golden(name):
    """Same pushed transitions, same CPython random state, same initial weights as the
    recorded reference run: indices bit-exact; q, y, loss, parameters, AdamW state 1e-4."""
    fx, cfg, data, buf, learner = build_from_fixture(name)
    random.setstate((3, tuple(int(x) for x in fx["mt_state_before"]), None))
    total = cfg["rounds"] * cfg["learn_calls"]
    # run in segments that end at the snapshot rounds (learn() semantics are unchanged:
    # _training_steps and the RNG state carry over between calls)
    cuts = sorted(set(cfg["snap_rounds"] + [total]))
    done, idx, q, y, mae = 0, [], [], [], []
    for c in cuts:
        learner._training_rounds = c - done
        rep = learner.learn(buf, trace=True)
        idx.append(rep["idx"].cpu().numpy()); q.append(rep["q"].cpu().numpy()); y.append(rep["y"].cpu().numpy())
        mae += rep["loss"]
        done = c
        if c in cfg["snap_rounds"]:
            assert_close(learner.flat_parameters.cpu().numpy(), fx[f"q_after_{c}"], f"{name} params after {c}")
            assert_close(learner.flat_target_parameters.cpu().numpy(), fx[f"qt_after_{c}"],
                         f"{name} target params after {c}")
    assert np.array_equal(np.concatenate(idx), fx["idx"]), "sampled indices differ from the reference"
    after = np.asarray(random.getstate()[1], dtype=np.uint64).astype(np.uint32)
    assert np.array_equal(after, fx["mt_state_after"]), "python random state not handed back correctly"
    assert_close(np.concatenate(q), fx["q"], f"{name} q")
    assert_close(np.concatenate(y), fx["y"], f"{name} y")
    assert_close(np.asarray(mae), fx["mae"], f"{name} loss")
    st = learner.adam_state()
    assert st["step"] == total
    assert_close(st["exp_avg"].cpu().numpy(), fx["exp_avg"], f"{name} exp_avg", atol=1e-7)
    assert_close(st["exp_avg_sq"].cpu().numpy(), fx["exp_avg_sq"], f"{name} exp_avg_sq", atol=1e-9)
    assert_close(st["max_exp_avg_sq"].cpu().numpy(), fx["max_exp_avg_sq"], f"{name} max_exp_avg_sq", atol=1e-9)
    # state_dict keys of the reference module tree (SURVEY.md appendix B)
    keys = set(learner.state_dict().keys())
    for net in ("_Q", "_Q_target"):
        for i in range(3):
            assert f"{net}._model.{i}.0.weight" in keys and f"{net}._model.{i}.0.bias" in keys
    info = learner.launch_info()
    assert info["launches"] == 1 and info["ctas"] >= 1


@pytest.mark.parametrize("rows", [2, 8, 16, 32])
def test_tiling_does_not_change_results_beyond_tolerance(rows):
    fx, cfg, data, buf, learner = build_from_fixture("dqn_cfg2_pool", rows_per_cta=rows)
    random.setstate((3, tuple(int(x) for x in fx["mt_state_before"]), None))
    learner._training_rounds = 10
    rep = learner.learn(buf, trace=True)
    assert np.array_equal(rep["idx"].cpu().numpy(), fx["idx"][:10])
    assert_close(rep["q"].cpu().numpy(), fx["q"][:10], f"rows={rows} q")
    assert_close(learner.flat_parameters.cpu().numpy(), fx["q_after_10"], f"rows={rows} params")
    assert learner.launch_info()["rows_per_cta"] == rows


def test_learn_is_deterministic():
    outs = []
    for _ in range(2):
        fx, cfg, data, buf, learner = build_from_fixture("ddqn_setbranch")
        random.setstate((3, tuple(int(x) for x in fx["mt_state_before"]), None))
        learner.learn(buf)
        outs.append(learner.flat_parameters.clone())
    assert torch.equal(outs[0], outs[1])


# --------------------------------------------------------------------------- learn_batch / q_values vs oracle
@pytest.mark.parametrize("double", [False, True])
def test_learn_batch_and_q_values_match_oracle(double):
    pearl_b200, _, OracleDQN, _, make_transitions = _imports()
    obs, A, hidden, B = 12, 6, (24, 20), 40
    d = make_transitions(B, obs, A, seed=77, dynamic=True)
    torch.manual_seed(3)
    cls = pearl_b200.B200DoubleDQN if double else pearl_b200.B200DeepQLearning
    learner = cls(state_dim=obs, action_space=_Space(A), hidden_dims=list(hidden), training_rounds=1,
                  batch_size=B, target_update_freq=3, soft_update_tau=0.3,
                  action_representation_module=pearl_b200.OneHotActionTensorRepresentationModule(A)).to("cuda")
    from oracle.pearl_oracle import flat
    orc = OracleDQN(obs, A, hidden, batch_size=B, target_update_freq=3, tau=0.3, double=double,
                    init_q=flat(learner._Q).cpu(), init_q_target=flat(learner._Q_target).cpu())
    # perturb the target so that online != target
    with torch.no_grad():
        for p, po in zip(learner._Q_target.parameters(), orc.Qt.parameters()):
            noise = torch.randn(p.shape) * 0.05
            p.add_(noise.to(p.device)); po.add_(noise)
    states = torch.from_numpy(d["state"])
    qv = learner.q_values(states).cpu()
    eye = torch.eye(A).unsqueeze(0).expand(B, A, A)
    with torch.no_grad():
        want = orc._q_values(orc.Q, states, eye)
    assert_close(qv.numpy(), want.numpy(), "q_values")
    # arbitrary (non-prefix) availability masks
    g = torch.Generator().manual_seed(1)
    mask = torch.rand((B, A), generator=g) < 0.4
    mask[mask.all(1), 0] = False  # keep at least one action available
    avail = torch.arange(A).float().view(1, A, 1).expand(B, A, 1).clone()
    batch = pearl_b200.TransitionBatch(
        state=states, action=torch.from_numpy(d["action"]).view(B, 1), reward=torch.from_numpy(d["reward"]),
        next_state=torch.from_numpy(d["next_state"]), terminated=torch.from_numpy(d["terminated"]),
        truncated=torch.from_numpy(d["truncated"]), next_available_actions=avail,
        next_unavailable_actions_mask=mask)
    for step in range(4):  # training_steps stays 0 in learn_batch (reference quirk): no target update
        got = learner.learn_batch(batch)["loss"]
        b = dict(state=states, action=orc._one_hot(batch.action), reward=batch.reward, terminated=batch.terminated,
                 next_state=batch.next_state, next_available_actions=orc._one_hot(avail),
                 next_unavailable_actions_mask=mask)
        want_loss = orc.learn_batch(b)
        assert abs(got - want_loss) <= RTOL * abs(want_loss) + 1e-6
    assert_close(learner.flat_parameters.cpu().numpy(), flat(orc.Q).numpy(), "params after learn_batch x4")
    assert_close(learner.flat_target_parameters.cpu().numpy(), flat(orc.Qt).numpy(), "target after learn_batch x4")


def test_empty_buffer_learn_returns_empty_report():
    pearl_b200 = _imports()[0]
    buf = pearl_b200.B200ReplayBuffer(8)
    learner = pearl_b200.B200DeepQLearning(
        state_dim=4, action_space=_Space(2), hidden_dims=[8, 8],
        action_representation_module=pearl_b200.OneHotActionTensorRepresentationModule(2)).to("cuda")
    assert learner.learn(buf) == {}


# --------------------------------------------------------------------------- full size (BASELINE cfg2)
@pytest.mark.parametrize("engine", ["simt", "tc"])
def test_full_size_cfg2_against_oracle_on_the_sampled_batches(engine):
    """obs=128, A=16, [64,64], B=256 on a 1e6-transition buffer (set branch of random.sample): the learner's own
    sampled indices (bit-exact vs the C oracle) select the batches the torch oracle replays.  Both engines: the
    cooperative fp32 SIMT kernel and the one-SM wgmma (3xTF32) kernel."""
    pearl_b200, c_oracle, OracleDQN, _, _ = _imports()
    n, obs, A, B, rounds = 1_000_000, 128, 16, 256, 12
    g = torch.Generator(device="cuda").manual_seed(4321)
    buf = pearl_b200.B200ReplayBuffer(n, rng="python")
    host = {}
    chunk = 250_000
    for s in range(0, n, chunk):
        st = torch.randn((chunk, obs), generator=g, device="cuda")
        ns = torch.randn((chunk, obs), generator=g, device="cuda")
        rw = torch.randn(chunk, generator=g, device="cuda")
        tm = torch.rand(chunk, generator=g, device="cuda") < 0.02
        ac = (torch.arange(s, s + chunk, device="cuda") % A).to(torch.int32)
        buf.push_batch(st, ac, rw, ns, tm, torch.zeros_like(tm), max_number_actions=A)
        host[s] = (st, ns, rw, tm, ac)
    assert len(buf) == n
    torch.manual_seed(1234)
    learner = pearl_b200.B200DeepQLearning(
        state_dim=obs, action_space=_Space(A), hidden_dims=[64, 64], training_rounds=rounds, batch_size=B,
        target_update_freq=10, soft_update_tau=0.75,
        action_representation_module=pearl_b200.OneHotActionTensorRepresentationModule(A), engine=engine).to("cuda")
    from oracle.pearl_oracle import flat
    orc = OracleDQN(obs, A, (64, 64), batch_size=B, target_update_freq=10, tau=0.75,
                    init_q=flat(learner._Q).cpu(), init_q_target=flat(learner._Q_target).cpu())
    random.seed(1234)
    mt = c_oracle.MT(state=np.asarray(random.getstate()[1], dtype=np.uint64).astype(np.uint32))
    rep = learner.learn(buf, trace=True)
    idx = rep["idx"].cpu().numpy()
    assert np.array_equal(idx, np.stack([mt.sample(n, B) for _ in range(rounds)]))

    full = [torch.cat([host[s][f] for s in sorted(host)]) for f in range(5)]
    host.clear()

    def rows(ix):
        ix = torch.from_numpy(ix.astype(np.int64)).cuda()
        return [f[ix].cpu() for f in full]

    eye = torch.eye(A).unsqueeze(0).expand(B, A, A)
    losses = []
    for r in range(rounds):
        st, ns, rw, tm, ac = rows(idx[r])
        orc.training_steps += 1
        b = dict(state=st, action=orc._one_hot(ac.long()), reward=rw, terminated=tm, next_state=ns,
                 next_available_actions=eye, next_unavailable_actions_mask=torch.zeros((B, A), dtype=torch.bool))
        losses.append(orc.learn_batch(b))
    assert_close(np.asarray(rep["loss"]), np.asarray(losses), "cfg2 loss")
    assert_close_adamw(learner.flat_parameters.cpu().numpy(), flat(orc.Q).numpy(), "cfg2 params after 12 rounds", 1e-3, rounds)
    assert_close_adamw(learner.flat_target_parameters.cpu().numpy(), flat(orc.Qt).numpy(), "cfg2 target params", 1e-3, rounds)


# --------------------------------------------------------------------------- tensor-core engine
def test_tc_engine_matches_reference_golden_cfg2():
    """The one-SM wgmma learner (3xTF32) on the cfg2-shaped fixture: same indices, q, y, loss,
    parameters, target parameters and AdamW state as the recorded reference run, 1e-4."""
    name = "dqn_cfg2_pool"
    fx, cfg, data, buf, learner = build_from_fixture(name)
    learner._engine = "tc"
    random.setstate((3, tuple(int(x) for x in fx["mt_state_before"]), None))
    cuts = sorted(set(cfg["snap_rounds"] + [cfg["rounds"]]))
    done, idx, q, y, mae = 0, [], [], [], []
    for c in cuts:
        learner._training_rounds = c - done
        rep = learner.learn(buf, trace=True)
        idx.append(rep["idx"].cpu().numpy()); q.append(rep["q"].cpu().numpy()); y.append(rep["y"].cpu().numpy())
        mae += rep["loss"]
        done = c
        if c in cfg["snap_rounds"]:
            assert_close(learner.flat_parameters.cpu().numpy(), fx[f"q_after_{c}"], f"tc params after {c}")
            assert_close(learner.flat_target_parameters.cpu().numpy(), fx[f"qt_after_{c}"], f"tc target after {c}")
    assert np.array_equal(np.concatenate(idx), fx["idx"])
    assert_close(np.concatenate(q), fx["q"], "tc q")
    assert_close(np.concatenate(y), fx["y"], "tc y")
    assert_close(np.asarray(mae), fx["mae"], "tc loss")
    st = learner.adam_state()
    assert_close(st["exp_avg"].cpu().numpy(), fx["exp_avg"], "tc exp_avg", atol=1e-7)
    assert_close(st["exp_avg_sq"].cpu().numpy(), fx["exp_avg_sq"], "tc exp_avg_sq", atol=1e-9)
    assert_close(st["max_exp_avg_sq"].cpu().numpy(), fx["max_exp_avg_sq"], "tc max_exp_avg_sq", atol=1e-9)


def _group_vs_simt(obs, A, B, dynamic=True, adamw_outliers=False):
    pearl_b200, _, _, _, make_transitions = _imports()
    n, rounds, L = 2000, 25, 5
    groups = {}
    for engine in ("simt", "tc"):
        learners, bufs = [], []
        for i in range(L):
            d = make_transitions(n, obs, A, seed=300 + i, dynamic=(dynamic and i % 2 == 1))
            buf = pearl_b200.B200ReplayBuffer(n, rng="device", dynamic_action_space=True)
            kw = {}
            if dynamic and i % 2 == 1:
                kw = dict(next_available_ids=torch.from_numpy(d["next_avail_ids"].astype(np.uint8)),
                          next_available_count=torch.from_numpy(d["next_avail_n"].astype(np.int32)))
            buf.push_batch(*(torch.from_numpy(d[k]) for k in ("state", "action", "reward", "next_state", "terminated", "truncated")),
                           max_number_actions=A, **kw)
            buf.seed(900 + i)
            torch.manual_seed(40 + i)
            learners.append(pearl_b200.B200DeepQLearning(
                state_dim=obs, action_space=_Space(A), hidden_dims=[64, 64], training_rounds=rounds, batch_size=B,
                target_update_freq=4, soft_update_tau=0.5,
                action_representation_module=pearl_b200.OneHotActionTensorRepresentationModule(A), engine=engine).to("cuda"))
            bufs.append(buf)
        if engine == "tc":
            reps = pearl_b200.B200LearnerGroup(learners, bufs).learn()
        else:
            reps = [l.learn(b) for l, b in zip(learners, bufs)]
        groups[engine] = (learners, bufs, reps)
    for i in range(L):
        ls, lt = groups["simt"][0][i], groups["tc"][0][i]
        assert np.array_equal(groups["simt"][1][i].get_rng_state(), groups["tc"][1][i].get_rng_state())
        assert_close(np.asarray(groups["tc"][2][i]["loss"]), np.asarray(groups["simt"][2][i]["loss"]), f"group loss {i}")
        close = (lambda g, w, what: assert_close_adamw(g, w, what, 1e-3, rounds)) if adamw_outliers else assert_close
        close(lt.flat_parameters.cpu().numpy(), ls.flat_parameters.cpu().numpy(), f"group params {i}")
        close(lt.flat_target_parameters.cpu().numpy(), ls.flat_target_parameters.cpu().numpy(), f"group target {i}")


def test_learner_group_equals_individual_simt_learners():
    """B200LearnerGroup (one launch, one SM per learner, tensor cores) vs the same learners trained one
    by one with the fp32 SIMT kernel: identical index streams, parameters within 1e-4; dynamic action
    sets and obs < 128 included."""
    _group_vs_simt(40, 8, 128)


@pytest.mark.parametrize("obs", [72, 96])
def test_learner_group_with_a_partial_second_k_pass(obs):
    """64 < obs < 128: layer 1 takes a second K pass shorter than 64 and the second warpgroup's share of dW1s is
    narrower than 64 columns (8 at obs 72, 32 at obs 96); two row tiles (batch 256).  Full action sets: with dynamic sets
    of 16 actions some first-step gradients are ~1e-7, where AdamW's eps makes the step depend on fp32 summation order,
    and 25 free-running rounds amplify that beyond an elementwise 1e-4; the dynamic path does not depend on obs and is
    covered at obs 40 above.  Parameters: elementwise 1e-4 with the bounded AdamW outliers of tests/_tol.py."""
    _group_vs_simt(obs, 16, 256, dynamic=False, adamw_outliers=True)


def test_tc_group_chunked_launch_is_bit_identical_to_short_calls():
    """One `group.learn()` of 80 rounds (index streams produced in chunks on a side stream, a 32-round and a
    48-round learner launch) and one of 300 rounds (four chunks: 32 rounds, then three launches of about 89); inside a
    launch the target network's small vectors stay cached in shared memory between soft updates and the target tiles
    are updated in tile order.  Each is compared with the same learners driven by calls of at most 20 / 50 rounds (one
    chunk each): same arithmetic in the same order, so losses, parameters, target parameters and AdamW state must be
    bit-identical — any state carried wrongly across a round or launch boundary shows up here.  Soft target updates
    (freq 4) fall on both sides of the boundaries."""
    for rounds, short in ((80, 20), (300, 50)):
        _chunked_vs_short_calls(rounds, short)


def _chunked_vs_short_calls(rounds, short):
    pearl_b200, _, _, _, make_transitions = _imports()
    obs, A, B, n, L = 128, 16, 256, 3000, 3
    out = {}
    for per_call in (rounds, short):
        learners, bufs = [], []
        for i in range(L):
            d = make_transitions(n, obs, A, seed=700 + i)
            buf = pearl_b200.B200ReplayBuffer(n, rng="device")
            buf.push_batch(*(torch.from_numpy(d[k]) for k in ("state", "action", "reward", "next_state", "terminated", "truncated")),
                           max_number_actions=A)
            buf.seed(70 + i)
            torch.manual_seed(7 + i)
            learners.append(pearl_b200.B200DeepQLearning(
                state_dim=obs, action_space=_Space(A), hidden_dims=[64, 64], training_rounds=rounds, batch_size=B,
                target_update_freq=4, soft_update_tau=0.5, max_rounds_per_call=per_call,
                action_representation_module=pearl_b200.OneHotActionTensorRepresentationModule(A), engine="tc").to("cuda"))
            bufs.append(buf)
        reps = pearl_b200.B200LearnerGroup(learners, bufs).learn()
        out[per_call] = (learners, bufs, reps)
    for i in range(L):
        la, lb = out[rounds][0][i], out[short][0][i]
        assert np.array_equal(out[rounds][1][i].get_rng_state(), out[short][1][i].get_rng_state())
        assert out[rounds][2][i]["loss"] == out[short][2][i]["loss"]
        assert torch.equal(la.flat_parameters, lb.flat_parameters)
        assert torch.equal(la.flat_target_parameters, lb.flat_target_parameters)
        sa, sb = la.adam_state(), lb.adam_state()
        for k in ("exp_avg", "exp_avg_sq", "max_exp_avg_sq"):
            assert torch.equal(sa[k], sb[k]), k


@pytest.mark.gpu
def test_group_push_matches_per_buffer_push():
    """B200LearnerGroup.push_batch (one library call, threaded packing) writes the same ring contents as per-buffer pushes,
    including the buffers that take the wrap-around path."""
    import pearl_b200
    from oracle.synth import make_transitions
    R, obs, A, cap = 5, 8, 4, 300
    bufs_a = [pearl_b200.B200ReplayBuffer(cap) for _ in range(R)]
    bufs_b = [pearl_b200.B200ReplayBuffer(cap) for _ in range(R)]

    class _L:   # the group only needs the learners for learn(); push goes through the buffers
        _n_actions = A
    group = pearl_b200.B200LearnerGroup([_L() for _ in range(R)], bufs_a)
    t = torch.from_numpy
    for step, n in enumerate((120, 130, 100, 7)):          # the third push wraps the ring
        d = [make_transitions(n, obs, A, seed=100 * step + i) for i in range(R)]
        stack = lambda k: torch.stack([t(d[i][k]) for i in range(R)])
        group.push_batch(stack("state"), stack("action"), stack("reward"), stack("next_state"), stack("terminated"), stack("truncated"))
        for i in range(R):
            bufs_b[i].push_batch(*(t(d[i][k]) for k in ("state", "action", "reward", "next_state", "terminated", "truncated")),
                                 max_number_actions=A)
    for a, b in zip(bufs_a, bufs_b):
        assert len(a) == len(b) == cap
        assert torch.equal(a._storage, b._storage)
        assert int(a._lib.prl_buf_head(a._handle)) == int(b._lib.prl_buf_head(b._handle))
