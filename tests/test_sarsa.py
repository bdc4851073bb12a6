"""DeepSARSA on the GPU (B200DeepSARSA over a B200SARSAReplayBuffer, csrc/sarsa.cu) against
(a) the recordings of the reference's PearlAgent(DeepSARSA, SARSAReplayBuffer) (tests/golden/sarsa_*.npz: the same push
    stream through the delayed-push cache, learn() + clear() at the recorded points, agent.learn_batch on sampled
    batches), elementwise 1e-4 (tests/_tol.py), with the sampled indices and CPython's `random` state bit-exact, graph
    replay on and off, and once with records that straddle the ring's end;
(b) oracle/sarsa_oracle.py at obs 128, 16 actions, [256, 256], batch 256 under contraction engines 0, 1 and 2;
plus bit-identity (run to run, graph vs eager, round chunking, learn vs learn_batch), the launch count, the graph cache,
lr changes on the same handle, the checkpoint views and the buffer's next-action storage and refusals."""
import copy
import ctypes as C
import os
import random

import numpy as np
import pytest
import torch

from conftest import GOLDEN
from oracle.pearl_oracle import flat, load_flat
from oracle.sarsa_oracle import OracleSARSA, one_hot

pytestmark = pytest.mark.gpu

from _tol import close as _close, close_params as _close_params  # noqa: E402
from test_iql import _close_net, _relu_boundary  # noqa: E402

LAUNCHES_PER_ROUND = 19     # load, soft update, 2 x (3 contractions + fold), target, 4 contractions + 2 small, AdamW, report


class _Space:
    def __init__(self, ids):
        ids = [int(i) for i in ids]
        self.n = len(ids)
        self.actions = [torch.tensor([i]) for i in ids]
        self.actions_batch = torch.tensor(ids).view(-1, 1)


def _learner(obs, A, hidden, **kw):
    import pearl_b200
    return pearl_b200.B200DeepSARSA(state_dim=obs, action_space=_Space(range(A)), hidden_dims=list(hidden),
                                    action_representation_module=pearl_b200.OneHotActionTensorRepresentationModule(A),
                                    **kw).to("cuda:0")


def _max_exp_avg_sq(fx):
    v = fx["adam_exp_avg_sq"].copy()
    v[fx["adam_max_exp_avg_sq_idx"]] = fx["adam_max_exp_avg_sq_val"]
    return v


def _replay(fx, graph, wrap=False):
    """The recorded run on the GPU; returns the learner, the buffer and (losses, sampled indices)."""
    import pearl_b200
    from pearl_b200 import _lib
    A, R, B = int(fx["n_actions"]), int(fx["rounds"]), int(fx["batch"])
    buf = pearl_b200.B200SARSAReplayBuffer(64 if wrap else int(fx["capacity"]))
    if wrap:   # records of the first call straddle the ring's end
        buf.push_batch(torch.zeros(1, int(fx["obs"])), torch.zeros(1, dtype=torch.int32), torch.zeros(1), torch.zeros(1, int(fx["obs"])),
                       torch.zeros(1, dtype=torch.bool), torch.zeros(1, dtype=torch.bool), max_number_actions=A,
                       next_action=torch.zeros(1, dtype=torch.int32))
        _lib.check(buf._lib.prl_buf_set_occupancy(buf.handle, 0, 64 - 7))
    pl = _learner(int(fx["obs"]), A, fx["hidden"].tolist(), learning_rate=float(fx["lr"]), discount_factor=float(fx["gamma"]),
                  training_rounds=R, batch_size=B, target_update_freq=int(fx["target_update_freq"]), soft_update_tau=float(fx["tau"]))
    pl.use_cuda_graph = graph
    load_flat(pl._Q, fx["init_q"])
    load_flat(pl._Q_target, fx["init_q"])
    random.setstate((3, tuple(int(x) for x in fx["rng_before"]), None))
    full, dyn = _Space(range(A)), bool(fx["dynamic"])
    learn_after = set(fx["learn_after"].tolist())
    losses, idx, calls, handles = [], [], 0, []
    for i in range(len(fx["push_action"])):
        nxt = _Space(fx["push_next_ids"][i][: int(fx["push_next_count"][i])]) if dyn else full
        buf.push(state=torch.from_numpy(fx["push_state"][i]), action=torch.tensor([int(fx["push_action"][i])]),
                 reward=float(fx["push_reward"][i]), terminated=bool(fx["push_terminated"][i]),
                 truncated=bool(fx["push_truncated"][i]), curr_available_actions=full,
                 next_state=torch.from_numpy(fx["push_next_state"][i]), next_available_actions=nxt, max_number_actions=A)
        if i in learn_after:
            pl.optimizer.param_groups[0]["lr"] = float(fx["call_lr"][calls])
            rep = pl.learn(buf, trace=True)                 # PearlAgent.learn: learn, then clear (on-policy)
            buf.clear()
            losses += rep.get("loss", [])
            if rep:
                idx += rep["idx"].reshape(-1).tolist()
                handles.append(pl._handle.value)
            _close(pl.flat_parameters.cpu().numpy(), fx["q_calls"][calls], f"online net after call {calls}")
            _close(pl.flat_target_parameters.cpu().numpy(), fx["qt_calls"][calls], f"target net after call {calls}")
            calls += 1
    for c in range(len(fx["q_calls"]) - calls):              # agent.learn_batch(buf.sample(batch))
        tb = buf.sample(B)
        assert tb.next_action.dtype == torch.int64 and tuple(tb.next_action.shape) == (B, 1)
        losses.append(pl.learn_batch(tb)["loss"])
        handles.append(pl._handle.value)
        _close(pl.flat_parameters.cpu().numpy(), fx["q_calls"][c], f"online net after batch {c}")
        _close(pl.flat_target_parameters.cpu().numpy(), fx["qt_calls"][c], f"target net after batch {c}")
    if calls:
        assert len(set(handles)) == 1, "an lr change or a new batch size re-created the C handle"
    return pl, buf, losses, idx


@pytest.mark.parametrize("graph", [True, False])
@pytest.mark.parametrize("case", ["sarsa_method", "sarsa_steps", "sarsa_lr", "sarsa_batch"])
def test_sarsa_matches_reference_recording(case, graph):
    fx = np.load(os.path.join(GOLDEN, f"{case}.npz"))
    pl, buf, losses, idx = _replay(fx, graph)
    if not bool(fx["learn_batch"]):
        assert idx == fx["idx"].tolist()                                            # bit-exact sampling
    assert random.getstate()[1] == tuple(int(x) for x in fx["rng_after"])            # CPython's random as the reference left it
    _close(losses, fx["loss"], "loss")
    st = pl.adam_state()
    assert st["step"] == int(fx["adam_step"])
    for k, want in (("exp_avg", fx["adam_exp_avg"]), ("exp_avg_sq", fx["adam_exp_avg_sq"]), ("max_exp_avg_sq", _max_exp_avg_sq(fx))):
        _close(st[k].cpu().numpy(), want, f"AdamW {k}", atol=1e-9)
    if case == "sarsa_steps":                  # the stale cache survived every clear() and was appended again
        assert buf.cache is not None


def test_sarsa_recording_on_a_wrapping_ring():
    fx = np.load(os.path.join(GOLDEN, "sarsa_method.npz"))
    pl, _, losses, idx = _replay(fx, True, wrap=True)
    assert idx == fx["idx"].tolist()
    _close(losses, fx["loss"], "loss")


def _data(n, obs, A, seed, p_term=0.1):
    rng = np.random.Generator(np.random.PCG64(seed))
    q8 = lambda x: (np.rint(x * 256) / 256).astype(np.float32)  # noqa: E731
    return dict(state=q8(rng.standard_normal((n, obs))), next_state=q8(rng.standard_normal((n, obs))),
                reward=q8(rng.standard_normal(n)), terminated=rng.random(n) < p_term, truncated=rng.random(n) < 0.05,
                action=rng.integers(0, A, size=n).astype(np.int32), next_action=rng.integers(0, A, size=n).astype(np.int32))


def _buffer(d, A, device=False, dynamic=False, **kw):
    import pearl_b200
    n = len(d["action"])
    buf = pearl_b200.B200SARSAReplayBuffer(n, **kw)
    t = (lambda x: torch.as_tensor(x).cuda()) if device else torch.as_tensor
    extra = {}
    if dynamic:
        ids = np.tile(np.arange(A), (n, 1))[:, ::-1].copy()
        extra = dict(next_available_ids=t(ids).to(torch.uint8), next_available_count=t(np.full(n, max(A - 1, 1))).to(torch.int32))
    buf.push_batch(t(d["state"]), t(d["action"]), t(d["reward"]), t(d["next_state"]), t(d["terminated"]), t(d["truncated"]),
                   max_number_actions=A, next_action=t(d["next_action"]), **extra)
    return buf


def _batch(d, i, A, one_hot_form=False):
    import pearl_b200
    g = lambda k: torch.from_numpy(np.asarray(d[k][i]))  # noqa: E731
    a, na = g("action").long().view(-1, 1), g("next_action").long().view(-1, 1)
    if one_hot_form:
        a, na = torch.eye(A)[a.view(-1)], torch.eye(A)[na.view(-1)]
    return pearl_b200.TransitionBatch(state=g("state"), action=a, reward=g("reward"), next_state=g("next_state"),
                                      next_action=na, terminated=g("terminated"), truncated=g("truncated"))


def _vecs(pl):
    st = pl.adam_state()
    return [pl.flat_parameters.cpu(), pl.flat_target_parameters.cpu()] + [st[k].cpu() for k in ("exp_avg", "exp_avg_sq", "max_exp_avg_sq")]


@pytest.mark.parametrize("engine", [0, 1, 2])
def test_sarsa_stress_shape_against_oracle(engine):
    """obs 128, 16 actions, [256, 256], batch 256, one learn_batch round at a time from the oracle's state (learn()
    equals learn_batch bit for bit, test_sarsa_learn_batch_equals_learn), target update every second round."""
    from pearl_b200 import _lib
    torch.manual_seed(7)
    threads = torch.get_num_threads()
    torch.set_num_threads(8)
    obs, A, H, n, B, R, lr = 128, 16, 256, 3000, 256, 4, 1e-3
    d = _data(n, obs, A, seed=11)
    orc = OracleSARSA(obs, A, (H, H), lr=lr, gamma=0.99, tau=0.1, target_update_freq=2)
    lib = _lib.load()
    prev = lib.prl_get_contraction_engine()
    _lib.check(lib.prl_set_contraction_engine(engine))
    try:
        pl = _learner(obs, A, (H, H), training_rounds=1, batch_size=B, learning_rate=lr, target_update_freq=2, soft_update_tau=0.1)
        rng = np.random.Generator(np.random.PCG64(19))
        for r in range(R):
            load_flat(pl._Q, flat(orc.Q))
            load_flat(pl._Q_target, flat(orc.Qt))
            st, params = pl.adam_state(), list(orc.Q.parameters())
            if params[0] in orc.opt.state:
                for key in ("exp_avg", "exp_avg_sq", "max_exp_avg_sq"):
                    st[key].copy_(torch.cat([orc.opt.state[p][key].reshape(-1) for p in params]))
            i = rng.choice(n, size=B, replace=False)
            orc.training_steps = pl._training_steps = r
            b = one_hot({k: torch.from_numpy(d[k][i]) for k in ("state", "action", "reward", "next_state", "next_action", "terminated")}, A)
            skip = _relu_boundary(orc.Q, torch.cat([b["state"], b["action"]], 1))
            rep = pl.learn_batch(_batch(d, i, A))
            loss = orc.learn_batch(b)
            _close(rep["loss"], loss, f"round {r} loss")
            _close_net(pl.flat_parameters.cpu().numpy(), orc.Q, skip, f"round {r} online", lr)
            _close_params(pl.flat_target_parameters.cpu().numpy(), flat(orc.Qt).numpy(), f"round {r} target", lr, 1)
    finally:
        _lib.check(lib.prl_set_contraction_engine(prev))
        torch.set_num_threads(threads)


def test_sarsa_is_bit_reproducible():
    """One call of R rounds == R one-round calls == chunks of 4; graph replay == plain launches; two runs agree."""
    n, obs, A, B, R = 1500, 24, 6, 128, 9
    d = _data(n, obs, A, seed=23)

    def run(per_call, graph):
        buf = _buffer(d, A, dynamic=True)
        torch.manual_seed(3)
        pl = _learner(obs, A, (64, 64), training_rounds=R, batch_size=B, max_rounds_per_call=per_call, target_update_freq=4)
        pl.use_cuda_graph = graph
        random.seed(29)
        rep = pl.learn(buf)
        rep["batch"] = pl.learn_batch(_batch(d, np.arange(B), A))
        return rep, _vecs(pl)

    base_rep, base = run(R, True)
    for per_call, graph in [(1, True), (R, False), (R, True), (4, True)]:
        rep, vecs = run(per_call, graph)
        assert rep == base_rep, (per_call, graph)
        for a, b in zip(vecs, base):
            assert torch.equal(a, b), (per_call, graph)


class _Foreign:
    def __init__(self, batches):
        self.batches = list(batches)

    def __len__(self):
        return 10 ** 6

    def sample(self, k):
        return self.batches.pop(0)


@pytest.mark.parametrize("one_hot_form", [True, False])
def test_sarsa_learn_batch_equals_learn(one_hot_form):
    """learn_batch on the rows a one-round learn() gathered, at the same training-step count, and learn() over a foreign
    buffer returning those rows, leave every vector bit-identical to learn() (target update included: freq 2)."""
    n, obs, A, B = 800, 12, 5, 96
    d = _data(n, obs, A, seed=43)
    buf = _buffer(d, A)

    def mk():
        torch.manual_seed(5)
        return _learner(obs, A, (64, 64), training_rounds=1, batch_size=B, target_update_freq=2)
    a, b, c = mk(), mk(), mk()
    random.seed(3)
    rep_a = a.learn(buf, trace=True)
    rows = rep_a["idx"][0].cpu().numpy()
    b._training_steps = 1
    rep_b = b.learn_batch(_batch(d, rows, A, one_hot_form))
    rep_c = c.learn(_Foreign([_batch(d, rows, A, one_hot_form)]))
    assert rep_a["loss"][0] == rep_b["loss"] == rep_c["loss"][0]
    for x, y, z in zip(_vecs(a), _vecs(b), _vecs(c)):
        assert torch.equal(x, y) and torch.equal(x, z)


def test_sarsa_launch_count_graph_cache_and_learning_rate():
    """19 launches per round; an lr change keeps the handle and its graph."""
    n, obs, A, B = 600, 8, 4, 64
    d = _data(n, obs, A, seed=31)
    buf = _buffer(d, A)
    pl = _learner(obs, A, (32, 32), training_rounds=5, batch_size=B)
    rep = pl.learn(buf, trace=True)
    assert rep["launches"] == 5 * LAUNCHES_PER_ROUND == pl.launch_info()["launches"]
    assert rep["graph_captures"] == 1
    h = pl._handle.value
    before = pl.flat_parameters.clone()
    pl.optimizer.param_groups[0]["lr"] = 0.0
    pl.learn(buf)
    assert pl._handle.value == h and torch.equal(pl.flat_parameters, before)
    pl.optimizer.param_groups[0]["lr"] = 1e-3
    pl.learn(buf)
    assert pl._handle.value == h and not torch.equal(pl.flat_parameters, before)
    assert pl.launch_info()["graph_captures"] == 1


def test_sarsa_graph_cache_on_policy_loop():
    """PearlAgent's on-policy loop on ONE buffer: push an episode, learn, clear.  Batch sizes seen before replay their
    graph: the capture count equals the number of distinct batch sizes."""
    import pearl_b200
    obs, A = 6, 3
    rng = np.random.Generator(np.random.PCG64(5))
    pl = _learner(obs, A, (32, 32), training_rounds=2, batch_size=32)
    buf = pearl_b200.B200SARSAReplayBuffer(1000)
    lengths = [10, 20, 10, 40, 20, 10, 40, 7]
    for L in lengths:
        d = _data(L, obs, A, seed=int(rng.integers(1 << 30)))
        buf.push_batch(d["state"], d["action"], d["reward"], d["next_state"], d["terminated"], d["truncated"],
                       max_number_actions=A, next_action=d["next_action"])
        pl.learn(buf)
        buf.clear()
    assert pl.launch_info()["graph_captures"] == len({min(L, 32) for L in lengths})


def test_sarsa_checkpoint_views_and_optimizer_load_state_dict():
    n, obs, A, B = 400, 6, 3, 32
    d = _data(n, obs, A, seed=53)
    pl = _learner(obs, A, (32, 32), training_rounds=2, batch_size=B)
    batch = _batch(d, np.arange(B), A)
    pl.learn_batch(batch)
    w, m = pl.flat_parameters, pl.adam_state()["exp_avg"]
    params = list(pl._Q.parameters())
    assert all(w.data_ptr() <= p.data_ptr() < w.data_ptr() + 4 * w.numel() for p in params)
    assert pl.optimizer.state[params[0]]["exp_avg"].data_ptr() == m.data_ptr()
    ck = copy.deepcopy((pl._Q.state_dict(), pl._Q_target.state_dict(), pl.optimizer.state_dict()))
    pl.learn_batch(batch)
    want = _vecs(pl)
    step = pl.adam_state()["step"]
    pl.learn_batch(batch)
    pl._Q.load_state_dict(ck[0])
    pl._Q_target.load_state_dict(ck[1])
    pl.optimizer.load_state_dict(ck[2])
    pl.learn_batch(batch)
    assert pl.adam_state()["step"] == step
    for x, y in zip(_vecs(pl), want):
        assert torch.equal(x, y)


def test_sarsa_q_values_and_act_equal_the_dqn_learner():
    import pearl_b200
    n, obs, A = 300, 10, 7
    d = _data(n, obs, A, seed=61)
    torch.manual_seed(9)
    pl = _learner(obs, A, (48, 40), batch_size=4)
    ref = pearl_b200.B200DeepQLearning(state_dim=obs, action_space=_Space(range(A)), hidden_dims=[48, 40],
                                       action_representation_module=pearl_b200.OneHotActionTensorRepresentationModule(A)).to("cuda:0")
    load_flat(ref._Q, flat(pl._Q).cpu())
    load_flat(ref._Q_target, flat(pl._Q_target).cpu())
    s = torch.from_numpy(d["state"])
    for rows in (1, 3, 64, 300):       # more rows than max_batch / A: chunks through the workspace
        for target in (False, True):
            _close(pl.q_values(s[:rows], target=target).cpu().numpy(), ref.q_values(s[:rows], target=target).cpu().numpy(),
                   f"q_values rows {rows} target {target}")
    for k in range(10):
        assert int(pl.act(s[k], _Space(range(A)), exploit=True)) == int(ref.act(s[k], _Space(range(A)), exploit=True))


def test_sarsa_buffer_storage():
    """Host and device push_batch (and the multi-buffer push) give bit-identical records; sample().next_action is the
    pushed one; the upgrade to dynamic sets keeps the next actions; state_dict round-trips records and the cache."""
    import pearl_b200
    from pearl_b200 import _lib
    from pearl_b200.replay_buffer import _stream_ptr
    n, obs, A = 50, 5, 7
    d = _data(n, obs, A, seed=71)
    host, dev = _buffer(d, A), _buffer(d, A, device=True)
    rec = lambda b: b.state_dict()["records"]  # noqa: E731
    assert torch.equal(rec(host), rec(dev))
    assert (rec(host)[:, host._layout.off_flags] >> 24 & 0xff).tolist() == d["next_action"].tolist()
    bufs = [pearl_b200.B200SARSAReplayBuffer(n) for _ in range(2)]
    for b in bufs:                              # allocate with one push, then clear
        b.push_batch(d["state"][:1], d["action"][:1], d["reward"][:1], d["next_state"][:1], d["terminated"][:1],
                     d["truncated"][:1], max_number_actions=A, next_action=d["next_action"][:1])
        b.clear()
    st = lambda k, dt: torch.from_numpy(np.stack([d[k], d[k]])).to(dt).contiguous()  # noqa: E731
    arrs = [st("state", torch.float32), st("action", torch.int32), st("reward", torch.float32), st("next_state", torch.float32),
            st("terminated", torch.uint8), st("truncated", torch.uint8), st("next_action", torch.int32)]
    lib = bufs[0]._lib
    _lib.check(lib.prl_buf_push_host_multi_sarsa((C.c_void_p * 2)(*[b.handle.value for b in bufs]), 2, n,
                                                 *[_lib.ptr(a) for a in arrs], _stream_ptr(bufs[0].device)))
    for b in bufs:
        assert torch.equal(rec(b), rec(host))
    # sample(): next_action [B, 1] int64 of the sampled rows
    random.seed(4)
    logical, _ = host.sample_indices(20, 1)
    random.seed(4)
    tb = host.sample(20)
    assert tb.next_action.dtype == torch.int64 and tuple(tb.next_action.shape) == (20, 1)
    assert tb.next_action.view(-1).cpu().tolist() == d["next_action"][logical[0].cpu().numpy()].tolist()
    # the upgrade to dynamic next-action sets re-packs the records and keeps the next actions
    ids = torch.zeros(1, A, dtype=torch.uint8)
    ids[0, :2] = torch.tensor([3, 1])
    host.push_batch(d["state"][:1], d["action"][:1], d["reward"][:1], d["next_state"][:1], d["terminated"][:1],
                    d["truncated"][:1], next_available_ids=ids, next_available_count=torch.tensor([2], dtype=torch.int32),
                    next_action=torch.tensor([5]))
    assert host._desc.flags & _lib.PRL_BUF_DYNAMIC_ACTIONS
    r = rec(host)
    want = d["next_action"][1:].tolist() + [5]
    assert (r[:, host._layout.off_flags] >> 24 & 0xff).tolist() == want
    assert (r[:, host._layout.off_flags] >> 8 & 0xffff).tolist()[-1] == 2
    # state_dict with a pending cache, mid-episode
    host.push(state=torch.zeros(obs), action=torch.tensor([2]), reward=1.0, terminated=False, truncated=False,
              next_state=torch.ones(obs), max_number_actions=A)
    sd = host.state_dict()
    other = pearl_b200.B200SARSAReplayBuffer(n)
    other.load_state_dict(sd)
    assert torch.equal(rec(other), rec(host)) and other.cache is not None and other.cache["action"] == 2
    other.clear()
    assert len(other) == 0 and other.cache is not None                   # clear() keeps the cache
    other.push(state=torch.ones(obs), action=torch.tensor([6]), reward=0.0, terminated=True, truncated=False,
               next_state=torch.zeros(obs), max_number_actions=A)
    tb = other.sample(2)
    assert sorted(tb.next_action.view(-1).tolist()) == [6, 6] and sorted(tb.action.view(-1).tolist()) == [2, 6]


def test_sarsa_buffer_and_learner_refusals():
    import pearl_b200
    from pearl_b200 import _lib
    from pearl_b200.replay_buffer import _stream_ptr
    n, obs, A, B = 64, 6, 4, 16
    d = _data(n, obs, A, seed=41)
    sarsa_buf = _buffer(d, A)
    t = lambda k, dt: torch.from_numpy(d[k]).to(dt).contiguous()  # noqa: E731
    args = [_lib.ptr(t("state", torch.float32)), _lib.ptr(t("action", torch.int32)), _lib.ptr(t("reward", torch.float32)),
            _lib.ptr(t("next_state", torch.float32)), _lib.ptr(t("terminated", torch.uint8)), _lib.ptr(t("truncated", torch.uint8)),
            None, None]
    lib = sarsa_buf._lib
    for fn in (lib.prl_buf_push_host, lib.prl_buf_push_device):     # the plain entries would store next action 0
        assert fn(sarsa_buf.handle, 4, *args, _stream_ptr(sarsa_buf.device)) == _lib.PRL_EINVAL
    assert lib.prl_buf_push_host_multi((C.c_void_p * 1)(sarsa_buf.handle.value), 1, 4, *args[:6],
                                       _stream_ptr(sarsa_buf.device)) == _lib.PRL_EINVAL
    plain = pearl_b200.B200ReplayBuffer(n)
    plain.push_batch(d["state"], d["action"], d["reward"], d["next_state"], d["terminated"], d["truncated"], max_number_actions=A)
    na = t("next_action", torch.int32)
    assert lib.prl_buf_push_host_sarsa(plain.handle, 4, *args, _lib.ptr(na), _stream_ptr(plain.device)) == _lib.PRL_EINVAL
    bad = na.clone()
    bad[2] = A
    assert lib.prl_buf_push_host_sarsa(sarsa_buf.handle, 4, *args, _lib.ptr(bad), _stream_ptr(plain.device)) == _lib.PRL_EINVAL
    assert len(sarsa_buf) == n
    with pytest.raises(ValueError, match="next_action"):
        sarsa_buf.push_batch(d["state"], d["action"], d["reward"], d["next_state"], d["terminated"], d["truncated"])
    pl = _learner(obs, A, (16, 16), training_rounds=2, batch_size=B)
    with pytest.raises(ValueError, match="B200SARSAReplayBuffer"):
        pl.learn(plain)
    per = pearl_b200.B200PrioritizedReplayBuffer(n)
    per.push_batch(d["state"], d["action"], d["reward"], d["next_state"], d["terminated"], d["truncated"], max_number_actions=A)
    with pytest.raises(NotImplementedError):
        pl.learn(per)
    with pytest.raises(AssertionError, match="next action"):
        pl.learn_batch(pearl_b200.TransitionBatch(state=torch.zeros(B, obs), action=torch.zeros(B, 1), reward=torch.zeros(B),
                                                  next_state=torch.zeros(B, obs), terminated=torch.zeros(B, dtype=torch.bool)))
    with pytest.raises(ValueError):
        pl.learn_batch(pearl_b200.TransitionBatch(state=torch.zeros(B, obs), action=torch.zeros(B, 1), reward=torch.zeros(B),
                                                  next_state=torch.zeros(B, obs), next_action=torch.full((B, 1), A),
                                                  terminated=torch.zeros(B, dtype=torch.bool)))
    pl.learn(sarsa_buf)
    dev = pl._device
    out = torch.zeros(4, dtype=torch.float32, device=dev)
    for buf, rounds, batch in ((plain, 1, B), (sarsa_buf, 1, B + 1), (sarsa_buf, 4097, B)):
        before = pl.flat_parameters.clone()
        rng0 = buf.get_rng_state()
        rc = pl._libh.prl_sarsa_learn(pl._handle, buf.handle, rounds, batch, 0, _lib.ptr(out), None, _stream_ptr(dev))
        assert rc == _lib.PRL_EINVAL, _lib.last_error()
        torch.cuda.synchronize()
        assert np.array_equal(buf.get_rng_state(), rng0), "the sampler ran"
        assert torch.equal(before, pl.flat_parameters), "a learner kernel ran"
