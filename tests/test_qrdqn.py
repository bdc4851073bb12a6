"""Quantile Regression DQN on the GPU (pearl_b200.B200QuantileRegressionDeepQLearning, csrc/qrdqn.cu) against
(a) the recordings of the reference's PearlAgent(QuantileRegressionDeepQLearning, BasicReplayBuffer)
    (tests/golden/qrdqn_*.npz: learn() with the same indices from CPython's `random.sample`, and agent.learn_batch() on
    sampled batches), elementwise 1e-4 (tests/_tol.py);
(b) oracle/qrdqn_oracle.py at a stress shape (obs 128, 16 actions, [256, 256], N = 200, batch 256, dynamic next sets,
    beta = 0.5), step by step from a re-synchronised state, under the SIMT engine and the tensor-core engine;
plus bit-identity (run to run, graph replay, round chunking, learn_batch vs learn), the launch count, a learning-rate
change on the same handle and the rejected inputs."""
import ctypes as C
import os
import random

import numpy as np
import pytest
import torch

from conftest import GOLDEN
from oracle.pearl_oracle import flat
from oracle.qrdqn_oracle import OracleQRDQN

pytestmark = pytest.mark.gpu

from _tol import close as _close, close_params as _close_params  # noqa: E402
from test_iql import _close_net, _relu_boundary  # noqa: E402

LAUNCHES_PER_ROUND = 19     # 11 contractions + 8 small kernels (DESIGN.md §3.4)


def _buffer(n, d, A, dynamic, **kw):
    import pearl_b200
    buf = pearl_b200.B200ReplayBuffer(n, **kw)
    t = torch.as_tensor
    extra = dict(next_available_ids=t(d["next_ids"]).to(torch.uint8), next_available_count=t(d["next_count"]).to(torch.int32)) \
        if dynamic else {}
    buf.push_batch(t(d["state"]), t(d["action"]).to(torch.int32), t(d["reward"]), t(d["next_state"]), t(d["terminated"]),
                   torch.zeros(n, dtype=torch.bool), max_number_actions=A, **extra)
    return buf


def _learner(obs, A, hidden, N, **kw):
    import pearl_b200
    return pearl_b200.B200QuantileRegressionDeepQLearning(state_dim=obs, n_actions=A, hidden_dims=list(hidden), num_quantiles=N, **kw)


def _batch(d, i, A, one_hot=True):
    """A TransitionBatch of rows i as the reference's preprocess_batch leaves it (one-hot actions and next slots) or with
    raw ids; next_unavailable_actions_mask from the stored counts."""
    import pearl_b200
    t = lambda k: torch.from_numpy(np.asarray(d[k][i]))  # noqa: E731
    a, nid = t("action").long(), t("next_ids").long()
    if one_hot:
        a, nid = torch.nn.functional.one_hot(a, A).float(), torch.nn.functional.one_hot(nid, A).float()
    else:
        a, nid = a.view(-1, 1), nid.view(len(i), A, 1).float()
    mask = torch.arange(A).view(1, A) >= t("next_count").view(-1, 1)
    return pearl_b200.TransitionBatch(state=t("state"), action=a, reward=t("reward"), next_state=t("next_state"),
                                      terminated=t("terminated"), next_available_actions=nid, next_unavailable_actions_mask=mask)


def _max_exp_avg_sq(fx):
    v = fx["adam_exp_avg_sq"].copy()
    v[fx["adam_max_exp_avg_sq_idx"]] = fx["adam_max_exp_avg_sq_val"]
    return v


@pytest.mark.parametrize("case", ["qrdqn_neutral", "qrdqn_variance", "qrdqn_lr", "qrdqn_batch"])
def test_qrdqn_matches_reference_recording(case):
    fx = np.load(os.path.join(GOLDEN, f"{case}.npz"))
    n, R, B, calls, A = int(fx["n"]), int(fx["rounds"]), int(fx["batch"]), int(fx["calls"]), int(fx["n_actions"])
    buf = _buffer(n, fx, A, bool(fx["dynamic"]))
    pl = _learner(int(fx["obs"]), A, fx["hidden"].tolist(), int(fx["num_quantiles"]), learning_rate=float(fx["lr"]),
                  discount_factor=float(fx["gamma"]), training_rounds=R, batch_size=B, target_update_freq=int(fx["target_update_freq"]),
                  soft_update_tau=float(fx["tau"]), variance_weighting_coefficient=float(fx["beta"]))
    pl.load_parameters(fx["init_q"])
    random.setstate((3, tuple(int(x) for x in fx["rng_before"]), None))
    losses, idx, handles = [], [], []
    for c in range(calls):
        pl.set_learning_rate(float(fx["call_lr"][c]))
        if bool(fx["learn_batch"]):         # agent.learn_batch(buf.sample(batch))
            logical, _ = buf.sample_indices(B, 1)
            i = logical[0].cpu().numpy()
            idx.append(i.tolist())
            losses.append(pl.learn_batch(_batch(fx, i, A))["loss"])
        else:
            trace = {}
            losses += pl.learn(buf, trace=trace)["loss"]
            idx += trace["idx"].tolist()
        handles.append(pl._handle.value)
        _close(pl.params.cpu().numpy(), fx["q_calls"][c], f"online net after call {c}")
        _close(pl.target_params.cpu().numpy(), fx["qt_calls"][c], f"target net after call {c}")
    assert len(set(handles)) == 1, "a learning-rate change re-created the C handle"
    assert pl._training_steps == (0 if bool(fx["learn_batch"]) else R * calls)
    assert idx == fx["idx"].tolist()                                                  # bit-exact sampling
    assert random.getstate()[1] == tuple(int(x) for x in fx["rng_after"])              # CPython's random as the reference left it
    _close(losses, fx["loss"], "loss")
    for i, want in enumerate((fx["adam_exp_avg"], fx["adam_exp_avg_sq"], _max_exp_avg_sq(fx))):
        _close(pl._state[i].cpu().numpy(), want, f"AdamW state {i}", atol=1e-9)


def _data(n, obs, A, seed, p_term=0.1):
    rng = np.random.Generator(np.random.PCG64(seed))
    q8 = lambda x: (np.rint(x * 256) / 256).astype(np.float32)  # noqa: E731
    d = dict(state=q8(rng.standard_normal((n, obs))), next_state=q8(rng.standard_normal((n, obs))), reward=q8(rng.standard_normal(n)),
             terminated=rng.random(n) < p_term, action=rng.integers(0, A, size=n).astype(np.int32))
    ids, cnt = np.zeros((n, A), np.int64), np.zeros(n, np.int32)
    for k in range(n):
        m = int(rng.integers(1, A + 1))
        ids[k, :m] = np.sort(rng.choice(A, size=m, replace=False))
        cnt[k] = m
    d.update(next_ids=ids, next_count=cnt)
    return d


def _adam_flat(opt, params, key):
    return torch.cat([opt.state[p][key].reshape(-1) for p in params])


@pytest.mark.parametrize("engine", [0, 2])
def test_qrdqn_stress_shape_against_oracle(engine):
    """obs 128, 16 actions, [256, 256], N = 200, batch 256, dynamic next sets, beta 0.5 (B*A = 4096 target rows: the
    automatic engine puts layers 2 and 3 of the target pass on the wgmma tiles), one learn_batch round at a time (learn()
    equals learn_batch bit for bit, test_qrdqn_learn_batch_equals_learn_bit_for_bit).  Each round starts from the oracle's
    state (parameters, target and AdamW moments); the loss and the parameters must agree elementwise to 1e-4 up to the
    counted AdamW outliers of `close_params`; the weight rows of hidden units at the ReLU boundary are held to one AdamW
    step instead (`_relu_boundary`, as in test_iql.py).  A slot whose risk value lies within fp32 summation noise (1e-4 relative)
    of its row's best could win under another summation order: such slots are masked on both sides (a non-prefix mask,
    which learn_batch compacts), so both pick the same greedy slot."""
    from pearl_b200 import TransitionBatch, _lib
    torch.manual_seed(7)
    threads = torch.get_num_threads()
    torch.set_num_threads(8)
    obs, A, H, N, n, B, R, lr, beta = 128, 16, 256, 200, 3000, 256, 6, 5e-4, 0.5
    d = _data(n, obs, A, seed=11)
    orc = OracleQRDQN(obs, A, (H, H), N, lr=lr, gamma=0.99, tau=0.05)
    lib = _lib.load()
    prev = lib.prl_get_contraction_engine()
    _lib.check(lib.prl_set_contraction_engine(engine))
    masked = 0
    try:
        pl = _learner(obs, A, (H, H), N, training_rounds=1, batch_size=B, learning_rate=lr, target_update_freq=2,
                      variance_weighting_coefficient=beta)
        pl.load_parameters(flat(orc.q), flat(orc.qt))
        rng = np.random.Generator(np.random.PCG64(19))
        for r in range(R):
            i = rng.choice(n, size=B, replace=False)
            t = lambda k: torch.from_numpy(np.asarray(d[k][i]))  # noqa: E731
            b = dict(state=t("state"), action=t("action"), reward=t("reward"), next_state=t("next_state"), terminated=t("terminated"),
                     next_ids=t("next_ids"), next_mask=torch.arange(A).view(1, A) >= t("next_count").view(-1, 1))
            _, g, rho = orc.target(b, beta)
            best = rho.gather(1, g.view(-1, 1))
            near = (best - rho <= 1e-4 * (1.0 + best.abs())) & ~b["next_mask"]
            near[torch.arange(B), g] = False
            masked += int(near.sum())
            b["next_mask"] = b["next_mask"] | near
            pl._training_steps = r
            skip = _relu_boundary(orc.q, torch.cat([b["state"], torch.nn.functional.one_hot(b["action"].long(), A).float()], dim=-1))
            rep = pl.learn_batch(TransitionBatch(state=b["state"], action=b["action"].long().view(-1, 1), reward=b["reward"],
                                                 next_state=b["next_state"], terminated=b["terminated"],
                                                 next_available_actions=b["next_ids"].float().view(B, A, 1),
                                                 next_unavailable_actions_mask=b["next_mask"]))
            loss = orc.learn_batch(b, beta, (r + 1) % 2 == 0)
            _close(rep["loss"], loss, f"round {r} loss")
            _close_net(pl.params.cpu().numpy(), orc.q, skip, f"round {r} online", lr)
            _close_params(pl.target_params.cpu().numpy(), flat(orc.qt).numpy(), f"round {r} target", lr, 1)
            pl.load_parameters(flat(orc.q), flat(orc.qt))
            params = list(orc.q.parameters())
            for k, key in enumerate(("exp_avg", "exp_avg_sq", "max_exp_avg_sq")):
                pl._state[k].copy_(_adam_flat(orc.opt, params, key))
        print(f"    {masked} near-tie slots masked over {R} rounds")
    finally:
        _lib.check(lib.prl_set_contraction_engine(prev))
        torch.set_num_threads(threads)


def _vecs(pl):
    return [pl.params.cpu(), pl.target_params.cpu()] + [s.cpu() for s in pl._state]


def test_qrdqn_is_bit_reproducible():
    """One call of R rounds == R one-round calls (max_rounds_per_call=1); CUDA-graph replay == plain launches; two runs
    agree.  Bit for bit: the launch sequence and every summation order are fixed."""
    n, obs, A, B, R, N = 1500, 24, 6, 128, 9, 51
    d = _data(n, obs, A, seed=23)

    def run(per_call, graph):
        buf = _buffer(n, d, A, True)
        pl = _learner(obs, A, (64, 64), N, training_rounds=R, batch_size=B, max_rounds_per_call=per_call, seed=3, target_update_freq=4,
                      variance_weighting_coefficient=1.5)
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


@pytest.mark.parametrize("one_hot", [True, False])
def test_qrdqn_learn_batch_equals_learn_bit_for_bit(one_hot):
    """learn_batch on the rows a one-round learn() gathered, at the same training-step count, leaves every vector
    bit-identical (target update included: freq 1)."""
    n, obs, A, B, N = 800, 12, 5, 96, 20
    d = _data(n, obs, A, seed=43)
    buf = _buffer(n, d, A, True)
    mk = lambda: _learner(obs, A, (64, 64), N, training_rounds=1, batch_size=B, seed=5, target_update_freq=1,  # noqa: E731
                          variance_weighting_coefficient=0.7)
    a, b = mk(), mk()
    random.seed(3)
    trace = {}
    rep_a = a.learn(buf, trace=trace)
    b._training_steps = 1            # learn() counted its round before the update check
    rep_b = b.learn_batch(_batch(d, trace["idx"][0].numpy(), A, one_hot=one_hot))
    assert rep_a["loss"][0] == rep_b["loss"]
    for x, y in zip(_vecs(a), _vecs(b)):
        assert torch.equal(x, y)


def test_qrdqn_launch_count_and_learning_rate_change():
    n, obs, A, B, N = 600, 8, 4, 64, 10
    d = _data(n, obs, A, seed=31)
    buf = _buffer(n, d, A, False)
    pl = _learner(obs, A, (32, 32), N, training_rounds=5, batch_size=B)
    trace = {}
    pl.learn(buf, trace=trace)
    assert trace["launches"] == 5 * LAUNCHES_PER_ROUND
    h = pl._handle.value
    before = pl.params.clone()
    pl.set_learning_rate(0.0)                       # lr 0: AdamW moves nothing, decay factor 1
    pl.learn(buf)
    assert pl._handle.value == h
    assert torch.equal(pl.params, before)
    pl.set_learning_rate(1e-3)
    pl.learn(buf)
    assert pl._handle.value == h and not torch.equal(pl.params, before)


def test_qrdqn_rejects_bad_inputs():
    import pearl_b200
    from pearl_b200 import _lib
    from pearl_b200.replay_buffer import _stream_ptr
    n, obs, A, B, N = 64, 6, 4, 16, 8
    d = _data(n, obs, A, seed=41)
    pl = _learner(obs, A, (16, 16), N, training_rounds=2, batch_size=B)
    assert pl.learn(pearl_b200.B200ReplayBuffer(16)) == {}                  # empty buffer: nothing to do
    with pytest.raises(NotImplementedError):                                # three hidden layers
        _learner(obs, A, (16, 16, 16), N)
    for bad_n in (0, 257):                                                  # num_quantiles outside [1, 256]
        with pytest.raises(ValueError):
            _learner(obs, A, (16, 16), bad_n)
    _learner(obs, A, (16, 16), 256)
    per = pearl_b200.B200PrioritizedReplayBuffer(n)
    per.push_batch(torch.from_numpy(d["state"]), torch.from_numpy(d["action"]), torch.from_numpy(d["reward"]),
                   torch.from_numpy(d["next_state"]), torch.from_numpy(d["terminated"]), torch.zeros(n, dtype=torch.bool),
                   max_number_actions=A)
    with pytest.raises(NotImplementedError):
        pl.learn(per)
    disc_buf = _buffer(n, d, A, False)
    cont_buf = pearl_b200.B200ReplayBuffer(n)
    cont_buf.is_action_continuous = True
    t = torch.from_numpy
    cont_buf.push_batch(t(d["state"]), torch.zeros(n, 2), t(d["reward"]), t(d["next_state"]), t(d["terminated"]),
                        torch.zeros(n, dtype=torch.bool))
    with pytest.raises(ValueError):
        pl.learn(cont_buf)
    dz = dict(d, state=np.zeros((n, obs + 1), np.float32), next_state=np.zeros((n, obs + 1), np.float32))
    other_obs = _buffer(n, dz, A, False)
    other_A = _buffer(n, dict(d, action=d["action"] % 3, next_ids=d["next_ids"][:, :3] % 3), A - 1, False)
    # the C entry point itself refuses these before the sampler or any learner kernel runs
    pl.learn(disc_buf)
    dev = pl._device
    out = torch.zeros(4, dtype=torch.float32, device=dev)
    for buf, rounds, batch in ((cont_buf, 1, B), (other_obs, 1, B), (other_A, 1, B), (disc_buf, 1, B + 1), (disc_buf, 1025, B)):
        before = [pl.params.clone(), pl.target_params.clone()]
        rng0 = buf.get_rng_state()
        rc = pl._lib.prl_qrdqn_learn(pl._handle, buf.handle, rounds, batch, 0, 0.0, _lib.ptr(out), C.c_void_p(0), _stream_ptr(dev))
        assert rc == _lib.PRL_EINVAL, _lib.last_error()
        torch.cuda.synchronize()
        assert np.array_equal(buf.get_rng_state(), rng0), "the sampler ran"
        assert all(torch.equal(x, y) for x, y in zip(before, [pl.params, pl.target_params])), "a learner kernel ran"
    x = torch.zeros((B + 1, obs), device=dev)
    i32 = torch.zeros(B + 1, dtype=torch.int32, device=dev)
    u8 = torch.zeros(B + 1, dtype=torch.uint8, device=dev)
    rc = pl._lib.prl_qrdqn_learn_batch(pl._handle, B + 1, _lib.ptr(x), _lib.ptr(i32), _lib.ptr(x[:, 0].contiguous()), _lib.ptr(x),
                                      _lib.ptr(u8), None, None, 0, 0.0, _lib.ptr(out), _stream_ptr(dev))
    assert rc == _lib.PRL_EINVAL
    # a shard of a multi-GPU buffer samples global slots: rejected before the sampler or any learner kernel runs
    sharded = pearl_b200.B200ReplayBuffer(n, rng="device")
    sharded.push_batch_sharded(0, 2, t(d["state"]), t(d["action"]), t(d["reward"]), t(d["next_state"]), t(d["terminated"]),
                               torch.zeros(n, dtype=torch.bool), max_number_actions=A)
    sharded.seed(5)
    rng0 = sharded.get_rng_state()
    params0 = pl.params.clone()
    with pytest.raises(ValueError, match="shard"):
        pl.learn(sharded)
    torch.cuda.synchronize()
    assert np.array_equal(sharded.get_rng_state(), rng0), "the sampler ran"
    assert torch.equal(params0, pl.params), "a learner kernel ran"
