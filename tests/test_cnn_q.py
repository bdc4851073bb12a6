"""The CNN DQN learner (csrc/cnnq.cu, pearl_b200/cnn_q.py) on the GPU: every recording of the reference
(tests/golden/cnnq_*.npz) with graphs on and off, the fp32 oracle (oracle/cnn_q_oracle.py) at Pong's shape for both
networks and both learners under the SIMT (0) and tensor-core (2) contraction engines, bit-identity run to run and
between graph replay and eager launches, the launch count, learning-rate changes, checkpoint views, act / q_values, and a
replay ring larger than 2^31 bytes."""
import copy
import os
import random

import numpy as np
import pytest
import torch

from _tol import close, close_params
from conftest import GOLDEN
from oracle import cnn_q_oracle as orc
from oracle.pearl_oracle import load_flat

pytestmark = pytest.mark.gpu

PONG = dict(input=(4, 84, 84), conv=[(32, 8, 4, 0), (64, 4, 2, 0), (64, 3, 1, 0)], hidden=[512], n_actions=6)
LEARN_CASES = ("cnnq_dqn", "cnnq_ddqn", "cnnq_mh_dqn", "cnnq_mh_ddqn", "cnnq_lr")


class _Space:
    def __init__(self, A):
        self.n = A
        self.actions = [torch.tensor([i]) for i in range(A)]
        self.actions_batch = torch.arange(A).view(A, 1)


def _net(spec):
    import pearl_b200
    C, H, W = spec["input"]
    cls = pearl_b200.CNNQValueMultiHeadNetwork if spec["multi"] else pearl_b200.CNNQValueNetwork
    return cls(input_width=W, input_height=H, input_channels_count=C, kernel_sizes=[c[1] for c in spec["conv"]],
               output_channels_list=[c[0] for c in spec["conv"]], strides=[c[2] for c in spec["conv"]],
               paddings=[c[3] for c in spec["conv"]], action_dim=spec["n_actions"], hidden_dims_fully_connected=list(spec["hidden"]),
               output_dim=spec["n_actions"] if spec["multi"] else 1)


def _learner(spec, double, init=None, **kw):
    import pearl_b200
    cls = pearl_b200.B200DoubleDQN if double else pearl_b200.B200DeepQLearning
    C, H, W = spec["input"]
    A = spec["n_actions"]
    pl = cls(state_dim=C * H * W, action_space=_Space(A), hidden_dims=list(spec["hidden"]), network_instance=_net(spec),
             action_representation_module=pearl_b200.OneHotActionTensorRepresentationModule(A), **kw).to("cuda:0")
    if init is not None:
        load_flat(pl._Q, init)
        load_flat(pl._Q_target, init)
    return pl


def _buffer(d, A, dynamic, **kw):
    import pearl_b200
    n = len(d["action"])
    buf = pearl_b200.B200ReplayBuffer(n, **kw)
    t = torch.as_tensor
    extra = dict(next_available_ids=t(d["next_ids"]).to(torch.uint8), next_available_count=t(d["next_count"]).to(torch.int32)) \
        if dynamic else {}
    buf.push_batch(t(np.asarray(d["state"])).float(), t(np.asarray(d["action"])).to(torch.int32), t(np.asarray(d["reward"])),
                   t(np.asarray(d["next_state"])).float(), t(np.asarray(d["terminated"])), torch.zeros(n, dtype=torch.bool),
                   max_number_actions=A, **extra)
    return buf


def _data(spec, n, seed, dynamic=False):
    rng = np.random.Generator(np.random.PCG64(seed))
    A = spec["n_actions"]
    d = dict(state=rng.integers(0, 256, (n,) + tuple(spec["input"]), dtype=np.uint8),
             next_state=rng.integers(0, 256, (n,) + tuple(spec["input"]), dtype=np.uint8),
             action=rng.integers(0, A, n).astype(np.int32), reward=rng.standard_normal(n).astype(np.float32),
             terminated=rng.random(n) < 0.15, next_ids=np.tile(np.arange(A), (n, 1)).astype(np.uint8), next_count=np.full(n, A, np.int32))
    if dynamic:
        for i in range(n):
            m = int(rng.integers(1, A + 1))
            d["next_ids"][i] = 0
            d["next_ids"][i, :m] = np.sort(rng.choice(A, size=m, replace=False))
            d["next_count"][i] = m
    return d


def _engine(engine):
    from pearl_b200 import _lib
    lib = _lib.init(0)
    prev = lib.prl_get_contraction_engine()
    _lib.check(lib.prl_set_contraction_engine(engine))
    return lib, prev


@pytest.mark.parametrize("graph", [True, False], ids=["graph", "eager"])
@pytest.mark.parametrize("case", LEARN_CASES)
def test_cnn_q_learn_matches_reference(case, graph):
    fx = np.load(os.path.join(GOLDEN, f"{case}.npz"))
    spec = orc.spec_of(fx)
    A, R, B = spec["n_actions"], int(fx["rounds"]), int(fx["batch"])
    buf = _buffer(fx, A, bool(fx["dynamic"]), rng="python")
    pl = _learner(spec, bool(fx["double"]), fx["init_q"], learning_rate=float(fx["lr"]), discount_factor=float(fx["gamma"]),
                  training_rounds=R, batch_size=B, target_update_freq=int(fx["target_update_freq"]), soft_update_tau=float(fx["tau"]))
    pl.use_cuda_graph = graph
    random.setstate((3, tuple(int(x) for x in fx["rng_before"]), None))
    for c in range(int(fx["calls"])):
        pl.optimizer.param_groups[0]["lr"] = float(fx["call_lr"][c])
        rep = pl.learn(buf, trace=True)
        assert rep["idx"].cpu().numpy().tolist() == fx["idx"][c * R:(c + 1) * R].tolist()
        close(rep["loss"], fx["loss"][c * R:(c + 1) * R], f"call {c} losses")
        close_params(pl.flat_parameters.cpu().numpy(), fx["q_calls"][c], f"call {c} online", float(fx["call_lr"][c]), (c + 1) * R)
        close_params(pl.flat_target_parameters.cpu().numpy(), fx["qt_calls"][c], f"call {c} target", float(fx["call_lr"][c]), (c + 1) * R)
    assert random.getstate()[1] == tuple(int(x) for x in fx["rng_after"])
    assert pl._training_steps == int(fx["training_steps"])
    st = pl.adam_state()
    assert st["step"] == int(fx["adam_step"])
    close(st["max_exp_avg_sq"].cpu().numpy(), fx["adam_max_exp_avg_sq"], "max_exp_avg_sq", rtol=2e-3, atol=1e-9)


@pytest.mark.parametrize("graph", [True, False], ids=["graph", "eager"])
@pytest.mark.parametrize("case", ("cnnq_batch_v", "cnnq_batch_mh"))
def test_cnn_q_learn_batch_matches_reference(case, graph):
    import pearl_b200
    fx = np.load(os.path.join(GOLDEN, f"{case}.npz"))
    spec = orc.spec_of(fx)
    A, B = spec["n_actions"], int(fx["batch"])
    pl = _learner(spec, bool(fx["double"]), fx["init_q"], learning_rate=float(fx["lr"]), discount_factor=float(fx["gamma"]),
                  training_rounds=1, batch_size=B, target_update_freq=int(fx["target_update_freq"]), soft_update_tau=float(fx["tau"]))
    pl.use_cuda_graph = graph
    for c, idx in enumerate(fx["idx"]):
        b = orc.batch_of(fx, idx)
        batch = pearl_b200.TransitionBatch(state=b["state"], action=torch.nn.functional.one_hot(b["action"], A).float(),
                                           reward=b["reward"], terminated=b["terminated"], next_state=b["next_state"])
        loss = pl.learn_batch(batch)["loss"]
        close(loss, fx["loss"][c], f"call {c} loss")
        close_params(pl.flat_parameters.cpu().numpy(), fx["q_calls"][c], f"call {c} online", float(fx["lr"]), c + 1)
        close_params(pl.flat_target_parameters.cpu().numpy(), fx["qt_calls"][c], f"call {c} target", float(fx["lr"]), c + 1)
    assert pl._training_steps == 0


@pytest.mark.parametrize("case", ("cnnq_act_v", "cnnq_act_mh"))
def test_cnn_q_act_and_q_values(case):
    fx = np.load(os.path.join(GOLDEN, f"{case}.npz"))
    spec = orc.spec_of(fx)
    A = spec["n_actions"]
    pl = _learner(spec, False, fx["init_q"])
    for i in range(len(fx["act"])):
        s = torch.from_numpy(fx["state"][i]).float().unsqueeze(0)
        assert int(pl.act(s, _Space(A), exploit=True)) == int(fx["act"][i])
        close(pl.q_values(s).cpu().numpy()[0], fx["q"][i], f"state {i} Q values")
    allq = pl.q_values(torch.from_numpy(fx["state"]).float()).cpu().numpy()
    close(allq, fx["q"], "batched Q values")
    with pytest.raises(ValueError, match="4-D"):
        pl.act(torch.from_numpy(fx["state"][0]).float(), _Space(A), exploit=True)


def _oracle_rounds(spec, double, d, idx, init, rounds, freq, lr, gamma=0.99, tau=0.1):
    st = dict(w=torch.from_numpy(init.copy()), wt=torch.from_numpy(init.copy()), step=0)
    st.update(m=torch.zeros_like(st["w"]), v=torch.zeros_like(st["w"]), vmax=torch.zeros_like(st["w"]))
    losses = []
    for r in range(rounds):
        losses.append(orc.round_step(spec, st, orc.batch_of(d, idx[r]), double=double, gamma=gamma, tau=tau, lr=lr,
                                     update_target=(r + 2) % freq == 0))
    return losses, st


@pytest.mark.parametrize("engine", [0, 2])
@pytest.mark.parametrize("multi,double", [(False, False), (False, True), (True, False), (True, True)],
                         ids=["dqn", "ddqn", "mh-dqn", "mh-ddqn"])
def test_cnn_q_pong_shape_matches_oracle(multi, double, engine):
    """Two rounds at Pong's shape, one learn() call each: round 1's gradient (recovered from exp_avg) against float64
    with the bound of test_gpu_cnn_q_shapes.py, both rounds' losses and the parameters after them against the fp32
    oracle (_close_steps)."""
    from oracle import cnn_q_fp64
    from test_gpu_cnn_q_shapes import C, OMB1, U
    torch.manual_seed(1)
    torch.set_num_threads(8)
    spec = dict(PONG, multi=multi)
    d = _data(spec, 96, seed=11, dynamic=double)
    lib, prev = _engine(engine)
    try:
        pl = _learner(spec, double, learning_rate=1e-4, training_rounds=1, batch_size=32, target_update_freq=2, soft_update_tau=0.1)
        assert sum(p.numel() for p in pl._Q.parameters()) == orc.param_count(spec)
        init = pl.flat_parameters.cpu().numpy().copy()
        buf = _buffer(d, 6, double, rng="python")
        rep = pl.learn(buf, trace=True)
        g = pl.adam_state()["exp_avg"].cpu().double() / OMB1
        wt1 = pl.flat_target_parameters.cpu().clone()
        rep2 = pl.learn(buf, trace=True)
        assert rep["launches"] == rep2["launches"] == _launches(spec, double)
    finally:
        lib.prl_set_contraction_engine(prev)
    idx = np.concatenate([rep["idx"].cpu().numpy(), rep2["idx"].cpu().numpy()])
    g64, scale, margin = cnn_q_fp64.step(spec, torch.from_numpy(init), wt1, orc.batch_of(d, idx[0]), double=double, gamma=0.99)
    R = 32 * 20 * 20
    bad = np.flatnonzero(((g - g64).abs() > (C + R * U / 32) * scale + 1e-30).numpy())
    ratio = ((g - g64).abs() / scale.clamp_min(1e-300)).numpy()
    ok = np.delete(ratio, bad)
    print(f"    round 1 gradient: max err / scale {float(ok.max()):.3e} outside the mask flips, bound {C + R * U / 32:.3e}; "
          f"smallest ReLU margin {margin:.1e}; elements past the bound: {bad.size} {bad[:8].tolist()}")
    # Pong's trunk has about 10^6 pre-activations per pass, and random data leave some within 1e-8 of their scale, where a
    # last-bit difference flips a ReLU mask: the gradient elements such a flip feeds are counted, at most 1e-4 of them
    # (test_gpu_cnn_q_shapes.py draws data without such pre-activations and holds every element)
    assert bad.size <= 1e-4 * g.numel(), f"{bad.size} gradient elements past the float64 bound"
    losses, st = _oracle_rounds(spec, double, d, idx, init, 2, 2, 1e-4)
    close(rep["loss"] + rep2["loss"], losses, "losses")
    _close_steps(pl, st, 1e-4, 2)


def _close_steps(pl, st, lr, rounds):
    """Parameters after `rounds` AdamW steps at Pong's shape.  The conv weight gradients sum 12 800 products with heavy
    cancellation, so an element whose gradient lies within rounding of zero can take its AdamW step (lr * m / sqrt(v),
    whatever the gradient's size) the other way than in the fp32 oracle: up to 0.5 % of the elements may differ, each by
    at most 2 lr per step (close_params); all others are held to 1e-4 relative plus 5 % of the steps taken.  The
    gradients themselves are held to float64 above and in test_gpu_cnn_q_shapes.py."""
    atol = 0.05 * lr * rounds
    close_params(pl.flat_parameters.cpu().numpy(), st["w"].numpy(), f"online after {rounds} rounds", lr, rounds, atol=atol, max_frac=5e-3)
    close_params(pl.flat_target_parameters.cpu().numpy(), st["wt"].numpy(), f"target after {rounds} rounds", lr, rounds, atol=atol,
                 max_frac=5e-3)


def _launches(spec, double):
    """Launches of one round (csrc/cnnq.cu): load, soft update; per trunk (target, online) an im2col and a product per
    layer and the feature transpose; the FC products and folds; the head (+ the broadcast kernel, multi-head); the
    backward FC products (+ the action-column gradient, vanilla); the feature transpose back, per conv layer a split
    weight-gradient product and its slice sum, below layer 1 a backward-data product and its col2im; AdamW; the report."""
    L, nf, multi = len(spec["conv"]), len(spec["hidden"]), spec["multi"]
    n = 2 + 2 * (2 * L + 1)
    if multi:
        n += 2 * (nf + 1) + 2
    else:
        n += (1 + 1 + nf) + (1 + 1 + nf) + (1 + nf if double else 0) + 1 + 1
    n += 2 * nf + 2 + 1 + 2 * L + 2 * (L - 1) + 2
    return n


def test_cnn_q_bit_identical_runs_and_graph_vs_eager():
    spec = dict(PONG, multi=False)
    d = _data(spec, 64, seed=5, dynamic=True)
    torch.manual_seed(3)
    init = _learner(spec, True).flat_parameters.cpu().numpy().copy()
    out = []
    for graph in (True, True, False):
        pl = _learner(spec, True, init, learning_rate=1e-4, training_rounds=3, batch_size=32, target_update_freq=2)
        pl.use_cuda_graph = graph
        buf = _buffer(d, 6, True, rng="device")
        buf.set_rng_state(np.arange(625, dtype=np.uint32) * 7 % 4096)
        rep = pl.learn(buf, trace=True)
        rep2 = pl.learn(buf, trace=True)
        out.append((rep["loss"] + rep2["loss"], pl.flat_parameters.cpu().numpy(), pl.flat_target_parameters.cpu().numpy()))
        assert rep2["launches"] == rep["launches"] == 3 * _launches(spec, True)
    for o in out[1:]:
        assert o[0] == out[0][0]
        assert np.array_equal(o[1], out[0][1]) and np.array_equal(o[2], out[0][2])


def test_cnn_q_set_lr_and_checkpoint_views():
    spec = dict(PONG, multi=True)
    d = _data(spec, 64, seed=6)
    torch.manual_seed(4)
    pl = _learner(spec, False, learning_rate=1e-4, training_rounds=1, batch_size=32, target_update_freq=100)
    buf = _buffer(d, 6, False, rng="python")
    random.seed(9)
    pl.learn(buf)
    handle = pl._handle.value
    # lr change: picked up through prl_cnnq_set_lr by the same handle, and the oracle agrees
    pl.optimizer.param_groups[0]["lr"] = 5e-4
    w0, wt0 = pl.flat_parameters.cpu().clone(), pl.flat_target_parameters.cpu().clone()
    ad = pl.adam_state()
    st = dict(w=w0, wt=wt0, m=ad["exp_avg"].cpu().clone(), v=ad["exp_avg_sq"].cpu().clone(), vmax=ad["max_exp_avg_sq"].cpu().clone(),
              step=ad["step"])
    rep = pl.learn(buf, trace=True)
    assert pl._handle.value == handle
    want = orc.round_step(spec, st, orc.batch_of(d, rep["idx"][0].cpu().numpy()), double=False, gamma=0.99, tau=0.1, lr=5e-4,
                          update_target=False)
    close(rep["loss"][0], want, "loss after the lr change")
    close_params(pl.flat_parameters.cpu().numpy(), st["w"].numpy(), "online after the lr change", 5e-4, 1)
    # checkpoint views: a state_dict round trip into the module and the optimizer is what the next call trains from
    sd, osd = {k: v.clone() for k, v in pl._Q.state_dict().items()}, copy.deepcopy(pl.optimizer.state_dict())
    pl.learn(buf)
    pl._Q.load_state_dict(sd)
    pl.optimizer.load_state_dict(osd)
    w1 = pl.flat_parameters.cpu().clone()
    assert torch.equal(w1, torch.cat([v.reshape(-1).cpu() for v in sd.values()]))
    assert pl.adam_state()["step"] == 2


def test_cnn_q_ring_past_2gb():
    """A Pong-shaped ring of 12 000 transitions (about 2.7 GB), pushed past the wrap: learn() trains on rows stored
    beyond byte offset 2^31 and matches the oracle."""
    import pearl_b200
    spec = dict(PONG, multi=False)
    cap, extra, chunk = 12000, 500, 500
    g = torch.Generator().manual_seed(0)
    base_s = torch.randint(0, 256, spec["input"], generator=g, dtype=torch.int32)
    base_n = torch.randint(0, 256, spec["input"], generator=g, dtype=torch.int32)
    n = cap + extra
    action = torch.randint(0, 6, (n,), generator=g, dtype=torch.int32)
    reward = torch.randn(n, generator=g)
    term = torch.rand(n, generator=g) < 0.1
    img = lambda base, i: ((base.unsqueeze(0) + 13 * i.view(-1, 1, 1, 1)) % 256).float()  # noqa: E731
    buf = pearl_b200.B200ReplayBuffer(cap, rng="python")
    for i0 in range(0, n, chunk):
        i = torch.arange(i0, min(n, i0 + chunk))
        buf.push_batch(img(base_s, i), action[i], reward[i], img(base_n, i), term[i], torch.zeros(len(i), dtype=torch.bool),
                       max_number_actions=6)
    assert len(buf) == cap and cap * buf.record_bytes > 2 ** 31
    torch.manual_seed(2)
    pl = _learner(spec, False, learning_rate=1e-4, training_rounds=2, batch_size=32, target_update_freq=2)
    init = pl.flat_parameters.cpu().numpy().copy()
    random.seed(17)
    rep = pl.learn(buf, trace=True)
    idx = rep["idx"].cpu().numpy()
    t = extra + idx                                      # the transition each logical index holds (oldest first)
    assert int((t % cap).max()) * buf.record_bytes >= 2 ** 31, "no row stored past byte offset 2^31 was sampled"
    rows = np.arange(n)
    d = dict(state=img(base_s, torch.from_numpy(rows[t.ravel()])).numpy().reshape(idx.size, *spec["input"]),
             next_state=img(base_n, torch.from_numpy(rows[t.ravel()])).numpy().reshape(idx.size, *spec["input"]),
             action=action.numpy()[t.ravel()], reward=reward.numpy()[t.ravel()], terminated=term.numpy()[t.ravel()],
             next_ids=np.tile(np.arange(6), (idx.size, 1)), next_count=np.full(idx.size, 6))
    losses, st = _oracle_rounds(spec, False, d, np.arange(idx.size).reshape(idx.shape), init, 2, 2, 1e-4)
    close(rep["loss"], losses, "losses")
    _close_steps(pl, st, 1e-4, 2)
