"""The CNN DQN restatement (oracle/cnn_q_oracle.py) against the recordings of the reference's DeepQLearning / DoubleDQN
with CNNQValueNetwork / CNNQValueMultiHeadNetwork (tests/golden/cnnq_*.npz), the fp64 oracle against the fp32 one, the
plugin's network parsing and refusals, the stand-in networks, and the act refusal of a 3-D state, all on the CPU."""
import os
import random

import numpy as np
import pytest
import torch

from conftest import GOLDEN
from oracle import cnn_q_fp64, cnn_q_oracle as orc

LEARN = ("cnnq_dqn", "cnnq_ddqn", "cnnq_mh_dqn", "cnnq_mh_ddqn", "cnnq_lr", "cnnq_batch_v", "cnnq_batch_mh")
PONG = dict(input_width=84, input_height=84, input_channels_count=4, kernel_sizes=[8, 4, 3], output_channels_list=[32, 64, 64],
            strides=[4, 2, 1], paddings=[0, 0, 0], action_dim=6, hidden_dims_fully_connected=[512])


@pytest.mark.parametrize("case", LEARN)
def test_cnn_q_oracle_reproduces_reference(case):
    torch.set_num_threads(1)
    fx = np.load(os.path.join(GOLDEN, f"{case}.npz"))
    if not bool(fx["learn_batch"]):
        st = random.getstate()
        try:
            random.setstate((3, tuple(int(x) for x in fx["rng_before"]), None))
            assert [random.sample(range(int(fx["n"])), int(fx["batch"])) for _ in range(len(fx["idx"]))] == fx["idx"].tolist()
            assert random.getstate()[1] == tuple(int(x) for x in fx["rng_after"])
        finally:
            random.setstate(st)
    got = orc.replay(fx)
    np.testing.assert_allclose(got["loss"], fx["loss"], rtol=1e-6, atol=1e-7)
    np.testing.assert_allclose(got["q_calls"], fx["q_calls"], rtol=1e-5, atol=1e-7)
    np.testing.assert_allclose(got["qt_calls"], fx["qt_calls"], rtol=1e-5, atol=1e-7)
    np.testing.assert_allclose(got["state"]["m"].numpy(), fx["adam_exp_avg"], rtol=1e-4, atol=1e-9)
    assert got["state"]["step"] == int(fx["adam_step"])


@pytest.mark.parametrize("case", ("cnnq_act_v", "cnnq_act_mh"))
def test_cnn_q_oracle_act_values(case):
    fx = np.load(os.path.join(GOLDEN, f"{case}.npz"))
    spec = orc.spec_of(fx)
    q = orc.q_all(spec, orc.unflat(spec, torch.from_numpy(fx["init_q"])), torch.from_numpy(fx["state"]).float())
    np.testing.assert_allclose(q.numpy(), fx["q"], rtol=1e-6, atol=1e-7)
    assert q.argmax(1).numpy().tolist() == fx["act"].tolist()
    assert bool(fx["act_3d_raised"])


@pytest.mark.parametrize("case", ("cnnq_ddqn", "cnnq_mh_ddqn"))
def test_cnn_q_fp64_matches_fp32_oracle(case):
    fx = np.load(os.path.join(GOLDEN, f"{case}.npz"))
    spec, w = orc.spec_of(fx), torch.from_numpy(fx["init_q"])
    b = orc.batch_of(fx, fx["idx"][0])
    g64, scale, margin = cnn_q_fp64.step(spec, w, w, b, double=True, gamma=float(fx["gamma"]))
    st = dict(w=w.clone(), wt=w.clone(), m=torch.zeros_like(w), v=torch.zeros_like(w), vmax=torch.zeros_like(w), step=0)
    orc.round_step(spec, st, b, double=True, gamma=float(fx["gamma"]), tau=0.1, lr=1e-3, update_target=False)
    assert bool((scale >= g64.abs() * (1 - 1e-12)).all())
    assert float(((st["grad"].double() - g64).abs() / scale.clamp_min(1e-300)).max()) < 1e-6
    assert margin > 0


def test_cnn_q_pong_param_count():
    import pearl_b200
    net = pearl_b200.CNNQValueNetwork(**PONG)
    assert sum(p.numel() for p in net.parameters()) == 1687713
    assert net._mlp_input_dims == 64 * 7 * 7 + 6
    mh = pearl_b200.CNNQValueMultiHeadNetwork(**dict(PONG, output_dim=6))
    assert mh._mlp_input_dims == 64 * 7 * 7
    spec = dict(input=(4, 84, 84), conv=[(32, 8, 4, 0), (64, 4, 2, 0), (64, 3, 1, 0)], hidden=[512], n_actions=6, multi=False)
    assert [(k, tuple(v.shape)) for k, v in net.state_dict().items()] == orc.param_shapes(spec)


def _plugin(net_cls, double=False, **kw):
    import pearl_b200
    cls = pearl_b200.B200DoubleDQN if double else pearl_b200.B200DeepQLearning
    A = 6

    class Space:
        n = A
        actions = [torch.tensor([i]) for i in range(A)]
        actions_batch = torch.arange(A).view(A, 1)
    net = kw.pop("net", None) or net_cls(**dict(PONG, output_dim=6 if net_cls is pearl_b200.CNNQValueMultiHeadNetwork else 1))
    return cls(state_dim=4 * 84 * 84, action_space=Space(), hidden_dims=[512], network_instance=net,
               action_representation_module=pearl_b200.OneHotActionTensorRepresentationModule(A), **kw), Space()


def test_cnn_q_shape_of_parses_both_networks():
    import pearl_b200
    from pearl_b200 import cnn_q
    for net_cls, multi in ((pearl_b200.CNNQValueNetwork, False), (pearl_b200.CNNQValueMultiHeadNetwork, True)):
        pl, _ = _plugin(net_cls)
        assert pl._variant is cnn_q
        assert pl._cnn == dict(input=(4, 84, 84), conv=[(32, 8, 4, 0), (64, 4, 2, 0), (64, 3, 1, 0)], hidden=[512], multi=multi)
        assert pl._obs_dim == 4 * 84 * 84
        cfg = cnn_q.make_cfg(pl, pl._adam_hparams(), 32)
        assert (cfg.n_conv, list(cfg.conv_out), cfg.n_fc, cfg.fc_hidden[0], cfg.multi_head) == (3, [32, 64, 64, 0], 1, 512, int(multi))


def test_cnn_q_refusals():
    import pearl_b200
    V, M = pearl_b200.CNNQValueNetwork, pearl_b200.CNNQValueMultiHeadNetwork
    with pytest.raises(NotImplementedError, match="batch norm"):
        _plugin(V, net=V(**dict(PONG, use_batch_norm_conv=True)))
    with pytest.raises(NotImplementedError, match="batch norm"):
        _plugin(M, net=M(**dict(PONG, output_dim=6, use_batch_norm_fully_connected=True)))
    five = dict(PONG, input_width=200, input_height=200, kernel_sizes=[3] * 5, output_channels_list=[4] * 5, strides=[2] * 5,
                paddings=[0] * 5)
    with pytest.raises(NotImplementedError, match="1 to 4 conv layers"):
        _plugin(V, net=V(**five))
    with pytest.raises(NotImplementedError, match="at most 2 hidden"):
        _plugin(V, net=V(**dict(PONG, hidden_dims_fully_connected=[8, 8, 8])))
    rect = V(**PONG)
    rect._model_cnn[0] = torch.nn.Conv2d(4, 32, (8, 4), stride=4)
    with pytest.raises(NotImplementedError, match="square"):
        _plugin(V, net=rect)
    with pytest.raises(NotImplementedError, match="conservative"):
        _plugin(V, is_conservative=True)
    with pytest.raises(NotImplementedError, match="engine='tc'"):
        _plugin(V, engine="tc")
    with pytest.raises(NotImplementedError, match="DeepSARSA"):
        A = 6
        pearl_b200.B200DeepSARSA(state_dim=4 * 84 * 84, action_space=None, hidden_dims=[512], network_instance=V(**PONG),
                                 action_representation_module=pearl_b200.OneHotActionTensorRepresentationModule(A))
    big = dict(PONG, action_dim=256)
    with pytest.raises(ValueError, match="at most 255"):
        pearl_b200.B200DeepQLearning(state_dim=4 * 84 * 84, action_space=None, hidden_dims=[512], network_instance=V(**big),
                                     action_representation_module=pearl_b200.OneHotActionTensorRepresentationModule(256))
    with pytest.raises(NotImplementedError, match="FC input"):
        _plugin(V, net=V(**dict(PONG, action_dim=5)))


def test_cnn_q_act_refuses_3d_state_before_any_device_call():
    """The learner is still on the CPU: a device call would raise RuntimeError; the 3-D state is refused first."""
    import pearl_b200
    pl, space = _plugin(pearl_b200.CNNQValueNetwork)
    with pytest.raises(ValueError, match="4-D"):
        pl.act(torch.zeros(4, 84, 84), space, exploit=True)
    with pytest.raises(ValueError, match="4-D"):
        pl.learn_batch(pearl_b200.TransitionBatch(state=torch.zeros(2, 4 * 84 * 84), action=torch.zeros(2, dtype=torch.long),
                                                  reward=torch.zeros(2), next_state=torch.zeros(2, 4 * 84 * 84)))
