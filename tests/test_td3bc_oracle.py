"""The CPU restatement of TD3BC (oracle/td3bc_oracle.py) and of TD3 / DDPG learn_batch (oracle/td3_oracle.py) against the
recordings of the reference's own PearlAgent(TD3BC | TD3 | DeepDeterministicPolicyGradient) learn() and learn_batch()
(tests/golden/td3bc_*.npz, {td3,ddpg}_batch.npz, oracle/gen_td3bc_golden.py)."""
import os

import numpy as np
import pytest
import torch

from conftest import GOLDEN
from oracle.pearl_oracle import flat
from oracle.td3bc_oracle import oracle_for, set_lrs

CASES = ["td3bc_learn", "td3bc_batch", "td3bc_lr", "td3_batch", "ddpg_batch"]


def replay(fx, orc):
    """Every call of the recording through the oracle: learn() = `rounds` x (count a step, learn_batch), learn_batch = one
    round at the recorded step count.  Returns the per-round losses."""
    t = torch.from_numpy
    al, cl = [], []
    k = j = 0
    for c, kind in enumerate(fx["call_kind"]):
        set_lrs(orc, *(float(x) for x in fx["call_lrs"][c]))
        if hasattr(orc, "alpha_bc"):
            orc.alpha_bc = float(fx["call_alpha"][c])
        orc.training_steps = int(fx["call_steps"][c])
        for _ in range(int(fx["rounds"]) if kind == 0 else 1):
            ix = fx["idx"][k].astype(np.int64)
            k += 1
            b = dict(state=t(fx["state"][ix]), action=t(fx["action"][ix]), reward=t(fx["reward"][ix]), next_state=t(fx["next_state"][ix]),
                     terminated=t(fx["terminated"][ix]))
            noise = None
            if len(fx["noise"]):
                noise = t(fx["noise"][j])
                j += 1
            if kind == 0:
                orc.training_steps += 1
            out = orc.learn_batch(b, noise)
            al.append(out["actor_loss"]); cl.append(out["critic_loss"])
    assert k == len(fx["idx"]) and j == len(fx["noise"])
    return al, cl


@pytest.mark.parametrize("case", CASES)
def test_oracle_reproduces_the_reference_recording(case):
    fx = np.load(os.path.join(GOLDEN, f"{case}.npz"))
    orc = oracle_for(fx)
    al, cl = replay(fx, orc)
    np.testing.assert_allclose(al, fx["actor_loss"], rtol=5e-6, atol=1e-7)
    np.testing.assert_allclose(cl, fx["critic_loss"], rtol=5e-6, atol=1e-7)
    for name, net in (("actor", orc.actor), ("actor_t", orc.actor_t), ("q1", orc.q[0]), ("q2", orc.q[1]), ("q1t", orc.qt[0]), ("q2t", orc.qt[1])):
        np.testing.assert_allclose(flat(net).numpy(), fx[f"{name}_after"], rtol=5e-6, atol=1e-7, err_msg=name)


def test_recordings_pin_the_quirks():
    """The recordings exercise what decides parity: an asymmetric box (the behaviour action is not scaled to it), learn_batch
    calls at an odd step count that repeat the last actor loss, and a handle re-created mid-delay."""
    fx = np.load(os.path.join(GOLDEN, "td3bc_batch.npz"))
    assert not np.allclose(fx["low"], -fx["high"])
    assert list(fx["call_steps"]) == [0, 0, 0, 3, 3, 3]
    assert len(set(fx["actor_loss"][2:].tolist())) == 1
    fx = np.load(os.path.join(GOLDEN, "td3bc_lr.npz"))
    assert fx["call_steps"][1] % 2 == 0 and fx["actor_loss"][2] == fx["actor_loss"][1]
    assert not np.array_equal(fx["call_lrs"][0], fx["call_lrs"][1]) and fx["call_alpha"][0] != fx["call_alpha"][1]
