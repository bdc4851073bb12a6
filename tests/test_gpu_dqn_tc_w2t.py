"""The online network's W2^T operand tiles of the tensor-core DQN learner (pearl_b200/csrc/dqn_tc.cu).

dH1 = dZ2 W2 takes its B operand from W2^T tiles kept in global memory next to the W2 tiles: hi = the fp32 value of
W2[j][k] at row k, column kperm(j) of the tile, lo = its residual below TF32.  AdamW writes them in its TMA sweep, the
scalar sweep (obs + A not a multiple of 4) and the kernel prologue rebuild them from the flat vector.  After a call both
must equal the transpose of the flat W2 exactly, also when the host replaced the parameters between calls.
"""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

HID = 64


class _Space:
    def __init__(self, n):
        self.n = n
        self.actions = [torch.tensor([i]) for i in range(n)]

    @property
    def actions_batch(self):
        return torch.stack(self.actions)


def _kperm(k):
    return (k & ~7) | ((k & 1) << 2) | ((k & 7) >> 1)


def _tile_index(r, k, K):
    return (r >> 3) * (K * 8) + (k >> 2) * 32 + (r & 7) * 4 + (k & 3)


def _tf32_lo(x):
    return x - (x.view(np.uint32) & np.uint32(0xFFFFE000)).view(np.float32)


def _setup(obs, A, rounds):
    import pearl_b200
    torch.manual_seed(obs * 100 + A)
    learner = pearl_b200.B200DeepQLearning(
        state_dim=obs, action_space=_Space(A), hidden_dims=[HID, HID], learning_rate=1e-3, training_rounds=rounds,
        batch_size=128, target_update_freq=3, soft_update_tau=0.5, engine="tc",
        action_representation_module=pearl_b200.OneHotActionTensorRepresentationModule(A)).to("cuda")
    n = 1024
    g = torch.Generator(device="cuda").manual_seed(obs + A)
    buf = pearl_b200.B200ReplayBuffer(n, rng="device")
    buf.push_batch(torch.randn((n, obs), generator=g, device="cuda"), (torch.arange(n, device="cuda") % A).to(torch.int32),
                   torch.randn(n, generator=g, device="cuda"), torch.randn((n, obs), generator=g, device="cuda"),
                   torch.rand(n, generator=g, device="cuda") < 0.05, torch.zeros(n, dtype=torch.bool, device="cuda"),
                   max_number_actions=A)
    buf.seed(obs + A)
    return learner, buf


def _check_w2t(learner, obs, A):
    k1 = (obs + 63) // 64 * 64
    net = 128 * k1 + 2 * HID * HID                      # one network's W1 and W2 tiles
    total = 2 * net + 2 * HID * HID                     # online, target, online W2^T
    ws = learner._flat["ws"]
    tiles = ws[ws.numel() - 4 * total:].view(torch.float32).cpu().numpy()
    w2t = tiles[net:net + 2 * HID * HID]
    D = obs + A
    w = learner.flat_parameters.cpu().numpy()
    w2 = w[HID * D + HID:HID * D + HID + HID * HID].reshape(HID, HID)   # [out j][in k]
    j, k = np.meshgrid(np.arange(HID), np.arange(HID), indexing="ij")
    idx = _tile_index(k, np.vectorize(_kperm)(j), HID)
    want_hi = np.zeros(HID * HID, np.float32)
    want_hi[idx.ravel()] = w2.ravel()
    assert np.array_equal(w2t[:HID * HID].view(np.uint32), want_hi.view(np.uint32)), "W2^T hi tile"
    assert np.array_equal(w2t[HID * HID:].view(np.uint32), _tf32_lo(want_hi).view(np.uint32)), "W2^T lo tile"


@pytest.mark.parametrize("obs,A", [(96, 16), (32, 16), (96, 2), (24, 2)],
                         ids=["obs96-A16-tma", "obs32-A16-tma", "obs96-A2-scalar", "obs24-A2-scalar"])
def test_w2t_tiles_follow_w2(obs, A):
    """A = 16 updates W1 | b1 | W2 in the TMA sweep, A = 2 in the scalar sweep; 5 rounds per call with soft updates."""
    learner, buf = _setup(obs, A, rounds=5)
    learner.learn(buf)
    _check_w2t(learner, obs, A)
    with torch.no_grad():   # the host replaces the parameters: the next call starts from tiles rebuilt from them
        p = learner.flat_parameters
        p.copy_(0.5 * p + 0.01 * torch.randn(p.shape, device=p.device))
    learner.learn(buf)
    _check_w2t(learner, obs, A)
