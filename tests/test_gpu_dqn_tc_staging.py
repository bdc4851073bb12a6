"""Work the tensor-core DQN learner (pearl_b200/csrc/dqn_tc.cu) stages a round ahead must not change what a round computes.

Within one launch, round r loads round r + 1's row scalars under its AdamW sweep and issues round r + 1's target tiles
after the sweep, unless a soft target update falls on round r + 1; the first round of every launch loads its own.  A
single-round learn() call never takes the staged paths, so a learner trained by multi-round calls must end bit-identical
to one trained by as many single-round calls: parameters, target parameters, AdamW state, losses, q and y.

The cases cover a soft update on every round (freq 1), on every second round (freq 2) and between staged rounds
(freq 10, where one also falls on the first round of a launch), one and two row tiles (batch 128 and 256), calls split
into several launches (max_rounds_per_call below training_rounds, and the chunked launches of a call of 64 rounds or
more), the TMA-fed and the scalar AdamW sweep, and parameters the host changes between two learn() calls.
"""
import pytest
import torch

pytestmark = pytest.mark.gpu

HID = 64
ROUNDS, PER_CALL = 88, 78   # calls of 78 rounds (two chunked launches) and 10; the call after 78 rounds starts at step 78


class _Space:
    def __init__(self, n):
        self.n = n
        self.actions = [torch.tensor([i]) for i in range(n)]

    @property
    def actions_batch(self):
        return torch.stack(self.actions)


def _learner(obs, A, B, freq, rounds, per_call):
    import pearl_b200
    torch.manual_seed(obs * 7 + A + B + freq)
    learner = pearl_b200.B200DeepQLearning(
        state_dim=obs, action_space=_Space(A), hidden_dims=[HID, HID], learning_rate=1e-3, discount_factor=0.99,
        training_rounds=rounds, batch_size=B, target_update_freq=freq, soft_update_tau=0.3, max_rounds_per_call=per_call,
        engine="tc", action_representation_module=pearl_b200.OneHotActionTensorRepresentationModule(A)).to("cuda")
    g = torch.Generator(device="cuda").manual_seed(obs + A)
    with torch.no_grad():   # the target network starts away from the online one
        for p in learner._Q_target.parameters():
            p.add_(0.05 * torch.randn(p.shape, generator=g, device=p.device))
    return learner


def _buffer(obs, A):
    import pearl_b200
    n = 1024
    g = torch.Generator(device="cuda").manual_seed(obs * 31 + A)
    buf = pearl_b200.B200ReplayBuffer(n, rng="device")
    buf.push_batch(torch.randn((n, obs), generator=g, device="cuda"), (torch.arange(n, device="cuda") % A).to(torch.int32),
                   torch.randn(n, generator=g, device="cuda"), torch.randn((n, obs), generator=g, device="cuda"),
                   torch.rand(n, generator=g, device="cuda") < 0.05, torch.zeros(n, dtype=torch.bool, device="cuda"),
                   max_number_actions=A)
    buf.seed(obs + A)
    return buf


def _train(learner, buf, calls, change):
    """`calls` learn() calls, the host changing the parameters after the first half of them; the reports concatenated."""
    rep = {"loss": [], "q": [], "y": [], "idx": []}
    for c in range(calls):
        if c == calls // 2:
            with torch.no_grad():
                learner.flat_parameters.copy_(0.5 * learner.flat_parameters + change)
        r = learner.learn(buf, trace=True)
        rep["loss"] += r["loss"]
        for k in ("q", "y", "idx"):
            rep[k].append(r[k])
    return rep["loss"], {k: torch.cat(rep[k]) for k in ("q", "y", "idx")}


@pytest.mark.parametrize("freq", [1, 2, 10])
@pytest.mark.parametrize("B", [128, 256])
@pytest.mark.parametrize("obs,A", [(96, 16), (24, 2)], ids=["obs96-A16-tma", "obs24-A2-scalar"])
def test_multi_round_calls_equal_single_round_calls(obs, A, B, freq):
    staged = _learner(obs, A, B, freq, ROUNDS, PER_CALL)
    single = _learner(obs, A, B, freq, 1, PER_CALL)
    assert torch.equal(staged.flat_parameters, single.flat_parameters)
    assert torch.equal(staged.flat_target_parameters, single.flat_target_parameters)
    g = torch.Generator(device="cuda").manual_seed(B + freq)
    change = 0.01 * torch.randn(staged.flat_parameters.shape, generator=g, device="cuda")

    loss_s, tr_s = _train(staged, _buffer(obs, A), 2, change)
    loss_1, tr_1 = _train(single, _buffer(obs, A), 2 * ROUNDS, change)

    assert torch.equal(tr_s["idx"], tr_1["idx"]), "the two learners sampled different rows"
    assert torch.equal(tr_s["y"], tr_1["y"]), "targets y"
    assert torch.equal(tr_s["q"], tr_1["q"]), "q values"
    assert loss_s == loss_1, "losses"
    assert torch.equal(staged.flat_parameters, single.flat_parameters), "parameters"
    assert torch.equal(staged.flat_target_parameters, single.flat_target_parameters), "target parameters"
    st_s, st_1 = staged.adam_state(), single.adam_state()
    assert st_s["step"] == st_1["step"] == 2 * ROUNDS
    for k in ("exp_avg", "exp_avg_sq", "max_exp_avg_sq"):
        assert torch.equal(st_s[k], st_1[k]), k
