"""The CUDA plugins in PearlAgent's loop (pearl/pearl_agent.py:55-330: reset -> act -> observe -> learn) against a recording
of the reference's own PearlAgent + DeepQLearning / DoubleDQN + BasicReplayBuffer on the same seeded environment
(tests/golden/agent_{dqn,ddqn}.npz, written by oracle/gen_agent_golden.py).  Pearl itself is not needed: the loop below does
what PearlAgent does with an identity history module.  The same comparison against a live Pearl, the checkpoint round trip
through `PearlAgent.state_dict()` and the actor-critic plugins under PearlAgent are tools/pearl_agent_check.py and
tools/pearl_agent_ac_check.py (they need facebookresearch/Pearl importable)."""
import hashlib
import os
import random

import numpy as np
import pytest
import torch

from conftest import GOLDEN


class _Space:
    def __init__(self, n):
        self.n = n
        self.actions = [torch.tensor([i]) for i in range(n)]

    @property
    def actions_batch(self):
        return torch.stack(self.actions)


class _ReplayedEGreedy:
    """epsilon_greedy_exploration.py:52-83 with the recorded choice: the draw from CPython's global stream is consumed as
    the reference's module consumes it (and must agree with the recording); the explored action itself came from the
    action space's private generator and is taken from the recording."""
    def __init__(self, eps, explored):
        self.eps, self.explored, self.t = eps, explored, 0

    def act(self, subjective_state, action_space, exploit_action, values=None, **kw):
        rec = int(self.explored[self.t])
        self.t += 1
        hit = random.random() < self.eps
        assert hit == (rec >= 0), "the global random stream is not where the reference's was"
        return action_space.actions[rec] if hit else exploit_action


def _sd(fx, prefix):
    return {k[len(prefix) + 1:]: torch.from_numpy(fx[k].copy()) for k in fx.files if k.startswith(prefix + "/")}


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["dqn", "ddqn"])
def test_plugins_reproduce_the_recorded_pearl_agent_run(kind):
    """Actions of all 90 steps identical (every sampled index and every exploration draw shares CPython's global stream, so
    they all have to line up), the global random state at the end identical, all 270 losses and the final Q / Q_target
    within 1e-4.  The learner state (Q, Q_target, AdamW) is reloaded from the recording before the learn() of every 15th
    step, through load_state_dict of the modules and of the torch optimizer."""
    import pearl_b200
    fx = np.load(os.path.join(GOLDEN, f"agent_{kind}.npz"))
    OBS, A, CAP, B, ROUNDS, STEPS, SYNC, FREQ, ENV_SEED, RUN_SEED = (int(x) for x in fx["config"])
    EPS, TAU = (float(x) for x in fx["config_f"])
    space = _Space(A)
    cls = pearl_b200.B200DoubleDQN if kind == "ddqn" else pearl_b200.B200DeepQLearning
    learner = cls(state_dim=OBS, action_space=space, hidden_dims=[64, 64], training_rounds=ROUNDS, batch_size=B,
                  target_update_freq=FREQ, soft_update_tau=TAU, exploration_module=_ReplayedEGreedy(EPS, fx["explored"]),
                  action_representation_module=pearl_b200.OneHotActionTensorRepresentationModule(A)).to("cuda:0")
    buf = pearl_b200.B200ReplayBuffer(CAP, rng="python")
    learner._Q.load_state_dict(_sd(fx, "init/q"))
    learner._Q_target.load_state_dict(_sd(fx, "init/q_target"))
    g = torch.Generator().manual_seed(ENV_SEED)
    obs = torch.randn((STEPS + 1, OBS), generator=g)
    rew = torch.randn(STEPS, generator=g)
    done = torch.rand(STEPS, generator=g) < 0.1
    random.seed(RUN_SEED)
    torch.manual_seed(RUN_SEED)
    actions, losses = [], []
    state = obs[0]
    for t in range(STEPS):
        a = learner.act(state, space, exploit=False)
        actions.append(int(torch.as_tensor(a).reshape(-1)[0]))
        buf.push(state=state, action=a, reward=float(rew[t]), terminated=bool(done[t]), truncated=False,
                 curr_available_actions=space, next_state=obs[t + 1], next_available_actions=space, max_number_actions=A)
        state = obs[t + 1]
        if t and t % SYNC == 0:
            learner._Q.load_state_dict(_sd(fx, f"sync{t}/q"))
            learner._Q_target.load_state_dict(_sd(fx, f"sync{t}/q_target"))
            osd = learner.optimizer.state_dict()
            n_params = len(osd["param_groups"][0]["params"])
            osd["state"] = {i: {k[len(f"sync{t}/opt/{i}/"):]: torch.from_numpy(fx[k].copy()) for k in fx.files
                                if k.startswith(f"sync{t}/opt/{i}/")} for i in range(n_params)}
            learner.optimizer.load_state_dict(osd)
        losses += list(learner.learn(buf).get("loss", []))
    assert actions == fx["actions"].tolist()
    assert np.array_equal(np.frombuffer(hashlib.sha1(repr(random.getstate()).encode()).digest(), np.uint8), fx["random_state_sha1"]), \
        "the global random state diverged"
    want = fx["losses"]
    assert len(losses) == len(want) > 0
    rel = np.abs(np.asarray(losses) - want) / (np.abs(want) + 1e-6)
    print(f"    {kind}: losses: max relative difference {rel.max():.3e} at gradient step {int(rel.argmax())} of {len(want)}")
    np.testing.assert_allclose(losses, want, rtol=1e-4, atol=1e-6)
    for name, module in (("q", learner._Q), ("q_target", learner._Q_target)):
        ref = _sd(fx, f"final/{name}")
        got = module.state_dict()
        assert list(got.keys()) == list(ref.keys())
        for k in ref:
            x, y = got[k].detach().cpu().double().numpy(), ref[k].double().numpy()
            err = np.abs(x - y)
            bad = err > 1e-6 + 1e-4 * np.abs(y)
            # elementwise 1e-4; AdamW eps-sensitive elements (gradient ~ 1e-8: the step depends on fp32 summation noise,
            # tests/_tol.py) are counted and bounded: at most 3 per tensor, each within 5 % of lr * gradient steps
            assert bad.sum() <= 3 and (not bad.any() or err[bad].max() <= 0.05 * 1e-3 * len(want)), (name, k, int(bad.sum()), float(err.max()))
