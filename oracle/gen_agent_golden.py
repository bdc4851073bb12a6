"""Record tests/golden/agent_{dqn,ddqn}.npz: the reference's own PearlAgent facade (pearl/pearl_agent.py:55-330) driving the
reference's DeepQLearning / DoubleDQN + BasicReplayBuffer on the CPU through reset -> act -> observe -> learn on a seeded
synthetic environment.  tests/test_pearl_agent_gpu.py replays the same loop on the CUDA plugins without Pearl installed.

    python oracle/gen_agent_golden.py <root of facebookresearch/Pearl>

Recorded per run: the action of every step and whether the epsilon-greedy module explored, every loss, CPython's global
random state at the end, the initial and final Q / Q_target, and the complete learner state (Q, Q_target, AdamW) BEFORE the
learn() of every SYNC-th step, from which the GPU run is restarted (one AdamW-sensitive element is enough to move every
later loss by up to 3e-3 over 270 un-resynchronised gradient steps; 45 stay within 1e-4)."""
import hashlib
import os
import random
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.dont_write_bytecode = True
sys.path[:0] = [os.path.join(ROOT, "oracle", "stubs"), sys.argv[1], ROOT]

import numpy as np  # noqa: E402
import torch  # noqa: E402

from pearl.action_representation_modules.one_hot_action_representation_module import OneHotActionTensorRepresentationModule  # noqa: E402
from pearl.api.action_result import ActionResult  # noqa: E402
from pearl.pearl_agent import PearlAgent  # noqa: E402
from pearl.policy_learners.exploration_modules.common.epsilon_greedy_exploration import EGreedyExploration  # noqa: E402
from pearl.policy_learners.sequential_decision_making.deep_q_learning import DeepQLearning  # noqa: E402
from pearl.policy_learners.sequential_decision_making.double_dqn import DoubleDQN  # noqa: E402
from pearl.replay_buffers.basic_replay_buffer import BasicReplayBuffer  # noqa: E402
from pearl.utils.instantiations.spaces.discrete_action import DiscreteActionSpace  # noqa: E402

OBS, A, CAP, B, ROUNDS, STEPS, SYNC = 12, 4, 300, 32, 3, 90, 15
EPS, FREQ, TAU, ENV_SEED, RUN_SEED, INIT_SEED = 0.3, 4, 0.6, 11, 99, 1001


class RecordingEGreedy(EGreedyExploration):
    """The reference's module; notes for every call whether it explored (the draw is peeked at, not consumed)."""
    explored = None

    def act(self, subjective_state, action_space, exploit_action, values=None, action_availability_mask=None, representation=None):
        st = random.getstate()
        hit = random.random() < self.curr_epsilon
        random.setstate(st)
        out = super().act(subjective_state, action_space, exploit_action, values, action_availability_mask, representation)
        self.explored.append(int(torch.as_tensor(out).reshape(-1)[0]) if hit else -1)
        return out


def environment():
    g = torch.Generator().manual_seed(ENV_SEED)
    obs = torch.randn((STEPS + 1, OBS), generator=g)
    rew = torch.randn(STEPS, generator=g)
    done = torch.rand(STEPS, generator=g) < 0.1
    return obs, rew, done


def flat_sd(prefix, sd, out):
    for k, v in sd.items():
        if torch.is_tensor(v):
            out[f"{prefix}/{k}"] = v.detach().cpu().numpy().copy()


def record(double):
    torch.manual_seed(INIT_SEED)
    space = DiscreteActionSpace([torch.tensor([i]) for i in range(A)], seed=123)
    expl = RecordingEGreedy(EPS)
    expl.explored = []
    learner = (DoubleDQN if double else DeepQLearning)(
        state_dim=OBS, action_space=space, hidden_dims=[64, 64], training_rounds=ROUNDS, batch_size=B, target_update_freq=FREQ,
        soft_update_tau=TAU, exploration_module=expl, action_representation_module=OneHotActionTensorRepresentationModule(A))
    agent = PearlAgent(policy_learner=learner, replay_buffer=BasicReplayBuffer(CAP), device_id=-1)
    out = {}
    flat_sd("init/q", learner._Q.state_dict(), out)
    flat_sd("init/q_target", learner._Q_target.state_dict(), out)
    obs, rew, done = environment()
    random.seed(RUN_SEED)
    torch.manual_seed(RUN_SEED)
    actions, losses = [], []
    agent.reset(obs[0], space)
    for t in range(STEPS):
        a = agent.act(exploit=False)
        actions.append(int(torch.as_tensor(a).reshape(-1)[0]))
        agent.observe(ActionResult(observation=obs[t + 1], reward=float(rew[t]), terminated=bool(done[t]), truncated=False))
        if t and t % SYNC == 0:
            flat_sd(f"sync{t}/q", learner._Q.state_dict(), out)
            flat_sd(f"sync{t}/q_target", learner._Q_target.state_dict(), out)
            osd = learner.optimizer.state_dict()
            for i, st in osd["state"].items():
                for k, v in st.items():
                    out[f"sync{t}/opt/{i}/{k}"] = torch.as_tensor(v).detach().cpu().numpy().copy()
        losses += list(agent.learn().get("loss", []))
        if bool(done[t]):
            agent.reset(obs[t + 1], space)
    flat_sd("final/q", learner._Q.state_dict(), out)
    flat_sd("final/q_target", learner._Q_target.state_dict(), out)
    out["actions"] = np.asarray(actions, np.int32)
    out["explored"] = np.asarray(expl.explored, np.int32)
    out["losses"] = np.asarray(losses, np.float64)
    out["random_state_sha1"] = np.frombuffer(hashlib.sha1(repr(random.getstate()).encode()).digest(), np.uint8)
    out["config"] = np.asarray([OBS, A, CAP, B, ROUNDS, STEPS, SYNC, FREQ, ENV_SEED, RUN_SEED], np.int64)
    out["config_f"] = np.asarray([EPS, TAU], np.float64)
    path = os.path.join(ROOT, "tests", "golden", "agent_ddqn.npz" if double else "agent_dqn.npz")
    np.savez_compressed(path, **out)
    print(path, os.path.getsize(path), "bytes;", len(losses), "losses;", sum(e >= 0 for e in expl.explored), "explored steps")


if __name__ == "__main__":
    for double in (False, True):
        record(double)
