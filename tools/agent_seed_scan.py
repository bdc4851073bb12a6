"""Developer tool (CPU only, needs /root/reference): how sensitive is the PearlAgent parity loop of tools/pearl_agent_check.py to the
initial weights?  For seeds [argv1, argv2) the REFERENCE agent is driven three times - unperturbed and with the initial Q
weights perturbed by 2e-7 relative - and the largest relative difference of the reported losses is printed for DeepQLearning
and DoubleDQN.  Quiet seeds stay at ~5e-7; chaotic ones (AdamW sign flips on near-zero gradients) reach 1e-4 .. 3e-3."""
import sys, os, random, copy
ROOT=os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0]=[os.path.join(ROOT,'oracle','stubs'),'/root/reference',ROOT]
import numpy as np, torch
from pearl.action_representation_modules.one_hot_action_representation_module import OneHotActionTensorRepresentationModule
from pearl.api.action_result import ActionResult
from pearl.pearl_agent import PearlAgent
from pearl.policy_learners.exploration_modules.common.epsilon_greedy_exploration import EGreedyExploration
from pearl.policy_learners.sequential_decision_making.deep_q_learning import DeepQLearning
from pearl.policy_learners.sequential_decision_making.double_dqn import DoubleDQN
from pearl.replay_buffers.basic_replay_buffer import BasicReplayBuffer
from pearl.utils.instantiations.spaces.discrete_action import DiscreteActionSpace
OBS, A, CAP, B, ROUNDS, STEPS = 12, 4, 300, 32, 3, 90
def make(double):
    space = DiscreteActionSpace([torch.tensor([i]) for i in range(A)], seed=123)
    kw = dict(state_dim=OBS, action_space=space, hidden_dims=[64, 64], training_rounds=ROUNDS, batch_size=B,
              target_update_freq=4, soft_update_tau=0.6, exploration_module=EGreedyExploration(0.3),
              action_representation_module=OneHotActionTensorRepresentationModule(A))
    return PearlAgent(policy_learner=(DoubleDQN if double else DeepQLearning)(**kw), replay_buffer=BasicReplayBuffer(CAP), device_id=-1), space
def drive(agent, space):
    g = torch.Generator().manual_seed(11)
    obs = torch.randn((STEPS + 1, OBS), generator=g); rew = torch.randn(STEPS, generator=g); done = torch.rand(STEPS, generator=g) < 0.1
    random.seed(99); torch.manual_seed(99)
    losses=[]; acts=[]
    agent.reset(obs[0], space)
    for t in range(STEPS):
        a = agent.act(exploit=False); acts.append(int(torch.as_tensor(a).reshape(-1)[0]))
        agent.observe(ActionResult(observation=obs[t + 1], reward=float(rew[t]), terminated=bool(done[t]), truncated=False))
        losses += list(agent.learn().get("loss", []))
        if bool(done[t]): agent.reset(obs[t + 1], space)
    return acts, np.asarray(losses)
for seed in range(int(sys.argv[1]), int(sys.argv[2])):
    out=[]
    for double in (False, True):
        res=[]
        for pert in (0, 1, 2):
            torch.manual_seed(1000 + seed)
            ag, sp = make(double)
            if pert:
                gp = torch.Generator().manual_seed(pert)
                with torch.no_grad():
                    for p in list(ag.policy_learner._Q.parameters()):
                        p.mul_(1 + 2e-7 * torch.randn(p.shape, generator=gp))
            res.append(drive(ag, sp))
        same_acts = res[0][0]==res[1][0]==res[2][0]
        rel = max(float((np.abs(res[0][1]-res[k][1])/(np.abs(res[0][1])+1e-6)).max()) for k in (1,2))
        out.append((same_acts, rel))
    print(seed, out, flush=True)
