"""Developer tool: a few SAC (configs[2] shape) and PPO (configs[3] shape) rounds with plain stream launches, for
`ncu --metrics gpu__time_duration.sum` launch lists; plus a TD3 round and the GAE pass of
the HBM-side table (16M transitions, episodes of 500)."""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

import pearl_b200

dev = torch.device("cuda", 0)
g = torch.Generator(device=dev).manual_seed(0)
rn = lambda *s: torch.randn(*s, device=dev, generator=g)
R = 3
obs, act, n, B = 376, 17, 100000, 512
buf = pearl_b200.B200ReplayBuffer(n, rng="device")
buf.is_action_continuous = True
buf.push_batch(rn(n, obs), rn(n, act).clamp(-1, 1), rn(n), rn(n, obs), torch.zeros(n, dtype=torch.bool, device=dev),
               torch.zeros(n, dtype=torch.bool, device=dev))
buf.seed(1)
sac = pearl_b200.B200ContinuousSoftActorCritic(state_dim=obs, low=[-1.0] * act, high=[1.0] * act, actor_hidden_dims=[256, 256],
                                               critic_hidden_dims=[256, 256], training_rounds=R, batch_size=B, seed=3)
sac.use_cuda_graph = False
print("sac", sac.learn(buf)["critic_loss"])
obs, A, n, B = 210, 16, 65536, 256
buf = pearl_b200.B200ReplayBuffer(n, rng="device")
buf.push_batch(rn(n, obs), torch.randint(0, A, (n,), device=dev, generator=g).to(torch.int32), rn(n), rn(n, obs),
               torch.rand(n, device=dev, generator=g) < 0.002, torch.zeros(n, dtype=torch.bool, device=dev), max_number_actions=A)
buf.seed(2)
ppo = pearl_b200.B200ProximalPolicyOptimization(state_dim=obs, n_actions=A, actor_hidden_dims=[64, 64], critic_hidden_dims=[64, 64],
                                                training_rounds=R, batch_size=B, epsilon=0.2, seed=4)
ppo.use_cuda_graph = False
print("ppo", ppo.learn(buf)["critic_loss"])
torch.cuda.synchronize()
del ppo, buf
obs, act, n, B = 17, 6, 100000, 256
buf = pearl_b200.B200ReplayBuffer(n, rng="device")
buf.is_action_continuous = True
buf.push_batch(rn(n, obs), rn(n, act).clamp(-1, 1), rn(n), rn(n, obs), torch.zeros(n, dtype=torch.bool, device=dev),
               torch.zeros(n, dtype=torch.bool, device=dev))
buf.seed(3)
td3 = pearl_b200.B200TD3(state_dim=obs, low=[-1.0] * act, high=[1.0] * act, actor_hidden_dims=[256, 256], critic_hidden_dims=[256, 256],
                         training_rounds=4, batch_size=B, seed=5)
td3.use_cuda_graph = False
print("td3", td3.learn(buf)["critic_loss"])
from pearl_b200.ppo import gae_and_lambda_returns
ng = 1 << 24
vals, rws = rn(ng), rn(ng)
te = ((torch.arange(ng, device=dev) % 500) == 499).to(torch.uint8)
tu = torch.zeros(ng, dtype=torch.uint8, device=dev)
for _ in range(2):
    gae_and_lambda_returns(vals, 0.1, rws, te, tu, 0.99, 0.95)
torch.cuda.synchronize()
