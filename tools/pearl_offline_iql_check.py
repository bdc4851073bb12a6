"""Developer check (needs facebookresearch/Pearl and a GPU) for B200ImplicitQLearning as a SUBCLASS of the reference's
ImplicitQLearning under the reference's own offline loop: `offline_learning()` (utils/functional_utils/train_and_eval/
offline_learning_and_evaluation.py:140-224) drives a PearlAgent through `agent.learn_batch(batch)` over a B200ReplayBuffer
filled by `load_offline_data` from transitions in the reference's offline-data format.  The plugin must (1) be an
ImplicitQLearning, (2) train on the GPU through that loop, (3) end bit-identical to the stand-alone CUDA learner fed the
same batches with the same torch.randint stream, and (4) keep its views: the agent's value net and its AdamW state are
the core's vectors.  The numerics against recordings of the reference are tests/test_iql.py; this file is about the
plugin boundary.  Needs facebookresearch/Pearl on sys.path (argv[1] = its root) plus the test-only gymnasium /
matplotlib stubs.

    python tools/pearl_offline_iql_check.py /path/to/Pearl
"""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.dont_write_bytecode = True
sys.path[:0] = [os.path.join(ROOT, "oracle", "stubs"), sys.argv[1], ROOT]

import numpy as np  # noqa: E402
import torch  # noqa: E402

import pearl_b200  # noqa: E402
from pearl_b200 import actor_critic as ac  # noqa: E402
from pearl.neural_networks.sequential_decision_making.actor_networks import VanillaContinuousActorNetwork  # noqa: E402
from pearl.pearl_agent import PearlAgent  # noqa: E402
from pearl.policy_learners.sequential_decision_making.implicit_q_learning import ImplicitQLearning  # noqa: E402
from pearl.utils.functional_utils.train_and_eval.offline_learning_and_evaluation import offline_learning  # noqa: E402
from pearl.utils.instantiations.spaces.box_action import BoxActionSpace  # noqa: E402

assert pearl_b200.HAVE_PEARL and ac.HAVE_REFERENCE_IQL
OBS, ACT, N, B, BATCHES, SEED = 17, 6, 5000, 256, 40, 11
DEV = torch.device("cuda", 0)


def transitions():
    """The offline-data format the reference's get_offline_data_in_buffer reads (a list of dicts)."""
    rng = np.random.Generator(np.random.PCG64(3))
    s, s2 = rng.standard_normal((N, OBS), dtype=np.float32), rng.standard_normal((N, OBS), dtype=np.float32)
    a, r, d = rng.uniform(-1, 1, (N, ACT)).astype(np.float32), rng.standard_normal(N, dtype=np.float32), rng.random(N) < 0.01
    return [dict(observation=torch.from_numpy(s[i]), action=torch.from_numpy(a[i]), reward=float(r[i]),
                 next_observation=torch.from_numpy(s2[i]), curr_available_actions=None, next_available_actions=None, done=bool(d[i]))
            for i in range(N)]


def main():
    space = BoxActionSpace(low=torch.full((ACT,), -1.0), high=torch.full((ACT,), 1.0))
    torch.manual_seed(0)
    pl = pearl_b200.B200ImplicitQLearning(state_dim=OBS, action_space=space, actor_network_type=VanillaContinuousActorNetwork,
                                          actor_hidden_dims=[256, 256], critic_hidden_dims=[256, 256],
                                          value_critic_hidden_dims=[256, 256], batch_size=B, expectile=0.7)
    assert isinstance(pl, ImplicitQLearning) and isinstance(pl, ac._B200ActorCriticMixin)
    buf = pearl_b200.B200ReplayBuffer(N, device=DEV)
    buf.is_action_continuous = True
    assert buf.load_offline_data(transitions()) == N
    agent = PearlAgent(policy_learner=pl, replay_buffer=buf, device_id=0)
    flat = lambda m: torch.cat([p.detach().reshape(-1) for p in m.parameters()]).clone()  # noqa: E731
    init = [flat(m) for m in (pl._actor, pl._critic._critic_1, pl._critic._critic_2, pl._value_network)]
    batches, losses = [], []

    def logger(loss, i, batch):
        batches.append(batch)
        losses.append(loss)
    offline_learning(agent, buf, number_of_batches=BATCHES, learning_logger=logger, seed=SEED)
    assert len(batches) == BATCHES and all(np.isfinite(list(v.values())).all() for v in losses)
    core = pl._b200
    assert pl._value_network._model[0][0].weight.data_ptr() == core.value_params.data_ptr(), "value net is not a view of the core"
    p0 = next(pl._value_network.parameters())
    assert pl._value_network_optimizer.state[p0]["exp_avg"].data_ptr() == core._value_state[0].data_ptr()
    assert int(pl._value_network_optimizer.state[p0]["step"]) == BATCHES and pl._training_steps == 0

    # the stand-alone learner on the same batches (as preprocess_batch left them) and the same randint stream
    ref = ac.IqlCore(state_dim=OBS, low=space.low, high=space.high, actor_hidden_dims=[256, 256], critic_hidden_dims=[256, 256],
                     value_critic_hidden_dims=[256, 256], batch_size=B, expectile=0.7, device=DEV)
    ref.load_parameters(*init)
    torch.manual_seed(SEED)       # offline_learning's set_seed(seed); the buffer samples from CPython's random, not torch
    for b in batches:
        ref.learn_batch(b)
    for name, got, want in (("actor", core.actor_params, ref.actor_params), ("critics", core.critic_params, ref.critic_params),
                            ("targets", core.critic_target_params, ref.critic_target_params), ("value", core.value_params, ref.value_params)):
        assert torch.equal(got, want), f"{name}: the plugin under offline_learning() differs from the stand-alone learner"
    print(f"offline_learning(): {BATCHES} batches through PearlAgent.learn_batch on the GPU; plugin == stand-alone learner bit for bit; "
          f"last losses {losses[-1]}")


if __name__ == "__main__":
    main()
