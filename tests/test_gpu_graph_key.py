"""A captured round bakes in the buffer's record layout and flags, not only its storage address.  Buffer storage is a
caller-owned tensor whose address a later buffer may reuse; a learner that outlives one buffer must not replay a graph
captured for the old layout over the new one.  Here two buffers share one storage tensor: a plain discrete layout
(obs 6, 5 actions: 20 words a record) and one with dynamic action sets (24 words).  A learner learns from the first and
then from the second with CUDA graphs on; losses, parameters and optimizer state must equal, bit for bit, the same
sequence with graphs off on a fresh learner."""
import ctypes as C
import random

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

OBS, A, B, R = 6, 5, 32, 3
CAP_PLAIN, CAP_DYNAMIC = 120, 100          # 120 x 20 words == 100 x 24 words: the same storage size


def _data(n, seed):
    g = np.random.default_rng(seed)
    cnt = g.integers(1, A + 1, n).astype(np.int32)
    ids = np.zeros((n, A), np.uint8)
    for i in range(n):
        ids[i, :cnt[i]] = np.sort(g.choice(A, cnt[i], replace=False))
    return dict(state=g.standard_normal((n, OBS)).astype(np.float32), action=g.integers(0, A, n).astype(np.int32),
                reward=g.standard_normal(n).astype(np.float32), next_state=g.standard_normal((n, OBS)).astype(np.float32),
                term=g.random(n) < 0.1, ids=ids, cnt=cnt)


def _push(buf, d, dynamic):
    t = torch.as_tensor
    buf.push_batch(t(d["state"]), t(d["action"]), t(d["reward"]), t(d["next_state"]), t(d["term"]),
                   torch.zeros(len(d["reward"]), dtype=torch.bool), next_available_ids=t(d["ids"]) if dynamic else None,
                   next_available_count=t(d["cnt"]) if dynamic else None, max_number_actions=A)


def _buffers():
    """Two prl_buf handles over one storage tensor: plain, then dynamic action sets."""
    import pearl_b200
    from pearl_b200 import _lib
    plain = pearl_b200.B200ReplayBuffer(CAP_PLAIN)
    _push(plain, _data(CAP_PLAIN, 1), False)
    dyn = pearl_b200.B200ReplayBuffer(CAP_DYNAMIC, dynamic_action_space=True)
    dyn._allocate(OBS, A, 1, True)
    assert (plain._layout.record_words, dyn._layout.record_words) == (20, 24)
    assert dyn._layout.storage_bytes == plain._layout.storage_bytes
    dyn._lib.prl_buf_destroy(dyn._handle)
    h = C.c_void_p(0)
    _lib.check(dyn._lib.prl_buf_create(C.byref(h), C.byref(dyn._desc), _lib.ptr(plain._storage), _lib.ptr(dyn._mt)))
    dyn._handle, dyn._storage = h, plain._storage
    return plain, dyn


def _state(pl):
    """Every device tensor the learner keeps (parameters, targets, optimizer state), except its scratch workspace."""
    out = []
    for k, v in sorted(vars(pl).items()):
        if k == "_workspace":
            continue
        for t in (v if isinstance(v, (list, tuple)) else [v]):
            if isinstance(t, torch.Tensor) and t.is_cuda:
                out.append(t.detach().clone())
    return out


def _run(make, graph):
    plain, dyn = _buffers()
    pl = make()
    pl.use_cuda_graph = graph
    random.seed(11)                                     # the buffer's sampling
    torch.manual_seed(11)                               # IQL's per-round random picks
    reps = [pl.learn(plain)]
    _push(dyn, _data(CAP_DYNAMIC, 2), True)             # overwrites the plain records in the shared storage
    reps.append(pl.learn(dyn))
    torch.cuda.synchronize()
    return reps, _state(pl)


def _learners():
    import pearl_b200
    h = [32, 32]
    return {
        "sac_discrete": lambda: pearl_b200.B200SoftActorCritic(OBS, A, h, h, actor_learning_rate=1e-3, critic_learning_rate=1e-3,
                                                               training_rounds=R, batch_size=B, seed=3),
        "iql": lambda: pearl_b200.B200ImplicitQLearning(OBS, None, h, h, h, n_actions=A, training_rounds=R, batch_size=B, seed=3),
        "reinforce": lambda: pearl_b200.B200REINFORCE(OBS, h, True, h, n_actions=A, actor_learning_rate=1e-3,
                                                      critic_learning_rate=1e-3, training_rounds=R, batch_size=B, seed=3),
        "ppo": lambda: pearl_b200.B200ProximalPolicyOptimization(OBS, None, h, h, actor_learning_rate=1e-3, critic_learning_rate=1e-3,
                                                                 training_rounds=R, batch_size=B, n_actions=A, seed=3),
        "qrdqn": lambda: pearl_b200.B200QuantileRegressionDeepQLearning(OBS, None, h, 8, learning_rate=1e-3, training_rounds=R,
                                                                        batch_size=B, target_update_freq=2, n_actions=A, seed=3),
    }


@pytest.mark.parametrize("name", ["sac_discrete", "iql", "reinforce", "ppo", "qrdqn"])
def test_graph_replay_follows_a_new_layout_at_the_same_address(name):
    make = _learners()[name]
    eager_reps, eager = _run(make, False)
    graph_reps, graph = _run(make, True)
    assert graph_reps == eager_reps
    assert len(graph) == len(eager) and len(graph) > 0
    for i, (a, b) in enumerate(zip(graph, eager)):
        assert torch.equal(a, b), f"{name}: state tensor {i} differs between graph replay and eager launches"
