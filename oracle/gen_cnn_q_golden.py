#!/usr/bin/env python
"""Record tests/golden/cnnq_*.npz by RUNNING THE REFERENCE's DeepQLearning / DoubleDQN with a CNNQValueNetwork or
CNNQValueMultiHeadNetwork network_instance (TEST INFRASTRUCTURE; same set-up and stubs as oracle/gen_golden.py, which
provides the import path).

    PYTHONDONTWRITEBYTECODE=1 python oracle/gen_cnn_q_golden.py

Recorded at a reduced image shape so the fixtures stay small: input 2 x 16 x 16, conv kernels [4, 3], channels [4, 8],
strides [2, 1], paddings [1, 0] (padding, overlapping windows and a stride above 1), FC [16].  Pixels are uint8 values,
pushed into a BasicReplayBuffer as float tensors; `pl.learn(buffer)` / `pl.learn_batch(...)` are called directly
(PearlAgent.act cannot drive a CNN learner: the reference's act adds a batch axis to 1-D states only).  Cases:
  cnnq_dqn       CNNQValueNetwork DeepQLearning, 4 actions, target_update_freq 3, two learn() calls: the target update
                 fires inside a call and across the boundary
  cnnq_ddqn      CNNQValueNetwork DoubleDQN, 6 actions, dynamic next-action sets
  cnnq_mh_dqn    CNNQValueMultiHeadNetwork DeepQLearning, 5 actions, two calls
  cnnq_mh_ddqn   CNNQValueMultiHeadNetwork DoubleDQN, 6 actions, dynamic next-action sets
  cnnq_lr        CNNQValueNetwork DeepQLearning, two calls; the learning rate changes in between
  cnnq_batch     pl.learn_batch() three times on sampled batches, both networks (cnnq_batch_v, cnnq_batch_mh)
  cnnq_act       act(exploit=True) on a [1, C, H, W] state and the Q values it ranks, both networks; act on a [C, H, W]
                 state raises
Recorded per learn case: the transitions, the sampled logical indices of every round, CPython's `random` state before and
after, per-round losses, the initial online net (the target is its deepcopy), the online and target nets after every
call and the AdamW state.  The generator asserts, for the multi-head network, that get_q_values returns [B, 1] for the
taken actions and that the loss broadcasts to [B, B] (MSELoss's size-mismatch warning; for DoubleDQN the next values
are [B, 1] as well, so the pair targets are V_i gamma (1 - terminated_j) + r_j), and for DoubleDQN that the best
available online next value beats the second best by more than 1e-3 (the initial action gaps are widened, _spread).
"""
from __future__ import annotations

import os
import random
import sys
import warnings

import numpy as np

sys.dont_write_bytecode = True
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from oracle.gen_golden import GOLDEN, flat_params, state_words  # noqa: E402  (sets up the reference import path and stubs)

import torch  # noqa: E402
from pearl.action_representation_modules.one_hot_action_representation_module import (  # noqa: E402
    OneHotActionTensorRepresentationModule,
)
from pearl.neural_networks.sequential_decision_making.q_value_networks import (  # noqa: E402
    CNNQValueMultiHeadNetwork, CNNQValueNetwork,
)
from pearl.policy_learners.sequential_decision_making.deep_q_learning import DeepQLearning  # noqa: E402
from pearl.policy_learners.sequential_decision_making.double_dqn import DoubleDQN  # noqa: E402
from pearl.replay_buffers.basic_replay_buffer import BasicReplayBuffer  # noqa: E402
from pearl.utils.instantiations.spaces.discrete_action import DiscreteActionSpace  # noqa: E402

MARGIN = 1e-3
SHAPE = dict(input=(2, 16, 16), kernels=[4, 3], channels=[4, 8], strides=[2, 1], paddings=[1, 0], fc=[16])


def _net(multi, n_act):
    C, H, W = SHAPE["input"]
    cls = CNNQValueMultiHeadNetwork if multi else CNNQValueNetwork
    return cls(input_width=W, input_height=H, input_channels_count=C, kernel_sizes=SHAPE["kernels"],
               output_channels_list=SHAPE["channels"], strides=SHAPE["strides"], paddings=SHAPE["paddings"], action_dim=n_act,
               hidden_dims_fully_connected=list(SHAPE["fc"]), output_dim=n_act if multi else 1)


def _learner(multi, double, n_act, lr, gamma, rounds, batch, freq, tau):
    full = DiscreteActionSpace(actions=list(torch.arange(n_act).view(-1, 1)))
    cls = DoubleDQN if double else DeepQLearning
    C, H, W = SHAPE["input"]
    return full, cls(state_dim=C * H * W, action_space=full, hidden_dims=list(SHAPE["fc"]), learning_rate=lr,
                     discount_factor=gamma, training_rounds=rounds, batch_size=batch, target_update_freq=freq,
                     soft_update_tau=tau, action_representation_module=OneHotActionTensorRepresentationModule(n_act),
                     network_instance=_net(multi, n_act))


def _data(n, n_act, seed, dynamic, p_term=0.15):
    rng = np.random.Generator(np.random.PCG64(seed))
    C, H, W = SHAPE["input"]
    d = dict(state=rng.integers(0, 256, (n, C, H, W), dtype=np.uint8), next_state=rng.integers(0, 256, (n, C, H, W), dtype=np.uint8),
             action=rng.integers(0, n_act, n).astype(np.int32), reward=rng.standard_normal(n).astype(np.float32),
             terminated=rng.random(n) < p_term)
    ids, cnt = np.tile(np.arange(n_act), (n, 1)), np.full(n, n_act)
    if dynamic:
        for i in range(n):
            m = int(rng.integers(1, n_act + 1))
            ids[i, :m] = np.sort(rng.choice(n_act, size=m, replace=False))
            ids[i, m:] = 0
            cnt[i] = m
    d.update(next_ids=ids.astype(np.uint8), next_count=cnt.astype(np.int32))
    return d


def _round_checks(pl, batch, multi, double):
    B = batch.state.shape[0]
    with torch.no_grad():
        q = pl._Q.get_q_values(batch.state, batch.action)
        assert tuple(q.shape) == ((B, 1) if multi else (B,)), f"taken-action Q shape {tuple(q.shape)}"
        if double:
            mask = batch.next_unavailable_actions_mask
            v = pl._Q.get_q_values(batch.next_state, batch.next_available_actions).view(B, -1).clone()
            v[mask] = -float("inf")
            top = torch.topk(v, 2, dim=-1).values
            two = (~mask).sum(-1) >= 2
            assert bool((top[two, 0] - top[two, 1] > MARGIN).all()), \
                f"greedy margin below {MARGIN}: {(top[two, 0] - top[two, 1]).min()}"


def _spy_learn_batch(pl, multi, double):
    orig = pl.learn_batch

    def spy(b):
        _round_checks(pl, b, multi, double)
        with warnings.catch_warnings(record=True) as ws:
            warnings.simplefilter("always")
            out = orig(b)
        broadcast = any("target size" in str(w.message) for w in ws)
        assert broadcast == multi, "the multi-head loss must (and the vanilla loss must not) broadcast to [B, B]"
        return out
    pl.learn_batch = spy


def _spread(pl, multi, factor=50.0):
    """Widens the initial gaps between the actions' values (the action columns of the first FC layer, or the head rows)
    so that DoubleDQN's argmax is decided by more than rounding; the target starts as the same net."""
    with torch.no_grad():
        fc = [m for m in pl._Q._model_fc.modules() if isinstance(m, torch.nn.Linear)]
        if multi:
            fc[-1].weight.mul_(factor)
            fc[-1].bias.mul_(factor)
        else:
            fc[0].weight[:, -pl.action_representation_module.max_number_actions:].mul_(factor)
    pl._Q_target.load_state_dict(pl._Q.state_dict())


def _adam(pl):
    params = list(pl._Q.parameters())
    st = pl._optimizer.state
    out = {f"adam_{k}": np.concatenate([st[p][k].numpy().ravel() for p in params])
           for k in ("exp_avg", "exp_avg_sq", "max_exp_avg_sq")}
    out["adam_step"] = float(st[params[0]]["step"])
    return out


def _save(name, out):
    path = os.path.join(GOLDEN, f"{name}.npz")
    np.savez_compressed(path, **out)
    print(f"{name}.npz: {os.path.getsize(path) // 1024} KB, loss", list(np.asarray(out.get("loss", []))[:3]))


def _config(multi, double, n_act, lr, gamma, rounds, batch, freq, tau, n):
    return dict(multi=multi, double=double, n_actions=n_act, lr=lr, gamma=gamma, rounds=rounds, batch=batch,
                target_update_freq=freq, tau=tau, n=n, input=np.asarray(SHAPE["input"]), kernels=np.asarray(SHAPE["kernels"]),
                channels=np.asarray(SHAPE["channels"]), strides=np.asarray(SHAPE["strides"]),
                paddings=np.asarray(SHAPE["paddings"]), fc=np.asarray(SHAPE["fc"]))


def _fill(buf, full, d, n_act):
    space = lambda row, m: DiscreteActionSpace(actions=[torch.tensor([int(a)]) for a in row[:m]])  # noqa: E731
    for i in range(len(d["action"])):
        buf.push(state=torch.from_numpy(d["state"][i].astype(np.float32)), action=torch.tensor(int(d["action"][i])),
                 reward=float(d["reward"][i]), terminated=bool(d["terminated"][i]), truncated=False, curr_available_actions=full,
                 next_state=torch.from_numpy(d["next_state"][i].astype(np.float32)),
                 next_available_actions=space(d["next_ids"][i], d["next_count"][i]), max_number_actions=n_act)


def gen_learn(name, *, multi, double, n_act, n=64, batch=16, rounds=4, calls=2, seed=0, data_seed=1, dynamic=False, lr=1e-3,
              new_lr=None, freq=3, tau=0.1, gamma=0.99, learn_batch_calls=0):
    torch.manual_seed(seed)
    random.seed(seed)
    torch.set_num_threads(1)
    full, pl = _learner(multi, double, n_act, lr, gamma, rounds, batch, freq, tau)
    if double:
        _spread(pl, multi)
    buf = BasicReplayBuffer(n)
    d = _data(n, n_act, data_seed, dynamic)
    _fill(buf, full, d, n_act)
    init = flat_params(pl._Q)
    assert np.array_equal(init, flat_params(pl._Q_target))
    idxs = []
    orig_sample = buf.sample

    def sample_spy(k):
        pos = {id(t): j for j, t in enumerate(buf.memory)}
        s0 = random.getstate()
        idxs.append([pos[id(t)] for t in random.sample(buf.memory, k)])
        random.setstate(s0)
        return orig_sample(k)
    buf.sample = sample_spy
    _spy_learn_batch(pl, multi, double)
    rs = random.getstate()
    losses, call_lr, q_calls, qt_calls = [], [], [], []
    for c in range(learn_batch_calls or calls):
        if c and new_lr is not None:
            pl._optimizer.param_groups[0]["lr"] = new_lr
        call_lr.append(pl._optimizer.param_groups[0]["lr"])
        if learn_batch_calls:
            losses.append(float(pl.learn_batch(pl.preprocess_batch(buf.sample(batch)))["loss"]))
        else:
            losses += [float(x) for x in pl.learn(buf)["loss"]]
        q_calls.append(flat_params(pl._Q))
        qt_calls.append(flat_params(pl._Q_target))
    out = dict(_config(multi, double, n_act, lr, gamma, rounds, batch, freq, tau, n), calls=learn_batch_calls or calls,
               learn_batch=bool(learn_batch_calls), dynamic=dynamic, call_lr=np.asarray(call_lr), **d,
               rng_before=state_words(rs), rng_after=state_words(random.getstate()), idx=np.asarray(idxs, dtype=np.int32),
               loss=np.asarray(losses), init_q=init, q_calls=np.stack(q_calls), qt_calls=np.stack(qt_calls),
               training_steps=int(pl._training_steps), **_adam(pl))
    _save(name, out)


def gen_act(name, *, multi, n_act, seed=0, data_seed=2):
    torch.manual_seed(seed)
    torch.set_num_threads(1)
    full, pl = _learner(multi, False, n_act, 1e-3, 0.99, 1, 4, 10, 0.1)
    d = _data(4, n_act, data_seed, False)
    qs, acts = [], []
    for i in range(4):
        s = torch.from_numpy(d["state"][i].astype(np.float32)).unsqueeze(0)
        acts.append(int(pl.act(s, full, exploit=True)))
        with torch.no_grad():
            qs.append(pl._Q.get_q_values(s, pl.action_representation_module(full.actions_batch).unsqueeze(0)).squeeze(0).numpy())
    try:
        pl.act(torch.from_numpy(d["state"][0].astype(np.float32)), full, exploit=True)
        raised = False
    except AssertionError:
        raised = True
    assert raised, "act on a [C, H, W] state no longer raises in the reference"
    _save(name, dict(_config(multi, False, n_act, 1e-3, 0.99, 1, 4, 10, 0.1, 4), state=d["state"], init_q=flat_params(pl._Q),
                     q=np.stack(qs), act=np.asarray(acts, np.int32), act_3d_raised=raised))


if __name__ == "__main__":
    gen_learn("cnnq_dqn", multi=False, double=False, n_act=4)
    gen_learn("cnnq_ddqn", multi=False, double=True, n_act=6, dynamic=True, data_seed=3, calls=1, rounds=5)
    gen_learn("cnnq_mh_dqn", multi=True, double=False, n_act=5, data_seed=4)
    gen_learn("cnnq_mh_ddqn", multi=True, double=True, n_act=6, dynamic=True, data_seed=5, calls=1, rounds=5)
    gen_learn("cnnq_lr", multi=False, double=False, n_act=4, data_seed=6, new_lr=3e-3, freq=10)
    gen_learn("cnnq_batch_v", multi=False, double=True, n_act=4, data_seed=7, freq=1, learn_batch_calls=3)
    gen_learn("cnnq_batch_mh", multi=True, double=False, n_act=4, data_seed=8, freq=1, learn_batch_calls=3)
    gen_act("cnnq_act_v", multi=False, n_act=5)
    gen_act("cnnq_act_mh", multi=True, n_act=5)
