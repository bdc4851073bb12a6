"""The conservative (CQL) path of B200DeepQLearning / B200DoubleDQN: Pearl's DeepQLearning / DoubleDQN built with
`is_conservative=True, conservative_alpha=alpha` (policy_learners/sequential_decision_making/deep_td_learning.py:269-360
with utils/functional_utils/learning/loss_fn_utils.py:17-71), on an H100 through `prl_cql_*` (csrc/cql.cu).

The DQN plugin (dqn.py) keeps its binding: `_Q`, `_Q_target` and the AdamW state are views into the flat vectors it
allocates, and a checkpoint or lr change is picked up the same way.  When `_is_conservative` is set, the plugin hands the
flat vectors to a `prl_cql` handle instead of a `prl_dqn` one and delegates `learn` (over a B200ReplayBuffer),
`learn_batch` and `q_values` to the functions here.  A round updates the target first (in the rounds the reference's
schedule flags), then takes one AdamW(amsgrad) step on mean (q - y)^2 + alpha * cql, with the reference's CQL term as it
computes it (include/pearl_b200.h).  alpha is read from `_conservative_alpha` on every call.  No CPU fallback."""
from __future__ import annotations

import ctypes as C

import torch

from . import _lib
from .replay_buffer import _stream_ptr


def check_config(pl, engine: str) -> None:
    """Refuses, at construction, the conservative configurations the CUDA learner does not run or the reference rejects."""
    if engine == "tc":
        raise NotImplementedError("engine='tc' has no conservative (CQL) kernel: use engine='auto' or 'simt'")
    alpha(pl)
    if pl._n_actions < 2:
        raise ValueError("conservative (CQL) updates need at least 2 actions: the reference's CQL term gathers column 1 "
                         "of the current-action values")


def alpha(pl) -> float:
    a = getattr(pl, "_conservative_alpha", None)
    if a is None:
        raise ValueError("conservative_alpha is None: the reference's CQL loss multiplies it with the CQL term")
    return float(a)


def make_cfg(pl, hp: dict, max_batch: int) -> _lib.CqlCfg:
    return _lib.CqlCfg(obs_dim=pl._obs_dim, n_actions=pl._n_actions, hidden1=pl._hidden[0], hidden2=pl._hidden[1],
                       double_dqn=int(pl._double), target_update_freq=int(pl._target_update_freq), max_batch=max_batch,
                       max_rounds=pl._max_rounds, lr=hp["lr"], beta1=hp["beta1"], beta2=hp["beta2"], eps=hp["eps"],
                       weight_decay=hp["weight_decay"], gamma=float(pl._discount_factor), tau=float(pl._soft_update_tau))


def learn(pl, replay_buffer, bs: int, rounds: int, trace: bool) -> dict:
    """PolicyLearner.learn over a B200ReplayBuffer: `rounds` x (sample -> round) through prl_cql_learn.  The ring holds no
    current action sets, so every round uses the full set, as B200ReplayBuffer.sample reports it."""
    from .per import B200PrioritizedReplayBuffer
    if isinstance(replay_buffer, B200PrioritizedReplayBuffer):
        raise NotImplementedError("conservative (CQL) updates sample uniformly: a B200PrioritizedReplayBuffer is not supported")
    pl._bind(bs)
    dev = pl._device
    if replay_buffer.device != dev:
        raise RuntimeError(f"replay buffer is on {replay_buffer.device}, learner on {dev}")
    a = alpha(pl)
    lib, h = pl._libh, pl._handle
    mae = torch.empty(rounds, dtype=torch.float32, device=dev)
    idx = torch.empty((rounds, bs), dtype=torch.int32, device=dev) if trace else None
    with torch.cuda.device(dev):
        stream = _stream_ptr(dev)
        _lib.check(lib.prl_cql_set_graph(h, int(pl.use_cuda_graph)))
        replay_buffer._rng_push()
        done = 0
        while done < rounds:
            r = min(pl._max_rounds, rounds - done)
            off = lambda t, w=1: C.c_void_p(0) if t is None else C.c_void_p(t.data_ptr() + 4 * done * w)  # noqa: E731
            _lib.check(lib.prl_cql_learn(h, replay_buffer.handle, r, bs, int(pl._training_steps), a, off(mae), off(idx, bs),
                                         stream))
            pl._training_steps += r
            done += r
        replay_buffer._rng_pull()
    pl._sync_step_tensors()
    report = {"loss": mae.cpu().tolist()}
    if trace:
        report.update(idx=idx, launches=int(lib.prl_cql_last_launches(h)))
    return report


def _ids(pl, t: torch.Tensor, one_hot_last: bool, what: str) -> torch.Tensor:
    a = pl._action_ids(t, one_hot_last)
    if bool(((a < 0) | (a >= pl._n_actions)).any()):
        raise ValueError(f"{what}: action ids must lie in [0, {pl._n_actions})")
    return a


def learn_batch(pl, batch) -> dict:
    """`DeepTDLearning.learn_batch` with the CQL term on a caller-supplied batch (raw ids, or the one-hot tensors the
    reference's preprocess_batch produces).  `curr_available_actions` (padding included: the reference's CQL term ignores
    `curr_unavailable_actions_mask`) defaults to every action; next-action slots that are masked are compacted away in
    order, which keeps DoubleDQN's first argmax."""
    B, A = len(batch), pl._n_actions
    if int(batch.state.shape[-1]) != pl._obs_dim:
        raise ValueError(f"batch.state has {int(batch.state.shape[-1])} features, the learner {pl._obs_dim}")
    pl._bind(B)
    dev = pl._device
    f32 = lambda t: t.to(device=dev, dtype=torch.float32).contiguous()  # noqa: E731
    state, next_state = f32(batch.state), f32(batch.next_state)
    reward = f32(batch.reward.reshape(B))
    term = batch.terminated.reshape(B).to(device=dev, dtype=torch.uint8).contiguous()
    i32 = lambda t: t.to(torch.int32).contiguous()  # noqa: E731
    action = i32(_ids(pl, batch.action.to(dev), batch.action.dim() == 2, "batch.action").reshape(B))
    cur = nid = cnt = None
    ca = getattr(batch, "curr_available_actions", None)
    if ca is not None:
        ca = ca.to(dev)
        cur = i32(_ids(pl, ca, ca.dim() == 3, "batch.curr_available_actions").reshape(B, A))
    na = getattr(batch, "next_available_actions", None)
    if na is not None:
        na = na.to(dev)
        nid = _ids(pl, na, na.dim() == 3, "batch.next_available_actions").reshape(B, A)
        mask = getattr(batch, "next_unavailable_actions_mask", None)
        mask = torch.zeros((B, A), dtype=torch.bool, device=dev) if mask is None else mask.to(dev).reshape(B, A).bool()
        order = torch.sort(mask.to(torch.int8), dim=1, stable=True).indices       # available slots first, in their order
        nid = i32(nid.gather(1, order))
        cnt = i32((~mask).sum(1))
    out = torch.empty(1, dtype=torch.float32, device=dev)
    lib, h, p = pl._libh, pl._handle, _lib.ptr
    with torch.cuda.device(dev):
        _lib.check(lib.prl_cql_set_graph(h, int(pl.use_cuda_graph)))
        _lib.check(lib.prl_cql_learn_batch(h, B, p(state), p(action), p(reward), p(next_state), p(term), p(cur), p(nid), p(cnt),
                                           int(pl._training_steps), alpha(pl), p(out), _stream_ptr(dev)))
    loss = out.item()  # also keeps the inputs alive until the round is done
    pl._sync_step_tensors()
    return {"loss": loss}


def q_values(pl, states: torch.Tensor, target: bool) -> torch.Tensor:
    pl._bind(1)
    dev = pl._device
    s = states.to(device=dev, dtype=torch.float32).reshape(-1, pl._obs_dim).contiguous()
    out = torch.empty((s.shape[0], pl._n_actions), dtype=torch.float32, device=dev)
    with torch.cuda.device(dev):
        _lib.check(pl._libh.prl_cql_q_values(pl._handle, s.shape[0], _lib.ptr(s), int(target), _lib.ptr(out), _stream_ptr(dev)))
    torch.cuda.current_stream(dev).synchronize()
    return out
