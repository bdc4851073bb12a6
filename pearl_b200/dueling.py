"""The dueling path of B200DeepQLearning / B200DoubleDQN: Pearl's DeepQLearning / DoubleDQN built with
`network_type=DuelingQValueNetwork` (or a DuelingQValueNetwork `network_instance`), on an H100 through `prl_duel_*`
(csrc/dueling.cu).

The DQN plugin (dqn.py) keeps its binding: `_Q`, `_Q_target` and the AdamW state are views into the flat vectors it
allocates, and a checkpoint or lr change is picked up the same way.  When the Q network is a dueling one, the plugin hands
the flat vectors to a `prl_duel` handle and delegates `learn` (over a B200ReplayBuffer), `learn_batch`, `q_values` and
`act` to the functions here.  The advantage mean of `get_q_values` runs over the set the reference's caller hands it
(include/pearl_b200.h): the current slots (padding included) in a round, all next slots (masked ones included) for the
target, the query alone when a batch has no current sets, and the available actions in `act`.  No CPU fallback."""
from __future__ import annotations

import ctypes as C

import torch

from . import _lib
from .cql import _ids
from .replay_buffer import _stream_ptr

_ARCHS = ("state_arch", "value_arch", "advantage_arch")


def is_dueling(qnet) -> bool:
    return all(isinstance(getattr(qnet, a, None), torch.nn.Module) for a in _ARCHS)


def shape_of(qnet, n_actions: int) -> tuple[int, dict]:
    """obs_dim and the widths of a DuelingQValueNetwork whose three MLPs are each Linear+ReLU, Linear+ReLU, Linear and
    whose parameters are registered state, value, advantage (torch's parameter order is the flat layout)."""
    names = [n for n, _ in qnet.named_children()]
    if names != list(_ARCHS):
        raise NotImplementedError(f"pearl_b200 fuses a dueling Q network made of {list(_ARCHS)} only; got {names}")
    lins = []
    for a in _ARCHS:
        mods = [m for m in getattr(qnet, a).modules() if not isinstance(m, torch.nn.Sequential) and m is not getattr(qnet, a)]
        if [type(m) for m in mods] != [torch.nn.Linear, torch.nn.ReLU, torch.nn.Linear, torch.nn.ReLU, torch.nn.Linear]:
            raise NotImplementedError(f"pearl_b200 fuses dueling MLPs of exactly two hidden Linear+ReLU layers and a Linear head; "
                                      f"{a} has {[type(m).__name__ for m in mods]}")
        lins.append(mods[0::2])
    st, va, ad = lins
    F = st[2].out_features
    ok = all(l[1].in_features == l[0].out_features and l[2].in_features == l[1].out_features for l in lins)
    if not ok or va[0].in_features != F or ad[0].in_features != F + n_actions or va[2].out_features != 1 or ad[2].out_features != 1:
        raise NotImplementedError("unexpected dueling Q-network shape")
    dims = dict(feature_dim=F, state_h1=st[0].out_features, state_h2=st[1].out_features, value_h1=va[0].out_features,
                value_h2=va[1].out_features, adv_h1=ad[0].out_features, adv_h2=ad[1].out_features)
    return st[0].in_features, dims


def check_config(pl, engine: str) -> None:
    """Refuses, at construction, the dueling configurations the CUDA learner does not run."""
    if engine == "tc":
        raise NotImplementedError("engine='tc' has no dueling kernel: use engine='auto' or 'simt'")
    if pl._conservative:
        raise NotImplementedError("conservative (CQL) updates of a dueling Q network are not supported")
    pl._adam_hparams()


def make_cfg(pl, hp: dict, max_batch: int) -> _lib.DuelCfg:
    return _lib.DuelCfg(obs_dim=pl._obs_dim, n_actions=pl._n_actions, **pl._duel_dims, double_dqn=int(pl._double),
                        target_update_freq=int(pl._target_update_freq), max_batch=max_batch, max_rounds=pl._max_rounds,
                        lr=hp["lr"], beta1=hp["beta1"], beta2=hp["beta2"], eps=hp["eps"], weight_decay=hp["weight_decay"],
                        gamma=float(pl._discount_factor), tau=float(pl._soft_update_tau))


def learn(pl, replay_buffer, bs: int, rounds: int, trace: bool) -> dict:
    """PolicyLearner.learn over a B200ReplayBuffer: `rounds` x (sample -> round) through prl_duel_learn.  The ring holds no
    current action sets, so every round's advantage mean runs over every action, as B200ReplayBuffer.sample reports."""
    from .per import B200PrioritizedReplayBuffer
    if isinstance(replay_buffer, B200PrioritizedReplayBuffer):
        raise NotImplementedError("dueling DQN samples uniformly: a B200PrioritizedReplayBuffer is not supported")
    pl._bind(bs)
    dev = pl._device
    if replay_buffer.device != dev:
        raise RuntimeError(f"replay buffer is on {replay_buffer.device}, learner on {dev}")
    lib, h = pl._libh, pl._handle
    mae = torch.empty(rounds, dtype=torch.float32, device=dev)
    idx = torch.empty((rounds, bs), dtype=torch.int32, device=dev) if trace else None
    with torch.cuda.device(dev):
        stream = _stream_ptr(dev)
        _lib.check(lib.prl_duel_set_graph(h, int(pl.use_cuda_graph)))
        replay_buffer._rng_push()
        done = 0
        while done < rounds:
            r = min(pl._max_rounds, rounds - done)
            off = lambda t, w=1: C.c_void_p(0) if t is None else C.c_void_p(t.data_ptr() + 4 * done * w)  # noqa: E731
            _lib.check(lib.prl_duel_learn(h, replay_buffer.handle, r, bs, int(pl._training_steps), off(mae), off(idx, bs), stream))
            pl._training_steps += r
            done += r
        replay_buffer._rng_pull()
    pl._sync_step_tensors()
    report = {"loss": mae.cpu().tolist()}
    if trace:
        report.update(idx=idx, launches=int(lib.prl_duel_last_launches(h)))
    return report


def learn_batch(pl, batch) -> dict:
    """`DeepTDLearning.learn_batch` on a caller-supplied batch (raw ids, or the one-hot tensors the reference's
    preprocess_batch produces).  `curr_available_actions` (padding included) sets the online advantage mean; without it the
    mean runs over the query action alone, as the reference's get_q_values does.  Every next slot enters the target's
    mean with the id it holds; `next_unavailable_actions_mask` only removes slots from the max / argmax."""
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
    cur = nid = mask = None
    ca = getattr(batch, "curr_available_actions", None)
    if ca is not None:
        ca = ca.to(dev)
        cur = i32(_ids(pl, ca, ca.dim() == 3, "batch.curr_available_actions").reshape(B, A))
    na = getattr(batch, "next_available_actions", None)
    if na is not None:
        na = na.to(dev)
        nid = i32(_ids(pl, na, na.dim() == 3, "batch.next_available_actions").reshape(B, A))
    nm = getattr(batch, "next_unavailable_actions_mask", None)
    if nm is not None:
        mask = nm.to(dev).reshape(B, A).to(torch.uint8).contiguous()
    out = torch.empty(1, dtype=torch.float32, device=dev)
    lib, h, p = pl._libh, pl._handle, _lib.ptr
    with torch.cuda.device(dev):
        _lib.check(lib.prl_duel_set_graph(h, int(pl.use_cuda_graph)))
        _lib.check(lib.prl_duel_learn_batch(h, B, p(state), p(action), p(reward), p(next_state), p(term), p(cur), p(nid), p(mask),
                                            int(pl._training_steps), p(out), _stream_ptr(dev)))
    loss = out.item()  # also keeps the inputs alive until the round is done
    pl._sync_step_tensors()
    return {"loss": loss}


def q_values(pl, states: torch.Tensor, target: bool, ids: torch.Tensor | None = None) -> torch.Tensor:
    """Q(s, .) at the ids [n, K] of every row (None: every action), the advantage mean over that row's K ids."""
    pl._bind(1)
    dev = pl._device
    s = states.to(device=dev, dtype=torch.float32).reshape(-1, pl._obs_dim).contiguous()
    n = s.shape[0]
    if ids is not None:
        ids = ids.to(device=dev, dtype=torch.int32).reshape(n, -1).contiguous()
        if bool(((ids < 0) | (ids >= pl._n_actions)).any()):
            raise ValueError(f"action ids must lie in [0, {pl._n_actions})")
    K = pl._n_actions if ids is None else ids.shape[1]
    out = torch.empty((n, K), dtype=torch.float32, device=dev)
    with torch.cuda.device(dev):
        _lib.check(pl._libh.prl_duel_q_values(pl._handle, n, _lib.ptr(s), _lib.ptr(ids), K, int(target), _lib.ptr(out),
                                              _stream_ptr(dev)))
    torch.cuda.current_stream(dev).synchronize()
    return out
