"""The multi-head path of B200DeepQLearning / B200DoubleDQN: Pearl's DeepQLearning / DoubleDQN built with
`network_type=VanillaQValueMultiHeadNetwork` (or such a `network_instance`), plain or with `is_conservative=True`, on an
H100 through `prl_mhq_*` (csrc/multihead.cu).

The DQN plugin (dqn.py) keeps its binding: `_Q`, `_Q_target` and the AdamW state are views into the flat vectors it
allocates, and a checkpoint or lr change is picked up the same way.  When the Q network is a multi-head one, the plugin
hands the flat vectors to a `prl_mhq` handle: `learn` (over a B200ReplayBuffer) runs through its prl_mhq_* entry points,
`learn_batch` and `q_values` through the functions here.  The network maps a state to one Q value per action; a query
slot holding id k reads head column k exactly (the reference's bmm with a one-hot slot), so a round needs one forward
pass per state (include/pearl_b200.h).  alpha is read from `_conservative_alpha` on every call.  No CPU fallback."""
from __future__ import annotations

import torch

from . import _lib
from ._batch import available_first, checked_ids
from ._compat import VanillaQValueMultiHeadNetwork
from .replay_buffer import _stream_ptr


def is_multihead(qnet) -> bool:
    """By class, not by shape: at one action a multi-head net has the shape of a one-hot vanilla net of one input less."""
    return isinstance(qnet, VanillaQValueMultiHeadNetwork)


def shape_of(qnet, n_actions: int) -> tuple[int, tuple[int, int]]:
    """obs_dim and the hidden widths of a VanillaQValueMultiHeadNetwork whose `_model` is Linear+ReLU, Linear+ReLU,
    Linear with n_actions outputs (torch's parameter order is the flat layout)."""
    model = getattr(qnet, "_model", None)
    if not isinstance(model, torch.nn.Module):
        raise NotImplementedError("pearl_b200 fuses a multi-head Q network whose layers are its `_model` MLP")
    mods = [m for m in model.modules() if not isinstance(m, torch.nn.Sequential)]
    kinds = [type(m) for m in mods]
    if torch.nn.LayerNorm in kinds:
        raise NotImplementedError("use_layer_norm=True: pearl_b200 fuses multi-head Q networks without layer norm")
    if kinds != [torch.nn.Linear, torch.nn.ReLU, torch.nn.Linear, torch.nn.ReLU, torch.nn.Linear]:
        raise NotImplementedError("pearl_b200 fuses multi-head Q networks of exactly two hidden Linear+ReLU layers and a Linear "
                                  f"head; got {[k.__name__ for k in kinds]}")
    l1, l2, l3 = mods[0::2]
    if l2.in_features != l1.out_features or l3.in_features != l2.out_features or l3.out_features != n_actions:
        raise NotImplementedError(f"unexpected multi-head Q-network shape: the head must have one output per action ({n_actions})")
    return l1.in_features, (l1.out_features, l2.out_features)


def check_config(pl, engine: str) -> None:
    """Refuses, at construction, the multi-head configurations the CUDA learner does not run or the reference rejects."""
    if engine == "tc":
        raise NotImplementedError("engine='tc' has no multi-head kernel: use engine='auto' or 'simt'")
    if pl._conservative:
        alpha(pl)
        if pl._n_actions < 2:
            raise ValueError("conservative (CQL) updates need at least 2 actions: the reference's CQL term gathers column 1 "
                             "of the current-action values")
    pl._adam_hparams()


def alpha(pl) -> float:
    if not pl._conservative:
        return 0.0
    a = getattr(pl, "_conservative_alpha", None)
    if a is None:
        raise ValueError("conservative_alpha is None: the reference's CQL loss multiplies it with the CQL term")
    return float(a)


def make_cfg(pl, hp: dict, max_batch: int) -> _lib.MhqCfg:
    return _lib.MhqCfg(obs_dim=pl._obs_dim, n_actions=pl._n_actions, hidden1=pl._hidden[0], hidden2=pl._hidden[1],
                       double_dqn=int(pl._double), conservative=int(pl._conservative),
                       target_update_freq=int(pl._target_update_freq), max_batch=max_batch, max_rounds=pl._max_rounds,
                       lr=hp["lr"], beta1=hp["beta1"], beta2=hp["beta2"], eps=hp["eps"], weight_decay=hp["weight_decay"],
                       gamma=float(pl._discount_factor), tau=float(pl._soft_update_tau))


def learn_batch(pl, batch) -> dict:
    """`DeepTDLearning.learn_batch` on a caller-supplied batch (raw ids, or the one-hot tensors the reference's
    preprocess_batch produces).  Conservative: `curr_available_actions` (padding included: the reference's CQL term
    ignores `curr_unavailable_actions_mask`) is required, as the reference asserts.  Next-action slots that are masked are
    compacted away in order, which keeps DoubleDQN's first argmax."""
    B, A = len(batch), pl._n_actions
    if int(batch.state.shape[-1]) != pl._obs_dim:
        raise ValueError(f"batch.state has {int(batch.state.shape[-1])} features, the learner {pl._obs_dim}")
    ca = getattr(batch, "curr_available_actions", None)
    if pl._conservative and ca is None:
        raise ValueError("a conservative (CQL) learn_batch needs batch.curr_available_actions, as the reference asserts")
    a = alpha(pl)
    pl._bind(B)
    dev = pl._device
    f32 = lambda t: t.to(device=dev, dtype=torch.float32).contiguous()  # noqa: E731
    state, next_state = f32(batch.state), f32(batch.next_state)
    reward = f32(batch.reward.reshape(B))
    term = batch.terminated.reshape(B).to(device=dev, dtype=torch.uint8).contiguous()
    i32 = lambda t: t.to(torch.int32).contiguous()  # noqa: E731
    action = i32(checked_ids(batch.action.to(dev), A, batch.action.dim() == 2, "batch.action").reshape(B))
    cur = nid = cnt = None
    if pl._conservative:
        ca = ca.to(dev)
        cur = i32(checked_ids(ca, A, ca.dim() == 3, "batch.curr_available_actions").reshape(B, A))
    na = getattr(batch, "next_available_actions", None)
    if na is not None:
        na = na.to(dev)
        nid = checked_ids(na, A, na.dim() == 3, "batch.next_available_actions").reshape(B, A)
        nid, cnt = available_first(nid, getattr(batch, "next_unavailable_actions_mask", None))
    out = torch.empty(1, dtype=torch.float32, device=dev)
    lib, h, p = pl._libh, pl._handle, _lib.ptr
    with torch.cuda.device(dev):
        _lib.check(lib.prl_mhq_set_graph(h, int(pl.use_cuda_graph)))
        _lib.check(lib.prl_mhq_learn_batch(h, B, p(state), p(action), p(reward), p(next_state), p(term), p(cur), p(nid), p(cnt),
                                           int(pl._training_steps), a, p(out), _stream_ptr(dev)))
    loss = out.item()  # also keeps the inputs alive until the round is done
    pl._sync_step_tensors()
    return {"loss": loss}


def q_values(pl, states: torch.Tensor, target: bool) -> torch.Tensor:
    """Q(s)[a] for every action id: [n, obs] -> [n, n_actions]."""
    pl._bind(1)
    dev = pl._device
    s = states.to(device=dev, dtype=torch.float32).reshape(-1, pl._obs_dim).contiguous()
    out = torch.empty((s.shape[0], pl._n_actions), dtype=torch.float32, device=dev)
    with torch.cuda.device(dev):
        _lib.check(pl._libh.prl_mhq_q_values(pl._handle, s.shape[0], _lib.ptr(s), int(target), _lib.ptr(out), _stream_ptr(dev)))
    torch.cuda.current_stream(dev).synchronize()
    return out
