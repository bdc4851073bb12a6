"""A caller-supplied TransitionBatch staged for the learn_batch paths of the discrete-action DQN family (dqn.py, cql.py,
dueling.py, multihead.py, sarsa.py, qrdqn.py): its action ids, its dense rows and action sets as the `prl_*_learn_batch`
entry points read them, and the call of one such round."""
from __future__ import annotations

import torch

from . import _lib
from .replay_buffer import _stream_ptr


def action_ids(a: torch.Tensor, n_actions: int, one_hot_last: bool) -> torch.Tensor:
    """Action ids from one-hot rows (the reference's preprocess_batch; `one_hot_last`: the trailing dimension holds them)
    or from raw ids (trailing dimension 1 or none)."""
    if a.is_floating_point() and a.dim() >= 2 and a.shape[-1] == n_actions and one_hot_last and n_actions > 1:
        return a.argmax(-1)
    if a.dim() >= 2 and a.shape[-1] == 1:
        a = a.squeeze(-1)
    return a.long()


def checked_ids(a: torch.Tensor, n_actions: int, one_hot_last: bool, what: str) -> torch.Tensor:
    """action_ids, refused unless every id lies in [0, n_actions)."""
    a = action_ids(a, n_actions, one_hot_last)
    if bool(((a < 0) | (a >= n_actions)).any()):
        raise ValueError(f"{what}: action ids must lie in [0, {n_actions})")
    return a


def available_first(ids: torch.Tensor, mask) -> tuple[torch.Tensor, torch.Tensor]:
    """The next-slot ids [B, A] with the available slots first, in their order, and the number of available slots per
    row, both int32.  `mask`: next_unavailable_actions_mask, None = every slot available.  The first argmax over the
    leading slots is then the first argmax with the unavailable ones at -inf."""
    B, A = ids.shape
    mask = torch.zeros((B, A), dtype=torch.bool, device=ids.device) if mask is None else mask.to(ids.device).reshape(B, A).bool()
    order = torch.sort(mask.to(torch.int8), dim=1, stable=True).indices
    return ids.gather(1, order).to(torch.int32).contiguous(), (~mask).sum(1).to(torch.int32).contiguous()


def check_features(batch, obs_dim: int) -> None:
    if int(batch.state.shape[-1]) != obs_dim:
        raise ValueError(f"batch.state has {int(batch.state.shape[-1])} features, the learner {obs_dim}")


def staged_ids(t: torch.Tensor, n_actions: int, shape: tuple, dev, what: str) -> torch.Tensor:
    """The checked ids of `t` (raw ids, or one-hot rows in one more dimension than `shape`) as an int32 tensor of
    `shape` on `dev`."""
    t = t.to(dev)
    return checked_ids(t, n_actions, t.dim() == len(shape) + 1, what).reshape(shape).to(torch.int32).contiguous()


def dense_rows(batch, B: int, n_actions: int, dev) -> tuple:
    """state, action ids, reward, next_state and terminated of the batch, in the order the learn_batch entry points take
    them."""
    f32 = lambda t: t.to(device=dev, dtype=torch.float32).contiguous()  # noqa: E731
    return (f32(batch.state), staged_ids(batch.action, n_actions, (B,), dev, "batch.action"), f32(batch.reward.reshape(B)),
            f32(batch.next_state), batch.terminated.reshape(B).to(device=dev, dtype=torch.uint8).contiguous())


def slot_ids(batch, field: str, B: int, n_actions: int, dev):
    """The ids [B, A] of the action set `field` (curr_available_actions / next_available_actions, padding included),
    None when the batch has no such set."""
    t = getattr(batch, field, None)
    return None if t is None else staged_ids(t, n_actions, (B, n_actions), dev, f"batch.{field}")


def next_available_first(batch, B: int, n_actions: int, dev) -> tuple:
    """available_first of the next action sets and next_unavailable_actions_mask; (None, None) without next sets: every
    action is available next."""
    nid = slot_ids(batch, "next_available_actions", B, n_actions, dev)
    return (None, None) if nid is None else available_first(nid, getattr(batch, "next_unavailable_actions_mask", None))


def call(set_graph, learn_batch, handle, use_graph: bool, dev, *args) -> float:
    """One round on a staged batch: the handle's graph switch, then learn_batch(handle, *args, out_loss, stream) on `dev`
    (tensors and None passed by address).  Returns the reported loss."""
    out = torch.empty(1, dtype=torch.float32, device=dev)
    arg = lambda a: _lib.ptr(a) if a is None or isinstance(a, torch.Tensor) else a  # noqa: E731
    with torch.cuda.device(dev):
        _lib.check(set_graph(handle, int(use_graph)))
        _lib.check(learn_batch(handle, *map(arg, args), _lib.ptr(out), _stream_ptr(dev)))
    return out.item()  # also keeps the inputs alive until the round is done


def plugin_call(pl, *args) -> dict:
    """`call` through the handle a DQN plugin learner binds (dqn.py); its AdamW step tensors then follow the handle."""
    loss = call(pl._c("set_graph"), pl._c("learn_batch"), pl._handle, pl.use_cuda_graph, pl._device, *args)
    pl._sync_step_tensors()
    return {"loss": loss}
