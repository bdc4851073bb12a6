"""Action ids of a caller-supplied TransitionBatch, shared by the learn_batch paths of the discrete-action DQN family
(dqn.py, cql.py, dueling.py, qrdqn.py)."""
from __future__ import annotations

import torch


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
