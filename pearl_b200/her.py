"""B200HindsightExperienceReplayBuffer — Pearl's HindsightExperienceReplayBuffer
(pearl/replay_buffers/sequential_decision_making/hindsight_experience_replay_buffer.py:25-154, "final" mode) on the
GPU-resident ring: every transition is pushed as it arrives; when an episode ends the trajectory is replayed with the goal
replaced by the episode's final state and the rewards (and optionally the terminal flags) recomputed by the user's
`reward_fn` / `terminated_fn` — the relabelled trajectory goes to the device ring as ONE `push_batch` instead of one
Python `push` per transition.  The callbacks are host Python (as in the reference) and see the same tensors."""
from __future__ import annotations

from typing import Callable, Optional

import torch

from .replay_buffer import B200ReplayBuffer


class B200HindsightExperienceReplayBuffer(B200ReplayBuffer):
    _stores_costs = False           # its records carry no cost word: `cost` is refused

    def __init__(self, capacity: int, goal_dim: int, reward_fn: Callable, terminated_fn: Optional[Callable] = None, **kwargs) -> None:
        super().__init__(capacity, **kwargs)
        self._goal_dim = int(goal_dim)
        self._reward_fn = reward_fn
        self._terminated_fn = terminated_fn
        self._trajectory: list = []

    def push(self, state, action, reward, terminated, truncated, curr_available_actions=None, next_state=None,
             next_available_actions=None, max_number_actions=None, cost=None) -> None:
        if next_state is None:
            raise AssertionError("next_state must be a tensor")
        if curr_available_actions is None or next_available_actions is None:
            raise ValueError(f"{type(self)} requires curr_available_actions / next_available_actions not to be None")
        super().push(state, action, reward, terminated, truncated, curr_available_actions, next_state, next_available_actions,
                     max_number_actions, cost)
        st = torch.as_tensor(state, dtype=torch.float32).reshape(-1).cpu().clone()
        ns = torch.as_tensor(next_state, dtype=torch.float32).reshape(-1).cpu().clone()
        n_act = max_number_actions if max_number_actions is not None else getattr(curr_available_actions, "n", None)
        self._trajectory.append((st, action, ns, bool(terminated), bool(truncated), n_act))
        if not (terminated or truncated):
            return
        goal = ns[: -self._goal_dim].clone()            # "final" mode (:129): the episode's last state is the new goal
        states, nexts, acts, rews, terms, truncs = [], [], [], [], [], []
        for (s, a, s2, te, tr, _) in self._trajectory:
            s, s2 = s.clone(), s2.clone()
            s[-self._goal_dim:] = goal
            s2[-self._goal_dim:] = goal
            states.append(s); nexts.append(s2); acts.append(a)
            rews.append(float(self._reward_fn(s, a)))
            terms.append(bool(te if self._terminated_fn is None else self._terminated_fn(s, a)))
            truncs.append(bool(tr))
        if self._is_action_continuous:
            action_t = torch.stack([torch.as_tensor(a, dtype=torch.float32).reshape(-1) for a in acts])
        else:
            action_t = torch.tensor([int(torch.as_tensor(a).reshape(-1)[0]) for a in acts], dtype=torch.int32)
        self.push_batch(torch.stack(states), action_t, torch.tensor(rews, dtype=torch.float32), torch.stack(nexts),
                        torch.tensor(terms), torch.tensor(truncs), max_number_actions=self._trajectory[-1][5])
        self._trajectory = []
