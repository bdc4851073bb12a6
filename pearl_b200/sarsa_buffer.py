"""B200SARSAReplayBuffer — GPU-resident drop-in for Pearl's SARSAReplayBuffer
(replay_buffers/sequential_decision_making/sarsa_replay_buffer.py:29-101).

SARSA needs the action the policy committed to in the next state, which is known only at the next push.  The reference
therefore delays a push: a non-terminal transition waits in a one-entry cache and is stored when a later push's state
equals its next state, with that push's action as `next_action`.  `SarsaPushCache` restates that state machine on the
host, quirks included:

  * match: a cached transition exists and its next_state equals the pushed state (torch.equal) -> the cached transition
    is stored with next_action = the pushed action;
  * a push that is neither terminated nor truncated becomes the new cache (a cache that did not match is dropped);
  * a terminated or truncated push is stored at once with next_action = its own action, and the cache is LEFT AS IT WAS:
    a stale cache survives the end of the episode and is stored if a later push's state happens to equal its next state;
  * truncated rows keep terminated = False, so their target bootstraps from Q'(s', a) with the row's own action;
  * clear() empties the stored transitions and keeps the cache (PearlAgent clears an on-policy learner's buffer after
    every learn()).

Stored transitions live in the device ring of B200ReplayBuffer with the committed next action in bits 24..31 of the
record's flags word (PRL_BUF_NEXT_ACTION); `sample()` returns it as `next_action`, int64 [B, 1], as the reference
collates it.  A match costs one host compare and one one-record push.  Nothing here needs Pearl.
"""
from __future__ import annotations

from typing import Optional

import torch

from . import _lib
from .replay_buffer import B200ReplayBuffer, _stream_ptr


class SarsaPushCache:
    """The reference's delayed-push state machine, host tensors only.  `step` takes one push and returns the complete
    SARSA tuples it releases, oldest first: dicts with state / next_state (float32 [obs]), action / next_action (int),
    reward (float), terminated / truncated (bool), next_ids (uint8 [A] or None) and next_count (int or None)."""

    def __init__(self) -> None:
        self.cache: Optional[dict] = None

    def step(self, state, action: int, reward: float, terminated: bool, truncated: bool, next_state, next_ids=None,
             next_count=None) -> list:
        state = torch.as_tensor(state, dtype=torch.float32).reshape(-1).cpu()
        next_state = torch.as_tensor(next_state, dtype=torch.float32).reshape(-1).cpu()
        row = dict(state=state.clone(), action=int(action), reward=float(reward), terminated=bool(terminated),
                   truncated=bool(truncated), next_state=next_state.clone(), next_ids=next_ids, next_count=next_count)
        out = []
        if self.cache is not None and torch.equal(self.cache["next_state"], state):
            out.append(dict(self.cache, next_action=int(action)))
        if not (terminated or truncated):
            self.cache = row
        else:
            out.append(dict(row, next_action=int(action)))
        return out

    def state_dict(self) -> dict:
        return {"cache": None if self.cache is None else dict(self.cache)}

    def load_state_dict(self, sd: dict) -> None:
        c = sd.get("cache")
        self.cache = None if c is None else dict(c)


class B200SARSAReplayBuffer(B200ReplayBuffer):
    """Drop-in for SARSAReplayBuffer: `push` has the reference's signature and delays transitions until their next
    action is known (SarsaPushCache); `push_batch(..., next_action=...)` stores complete SARSA tuples directly (offline
    data, tests, benchmarks).  Discrete actions only."""

    _record_flags = _lib.PRL_BUF_NEXT_ACTION
    _stores_costs = False           # its records carry no cost word: `cost` is refused

    def __init__(self, capacity: int, device=None, dynamic_action_space: bool = False, rng: str = "python") -> None:
        super().__init__(capacity, device=device, dynamic_action_space=dynamic_action_space, rng=rng)
        self._sarsa = SarsaPushCache()
        self._next_action_src = None     # the prepared next-action ids of the push in progress (see _push_records)

    @property
    def cache(self) -> Optional[dict]:
        """The transition waiting for its next action (None when there is none)."""
        return self._sarsa.cache

    # ------------------------------------------------------------------ write side
    def push(self, state, action, reward, terminated, truncated, curr_available_actions=None,
             next_state=None, next_available_actions=None, max_number_actions=None, cost=None) -> None:
        """One transition, same signature as the reference (sarsa_replay_buffer.py:29-101 behind
        tensor_based_replay_buffer.py:55-133)."""
        if cost is not None:
            raise NotImplementedError("B200SARSAReplayBuffer does not store costs")
        if self._is_action_continuous:
            raise NotImplementedError("B200SARSAReplayBuffer stores discrete actions (DeepSARSA's one-hot Q network)")
        if next_state is None:
            raise ValueError("SARSA needs the next state of every transition")
        if max_number_actions is None:
            if curr_available_actions is None:
                raise AssertionError("curr_available_actions is needed to infer max_number_actions")
            max_number_actions = curr_available_actions.n
        ids = cnt = None
        if next_available_actions is not None:
            a_ids = next_available_actions.actions_batch.reshape(next_available_actions.n, -1)[:, 0].to(torch.int64).cpu()
            if not (a_ids.numel() == max_number_actions and bool((a_ids == torch.arange(max_number_actions)).all())):
                ids = torch.zeros(max_number_actions, dtype=torch.uint8)
                ids[: a_ids.numel()] = a_ids.to(torch.uint8)
                cnt = int(a_ids.numel())
        act = int(torch.as_tensor(action).reshape(-1)[0])
        done = self._sarsa.step(state, act, float(reward), bool(terminated), bool(truncated), next_state, ids, cnt)
        if done:
            self._push_rows(done, max_number_actions)

    def _push_rows(self, rows: list, max_number_actions: int) -> None:
        dyn = any(r["next_ids"] is not None for r in rows)
        A = self.n_actions or max_number_actions
        ids = cnt = None
        if dyn:
            ids = torch.stack([r["next_ids"] if r["next_ids"] is not None else torch.arange(A, dtype=torch.uint8) for r in rows])
            cnt = torch.tensor([r["next_count"] if r["next_count"] is not None else A for r in rows], dtype=torch.int32)
        self.push_batch(torch.stack([r["state"] for r in rows]), torch.tensor([r["action"] for r in rows], dtype=torch.int32),
                        torch.tensor([r["reward"] for r in rows], dtype=torch.float32),
                        torch.stack([r["next_state"] for r in rows]), torch.tensor([r["terminated"] for r in rows]),
                        torch.tensor([r["truncated"] for r in rows]), next_available_ids=ids, next_available_count=cnt,
                        max_number_actions=max_number_actions,
                        next_action=torch.tensor([r["next_action"] for r in rows], dtype=torch.int32))

    def push_batch(self, state, action, reward, next_state, terminated, truncated, next_available_ids=None,
                   next_available_count=None, max_number_actions=None, next_action=None) -> None:
        """B200ReplayBuffer.push_batch of n complete SARSA tuples: `next_action` [n] ints, the committed next action of
        every transition (required).  Bypasses the delayed-push cache."""
        if self._is_action_continuous:
            raise NotImplementedError("B200SARSAReplayBuffer stores discrete actions (DeepSARSA's one-hot Q network)")
        n = torch.as_tensor(state).shape[0]
        if n == 0:
            return
        if next_action is None:
            raise ValueError("B200SARSAReplayBuffer.push_batch needs next_action: the committed next action of every transition")
        na = torch.as_tensor(next_action).reshape(-1)
        if na.numel() != n:
            raise ValueError(f"next_action has {na.numel()} entries for {n} transitions")
        A = self.n_actions or max_number_actions
        if A is not None and bool(((na < 0) | (na >= A)).any()):
            raise ValueError(f"next_action ids must lie in [0, {A})")
        dev = self._device if torch.as_tensor(state).is_cuda else torch.device("cpu")
        # kept for _push_records; restored afterwards because an upgrade to dynamic sets re-pushes the stored content
        prev, self._next_action_src = self._next_action_src, na.to(device=dev, dtype=torch.int32).contiguous()
        try:
            super().push_batch(state, action, reward, next_state, terminated, truncated, next_available_ids=next_available_ids,
                               next_available_count=next_available_count, max_number_actions=max_number_actions)
        finally:
            self._next_action_src = prev

    def _push_records(self, on_dev: bool, n: int, fields: list) -> None:
        fn = self._lib.prl_buf_push_device_sarsa if on_dev else self._lib.prl_buf_push_host_sarsa
        _lib.check(fn(self._handle, n, *fields, _lib.ptr(self._next_action_src), _stream_ptr(self._device)))

    def _upgrade_to_dynamic(self) -> None:
        """Re-create the storage with per-transition action lists, keeping the content and its next actions."""
        n = self.local_len()
        old = nxt = None
        if n:
            head = int(self._lib.prl_buf_head(self._handle))
            slot = ((torch.arange(n, device=self._device) + head) % self.capacity).to(torch.int32)
            old = self._gather_slots(slot)
            nxt = self._next_actions(slot)
        self._lib.prl_buf_destroy(self._handle)
        self._allocate(self.obs_dim, self.n_actions, self.act_dim, True)
        if old is not None:
            cnt = (~old["mask"].bool()).sum(1).to(torch.int32)
            self.push_batch(old["state"], old["action"].to(torch.int32), old["reward"], old["next_state"],
                            old["terminated"], old["truncated"], next_available_ids=old["avail"].to(torch.uint8),
                            next_available_count=cnt, next_action=nxt)

    # ------------------------------------------------------------------ read side
    def _next_actions(self, slot: torch.Tensor) -> torch.Tensor:
        """The committed next action at ring slots `slot`: int64 [k] on the buffer's device."""
        slot = slot.to(torch.int32).contiguous()
        out = torch.empty(slot.numel(), dtype=torch.int64, device=self._device)
        with torch.cuda.device(self._device):
            _lib.check(self._lib.prl_buf_gather_next_action(self.handle, _lib.ptr(slot), slot.numel(), _lib.ptr(out),
                                                            _stream_ptr(self._device)))
        return out

    def sample(self, batch_size: int):
        """SARSAReplayBuffer.sample: the TransitionBatch of B200ReplayBuffer.sample plus next_action, int64 [B, 1]."""
        _, slot = self.sample_indices(batch_size, 1)
        tb = self._batch_of_slots(slot[0])
        tb.next_action = self._next_actions(slot[0]).unsqueeze(-1)
        return tb.to(self._device_for_batches)

    # ------------------------------------------------------------------ snapshot
    def state_dict(self) -> dict:
        """B200ReplayBuffer.state_dict (the raw records carry the next actions) plus the delayed-push cache, so a snapshot
        taken mid-episode resumes the same way."""
        out = super().state_dict()
        out["sarsa"] = self._sarsa.state_dict()
        return out

    def load_state_dict(self, sd: dict) -> None:
        super().load_state_dict(sd)
        self._sarsa.load_state_dict(sd.get("sarsa", {}))
