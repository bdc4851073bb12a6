"""B200PrioritizedReplayBuffer — GPU-resident ring replay with a proportional prioritized sampler
(sum tree + min tree in HBM).  The reference has no prioritized replay (SURVEY.md §0.3); the behaviour
is specified by oracle/per_oracle.py (Schaul et al. 2016) and delivered through the reference's own
`TransitionBatch.weight` field (pearl/replay_buffers/transition.py:128)."""
from __future__ import annotations

import ctypes as C

import torch

from . import _lib
from ._compat import TransitionBatch
from .replay_buffer import B200ReplayBuffer, _stream_ptr


class B200PrioritizedReplayBuffer(B200ReplayBuffer):
    _stores_costs = False           # its records carry no cost word: `cost` is refused

    def __init__(self, capacity: int, alpha: float = 0.6, beta: float = 0.4, eps: float = 1e-6, seed: int = 0,
                 **kwargs) -> None:
        super().__init__(capacity, **kwargs)
        self.alpha, self.beta, self.eps, self.per_seed = float(alpha), float(beta), float(eps), int(seed)
        self._per = C.c_void_p(0)
        self.sum_tree = self.min_tree = self._max_priority = None
        self.last_slots = None

    def __del__(self):
        try:
            if getattr(self, "_per", None) and self._per.value:
                self._lib.prl_per_destroy(self._per)
                self._per = C.c_void_p(0)
        except Exception:
            pass
        super().__del__()

    def _allocate(self, obs_dim, n_actions, act_dim, dynamic) -> None:
        super()._allocate(obs_dim, n_actions, act_dim, dynamic)
        if self._per.value:
            self._lib.prl_per_destroy(self._per)
        n = int(self._lib.prl_per_tree_floats(self.capacity))
        self.sum_tree = torch.empty(n, dtype=torch.float32, device=self._device)
        self.min_tree = torch.empty(n, dtype=torch.float32, device=self._device)
        self._max_priority = torch.empty(1, dtype=torch.float32, device=self._device)
        cfg = _lib.PerCfg(self.capacity, self.alpha, self.beta, self.eps, self.per_seed)
        h = C.c_void_p(0)
        with torch.cuda.device(self._device):
            _lib.check(self._lib.prl_per_create(C.byref(h), C.byref(cfg), _lib.ptr(self.sum_tree), _lib.ptr(self.min_tree),
                                                _lib.ptr(self._max_priority), _stream_ptr(self._device)))
        self._per = h

    @property
    def per_handle(self) -> C.c_void_p:
        if not self._per.value:
            raise RuntimeError("replay buffer is empty: nothing has been pushed yet")
        return self._per

    def push_batch(self, state, *args, **kwargs) -> None:
        n = torch.as_tensor(state).shape[0]
        super().push_batch(state, *args, **kwargs)
        if n:
            # the slot of the first new row, derived AFTER the push: a push that upgrades the storage to dynamic
            # action sets re-creates the trees and re-pushes the old content from slot 0 (at max priority; learned
            # priorities do not survive the upgrade), so a position taken before the push would be stale
            first = (int(self._lib.prl_buf_head(self._handle)) + len(self) - min(n, self.capacity)) % self.capacity
            n = min(n, self.capacity)
            with torch.cuda.device(self._device):
                _lib.check(self._lib.prl_per_push(self.per_handle, first, n, _stream_ptr(self._device)))

    def clear(self) -> None:
        raise NotImplementedError("clear() on a prioritized buffer is not supported")

    def sample_prioritized(self, batch_size: int):
        """(slots i32[B], weights f32[B]) on the device."""
        if batch_size > len(self):
            raise ValueError(f"Can't get a batch of size {batch_size} from a replay buffer with only {len(self)} elements")
        slots = torch.empty(batch_size, dtype=torch.int32, device=self._device)
        w = torch.empty(batch_size, dtype=torch.float32, device=self._device)
        with torch.cuda.device(self._device):
            _lib.check(self._lib.prl_per_sample(self.per_handle, batch_size, _lib.ptr(slots), _lib.ptr(w),
                                                _stream_ptr(self._device)))
        return slots, w

    def sample(self, batch_size: int) -> TransitionBatch:
        slots, w = self.sample_prioritized(batch_size)
        self.last_slots = slots
        g = self._gather_slots(slots)
        A = self.n_actions
        curr = torch.arange(A, dtype=torch.float32, device=self._device).view(1, A, 1).expand(batch_size, A, 1).contiguous()
        tb = TransitionBatch(
            state=g["state"], action=g["action"].unsqueeze(-1), reward=g["reward"], next_state=g["next_state"],
            curr_available_actions=curr,
            curr_unavailable_actions_mask=torch.zeros((batch_size, A), dtype=torch.bool, device=self._device),
            next_available_actions=g["avail"].unsqueeze(-1), next_unavailable_actions_mask=g["mask"],
            terminated=g["terminated"], truncated=g["truncated"], weight=w)
        return tb.to(self._device_for_batches)

    def update_priorities(self, slots: torch.Tensor, td_errors: torch.Tensor) -> torch.Tensor:
        slots = slots.to(device=self._device, dtype=torch.int32).contiguous()
        td = td_errors.to(device=self._device, dtype=torch.float32).contiguous()
        out = torch.empty_like(td)
        with torch.cuda.device(self._device):
            _lib.check(self._lib.prl_per_set_priorities(self.per_handle, _lib.ptr(slots), _lib.ptr(td), slots.numel(),
                                                        _lib.ptr(out), _stream_ptr(self._device)))
        return out
