"""B200ReplayBuffer — GPU-resident drop-in for Pearl's BasicReplayBuffer.

Mirrors the plugin surface of `pearl.replay_buffers.replay_buffer.ReplayBuffer`
(replay_buffer.py:18-91) and the behaviour of `TensorBasedReplayBuffer` /
`BasicReplayBuffer` (tensor_based_replay_buffer.py:55-133,253-288;
basic_replay_buffer.py:17-48): FIFO eviction at `capacity`, `sample()` draws
WITHOUT replacement with CPython's `random.sample` index stream (bit-exact,
produced on the GPU) and returns a `TransitionBatch` with the reference's
field shapes / dtypes on `device_for_batches`.

Python holds torch tensors purely as containers (record storage, MT19937
state, batch outputs); all work happens in libpearlb200.so.  Unlike the
reference, transitions live in HBM (the reference keeps them on the CPU and a
unit test asserts it, test_replay_buffer.py:46-82 — a deliberate difference).
"""
from __future__ import annotations

import ctypes as C
import os
import random
from typing import Optional

import numpy as np
import torch

from . import _lib
from ._compat import ReplayBuffer, TransitionBatch


def _stream_ptr(device) -> C.c_void_p:
    return C.c_void_p(torch.cuda.current_stream(device).cuda_stream)


class B200ReplayBuffer(ReplayBuffer):
    _record_flags = 0               # PRL_BUF_* bits a subclass adds to every record layout it allocates
    _stores_costs = True            # False: a subclass that refuses `cost` (its records have no cost word)

    def __init__(self, capacity: int, device: Optional[torch.device | str | int] = None,
                 dynamic_action_space: bool = False, rng: str = "python") -> None:
        """
        Args:
            capacity: maximum number of transitions (oldest evicted first).
            device: CUDA device holding the buffer (default: current device).
            dynamic_action_space: store a per-transition list of next available
                actions (needed only if the action set changes between steps);
                switched on automatically by the first push that needs it.
            rng: "python" — every `sample()` / `learn()` continues the global
                `random` module's MT19937 stream and hands the advanced state
                back, exactly like the reference; "device" — the buffer keeps a
                private MT19937 stream (seed it with `seed()`), avoiding two
                small host<->device copies per call.
        """
        super().__init__()
        if not torch.cuda.is_available():
            raise RuntimeError("B200ReplayBuffer needs a CUDA device: pearl_b200 has no CPU path")
        if rng not in ("python", "device"):
            raise ValueError("rng must be 'python' or 'device'")
        self.capacity = int(capacity)
        self._device = torch.device("cuda", torch.cuda.current_device()) if device is None else torch.device(
            device if not isinstance(device, int) else f"cuda:{device}")
        if self._device.type != "cuda":
            raise RuntimeError("B200ReplayBuffer lives on a CUDA device")
        if self._device.index is None:
            self._device = torch.device("cuda", torch.cuda.current_device())
        self._device_for_batches = self._device
        self._lib = _lib.init(self._device.index)
        self._rng_mode = rng
        self._want_dynamic = bool(dynamic_action_space)
        self._has_cost = False        # decided by the first push, as the reference decides from transitions[0].cost
        self._handle = C.c_void_p(0)
        self._storage = None
        self._mt = torch.zeros(625, dtype=torch.int32, device=self._device)
        self._mt_host = np.zeros(625, dtype=np.uint32)
        self._layout = None
        self._desc = None
        self.obs_dim = self.n_actions = self.act_dim = None
        # rng="device": never leave the private MT19937 stream uninitialised (an all-zero state twists to zeros for
        # ever and the set-branch sampler would spin on duplicates); a distinct stream per buffer until seed() is called
        self._pending_seed = int.from_bytes(os.urandom(8), "little") if rng == "device" else None
        self._shard = None            # (rank, world) when this buffer is one shard of a logical multi-GPU buffer
        self._g_pushed = 0            # pushes to the logical buffer so far

    # ------------------------------------------------------------------ plumbing
    def __del__(self):
        try:
            if getattr(self, "_handle", None) and self._handle.value:
                self._lib.prl_buf_destroy(self._handle)
                self._handle = C.c_void_p(0)
        except Exception:
            pass

    @property
    def device_for_batches(self) -> torch.device:
        return self._device_for_batches

    @device_for_batches.setter
    def device_for_batches(self, new_device_for_batches: torch.device) -> None:
        self._device_for_batches = torch.device(new_device_for_batches)

    @property
    def device(self) -> torch.device:
        return self._device

    @property
    def handle(self) -> C.c_void_p:
        if not self._handle.value:
            raise RuntimeError("replay buffer is empty: nothing has been pushed yet")
        return self._handle

    @property
    def has_cost(self) -> bool:
        """True when the records store a cost (the first push carried one); sample() then fills TransitionBatch.cost."""
        return self._has_cost

    @property
    def record_bytes(self) -> int:
        return 0 if self._layout is None else 4 * self._layout.record_words

    def _allocate(self, obs_dim: int, n_actions: int, act_dim: int, dynamic: bool) -> None:
        flags = _lib.PRL_BUF_CONTINUOUS if self._is_action_continuous else _lib.PRL_BUF_DISCRETE
        if dynamic:
            flags |= _lib.PRL_BUF_DYNAMIC_ACTIONS
        if self._has_cost:
            flags |= _lib.PRL_BUF_COST
        flags |= self._record_flags
        desc = _lib.BufDesc(self.capacity, obs_dim, act_dim, n_actions, flags)
        lay = _lib.BufLayout()
        _lib.check(self._lib.prl_buf_layout_of(C.byref(desc), C.byref(lay)))
        with torch.cuda.device(self._device):
            storage = torch.empty(lay.storage_bytes // 4, dtype=torch.int32, device=self._device)
        handle = C.c_void_p(0)
        _lib.check(self._lib.prl_buf_create(C.byref(handle), C.byref(desc), _lib.ptr(storage), _lib.ptr(self._mt)))
        self._storage, self._handle, self._layout, self._desc = storage, handle, lay, desc
        self.obs_dim, self.n_actions, self.act_dim = obs_dim, n_actions, act_dim
        if self._pending_seed is not None:
            self.seed(self._pending_seed)

    def _upgrade_to_dynamic(self) -> None:
        """Re-create the storage with per-transition action lists, keeping the content."""
        n = self.local_len()
        old = None
        if n:
            old = self._gather_logical(torch.arange(n, dtype=torch.int32, device=self._device))
        self._lib.prl_buf_destroy(self._handle)
        self._allocate(self.obs_dim, self.n_actions, self.act_dim, True)
        if old is not None:
            cnt = (~old["mask"].bool()).sum(1).to(torch.int32)
            self.push_batch(old["state"], old["action"].to(torch.int32), old["reward"], old["next_state"],
                            old["terminated"], old["truncated"],
                            next_available_ids=old["avail"].to(torch.uint8), next_available_count=cnt, cost=old.get("cost"))

    # ------------------------------------------------------------------ RNG
    def seed(self, seed: int) -> None:
        """`random.seed(seed)` for the buffer's private stream (rng='device')."""
        if not self._handle.value:
            self._pending_seed = seed
            return
        s = abs(int(seed))
        key = []
        while True:
            key.append(s & 0xFFFFFFFF)
            s >>= 32
            if s == 0:
                break
        arr = np.asarray(key, dtype=np.uint32)
        _lib.check(self._lib.prl_rng_seed(self._handle, C.c_void_p(arr.ctypes.data), len(key),
                                          _stream_ptr(self._device)))
        self._pending_seed = None

    def set_rng_state(self, words) -> None:
        """words: 625 uint32 = random.getstate()[1]."""
        self._mt_host[:] = np.asarray(words, dtype=np.uint64).astype(np.uint32)
        _lib.check(self._lib.prl_rng_set_state(self.handle, C.c_void_p(self._mt_host.ctypes.data),
                                               _stream_ptr(self._device)))

    def get_rng_state(self) -> np.ndarray:
        _lib.check(self._lib.prl_rng_get_state(self.handle, C.c_void_p(self._mt_host.ctypes.data),
                                               _stream_ptr(self._device)))
        return self._mt_host.copy()

    def _rng_push(self) -> None:
        if self._rng_mode == "python":
            self.set_rng_state(random.getstate()[1])

    def _rng_pull(self) -> None:
        if self._rng_mode == "python":
            st = self.get_rng_state()
            ver, _, gauss_next = random.getstate()   # random.sample never touches the cached Gaussian: keep it
            random.setstate((ver, tuple(int(x) for x in st), gauss_next))

    # ------------------------------------------------------------------ write side
    def push(self, state, action, reward, terminated, truncated, curr_available_actions=None,
             next_state=None, next_available_actions=None, max_number_actions=None, cost=None) -> None:
        """One transition, same signature as the reference (tensor_based_replay_buffer.py:55-69)."""
        if cost is not None and not self._stores_costs:
            raise NotImplementedError(f"{type(self).__name__} does not store costs")
        st = torch.as_tensor(state, dtype=torch.float32).reshape(-1).cpu()
        nst = None if next_state is None else torch.as_tensor(next_state, dtype=torch.float32).reshape(-1).cpu()
        ids = cnt = None
        if self._is_action_continuous:
            act = torch.as_tensor(action, dtype=torch.float32).reshape(1, -1).cpu()
        else:
            if max_number_actions is None:
                if curr_available_actions is None:
                    raise AssertionError("curr_available_actions is needed to infer max_number_actions")
                max_number_actions = curr_available_actions.n
            act = torch.as_tensor(action).reshape(-1)[:1].to(torch.int32).cpu()
            if next_available_actions is not None:
                a_ids = next_available_actions.actions_batch.reshape(next_available_actions.n, -1)[:, 0]
                a_ids = a_ids.to(torch.int64).cpu()
                full = a_ids.numel() == max_number_actions and bool(
                    (a_ids == torch.arange(max_number_actions)).all())
                if not full:
                    ids = torch.zeros(1, max_number_actions, dtype=torch.uint8)
                    ids[0, : a_ids.numel()] = a_ids.to(torch.uint8)
                    cnt = torch.tensor([a_ids.numel()], dtype=torch.int32)
        self.push_batch(st.unsqueeze(0), act, torch.tensor([float(reward)], dtype=torch.float32),
                        None if nst is None else nst.unsqueeze(0),
                        torch.tensor([bool(terminated)]), torch.tensor([bool(truncated)]),
                        next_available_ids=ids, next_available_count=cnt,
                        max_number_actions=max_number_actions,
                        cost=None if cost is None else torch.tensor([float(cost)], dtype=torch.float32))

    def push_batch(self, state, action, reward, next_state, terminated, truncated,
                   next_available_ids=None, next_available_count=None, max_number_actions=None, cost=None) -> None:
        """Vectorised push of n transitions (host or device tensors, struct-of-arrays).

        state/next_state [n, obs]; action [n] ints (discrete) or [n, act_dim] floats;
        reward [n]; terminated/truncated [n] bool; optional next_available_ids
        [n, A] uint8 + next_available_count [n] int32 (omit when every action is
        available); cost [n] floats (the first push decides whether the buffer
        stores costs, and every later push must agree).  Host tensors are staged
        through pinned memory inside the library; device tensors are packed by a
        kernel.
        """
        if cost is not None and not self._stores_costs:
            raise NotImplementedError(f"{type(self).__name__} does not store costs")
        state = torch.as_tensor(state)
        n = state.shape[0]
        if n == 0:
            return
        on_dev = state.is_cuda
        dev = self._device if on_dev else torch.device("cpu")

        def prep(x, dtype):
            return None if x is None else torch.as_tensor(x).to(device=dev, dtype=dtype).contiguous()

        state = prep(state.reshape(n, -1), torch.float32)
        next_state = prep(None if next_state is None else torch.as_tensor(next_state).reshape(n, -1), torch.float32)
        reward = prep(torch.as_tensor(reward).reshape(n), torch.float32)
        terminated = prep(torch.as_tensor(terminated).reshape(n), torch.uint8)
        truncated = prep(torch.as_tensor(truncated).reshape(n), torch.uint8)
        if self._is_action_continuous:
            action = prep(torch.as_tensor(action).reshape(n, -1), torch.float32)
            n_act, act_dim = 0, action.shape[1]
        else:
            action = prep(torch.as_tensor(action).reshape(n), torch.int32)
            act_dim = 1
            n_act = self.n_actions if self.n_actions else max_number_actions
            if n_act is None:
                if next_available_ids is not None:
                    n_act = torch.as_tensor(next_available_ids).shape[1]
                else:
                    raise ValueError("max_number_actions is required for the first discrete push")
        ids = prep(next_available_ids, torch.uint8)
        cnt = prep(next_available_count, torch.int32)
        cost = prep(None if cost is None else torch.as_tensor(cost).reshape(n), torch.float32)
        if not self._handle.value:
            self._has_cost = cost is not None
            self._allocate(state.shape[1], n_act, act_dim, self._want_dynamic or ids is not None)
        elif (cost is not None) != self._has_cost:
            raise ValueError("this buffer stores costs: every push needs one" if self._has_cost else
                             "this buffer stores no costs (its first push had none): a push with costs is refused")
        if state.shape[1] != self.obs_dim:
            raise ValueError(f"state has {state.shape[1]} features, buffer stores {self.obs_dim}")
        if ids is not None and not (self._desc.flags & _lib.PRL_BUF_DYNAMIC_ACTIONS):
            self._upgrade_to_dynamic()
        with torch.cuda.device(self._device):
            fields = [_lib.ptr(state), _lib.ptr(action), _lib.ptr(reward), _lib.ptr(next_state), _lib.ptr(terminated),
                      _lib.ptr(truncated), _lib.ptr(ids), _lib.ptr(cnt)]
            if cost is not None:
                fn = self._lib.prl_buf_push_device_cost if on_dev else self._lib.prl_buf_push_host_cost
                _lib.check(fn(self._handle, n, *fields, _lib.ptr(cost), _stream_ptr(self._device)))
            else:
                self._push_records(on_dev, n, fields)
        if on_dev:  # keep the sources alive until the pack kernel has run
            torch.cuda.current_stream(self._device).synchronize()

    def _push_records(self, on_dev: bool, n: int, fields: list) -> None:
        """The library push of n prepared transitions (`fields`: the pointer arguments of prl_buf_push_host / _device)."""
        fn = self._lib.prl_buf_push_device if on_dev else self._lib.prl_buf_push_host
        _lib.check(fn(self._handle, n, *fields, _stream_ptr(self._device)))

    # ------------------------------------------------------------------ multi-GPU sharding (SURVEY.md 8e)
    def set_shard(self, rank: int, world: int, global_pushed: int) -> None:
        """Declare this buffer rank `rank`'s shard of ONE logical buffer of `world * capacity` transitions: the
        transition with global write counter g lives on rank g mod world at local slot (g div world) mod capacity
        (pearl_b200.dist.shard_owner).  The local content must be exactly this rank's share, pushed in order."""
        _lib.check(self._lib.prl_buf_set_shard(self.handle, int(rank), int(world), int(global_pushed)))
        self._shard = (int(rank), int(world)) if world > 1 else None
        self._g_pushed = int(global_pushed)

    def push_batch_sharded(self, rank: int, world: int, state, action, reward, next_state, terminated, truncated,
                           **kwargs) -> None:
        """Every rank calls this with the SAME global batch (a replicated producer); the rank keeps the rows it owns.
        `len()` of a sharded buffer is the population of the logical buffer, and `learn()` of a learner with a
        communicator draws the same `batch` global indices on every rank as one GPU would."""
        state = torch.as_tensor(state)
        n = state.shape[0]
        first = (rank - self._g_pushed) % world
        pick = lambda x: None if x is None else torch.as_tensor(x)[first::world]
        if first < n:
            self.push_batch(pick(state), pick(action), pick(reward), pick(next_state), pick(terminated), pick(truncated),
                            **{k: pick(v) if torch.is_tensor(v) else v for k, v in kwargs.items()})
        if self._handle.value:
            self.set_shard(rank, world, self._g_pushed + n)
        else:
            self._g_pushed += n

    def local_len(self) -> int:
        return int(self._lib.prl_buf_len(self._handle)) if self._handle.value else 0

    # ------------------------------------------------------------------ snapshot / offline data (SURVEY.md 8f rank 4)
    def state_dict(self) -> dict:
        """Snapshot of the buffer: the stored records in FIFO order (oldest first, raw record words as the kernels keep
        them), the layout needed to re-create the storage, and the sampler's MT19937 stream.  The reference never
        serialises replay-buffer contents (the buffer is not a Module; `PearlAgent.compare` only checks its type,
        pearl_agent.py:313-318) — this is what makes a GPU training job resumable."""
        if self._shard:
            raise NotImplementedError("snapshot a sharded buffer shard by shard with set_shard cleared")
        n = self.local_len()
        out = dict(capacity=self.capacity, len=n, is_action_continuous=bool(self._is_action_continuous),
                   obs_dim=self.obs_dim, n_actions=self.n_actions, act_dim=self.act_dim, rng_mode=self._rng_mode,
                   cost=self._has_cost)
        if n:
            W = self._layout.record_words
            head = int(self._lib.prl_buf_head(self._handle))
            rec = self._storage[: self.capacity * W].view(self.capacity, W)
            order = (torch.arange(n, device=self._device) + head) % self.capacity
            out.update(records=rec[order].cpu(), record_words=W, dynamic=bool(self._desc.flags & _lib.PRL_BUF_DYNAMIC_ACTIONS),
                       mt_state=torch.from_numpy(self.get_rng_state().astype(np.int64)))
        return out

    def load_state_dict(self, sd: dict) -> None:
        """Restore a snapshot taken by `state_dict()` (the contents land at logical positions 0 .. len-1)."""
        if int(sd["capacity"]) != self.capacity:
            raise ValueError(f"snapshot of a buffer of capacity {sd['capacity']}, this one holds {self.capacity}")
        self._is_action_continuous = bool(sd["is_action_continuous"])
        n = int(sd["len"])
        if self._handle.value:
            self.clear()
        if n == 0:
            return
        has_cost = bool(sd.get("cost", False))      # a snapshot from before costs were stored is a plain buffer
        if has_cost and not self._stores_costs:
            raise NotImplementedError(f"{type(self).__name__} does not store costs")
        if (not self._handle.value or bool(self._desc.flags & _lib.PRL_BUF_DYNAMIC_ACTIONS) != bool(sd["dynamic"])
                or has_cost != self._has_cost):
            if self._handle.value:
                self._lib.prl_buf_destroy(self._handle)
                self._handle = C.c_void_p(0)
            self._has_cost = has_cost
            self._allocate(int(sd["obs_dim"]), int(sd["n_actions"] or 0), int(sd["act_dim"]), bool(sd["dynamic"]))
        W = self._layout.record_words
        if int(sd["record_words"]) != W:
            raise ValueError("snapshot record layout does not match this build")
        self._storage[: n * W].copy_(sd["records"].reshape(-1).to(self._device))
        _lib.check(self._lib.prl_buf_set_occupancy(self._handle, n, 0))
        self.set_rng_state(sd["mt_state"].numpy().astype(np.uint32))

    def load_offline_data(self, transitions, max_number_actions_if_discrete: Optional[int] = None, chunk: int = 65536) -> int:
        """The reference's `get_offline_data_in_buffer` (utils/functional_utils/train_and_eval/
        offline_learning_and_evaluation.py:39-137) for a device-resident buffer: `transitions` is the iterable of dicts a `.pt` offline
        data file holds (`observation, action, reward, next_observation, curr_available_actions, next_available_actions,
        done`); they are packed into the device ring `chunk` at a time instead of one Python push each.  Discrete action
        sets must be the full `range(max_number_actions)` (a `Discrete(n)` space or a DiscreteActionSpace of all ids), as in
        the reference's offline benchmarks.  Returns the number of transitions loaded."""
        if self._is_action_continuous:
            if max_number_actions_if_discrete is not None:
                raise ValueError("is_action_continuous = True requires max_number_actions to be None")
        elif max_number_actions_if_discrete is None:
            raise ValueError("is_action_continuous = False requires max_number_actions to be an integer value")
        cols = dict(s=[], a=[], r=[], ns=[], d=[])
        total = 0

        def flush():
            nonlocal total
            if not cols["s"]:
                return
            n = len(cols["s"])
            st = torch.stack([torch.as_tensor(x, dtype=torch.float32).reshape(-1) for x in cols["s"]])
            ns = torch.stack([torch.as_tensor(x, dtype=torch.float32).reshape(-1) for x in cols["ns"]])
            if self._is_action_continuous:
                ac = torch.stack([torch.as_tensor(x, dtype=torch.float32).reshape(-1) for x in cols["a"]])
            else:
                ac = torch.tensor([int(torch.as_tensor(x).reshape(-1)[0]) for x in cols["a"]], dtype=torch.int32)
            self.push_batch(st, ac, torch.tensor([float(x) for x in cols["r"]]), ns,
                            torch.tensor([bool(x) for x in cols["d"]]), torch.zeros(n, dtype=torch.bool),
                            max_number_actions=max_number_actions_if_discrete)
            total += n
            for v in cols.values():
                v.clear()

        for t in transitions:
            if not self._is_action_continuous:
                for key in ("curr_available_actions", "next_available_actions"):
                    sp = t.get(key)
                    if sp is not None and int(getattr(sp, "n", max_number_actions_if_discrete)) != max_number_actions_if_discrete:
                        raise NotImplementedError("offline transitions with partial action sets: push them one by one")
            cols["s"].append(t["observation"]); cols["a"].append(t["action"]); cols["r"].append(t["reward"])
            cols["ns"].append(t["next_observation"]); cols["d"].append(t["done"])
            if len(cols["s"]) >= chunk:
                flush()
        flush()
        return total

    # ------------------------------------------------------------------ read side
    def __len__(self) -> int:
        if not self._handle.value:
            return 0
        return int(self._lib.prl_buf_global_len(self._handle)) if self._shard else int(self._lib.prl_buf_len(self._handle))

    def clear(self) -> None:
        if self._handle.value:
            _lib.check(self._lib.prl_buf_clear(self._handle))
            if self._shard:
                self.set_shard(self._shard[0], self._shard[1], 0)

    def sample_indices(self, batch_size: int, rounds: int = 1):
        """(logical, slot) int32 [rounds, batch] tensors on the device; logical index 0 = oldest."""
        if batch_size > len(self):
            raise ValueError(f"Can't get a batch of size {batch_size} from a replay buffer with "
                             f"only {len(self)} elements")
        logical = torch.empty((rounds, batch_size), dtype=torch.int32, device=self._device)
        slot = torch.empty((rounds, batch_size), dtype=torch.int32, device=self._device)
        if batch_size == 0 or rounds == 0:
            return logical, slot
        with torch.cuda.device(self._device):
            self._rng_push()
            _lib.check(self._lib.prl_buf_sample_indices(self.handle, rounds, batch_size, _lib.ptr(logical),
                                                        _lib.ptr(slot), _stream_ptr(self._device)))
            self._rng_pull()
        return logical, slot

    def _gather_slots(self, slot: torch.Tensor) -> dict:
        if self._shard:
            raise NotImplementedError("a sharded buffer holds 1 / world of the sampled rows: use learn() of a learner "
                                      "with a communicator (the gradient, not the batch, crosses NVLink)")
        k = slot.numel()
        dev = self._device
        A = self.n_actions or 0
        out = dict(
            state=torch.empty((k, self.obs_dim), dtype=torch.float32, device=dev),
            next_state=torch.empty((k, self.obs_dim), dtype=torch.float32, device=dev),
            reward=torch.empty((k,), dtype=torch.float32, device=dev),
            terminated=torch.empty((k,), dtype=torch.bool, device=dev),
            truncated=torch.empty((k,), dtype=torch.bool, device=dev),
        )
        if self._is_action_continuous:
            out["action"] = torch.empty((k, self.act_dim), dtype=torch.float32, device=dev)
            out["avail"] = out["mask"] = None
        else:
            out["action"] = torch.empty((k,), dtype=torch.int64, device=dev)
            out["avail"] = torch.empty((k, A), dtype=torch.float32, device=dev)
            out["mask"] = torch.empty((k, A), dtype=torch.bool, device=dev)
        with torch.cuda.device(dev):
            _lib.check(self._lib.prl_buf_gather(
                self.handle, _lib.ptr(slot.contiguous()), k, _lib.ptr(out["state"]), _lib.ptr(out["action"]),
                _lib.ptr(out["reward"]), _lib.ptr(out["next_state"]), _lib.ptr(out["terminated"]),
                _lib.ptr(out["truncated"]), _lib.ptr(out["avail"]), _lib.ptr(out["mask"]),
                _stream_ptr(dev)))
            if self._has_cost:
                out["cost"] = torch.empty((k,), dtype=torch.float32, device=dev)
                _lib.check(self._lib.prl_buf_gather_cost(self.handle, _lib.ptr(slot.contiguous()), k, _lib.ptr(out["cost"]),
                                                         _stream_ptr(dev)))
        return out

    def _gather_logical(self, logical: torch.Tensor) -> dict:
        head = int(self._lib.prl_buf_head(self._handle))
        slot = ((logical.to(torch.int64) + head) % self.capacity).to(torch.int32)
        return self._gather_slots(slot)

    def sample(self, batch_size: int) -> TransitionBatch:
        """`TensorBasedReplayBuffer.sample` (tensor_based_replay_buffer.py:253-282)."""
        _, slot = self.sample_indices(batch_size, 1)
        return self._batch_of_slots(slot[0]).to(self._device_for_batches)

    def _batch_of_slots(self, slot: torch.Tensor) -> TransitionBatch:
        """The TransitionBatch of the records at ring slots `slot`, on the buffer's device."""
        batch_size = slot.numel()
        g = self._gather_slots(slot)
        if self._is_action_continuous:
            tb = TransitionBatch(state=g["state"], action=g["action"], reward=g["reward"],
                                 next_state=g["next_state"], terminated=g["terminated"],
                                 truncated=g["truncated"], cost=g.get("cost"))
        else:
            A = self.n_actions
            curr = torch.arange(A, dtype=torch.float32, device=self._device).view(1, A, 1).expand(
                batch_size, A, 1).contiguous()
            tb = TransitionBatch(
                state=g["state"], action=g["action"].unsqueeze(-1), reward=g["reward"],
                next_state=g["next_state"],
                curr_available_actions=curr,
                curr_unavailable_actions_mask=torch.zeros((batch_size, A), dtype=torch.bool, device=self._device),
                next_available_actions=g["avail"].unsqueeze(-1),
                next_unavailable_actions_mask=g["mask"],
                terminated=g["terminated"], truncated=g["truncated"], cost=g.get("cost"))
        return tb
