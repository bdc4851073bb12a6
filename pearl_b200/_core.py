"""The host code the flat-vector learner cores share (sac, sac_discrete, td3, iql, ppo, reinforce, qrdqn; the handle
lifecycle also serves rc_safety's cost-critic step): the device and generator, the C handle and the AdamW step counts it
is created at, the chunked round loop of `learn()`, and the reference initialisation of the flat parameter vectors.

A core names its C prefix in `_ABI` ("prl_sac"); the base calls that prefix's `_destroy`, `_workspace_bytes`, `_set_graph`
and `_last_launches` entries and its step-count entries (`_STEPS`: `_adam_step`, or TD3's `_actor_adam_step` and
`_critic_adam_step`).  The core keeps its vectors, its `_cfg(max_batch)` and its `_create(h, cfg)`,
which passes its pointer list to `<prefix>_create`.
"""
from __future__ import annotations

import ctypes as C
from typing import Callable, Optional

import torch

from . import _lib
from .replay_buffer import B200ReplayBuffer


def _bounds(action_space, low, high, device):
    if action_space is not None:
        low, high = getattr(action_space, "low"), getattr(action_space, "high")
    if low is None or high is None:
        raise ValueError("continuous SAC needs a box action space (`action_space.low/.high`) or explicit low/high")
    lo = torch.as_tensor(low, dtype=torch.float32).reshape(-1).to(device).contiguous()
    hi = torch.as_tensor(high, dtype=torch.float32).reshape(-1).to(device).contiguous()
    if lo.shape != hi.shape:
        raise ValueError("low / high shapes differ")
    return lo, hi


def fill_like_reference(vec: torch.Tensor, shapes: list, gen: torch.Generator, xavier: bool = True) -> None:
    """Fills `vec` layer by layer in `shapes` order ((out, in) weights, (out,) biases).  xavier: Xavier-uniform weights and
    biases 0.01 (neural_networks/common/utils.py xavier_init_weights).  Otherwise torch's default nn.Linear
    initialisation: weights and biases U(-1/sqrt(fan_in), 1/sqrt(fan_in))."""
    off, fan_in = 0, 1
    for shp in shapes:
        n = shp[0] * (shp[1] if len(shp) == 2 else 1)
        if len(shp) == 2:
            fan_in = shp[1]
        if xavier and len(shp) == 1:
            vec[off:off + n].fill_(0.01)
        else:
            bound = (6.0 / (shp[0] + shp[1])) ** 0.5 if xavier else fan_in ** -0.5
            vec[off:off + n].uniform_(-bound, bound, generator=gen)
        off += n
    assert off == vec.numel()


class Handle:
    """A C handle and the AdamW step counts the next one is created at (`_adam_steps`: one count, or one per entry of
    `_STEPS`).  The moments and parameters live in the learner's vectors, so a handle can be dropped at any time."""
    _ABI = ""
    _STEPS = ("_adam_step",)
    _ONE_STEP = ""          # restart()'s refusal of differing counts where the learner keeps one

    def adam_steps(self) -> tuple:
        """The AdamW step counts: the live handle's, else the ones the next handle starts at."""
        if not self._handle.value:
            return self._adam_steps
        return tuple(int(getattr(self._lib, self._ABI + s)(self._handle)) for s in self._STEPS)

    def restart(self, steps: Optional[tuple] = None) -> None:
        """Drop the C handle; the next call re-creates it at `steps` (default: the current counts).  One count per
        optimizer may be given to a learner that keeps one; they must agree."""
        steps = self.adam_steps() if steps is None else tuple(int(s) for s in steps)
        n = len(self._adam_steps)
        if len(steps) > n and len(set(steps)) != 1:
            raise NotImplementedError(self._ONE_STEP)
        if self._handle.value:
            getattr(self._lib, self._ABI + "_destroy")(self._handle)
            self._handle = C.c_void_p(0)
        self._adam_steps = steps[:n]

    def __del__(self):
        try:
            if getattr(self, "_handle", None) and self._handle.value:
                getattr(self._lib, self._ABI + "_destroy")(self._handle)
                self._handle = C.c_void_p(0)
        except Exception:
            pass


class FlatCore(Handle):
    """The device, generator, batch binding and round loop of a learner core (see the module docstring)."""

    def _open(self, device, training_rounds: int, batch_size: int, max_rounds_per_call: int, seed: Optional[int]) -> None:
        """The state every core has; `cuda` without an index is the current device."""
        self._device = torch.device("cuda", torch.cuda.current_device()) if device is None else torch.device(device)
        if self._device.index is None:
            self._device = torch.device("cuda", torch.cuda.current_device())
        self._lib = _lib.init(self._device.index)
        self._training_rounds, self._batch_size = int(training_rounds), int(batch_size)
        self._max_rounds = max(int(max_rounds_per_call), 1)
        self._training_steps = 0
        self.use_cuda_graph = True       # False: plain stream launches (profilers)
        self._handle = C.c_void_p(0)
        self._bound_batch = 0
        self._adam_steps = (0,) * len(self._STEPS)
        self._gen = torch.Generator(device=self._device)
        if seed is not None:
            self._gen.manual_seed(int(seed))

    @property
    def batch_size(self) -> int:
        return self._batch_size

    @property
    def training_rounds(self) -> int:
        return self._training_rounds

    def _fill(self, vec: torch.Tensor, shapes: list, xavier: bool = True) -> None:
        fill_like_reference(vec, shapes, self._gen, xavier)

    def _load(self, *pairs) -> None:
        """(flat vector, values) pairs: values in `torch.nn.Module.parameters()` order, flattened and copied in as fp32."""
        for dst, values in pairs:
            dst.copy_(torch.as_tensor(values, dtype=torch.float32).reshape(-1).to(self._device))

    def _workspace_bytes(self, cfg) -> int:
        return int(getattr(self._lib, self._ABI + "_workspace_bytes")(C.byref(cfg)))

    def _create(self, h: C.c_void_p, cfg) -> int:
        raise NotImplementedError

    def _bind(self, need_batch: int) -> None:
        """A handle for batches of up to `need_batch` rows (at least `batch_size`), re-created at the current step counts
        when the bound one is smaller."""
        if self._handle.value and need_batch <= self._bound_batch:
            return
        self.restart()
        cfg = self._cfg(max(need_batch, self._batch_size if self._batch_size > 0 else need_batch))
        self._workspace = torch.empty(self._workspace_bytes(cfg), dtype=torch.uint8, device=self._device)
        h = C.c_void_p(0)
        with torch.cuda.device(self._device):
            _lib.check(self._create(h, cfg))
        self._handle, self._bound_batch = h, cfg.max_batch

    def _batch(self, n: int) -> int:
        """Rows per round from a buffer of n transitions: all of them when batch_size is -1 or larger than n."""
        return n if (self._batch_size == -1 or n < self._batch_size) else self._batch_size

    def _accepts(self, replay_buffer, continuous: bool, refusal: str, holds: str = "ring") -> bool:
        """Refuses a buffer of another type (TypeError) or action kind (ValueError `refusal`); False when it is empty."""
        if not isinstance(replay_buffer, B200ReplayBuffer):
            raise TypeError(f"{type(self).__name__} learns from a B200ReplayBuffer (GPU-resident {holds})")
        if len(replay_buffer) == 0:
            return False
        if bool(replay_buffer.is_action_continuous) != continuous:
            raise ValueError(refusal)
        return True

    def _rounds(self, replay_buffer: B200ReplayBuffer, B: int, trace: Optional[dict], n_rows: int, rows: dict,
                chunk: Callable) -> dict:
        """`training_rounds` rounds in chunks of at most `_max_rounds`.  `chunk(r, done, out, idx)` makes one chunk's learn
        call and returns its status: r rounds after `done` of this call, at training step `_training_steps`, writing
        `out` [n_rows, r] and, when traced, the sampled rows `idx` [r, B].  The report maps each key of `rows` to the
        values of its row of `out`; `trace` gets the sampled rows and the last chunk's launch count."""
        R, dev = self._training_rounds, self._device
        report = {k: [] for k in rows}
        idx_all, done = [], 0
        while done < R:
            r = min(self._max_rounds, R - done)
            out = torch.empty((n_rows, r), dtype=torch.float32, device=dev)
            idx = torch.empty((r, B), dtype=torch.int32, device=dev) if trace is not None else None
            replay_buffer._rng_push()
            with torch.cuda.device(dev):
                _lib.check(getattr(self._lib, self._ABI + "_set_graph")(self._handle, int(self.use_cuda_graph)))
                _lib.check(chunk(r, done, out, idx))
            replay_buffer._rng_pull()
            host = out.cpu()
            for k, row in rows.items():
                report[k] += host[row].tolist()
            if idx is not None:
                idx_all.append(idx.cpu())
            self._training_steps += r
            done += r
        if trace is not None:
            trace["idx"] = torch.cat(idx_all)
            trace["launches"] = int(getattr(self._lib, self._ABI + "_last_launches")(self._handle))
        return report
