"""Random draws made on the host and staged to the device.

The exploration modules that sample (SquareCB / FastCB, Thompson sampling) draw from torch's default CPU generator,
exactly the draws the reference makes, so a seeded run stays in step with a reference run.  The draws reach the device
through one pinned buffer per learner.
"""
from __future__ import annotations

import torch


class PinnedDraws:
    """A pinned host buffer and a device buffer, grown on demand.  `put` copies host draws to the device asynchronously on
    the current stream; it waits for its previous copy before it overwrites the pinned buffer."""

    def __init__(self) -> None:
        self.pin = self.dev = self.done = None

    def put(self, draws: torch.Tensor, dev: torch.device) -> torch.Tensor:
        n = draws.numel()
        if self.done is not None:
            self.done.synchronize()
        if self.pin is None or self.pin.numel() < n or self.dev.device != dev:
            m = max(n, 64)
            self.pin = torch.empty(m, dtype=torch.float32, pin_memory=True)
            self.dev = torch.empty(m, dtype=torch.float32, device=dev)
            self.done = None
        self.pin[:n].copy_(draws.reshape(-1))
        out = self.dev[:n]
        with torch.cuda.device(dev):
            out.copy_(self.pin[:n], non_blocking=True)
            self.done = torch.cuda.Event()
            self.done.record()
        return out
