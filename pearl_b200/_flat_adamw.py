"""The parameter and optimizer plumbing the neural contextual-bandit plugins share (neural_linear.py, neural_bandit.py):
the model's parameters as views of one flat device vector, the AdamW state as views of three more, the learning rate
read from the optimizer, the row layout learn() folds from the stored action ids, and the refusals every such learner
makes.

A plugin keeps its runtime in a dict attribute named by `_RT` (keys handle, lib, flat, state, step) and names its C
prefix in `_ABI` ("prl_nlb"), whose `_adam_step` / `_set_adam_step` entries the helpers call.
"""
from __future__ import annotations

import torch

from . import _lib
from ._compat import BinaryActionTensorRepresentationModule, OneHotActionTensorRepresentationModule
from .bandit import _refuse_distributed


class FlatAdamW:
    _RT = ""
    _ABI = ""

    def _rt(self) -> dict:
        return self.__dict__[self._RT]

    def _lr(self) -> float:
        """lr of the AdamW(amsgrad=True) the reference constructs; other optimizers or settings are refused."""
        opt = self._optimizer
        groups = [g for g in opt.param_groups if len(g["params"])]
        g = groups[0] if isinstance(opt, torch.optim.AdamW) and len(groups) == 1 else None
        if (g is None or not g.get("amsgrad", False) or g.get("maximize", False) or tuple(g["betas"]) != (0.9, 0.999)
                or float(g["eps"]) != 1e-8 or float(g["weight_decay"]) != 0.01):
            raise NotImplementedError("the fused update implements torch.optim.AdamW(amsgrad=True) with default betas / eps / "
                                      "weight_decay over the model's parameters")
        return float(g["lr"])

    def _adopt(self, dev: torch.device) -> torch.Tensor:
        """The flat parameter vector, with the model's parameters re-pointed at views of it (copied in when they are not
        views of it already: first use, `.to()`, or parameters replaced)."""
        nl, params = self._rt(), list(self.model.parameters())
        flat = nl["flat"]
        if flat is None or flat.device != dev or params[0].data_ptr() != flat.data_ptr():
            n = sum(p.numel() for p in params)
            flat = torch.empty(n, dtype=torch.float32, device=dev)
            off = 0
            for p in params:
                k = p.numel()
                flat[off:off + k].copy_(p.detach().reshape(-1).to(device=dev, dtype=torch.float32))
                p.data = flat[off:off + k].view(p.shape)
                off += k
            nl["flat"] = flat
        return flat

    def _bind_optimizer(self, dev: torch.device, n_opt: int) -> None:
        """`optimizer.state` as views of the flat AdamW vectors for the first n_opt parameters (the ones that get a
        gradient; torch keeps no state for the others).  State that is there and is not ours (built by torch, or loaded
        with optimizer.load_state_dict) is imported first."""
        nl, params, st = self._rt(), list(self.model.parameters()), self._optimizer.state
        n = sum(p.numel() for p in params)
        state = nl["state"]
        if state is None or state[0].device != dev:
            state = [torch.zeros(n, dtype=torch.float32, device=dev) for _ in range(3)]
            nl["state"] = state
        used = params[:n_opt]
        if all(p in st and "exp_avg" in st[p] for p in used) and st[used[0]]["exp_avg"].data_ptr() == state[0].data_ptr():
            return
        if all(p in st and "exp_avg" in st[p] for p in used):
            cat = lambda key: torch.cat([st[p][key].detach().reshape(-1).to(dev, torch.float32) for p in used])  # noqa: E731
            m = sum(p.numel() for p in used)
            state[0][:m].copy_(cat("exp_avg"))
            state[1][:m].copy_(cat("exp_avg_sq"))
            state[2][:m].copy_(cat("max_exp_avg_sq") if all("max_exp_avg_sq" in st[p] for p in used) else cat("exp_avg_sq"))
            nl["step"] = int(float(st[used[0]]["step"]))
            if nl["handle"].value:
                _lib.check(getattr(nl["lib"], self._ABI + "_set_adam_step")(nl["handle"], nl["step"]))
        off = 0
        for i, p in enumerate(params):
            k = p.numel()
            if i < n_opt:
                st[p] = dict(step=torch.tensor(float(nl["step"]), dtype=torch.float32), exp_avg=state[0][off:off + k].view(p.shape),
                             exp_avg_sq=state[1][off:off + k].view(p.shape), max_exp_avg_sq=state[2][off:off + k].view(p.shape))
            else:
                st.pop(p, None)
            off += k

    def _after_step(self) -> None:
        nl = self._rt()
        nl["step"] = int(getattr(nl["lib"], self._ABI + "_adam_step")(nl["handle"]))
        for s in self._optimizer.state.values():
            if "step" in s:
                s["step"].fill_(float(nl["step"]))

    def _representation(self) -> tuple[int, int]:
        """(action_rep, action_dim) of the rows learn folds from the stored action ids."""
        if self._state_features_only:
            return 0, 0
        mod = self.action_representation_module
        if isinstance(mod, OneHotActionTensorRepresentationModule):
            return 1, int(mod.max_number_actions)
        if isinstance(mod, BinaryActionTensorRepresentationModule):
            return 2, int(mod.representation_dim)
        raise NotImplementedError(f"learn over a replay buffer folds the stored action id into the row as a one-hot or "
                                  f"binary representation; {type(mod).__name__} is not supported")

    def _check_learner(self) -> None:
        _refuse_distributed()
        h = getattr(self, "_history_summarization_module", None)
        if h is not None and any(True for _ in h.parameters()):
            raise NotImplementedError("a history summarization module with parameters: the CUDA bandit learner reads the "
                                      "stored states as they are")
