"""B200NeuralBandit — Pearl's NeuralBandit (policy_learners/contextual_bandits/neural_bandit.py: a value network fitted to the
observed rewards) with its learning, scoring and SquareCB / FastCB / greedy action choice on an H100 through `prl_nb_*`
(csrc/neural_bandit.cu, include/pearl_b200.h).

When Pearl is importable this is the reference class with `learn`, `learn_batch`, `act` and `get_scores` replaced: the
reference constructor runs unchanged, so `PearlAgent` accepts it as it is and `state_dict()` / `compare()` are the
reference's own.  Without Pearl it subclasses a stand-in (_compat.py) with the same constructor, defaults and state_dict
keys.

The network's parameters are views of one flat device vector and the optimizer's AdamW state views of three more
(_flat_adamw.py).  A state loaded with `load_state_dict` is what the next call reads, and the learning rate is read from
`optimizer.param_groups` on every call.  No CPU fallback.

    learn(B200ReplayBuffer)   PolicyLearner.learn: training_rounds x (sample, the row as learn_batch builds it, one round)
    learn_batch(batch)        one round on a caller's batch; batch.action is the already represented action matrix
    act                       NoExploration: the first maximum over the available actions, as action vectors;
                              SquareCBExploration / FastCBExploration: one state, the sampled action INDEX as a 0-d
                              torch.int32 CPU tensor, the availability mask ignored, as the reference returns and does
    get_scores                the network's raw output, [batch, A]
SquareCB / FastCB draw the A exponentials of the reference's Categorical(p).sample() from torch's default CPU generator,
exactly as many per call, so the generator stays in step with a reference run; nothing else here touches it.
"""
from __future__ import annotations

import ctypes as C
from typing import Any, Optional

import torch

from . import _lib
from ._draws import PinnedDraws
from ._compat import (FastCBExploration, LossType, NoExploration, SquareCBExploration, TiebreakingStrategy,
                      _RefNeuralBandit)
from ._flat_adamw import FlatAdamW
from .bandit import _refuse_distributed
from .per import B200PrioritizedReplayBuffer
from .replay_buffer import B200ReplayBuffer, _stream_ptr

SCORE_ROWS = 4096          # feature rows the workspace holds per scoring chunk
_LOSS = {LossType.MSE: 0, LossType.MAE: 1}


class B200NeuralBandit(FlatAdamW, _RefNeuralBandit):
    _RT, _ABI = "_nb", "prl_nb"

    def __init__(self, feature_dim: int, hidden_dims: list, exploration_module, output_dim: int = 1, training_rounds: int = 100,
                 batch_size: int = 128, learning_rate: float = 0.001, state_features_only: bool = False, loss_type=LossType.MSE,
                 action_representation_module=None, *, max_rounds_per_call: int = 1024) -> None:
        hidden_dims = list(hidden_dims)
        if len(hidden_dims) != 2:
            raise NotImplementedError(f"hidden_dims={hidden_dims}: the CUDA NeuralBandit is built for two hidden layers")
        if output_dim != 1:
            raise NotImplementedError(f"output_dim={output_dim}: the CUDA NeuralBandit has one output (the reference's "
                                      "learn_batch views the prediction as the reward's shape, which needs one)")
        if (LossType(loss_type) if isinstance(loss_type, str) else loss_type) is LossType.CROSS_ENTROPY:
            raise NotImplementedError("LossType.CROSS_ENTROPY: the reference applies binary_cross_entropy to the raw linear "
                                      "output and raises once a prediction leaves [0, 1], which would need a host check "
                                      "every round; the CUDA NeuralBandit implements MSE and MAE")
        super().__init__(feature_dim=feature_dim, hidden_dims=hidden_dims, exploration_module=exploration_module,
                         output_dim=output_dim, training_rounds=training_rounds, batch_size=batch_size,
                         learning_rate=learning_rate, state_features_only=state_features_only, loss_type=loss_type,
                         action_representation_module=action_representation_module)
        object.__setattr__(self, "_nb", dict(handle=C.c_void_p(0), key=None, batch=0, ws=None, lib=None, lr=None, flat=None,
                                             state=None, step=0, draws=PinnedDraws(), prob=None))
        self._hidden = (int(hidden_dims[0]), int(hidden_dims[1]))
        self.max_rounds_per_call = max(int(max_rounds_per_call), 1)
        self.use_cuda_graph = True       # False: plain stream launches (profilers)

    def __del__(self):
        try:
            nb = self.__dict__.get("_nb")
            if nb and nb["handle"].value:
                nb["lib"].prl_nb_destroy(nb["handle"])
                nb["handle"] = C.c_void_p(0)
        except Exception:
            pass

    # ------------------------------------------------------------------ binding
    def _device_of(self, hint: Optional[torch.device] = None) -> torch.device:
        dev = next(self.model.parameters()).device
        if dev.type != "cuda":
            dev = hint if hint is not None else torch.device("cuda", torch.cuda.current_device())
            self.model.to(dev)
        return dev

    def _bind(self, dev: torch.device, obs: int, act_dim: int, rep: int, n_actions: int, batch: int, any_rep: bool = False) -> dict:
        """The prl_nb handle over the current parameter and AdamW buffers for this row layout, re-created when a buffer
        moved, the layout or a setting changed or the batch outgrew it.  learn_batch and scoring read only the widths
        (any_rep), so any handle of the same widths serves them."""
        nb = self._nb
        if obs + act_dim != self._feature_dim:
            raise ValueError(f"state ({obs}) + action features ({act_dim}) != feature_dim ({self._feature_dim})")
        if self.loss_type not in _LOSS:
            raise NotImplementedError(f"{self.loss_type}: the CUDA NeuralBandit implements MSE and MAE")
        flat = self._adopt(dev)
        self._bind_optimizer(dev, len(list(self.model.parameters())))
        lr = self._lr()
        key = (obs, act_dim, rep, n_actions, _LOSS[self.loss_type], self.max_rounds_per_call, flat.data_ptr(),
               nb["state"][0].data_ptr())
        same = (lambda k: k[:2] + k[4:] == key[:2] + key[4:]) if any_rep else (lambda k: k == key)  # noqa: E731
        if nb["handle"].value and same(nb["key"]) and batch <= nb["batch"]:
            if lr != nb["lr"]:
                _lib.check(nb["lib"].prl_nb_set_lr(nb["handle"], lr))
                nb["lr"] = lr
            return nb
        lib = _lib.init(dev.index)
        if nb["handle"].value:
            nb["step"] = int(lib.prl_nb_adam_step(nb["handle"]))
            lib.prl_nb_destroy(nb["handle"])
            nb["handle"] = C.c_void_p(0)
        B = max(batch, self._batch_size if self._batch_size > 0 else batch, 1)
        h1, h2 = self._hidden
        cfg = _lib.NbCfg(obs, n_actions, act_dim, rep, h1, h2, _LOSS[self.loss_type], B, self.max_rounds_per_call, SCORE_ROWS,
                         lr, 0.9, 0.999, 1e-8, 0.01)
        nbytes = int(lib.prl_nb_workspace_bytes(C.byref(cfg)))
        if nbytes < 0:
            raise ValueError(_lib.last_error())
        ws = torch.empty(nbytes, dtype=torch.uint8, device=dev)
        h, p = C.c_void_p(0), _lib.ptr
        st = nb["state"]
        with torch.cuda.device(dev):
            _lib.check(lib.prl_nb_create(C.byref(h), C.byref(cfg), p(flat), p(st[0]), p(st[1]), p(st[2]), nb["step"], p(ws)))
        nb.update(handle=h, key=key, batch=B, ws=ws, lib=lib, lr=lr)
        return nb

    # ------------------------------------------------------------------ PolicyLearner.learn (policy_learner.py)
    def learn(self, replay_buffer: B200ReplayBuffer, trace: Optional[dict] = None) -> dict[str, Any]:
        if not isinstance(replay_buffer, B200ReplayBuffer):
            raise TypeError("B200NeuralBandit learns from a B200ReplayBuffer (GPU-resident ring)")
        if isinstance(replay_buffer, B200PrioritizedReplayBuffer):
            raise NotImplementedError("NeuralBandit samples uniformly, as the reference: a B200PrioritizedReplayBuffer "
                                      "is not supported")
        if replay_buffer._shard is not None:
            raise NotImplementedError("a sharded replay buffer: the CUDA bandit learner samples local buffers only")
        self._check_learner()
        n = len(replay_buffer)
        if n == 0:
            return {}
        if bool(replay_buffer.is_action_continuous):
            raise NotImplementedError("a replay buffer with continuous actions: the CUDA NeuralBandit folds discrete "
                                      "action ids into its rows")
        rep, act_dim = self._representation()
        B = n if (self._batch_size == -1 or n < self._batch_size) else self._batch_size
        dev = replay_buffer.device
        self._device_of(dev)
        nb = self._bind(dev, int(replay_buffer.obs_dim), act_dim, rep, int(replay_buffer.n_actions), B)
        R, lib = self._training_rounds, nb["lib"]
        out = torch.empty((3, R, B), dtype=torch.float32, device=dev)      # prediction, label, weight
        loss = torch.empty(R, dtype=torch.float32, device=dev)
        idx = torch.empty((R, B), dtype=torch.int32, device=dev) if trace is not None else None
        done = 0
        while done < R:
            r = min(self.max_rounds_per_call, R - done)
            replay_buffer._rng_push()
            with torch.cuda.device(dev):
                _lib.check(lib.prl_nb_set_graph(nb["handle"], int(self.use_cuda_graph)))
                _lib.check(lib.prl_nb_learn(nb["handle"], replay_buffer.handle, r, B, _lib.ptr(out[0, done]), _lib.ptr(out[1, done]),
                                            _lib.ptr(out[2, done]), _lib.ptr(loss[done:]),
                                            _lib.ptr(idx[done]) if idx is not None else None, _stream_ptr(dev)))
            replay_buffer._rng_pull()
            done += r
        self._training_steps += R
        self._after_step()
        if trace is not None:
            trace["idx"] = idx.cpu()
            trace["launches"] = int(lib.prl_nb_last_launches(nb["handle"]))
        return {"label": list(out[1]), "prediction": [p.view(B, 1) for p in out[0]], "weight": list(out[2]), "loss": list(loss)}

    # ------------------------------------------------------------------ NeuralBandit.learn_batch
    def learn_batch(self, batch) -> dict[str, Any]:
        self._check_learner()
        dev = self._device_of(batch.state.device if batch.state.is_cuda else None)
        f32 = lambda t: t.to(device=dev, dtype=torch.float32).contiguous()  # noqa: E731
        B = int(batch.state.shape[0])
        rows = lambda t: t.reshape(B, -1) if t.numel() else t.reshape(B, 0)  # noqa: E731
        state = f32(rows(batch.state))
        action = None if self._state_features_only else f32(rows(batch.action))
        reward = f32(batch.reward.reshape(B))
        weight = None if batch.weight is None else f32(batch.weight.reshape(B))
        act_dim = 0 if action is None else int(action.shape[1])
        nb = self._bind(dev, int(state.shape[1]), act_dim, 0, 0, B, any_rep=True)
        pred = torch.empty((B, 1), dtype=torch.float32, device=dev)
        loss = torch.empty((), dtype=torch.float32, device=dev)
        with torch.cuda.device(dev):
            _lib.check(nb["lib"].prl_nb_set_graph(nb["handle"], int(self.use_cuda_graph)))
            _lib.check(nb["lib"].prl_nb_learn_batch(nb["handle"], B, _lib.ptr(state), _lib.ptr(action), _lib.ptr(reward),
                                                    _lib.ptr(weight), _lib.ptr(pred), _lib.ptr(loss), _stream_ptr(dev)))
        self._after_step()
        return {"label": batch.reward, "prediction": pred,
                "weight": batch.weight if batch.weight is not None else torch.ones_like(batch.reward), "loss": loss}

    # ------------------------------------------------------------------ act / get_scores
    def _rows(self, subjective_state, action_space):
        """(device, the action features or None, the states [n, obs], the bound runtime)."""
        _refuse_distributed()
        dev = self._device_of(subjective_state.device if torch.is_tensor(subjective_state) and subjective_state.is_cuda else None)
        S = int(action_space.n)
        if self._state_features_only:
            feats, act_dim = None, 0
        else:
            feats = self.action_representation_module(torch.stack(list(action_space.actions)).to(dev))
            feats = feats.reshape(S, -1).to(torch.float32).contiguous()
            act_dim = int(feats.shape[1])
        obs = self._feature_dim - act_dim
        states = torch.as_tensor(subjective_state).to(device=dev, dtype=torch.float32).reshape(-1, obs).contiguous()
        return dev, feats, states, self._bind(dev, obs, act_dim, 0, 0, 1, any_rep=True)

    def _explorer(self) -> int:
        """0: NoExploration, 1: SquareCBExploration, 2: FastCBExploration; anything else is refused."""
        ex = self.exploration_module
        if isinstance(ex, FastCBExploration):
            kind = 2
        elif isinstance(ex, SquareCBExploration):
            kind = 1
        elif isinstance(ex, NoExploration):
            kind = 0
        else:
            raise NotImplementedError(f"act with {type(ex).__name__}: the CUDA NeuralBandit acts with SquareCBExploration, "
                                      "FastCBExploration or NoExploration")
        if getattr(ex, "randomized_tiebreaking", False) not in (False, None, TiebreakingStrategy.NO_TIEBREAKING):
            raise NotImplementedError("randomized tie-breaking: the CUDA NeuralBandit picks the first maximum")
        return kind

    def act(self, subjective_state, available_action_space, action_availability_mask: Optional[torch.Tensor] = None,
            exploit: bool = False):
        kind = self._explorer()
        S = int(available_action_space.n)
        dev, feats, states, nb = self._rows(subjective_state, available_action_space)
        n = int(states.shape[0])
        if kind and n != 1:
            raise NotImplementedError("SquareCB / FastCB act over more than one state: the reference broadcasts the per-state "
                                      "maxima against the action axis there, which fails or computes unrelated gaps")
        values = torch.empty((n, S), dtype=torch.float32, device=dev)
        index = torch.empty(n, dtype=torch.int32, device=dev)
        ex, E, prob = self.exploration_module, None, None
        if kind:
            # the draws torch's one-sample multinomial makes inside Categorical(p).sample(), from the same generator
            E = nb["draws"].put(torch.empty(S).exponential_(), dev)
            nb["prob"] = prob = torch.empty(S, dtype=torch.float32, device=dev)
        m = None
        if kind == 0 and action_availability_mask is not None:
            m = torch.as_tensor(action_availability_mask).to(dev).reshape(n, S).ne(0).to(torch.uint8).contiguous()
        gamma, lb, ub, clamp = ((float(ex._gamma), float(ex.reward_lb), float(ex.reward_ub), int(bool(ex.clamp_values)))
                                if kind else (0.0, 0.0, 0.0, 0))
        with torch.cuda.device(dev):
            _lib.check(nb["lib"].prl_nb_act(nb["handle"], n, _lib.ptr(states), S, _lib.ptr(feats), kind, gamma, lb, ub, clamp,
                                            _lib.ptr(E), _lib.ptr(m), _lib.ptr(values), _lib.ptr(prob), _lib.ptr(index),
                                            _stream_ptr(dev)))
        if kind:
            return index.cpu().reshape(())      # the index as the reference returns it; the copy is the one host sync
        actions_batch = torch.stack(list(available_action_space.actions)).to(dev)
        return torch.nn.functional.embedding(index.long(), actions_batch.reshape(S, -1))

    @torch.no_grad()
    def get_scores(self, subjective_state, action_space_to_score, exploit: bool = False) -> torch.Tensor:
        assert not exploit, "exploit=True is not yet implemented for NeuralBandit.get_scores"
        dev, feats, states, nb = self._rows(subjective_state, action_space_to_score)
        n, S = int(states.shape[0]), int(action_space_to_score.n)
        scores = torch.empty((n, S), dtype=torch.float32, device=dev)
        with torch.cuda.device(dev):
            _lib.check(nb["lib"].prl_nb_scores(nb["handle"], n, _lib.ptr(states), S, _lib.ptr(feats), _lib.ptr(scores),
                                               _stream_ptr(dev)))
        return scores.squeeze(-1)
