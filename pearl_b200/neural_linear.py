"""B200NeuralLinearBandit — Pearl's NeuralLinearBandit (policy_learners/contextual_bandits/neural_linear_bandit.py: an MLP
learns features, LinUCB runs on them) with its learning and scoring on an H100 through `prl_nlb_*` (csrc/neural_linear.cu,
include/pearl_b200.h).

When Pearl is importable this is the reference class with `learn`, `learn_batch`, `act` and `get_scores` replaced: the
reference constructor runs unchanged, so `PearlAgent` accepts it as it is and `state_dict()` / `compare()` are the
reference's own.  Without Pearl it subclasses a stand-in (_compat.py) with the same constructor, module tree and
state_dict keys.

The network's parameters (and linear_layer_e2e's weight) are views of one flat device vector, and the optimizer's AdamW
state (`exp_avg`, `exp_avg_sq`, `max_exp_avg_sq`, `step`) views of three more (_flat_adamw.py); the ridge
buffers of `model._linear_regression_layer` are the device memory the kernels update.  A state loaded with
`load_state_dict` is what the next call reads, and the learning rate is read from `optimizer.param_groups` on every call.
`last_sum_weight_when_discounted` lives on the device, as in bandit.py.  No CPU fallback.

    learn(B200ReplayBuffer)   PolicyLearner.learn: training_rounds x (sample, the row as learn_batch builds it, one round)
    learn_batch(batch)        one round on a caller's batch; batch.action is the already represented action matrix
    act / get_scores          UCB on the network's output (UCBExploration, NO_TIEBREAKING), or Thompson sampling
                              (ThompsonSamplingExplorationLinear's default mode): [1, nn_output] . theta with theta ~
                              N(coefs, (A + lambda I)^-1), prl_cb_ts_sample / prl_nlb_ts_scores
"""
from __future__ import annotations

import ctypes as C
from typing import Any, Optional

import torch

from . import _lib
from ._compat import LossType, _RefNeuralLinearBandit
from ._draws import PinnedDraws
from ._flat_adamw import FlatAdamW
from .bandit import MAX_RIDGE_WIDTH, _explorer, _refuse_distributed, _ts_failed
from .per import B200PrioritizedReplayBuffer
from .replay_buffer import B200ReplayBuffer, _stream_ptr

SCORE_ROWS = 4096          # feature rows the workspace holds per scoring chunk
_LOSS = {LossType.MSE: 0, LossType.MAE: 1, LossType.CROSS_ENTROPY: 2}


class B200NeuralLinearBandit(FlatAdamW, _RefNeuralLinearBandit):
    _RT, _ABI = "_nl", "prl_nlb"

    def __init__(self, feature_dim: int, hidden_dims: list, exploration_module=None, action_representation_module=None,
                 training_rounds: int = 100, batch_size: int = 128, learning_rate: float = 0.0003,
                 l2_reg_lambda_linear: float = 1.0, gamma: float = 1.0, apply_discounting_interval: float = 0.0,
                 force_pinv: bool = False, state_features_only: bool = True, loss_type=LossType.MSE,
                 output_activation_name: str = "linear", use_batch_norm: bool = False, use_layer_norm: bool = False,
                 hidden_activation: str = "relu", last_activation: Optional[str] = None, dropout_ratio: float = 0.0,
                 use_skip_connections: bool = False, nn_e2e: bool = True, separate_uncertainty: bool = False, *,
                 max_rounds_per_call: int = 1024) -> None:
        hidden_dims = list(hidden_dims)
        if len(hidden_dims) != 2:
            raise NotImplementedError(f"hidden_dims={hidden_dims}: the CUDA NeuralLinearBandit is built for two hidden layers")
        if int(hidden_dims[-1]) > MAX_RIDGE_WIDTH:
            raise NotImplementedError(f"hidden_dims[-1]={hidden_dims[-1]}: the CUDA ridge solve supports at most "
                                      f"{MAX_RIDGE_WIDTH} features (d = hidden_dims[-1] + 1 <= 128)")
        if dropout_ratio > 0:
            raise NotImplementedError(f"dropout_ratio={dropout_ratio}: the CUDA NeuralLinearBandit has no dropout")
        if use_batch_norm or use_layer_norm:
            raise NotImplementedError("batch norm or layer norm: the CUDA NeuralLinearBandit's hidden layers are Linear + ReLU")
        if hidden_activation != "relu":
            raise NotImplementedError(f"hidden_activation={hidden_activation!r}: the CUDA NeuralLinearBandit implements relu")
        if last_activation is not None:
            raise NotImplementedError(f"last_activation={last_activation!r}: the CUDA NeuralLinearBandit's last layer is linear")
        if output_activation_name not in ("linear", "sigmoid"):
            raise NotImplementedError(f"output_activation_name={output_activation_name!r}: the CUDA NeuralLinearBandit "
                                      "implements linear and sigmoid")
        if force_pinv:
            raise NotImplementedError("force_pinv=True: the CUDA ridge solve inverts A + lambda I directly, with no "
                                      "pseudo-inverse")
        if not l2_reg_lambda_linear > 0:
            raise NotImplementedError(f"l2_reg_lambda_linear={l2_reg_lambda_linear}: the CUDA ridge solve needs a positive "
                                      "lambda (the reference's pinv fallback, which a singular A can reach, is not implemented)")
        super().__init__(feature_dim=feature_dim, hidden_dims=hidden_dims, exploration_module=exploration_module,
                         action_representation_module=action_representation_module, training_rounds=training_rounds,
                         batch_size=batch_size, learning_rate=learning_rate, l2_reg_lambda_linear=l2_reg_lambda_linear,
                         gamma=gamma, apply_discounting_interval=apply_discounting_interval, force_pinv=force_pinv,
                         state_features_only=state_features_only, loss_type=loss_type,
                         output_activation_name=output_activation_name, use_batch_norm=use_batch_norm,
                         use_layer_norm=use_layer_norm, hidden_activation=hidden_activation, last_activation=last_activation,
                         dropout_ratio=dropout_ratio, use_skip_connections=use_skip_connections, nn_e2e=nn_e2e,
                         separate_uncertainty=separate_uncertainty)
        object.__setattr__(self, "_nl", dict(handle=C.c_void_p(0), key=None, batch=0, ws=None, lib=None, lr=None, flat=None,
                                             state=None, step=0, draws=PinnedDraws()))
        self._hidden = (int(hidden_dims[0]), int(hidden_dims[1]))
        self._skip = bool(use_skip_connections)
        self._sigmoid = output_activation_name == "sigmoid"
        self.max_rounds_per_call = max(int(max_rounds_per_call), 1)
        self.use_cuda_graph = True       # False: plain stream launches (profilers)

    # ------------------------------------------------------------------ last_sum_weight_when_discounted on the device
    @property
    def last_sum_weight_when_discounted(self) -> float:
        return float(self.__dict__["_last_discount"].item())

    @last_sum_weight_when_discounted.setter
    def last_sum_weight_when_discounted(self, value: float) -> None:
        t = self.__dict__.get("_last_discount")
        dev = t.device if t is not None else torch.device("cpu")
        object.__setattr__(self, "_last_discount", torch.tensor([float(value)], dtype=torch.float64, device=dev))

    def __del__(self):
        try:
            nl = self.__dict__.get("_nl")
            if nl and nl["handle"].value:
                nl["lib"].prl_nlb_destroy(nl["handle"])
                nl["handle"] = C.c_void_p(0)
        except Exception:
            pass

    # ------------------------------------------------------------------ binding
    def _device_of(self, hint: Optional[torch.device] = None) -> torch.device:
        dev = self.model._linear_regression_layer._A.device
        if dev.type != "cuda":
            dev = hint if hint is not None else torch.device("cuda", torch.cuda.current_device())
            self.model.to(dev)
        return dev

    def _bind(self, dev: torch.device, obs: int, act_dim: int, rep: int, n_actions: int, batch: int, any_rep: bool = False) -> dict:
        """The prl_nlb handle over the current parameter, AdamW and ridge buffers for this row layout, re-created when a
        buffer moved, the layout or a setting changed or the batch outgrew it.  learn_batch and scoring read only the
        widths (any_rep), so any handle of the same widths serves them: an agent that mixes learn() and learn_batch()
        keeps one handle."""
        m, nl = self.model, self._nl
        if obs + act_dim != self._feature_dim:
            raise ValueError(f"state ({obs}) + action features ({act_dim}) != feature_dim ({self._feature_dim})")
        if self.loss_type is LossType.CROSS_ENTROPY:
            assert self._sigmoid, "the cross-entropy loss needs output_activation_name='sigmoid'"
        lin = m._linear_regression_layer
        for name in ("_A", "_b", "_sum_weight", "_inv_A", "_coefs"):
            t = getattr(lin, name)
            if t.dtype != torch.float32 or t.device != dev or not t.is_contiguous():
                setattr(lin, name, t.to(device=dev, dtype=torch.float32).contiguous())
        last = self.__dict__["_last_discount"]
        if last.device != dev:
            object.__setattr__(self, "_last_discount", last.to(dev))
        e2e = bool(m.nn_e2e)
        flat = self._adopt(dev)
        n_params = len(list(m.parameters()))
        self._bind_optimizer(dev, n_params if e2e else n_params - 1)
        lr = self._lr()
        bufs = (lin._A, lin._b, lin._sum_weight, lin._inv_A, lin._coefs, self.__dict__["_last_discount"])
        key = (obs, act_dim, rep, n_actions, e2e, _LOSS[self.loss_type], float(lin.l2_reg_lambda), float(lin.gamma),
               float(self.apply_discounting_interval), self.max_rounds_per_call, flat.data_ptr(),
               nl["state"][0].data_ptr()) + tuple(t.data_ptr() for t in bufs)
        same = (lambda k: k[:2] + k[4:] == key[:2] + key[4:]) if any_rep else (lambda k: k == key)  # noqa: E731
        if nl["handle"].value and same(nl["key"]) and batch <= nl["batch"]:
            if lr != nl["lr"]:
                _lib.check(nl["lib"].prl_nlb_set_lr(nl["handle"], lr))
                nl["lr"] = lr
            return nl
        lib = _lib.init(dev.index)
        if nl["handle"].value:
            nl["step"] = int(lib.prl_nlb_adam_step(nl["handle"]))
            lib.prl_nlb_destroy(nl["handle"])
            nl["handle"] = C.c_void_p(0)
        B = max(batch, self._batch_size if self._batch_size > 0 else batch, 1)
        h1, h2 = self._hidden
        cfg = _lib.NlbCfg(obs, n_actions, act_dim, rep, h1, h2, int(self._skip), int(e2e), _LOSS[self.loss_type], int(self._sigmoid),
                          B, self.max_rounds_per_call, SCORE_ROWS, lr, 0.9, 0.999, 1e-8, 0.01, float(lin.l2_reg_lambda),
                          float(lin.gamma), float(self.apply_discounting_interval))
        nbytes = int(lib.prl_nlb_workspace_bytes(C.byref(cfg)))
        if nbytes < 0:
            raise ValueError(_lib.last_error())
        ws = torch.empty(nbytes, dtype=torch.uint8, device=dev)
        h, p = C.c_void_p(0), _lib.ptr
        st = nl["state"]
        with torch.cuda.device(dev):
            _lib.check(lib.prl_nlb_create(C.byref(h), C.byref(cfg), p(flat), p(st[0]), p(st[1]), p(st[2]), nl["step"],
                                          *(p(t) for t in bufs), p(ws)))
        nl.update(handle=h, key=key, batch=B, ws=ws, lib=lib, lr=lr)
        return nl

    # ------------------------------------------------------------------ PolicyLearner.learn (policy_learner.py:162-195)
    def learn(self, replay_buffer: B200ReplayBuffer, trace: Optional[dict] = None) -> dict[str, Any]:
        if not isinstance(replay_buffer, B200ReplayBuffer):
            raise TypeError("B200NeuralLinearBandit learns from a B200ReplayBuffer (GPU-resident ring)")
        if isinstance(replay_buffer, B200PrioritizedReplayBuffer):
            raise NotImplementedError("NeuralLinearBandit samples uniformly, as the reference: a B200PrioritizedReplayBuffer "
                                      "is not supported")
        if replay_buffer._shard is not None:
            raise NotImplementedError("a sharded replay buffer: the CUDA bandit learner samples local buffers only")
        self._check_learner()
        n = len(replay_buffer)
        if n == 0:
            return {}
        if bool(replay_buffer.is_action_continuous):
            raise ValueError("NeuralLinearBandit learns from a replay buffer with discrete actions")
        rep, act_dim = self._representation()
        B = n if (self._batch_size == -1 or n < self._batch_size) else self._batch_size
        dev = replay_buffer.device
        self._device_of(dev)
        nl = self._bind(dev, int(replay_buffer.obs_dim), act_dim, rep, int(replay_buffer.n_actions), B)
        R, lib = self._training_rounds, nl["lib"]
        out = torch.empty((3, R, B), dtype=torch.float32, device=dev)      # prediction, label, weight
        stats = torch.empty((2, R), dtype=torch.float32, device=dev)       # loss, mu_scores
        idx = torch.empty((R, B), dtype=torch.int32, device=dev) if trace is not None else None
        done = 0
        while done < R:
            r = min(self.max_rounds_per_call, R - done)
            replay_buffer._rng_push()
            with torch.cuda.device(dev):
                _lib.check(lib.prl_nlb_set_graph(nl["handle"], int(self.use_cuda_graph)))
                _lib.check(lib.prl_nlb_learn(nl["handle"], replay_buffer.handle, r, B, _lib.ptr(out[0, done]), _lib.ptr(out[1, done]),
                                             _lib.ptr(out[2, done]), _lib.ptr(stats[0, done:]), _lib.ptr(stats[1, done:]),
                                             _lib.ptr(idx[done]) if idx is not None else None, _stream_ptr(dev)))
            replay_buffer._rng_pull()
            done += r
        self._training_steps += R
        self._after_step()
        if trace is not None:
            trace["idx"] = idx.cpu()
            trace["launches"] = int(lib.prl_nlb_last_launches(nl["handle"]))
        return {"label": [y.view(B, 1) for y in out[1]], "prediction": [p.view(B, 1) for p in out[0]],
                "weight": [w.view(B, 1) for w in out[2]], "loss": list(stats[0]), "mu_scores": list(stats[1])}

    # ------------------------------------------------------------------ NeuralLinearBandit.learn_batch
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
        zero = False
        if weight is not None:      # the one host reduction, made only when a weight is given
            neg, nonzero = torch.stack([(weight < 0).any(), (weight != 0).any()]).tolist()
            if neg:
                raise NotImplementedError("negative weights: A + lambda I can then be singular, where the reference falls "
                                          "back to a pseudo-inverse, which the CUDA ridge solve does not implement")
            zero = not nonzero
        if self.loss_type is LossType.CROSS_ENTROPY:     # the reference asserts the labels are probabilities
            assert bool(((reward >= 0) & (reward <= 1)).all()), "cross-entropy labels must lie in [0, 1]"
        act_dim = 0 if action is None else int(action.shape[1])
        nl = self._bind(dev, int(state.shape[1]), act_dim, 0, 0, B, any_rep=True)
        pred = torch.empty((B, 1), dtype=torch.float32, device=dev)
        stats = torch.empty(2, dtype=torch.float32, device=dev)
        with torch.cuda.device(dev):
            _lib.check(nl["lib"].prl_nlb_set_graph(nl["handle"], int(self.use_cuda_graph)))
            _lib.check(nl["lib"].prl_nlb_learn_batch(nl["handle"], B, _lib.ptr(state), _lib.ptr(action), _lib.ptr(reward),
                                                     _lib.ptr(weight), int(zero), _lib.ptr(pred), _lib.ptr(stats[0:]),
                                                     _lib.ptr(stats[1:]), _stream_ptr(dev)))
        self._after_step()
        return {"label": batch.reward, "prediction": pred,
                "weight": batch.weight if batch.weight is not None else torch.ones_like(batch.reward),
                "loss": stats[0], "mu_scores": stats[1]}

    # ------------------------------------------------------------------ act / get_scores
    def _scores(self, subjective_state, action_space, alpha: float, mode: int, mask=None, want_index: bool = False,
                ts: bool = False):
        """UCB scores in `mode` (prl_nlb_scores), or with ts Thompson scores [1, nn_output] . theta, theta sampled from
        N(coefs, (A + lambda I)^-1) with d standard normals from torch's default CPU generator (mode 1: through the
        output activation)."""
        _refuse_distributed()
        dev = self._device_of(subjective_state.device if torch.is_tensor(subjective_state) and subjective_state.is_cuda else None)
        S = int(action_space.n)
        if self._state_features_only:
            feats = None
            act_dim = 0
        else:
            feats = self.action_representation_module(torch.stack(list(action_space.actions)).to(dev))
            feats = feats.reshape(S, -1).to(torch.float32).contiguous()
            act_dim = int(feats.shape[1])
        obs = self._feature_dim - act_dim
        states = torch.as_tensor(subjective_state).to(device=dev, dtype=torch.float32).reshape(-1, obs).contiguous()
        n = int(states.shape[0])
        nl = self._bind(dev, obs, act_dim, 0, 0, 1, any_rep=True)
        scores = torch.empty((n, S), dtype=torch.float32, device=dev)
        index = torch.empty(n, dtype=torch.int32, device=dev) if want_index else None
        m = None if mask is None else torch.as_tensor(mask).to(dev).reshape(n, S).ne(0).to(torch.uint8).contiguous()
        lib, h, p = nl["lib"], nl["handle"], _lib.ptr
        with torch.cuda.device(dev):
            if not ts:
                _lib.check(lib.prl_nlb_scores(h, n, p(states), S, p(feats), float(alpha), mode, p(m), p(scores), p(index),
                                              _stream_ptr(dev)))
                return scores, index
            d = self._hidden[1] + 1
            eps = nl["draws"].put(torch.empty(d).normal_(), dev)       # MultivariateNormal.sample(): d standard normals
            theta = torch.empty(d, dtype=torch.float32, device=dev)
            status = torch.empty(1, dtype=torch.int32, device=dev)
            lin = self.model._linear_regression_layer
            _lib.check(lib.prl_cb_ts_sample(d, float(lin.l2_reg_lambda), p(lin._A), p(lin._coefs), p(eps), p(theta), p(status),
                                            _stream_ptr(dev)))
            _lib.check(lib.prl_nlb_ts_scores(h, n, p(states), S, p(feats), p(theta), int(mode == 1), p(m), p(scores), p(index),
                                             _stream_ptr(dev)))
        _ts_failed(status, False)
        return scores, index

    def act(self, subjective_state, available_action_space, action_availability_mask: Optional[torch.Tensor] = None,
            exploit: bool = False):
        kind, arg = _explorer(self.exploration_module, "NeuralLinearBandit", efficient_ok=False)
        _, index = self._scores(subjective_state, available_action_space, arg if kind == "ucb" else 0.0, 0,
                                action_availability_mask, True, ts=kind == "ts")
        actions_batch = torch.stack(list(available_action_space.actions)).to(index.device)
        return torch.nn.functional.embedding(index.long(), actions_batch.reshape(int(available_action_space.n), -1))

    @torch.no_grad()
    def get_scores(self, subjective_state, action_space_to_score, exploit: bool = False) -> torch.Tensor:
        assert not exploit, "exploit=True is not yet implemented for NeuralLinearBandit.get_scores"
        kind, arg = _explorer(self.exploration_module, "NeuralLinearBandit", efficient_ok=False)
        scores, _ = self._scores(subjective_state, action_space_to_score, arg if kind == "ucb" else 0.0,
                                 2 if self.separate_uncertainty else 1, ts=kind == "ts")
        return scores.squeeze(-1)
