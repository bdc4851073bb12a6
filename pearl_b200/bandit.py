"""B200LinearBandit — Pearl's LinearBandit (policy_learners/contextual_bandits/linear_bandit.py, LinUCB on the ridge
regression of neural_networks/contextual_bandit/linear_regression.py) with its learning and scoring on an H100 through
`prl_cb_*` (csrc/bandit.cu, include/pearl_b200.h).

When Pearl is importable this is the reference class with `learn`, `learn_batch`, `act` and `get_scores` replaced: the
reference constructor runs unchanged, so `PearlAgent` accepts it as it is and `state_dict()` / `compare()` are the
reference's own.  Without Pearl it subclasses a stand-in (_compat.py) with the same constructor and state_dict keys.

The ridge buffers `model._A`, `_b`, `_sum_weight`, `_inv_A` and `_coefs` are the device memory the kernels update in
place: nothing is copied per call, and a state loaded with `load_state_dict` is what the next call reads.
`last_sum_weight_when_discounted` lives on the device too (the discounting decision is taken there) and is read back only
when the attribute is accessed.  No CPU fallback.

    learn(B200ReplayBuffer)   PolicyLearner.learn: training_rounds x (sample, fold the stored action id into the row as the
                              one-hot or binary representation module would, learn_batch), one prl_cb_learn per chunk
    learn_batch(batch)        one round on a caller's batch; batch.action is the already represented action matrix
    act / get_scores          UCB scores mu + alpha sigma (UCBExploration, NO_TIEBREAKING), prl_cb_scores; or Thompson
                              sampling (ThompsonSamplingExplorationLinear): x . theta with theta ~ N(coefs, (A + lambda
                              I)^-1) (prl_cb_ts_sample), or with efficient sampling mu + z sigma per score
                              (prl_cb_ts_scores).  The standard normals come from torch's default CPU generator, the
                              draws the reference makes; one status word is copied back per call.
"""
from __future__ import annotations

import ctypes as C
from typing import Any, Optional

import torch

from . import _lib
from ._compat import (BinaryActionTensorRepresentationModule, OneHotActionTensorRepresentationModule,
                      ThompsonSamplingExplorationLinear, TiebreakingStrategy, UCBExploration, _RefLinearBandit)
from ._draws import PinnedDraws
from .per import B200PrioritizedReplayBuffer
from .replay_buffer import B200ReplayBuffer, _stream_ptr

MAX_RIDGE_WIDTH = 127      # d = width + 1 (the intercept) <= 128: the solve's fp64 matrix fills 128 KB of shared memory


def _explorer(ex, learner: str, efficient_ok: bool = True) -> tuple[str, Any]:
    """("ucb", alpha) for UCBExploration, ("ts", enable_efficient_sampling) for ThompsonSamplingExplorationLinear; the
    rest is refused.  The disjoint Thompson explorer subclasses the joint one, so the class is matched exactly."""
    if isinstance(ex, UCBExploration):
        if ex.randomized_tiebreaking != TiebreakingStrategy.NO_TIEBREAKING:
            raise NotImplementedError("randomized tie-breaking: the CUDA bandit learner picks the first maximum "
                                      "(TiebreakingStrategy.NO_TIEBREAKING)")
        return "ucb", float(ex._alpha)
    if type(ex) is ThompsonSamplingExplorationLinear:
        # the reference passes the explorer's flag on as a tie-breaking strategy: a bool selects the first maximum there
        if ex.randomized_tiebreaking in (TiebreakingStrategy.PER_ROW_TIEBREAKING, TiebreakingStrategy.BATCH_TIEBREAKING):
            raise NotImplementedError("randomized tie-breaking: the CUDA bandit learner picks the first maximum "
                                      "(TiebreakingStrategy.NO_TIEBREAKING)")
        efficient = bool(ex._enable_efficient_sampling)
        if efficient and not efficient_ok:
            raise NotImplementedError(f"ThompsonSamplingExplorationLinear(enable_efficient_sampling=True) on {learner}: the "
                                      "reference fails its own shape assertion there (the network's output reaches the "
                                      "explorer flattened), so there is nothing to reproduce; use the default sampling")
        return "ts", efficient
    raise NotImplementedError(f"act / get_scores with {type(ex).__name__}: the CUDA bandit learner scores with "
                              "UCBExploration or ThompsonSamplingExplorationLinear")


def _ts_failed(status: torch.Tensor, efficient: bool) -> None:
    """Raise as the reference does when the sampler found A + lambda I not positive definite, or the efficient scores a
    NaN sigma.  The status read is the Thompson path's one device-to-host copy."""
    if int(status.item()) == 0:
        return
    if efficient:
        raise RuntimeError("normal expects all elements of std >= 0.0")
    raise ValueError("Thompson sampling: the precision matrix A + lambda I is not positive definite")


def _refuse_distributed() -> None:
    if torch.distributed.is_available() and torch.distributed.is_initialized():
        raise NotImplementedError("torch.distributed is initialized: the reference would all-reduce the ridge statistics, "
                                  "which the CUDA bandit learner does not implement")


class B200LinearBandit(_RefLinearBandit):
    def __init__(self, feature_dim: int, exploration_module=None, l2_reg_lambda: float = 1.0, gamma: float = 1.0,
                 apply_discounting_interval: float = 0.0, force_pinv: bool = False, training_rounds: int = 100,
                 batch_size: int = 128, action_representation_module=None, initial_coefs: Optional[torch.Tensor] = None, *,
                 max_rounds_per_call: int = 1024) -> None:
        if force_pinv:
            raise NotImplementedError("force_pinv=True: the CUDA ridge solve inverts A + lambda I directly, with no "
                                      "pseudo-inverse")
        if not l2_reg_lambda > 0:
            raise NotImplementedError(f"l2_reg_lambda={l2_reg_lambda}: the CUDA ridge solve needs l2_reg_lambda > 0 (the "
                                      "reference's pinv fallback, which a singular A can reach, is not implemented)")
        if int(feature_dim) > MAX_RIDGE_WIDTH:
            raise NotImplementedError(f"feature_dim={feature_dim}: the CUDA ridge solve supports at most {MAX_RIDGE_WIDTH} "
                                      "features (d = feature_dim + 1 <= 128)")
        super().__init__(feature_dim=feature_dim, exploration_module=exploration_module, l2_reg_lambda=l2_reg_lambda,
                         gamma=gamma, apply_discounting_interval=apply_discounting_interval, force_pinv=force_pinv,
                         training_rounds=training_rounds, batch_size=batch_size,
                         action_representation_module=action_representation_module, initial_coefs=initial_coefs)
        object.__setattr__(self, "_cb", dict(handle=C.c_void_p(0), key=None, batch=0, ws=None, lib=None, draws=PinnedDraws()))
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
            cb = self.__dict__.get("_cb")
            if cb and cb["handle"].value:
                cb["lib"].prl_cb_destroy(cb["handle"])
                cb["handle"] = C.c_void_p(0)
        except Exception:
            pass

    # ------------------------------------------------------------------ binding
    def _device_of(self, hint: Optional[torch.device] = None) -> torch.device:
        dev = self.model._A.device
        if dev.type != "cuda":
            dev = hint if hint is not None else torch.device("cuda", torch.cuda.current_device())
            self.model.to(dev)
        return dev

    def _bind(self, dev: torch.device, obs: int, act_dim: int, rep: int, n_actions: int, batch: int, scoring: bool = False) -> dict:
        """The prl_cb handle over the model's current buffers for this row layout, re-created when a buffer moved
        (a reference method that reassigns one, `.to()`), the layout changed or the batch outgrew it.  Scoring reads only
        the feature widths, so any handle of the same widths serves it (act -> learn per step keeps one handle)."""
        m, cb = self.model, self._cb
        if obs + act_dim != self._feature_dim:
            raise ValueError(f"state ({obs}) + action features ({act_dim}) != feature_dim ({self._feature_dim})")
        for name in ("_A", "_b", "_sum_weight", "_inv_A", "_coefs"):
            t = getattr(m, name)
            if t.dtype != torch.float32 or t.device != dev or not t.is_contiguous():
                setattr(m, name, t.to(device=dev, dtype=torch.float32).contiguous())
        last = self.__dict__["_last_discount"]
        if last.device != dev:
            object.__setattr__(self, "_last_discount", last.to(dev))
        bufs = (m._A, m._b, m._sum_weight, m._inv_A, m._coefs, self.__dict__["_last_discount"])
        key = (obs, act_dim, rep, n_actions, float(m.l2_reg_lambda), float(m.gamma), float(self.apply_discounting_interval),
               self.max_rounds_per_call) + tuple(t.data_ptr() for t in bufs)
        same = (lambda k: k[:2] + k[4:] == key[:2] + key[4:]) if scoring else (lambda k: k == key)  # noqa: E731
        if cb["handle"].value and same(cb["key"]) and batch <= cb["batch"]:
            return cb
        lib = _lib.init(dev.index)
        if cb["handle"].value:
            lib.prl_cb_destroy(cb["handle"])
            cb["handle"] = C.c_void_p(0)
        B = max(batch, self._batch_size if self._batch_size > 0 else batch, 1)
        cfg = _lib.CbCfg(obs, n_actions, act_dim, rep, B, self.max_rounds_per_call, float(m.l2_reg_lambda), float(m.gamma),
                         float(self.apply_discounting_interval))
        nbytes = int(lib.prl_cb_workspace_bytes(C.byref(cfg)))
        if nbytes < 0:
            raise ValueError(_lib.last_error())
        ws = torch.empty(nbytes, dtype=torch.uint8, device=dev)
        h = C.c_void_p(0)
        with torch.cuda.device(dev):
            _lib.check(lib.prl_cb_create(C.byref(h), C.byref(cfg), *(_lib.ptr(t) for t in bufs), _lib.ptr(ws)))
        cb.update(handle=h, key=key, batch=B, ws=ws, lib=lib)
        return cb

    def _representation(self) -> tuple[int, int]:
        """(action_rep, action_dim) of the action representation module for rows folded from stored ids."""
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

    # ------------------------------------------------------------------ PolicyLearner.learn (policy_learner.py:162-195)
    def learn(self, replay_buffer: B200ReplayBuffer, trace: Optional[dict] = None) -> dict[str, Any]:
        if not isinstance(replay_buffer, B200ReplayBuffer):
            raise TypeError("B200LinearBandit learns from a B200ReplayBuffer (GPU-resident ring)")
        if isinstance(replay_buffer, B200PrioritizedReplayBuffer):
            raise NotImplementedError("LinearBandit samples uniformly, as the reference: a B200PrioritizedReplayBuffer is "
                                      "not supported")
        if replay_buffer._shard is not None:
            raise NotImplementedError("a sharded replay buffer: the CUDA bandit learner samples local buffers only")
        self._check_learner()
        n = len(replay_buffer)
        if n == 0:
            return {}
        if bool(replay_buffer.is_action_continuous):
            raise ValueError("LinearBandit learns from a replay buffer with discrete actions")
        rep, act_dim = self._representation()
        B = n if (self._batch_size == -1 or n < self._batch_size) else self._batch_size
        dev = replay_buffer.device
        self._device_of(dev)
        cb = self._bind(dev, int(replay_buffer.obs_dim), act_dim, rep, int(replay_buffer.n_actions), B)
        R, lib = self._training_rounds, cb["lib"]
        out = torch.empty((3, R, B), dtype=torch.float32, device=dev)      # prediction, label, weight
        idx = torch.empty((R, B), dtype=torch.int32, device=dev) if trace is not None else None
        done = 0
        while done < R:
            r = min(self.max_rounds_per_call, R - done)
            replay_buffer._rng_push()
            with torch.cuda.device(dev):
                _lib.check(lib.prl_cb_set_graph(cb["handle"], int(self.use_cuda_graph)))
                _lib.check(lib.prl_cb_learn(cb["handle"], replay_buffer.handle, r, B, _lib.ptr(out[0, done]), _lib.ptr(out[1, done]),
                                            _lib.ptr(out[2, done]), _lib.ptr(idx[done]) if idx is not None else None,
                                            _stream_ptr(dev)))
            replay_buffer._rng_pull()
            done += r
        self._training_steps += R
        if trace is not None:
            trace["idx"] = idx.cpu()
            trace["launches"] = int(lib.prl_cb_last_launches(cb["handle"]))
        return {"label": list(out[1]), "prediction": [p.view(B, 1) for p in out[0]], "weight": list(out[2])}

    # ------------------------------------------------------------------ LinearBandit.learn_batch (linear_bandit.py:141-164)
    def learn_batch(self, batch) -> dict[str, Any]:
        self._check_learner()
        dev = self._device_of(batch.state.device if batch.state.is_cuda else None)
        f32 = lambda t: t.to(device=dev, dtype=torch.float32).contiguous()  # noqa: E731
        B = int(batch.state.shape[0])
        rows = lambda t: t.reshape(B, -1) if t.numel() else t.reshape(B, 0)  # noqa: E731
        state, action = f32(rows(batch.state)), f32(rows(batch.action))
        reward = f32(batch.reward.reshape(B))
        weight = None if batch.weight is None else f32(batch.weight.reshape(B))
        if weight is not None and bool((weight < 0).any()):      # the one host reduction, made only when a weight is given
            raise NotImplementedError("negative weights: A + lambda I can then be singular, where the reference falls back "
                                      "to a pseudo-inverse, which the CUDA ridge solve does not implement")
        cb = self._bind(dev, int(state.shape[1]), int(action.shape[1]), 0, 0, B)
        pred = torch.empty((B, 1), dtype=torch.float32, device=dev)
        with torch.cuda.device(dev):
            _lib.check(cb["lib"].prl_cb_set_graph(cb["handle"], int(self.use_cuda_graph)))
            _lib.check(cb["lib"].prl_cb_learn_batch(cb["handle"], B, _lib.ptr(state), _lib.ptr(action), _lib.ptr(reward),
                                                    _lib.ptr(weight), _lib.ptr(pred), _stream_ptr(dev)))
        return {"label": batch.reward, "prediction": pred,
                "weight": batch.weight if batch.weight is not None else torch.ones_like(batch.reward)}

    # ------------------------------------------------------------------ act / get_scores (linear_bandit.py:168-223)
    def _scores(self, subjective_state, action_space, alpha: float, with_sigma: bool, mask=None, want_index: bool = False,
                ts: Optional[bool] = None):
        """UCB scores (ts None), or Thompson scores: from sampled coefficients (ts False) or, with efficient sampling (ts
        True), one draw per score.  The draws come from torch's default CPU generator, as many as the reference makes."""
        _refuse_distributed()
        dev = self._device_of(subjective_state.device if torch.is_tensor(subjective_state) and subjective_state.is_cuda else None)
        feats = self.action_representation_module(torch.stack(list(action_space.actions)).to(dev))
        S = int(action_space.n)
        feats = feats.reshape(S, -1).to(torch.float32).contiguous()
        obs = self._feature_dim - int(feats.shape[1])
        states = torch.as_tensor(subjective_state).to(device=dev, dtype=torch.float32).reshape(-1, obs).contiguous()
        n = int(states.shape[0])
        cb = self._bind(dev, obs, int(feats.shape[1]), 0, 0, 1, scoring=True)
        scores = torch.empty((n, S), dtype=torch.float32, device=dev)
        index = torch.empty(n, dtype=torch.int32, device=dev) if want_index else None
        m = None if mask is None else torch.as_tensor(mask).to(dev).reshape(n, S).ne(0).to(torch.uint8).contiguous()
        lib, h, p = cb["lib"], cb["handle"], _lib.ptr
        with torch.cuda.device(dev):
            if ts is None:
                _lib.check(lib.prl_cb_scores(h, n, p(states), S, p(feats), float(alpha), int(with_sigma), p(m), p(scores),
                                             p(index), _stream_ptr(dev)))
                return scores, index
            status = torch.empty(1, dtype=torch.int32, device=dev)
            theta = z = None
            if ts:      # torch.normal(mean, std): one standard normal per score, row-major
                z = cb["draws"].put(torch.empty(n, S).normal_(), dev)
            else:       # MultivariateNormal.sample(): d standard normals
                d = self._feature_dim + 1
                eps = cb["draws"].put(torch.empty(d).normal_(), dev)
                theta = torch.empty(d, dtype=torch.float32, device=dev)
                _lib.check(lib.prl_cb_ts_sample(d, float(self.model.l2_reg_lambda), p(self.model._A), p(self.model._coefs), p(eps),
                                                p(theta), p(status), _stream_ptr(dev)))
            _lib.check(lib.prl_cb_ts_scores(h, n, p(states), S, p(feats), p(theta), p(z), p(m), p(scores), p(index),
                                            p(status) if ts else None, _stream_ptr(dev)))
        _ts_failed(status, ts)
        return scores, index

    def act(self, subjective_state, available_action_space, action_availability_mask: Optional[torch.Tensor] = None,
            exploit: bool = False):
        kind, arg = _explorer(self.exploration_module, "LinearBandit")
        ts = arg if kind == "ts" else None
        _, index = self._scores(subjective_state, available_action_space, arg if ts is None else 0.0, True,
                                action_availability_mask, True, ts=ts)
        actions_batch = torch.stack(list(available_action_space.actions)).to(index.device)
        return torch.nn.functional.embedding(index.long(), actions_batch.reshape(int(available_action_space.n), -1))

    def get_scores(self, subjective_state, action_space_to_score, exploit: bool = False) -> torch.Tensor:
        if exploit:         # the model's mu, bypassing the explorer
            scores, _ = self._scores(subjective_state, action_space_to_score, 0.0, False)
            return scores.squeeze(-1)
        kind, arg = _explorer(self.exploration_module, "LinearBandit")
        if kind == "ts":
            scores, _ = self._scores(subjective_state, action_space_to_score, 0.0, False, ts=arg)
        else:
            scores, _ = self._scores(subjective_state, action_space_to_score, arg, True)
        return scores.squeeze(-1)
