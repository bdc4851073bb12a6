"""B200DisjointBanditContainer and B200DisjointLinearBandit — Pearl's disjoint linear bandits (policy_learners/
contextual_bandits/disjoint_bandit.py with LinearBandit arms, and disjoint_linear_bandit.py): one ridge regression per
arm, every arm's statistics and solve in the same launches through `prl_dcb_*` (csrc/disjoint_bandit.cu,
include/pearl_b200.h).

When Pearl is importable these are the reference classes with `learn`, `learn_batch`, `act` and `get_scores` replaced;
otherwise they subclass stand-ins (_compat.py) with the same constructors and state_dict keys.

Each arm's LinearRegression buffers (`_A`, `_b`, `_sum_weight`, `_inv_A`, `_coefs`) are views into flat device arrays
A[K][d][d], b[K][d], sum_weight[K], inv_A[K][d][d], coefs[K][d] that the kernels update in place, so a state loaded with
`load_state_dict` is what the next call reads.  A buffer that was reassigned (reference code, `.to()`) is copied back
into the flat array before the next launch.  The container's arms keep `last_sum_weight_when_discounted`: a
B200LinearBandit arm reads it from the flat device array, a reference LinearBandit arm gets it written back after each
learning call.  No CPU fallback.

    learn(B200ReplayBuffer)   PolicyLearner.learn: training_rounds x (sample, route each row to the arm of its stored
                              action id, per-arm ridge update), one prl_dcb_learn per chunk of rounds; the per-round arm
                              counts are copied back once per call to slice the container's report
    learn_batch(batch)        one round on a caller's batch (PearlAgent.learn_batch / offline_learning)
    act / get_scores          DisjointUCBExploration (mu_k + alpha sigma_k) or ThompsonSamplingExplorationLinearDisjoint
                              (one draw per arm from torch's default CPU generator, in arm order, as the reference makes
                              them), NO_TIEBREAKING; DisjointLinearBandit.get_scores raises, as the reference's does
"""
from __future__ import annotations

import ctypes as C
from typing import Any, Optional

import torch

from . import _lib
from ._compat import (DisjointUCBExploration, IdentityActionRepresentationModule, ThompsonSamplingExplorationLinearDisjoint,
                      TiebreakingStrategy, _RefDisjointBanditContainer, _RefDisjointLinearBandit, _RefLinearBandit)
from ._draws import PinnedDraws
from .bandit import (B200LinearBandit, _check_history, _check_ridge, _refuse_distributed, _refuse_negative_weights,
                     _ts_failed)
from .per import B200PrioritizedReplayBuffer
from .replay_buffer import B200ReplayBuffer, _stream_ptr

MAX_ARMS = 1024
_BUFS = ("_A", "_b", "_sum_weight", "_inv_A", "_coefs")


def _disjoint_explorer(ex, learner: str) -> tuple[str, float]:
    """("ucb", alpha) for DisjointUCBExploration, ("ts", 0) for ThompsonSamplingExplorationLinearDisjoint with the
    default sampling; the rest is refused."""
    if isinstance(ex, DisjointUCBExploration):
        if ex.randomized_tiebreaking != TiebreakingStrategy.NO_TIEBREAKING:
            raise NotImplementedError("randomized tie-breaking: the CUDA bandit learner picks the first maximum "
                                      "(TiebreakingStrategy.NO_TIEBREAKING)")
        return "ucb", float(ex._alpha)
    if type(ex) is ThompsonSamplingExplorationLinearDisjoint:
        if ex.randomized_tiebreaking in (TiebreakingStrategy.PER_ROW_TIEBREAKING, TiebreakingStrategy.BATCH_TIEBREAKING):
            raise NotImplementedError("randomized tie-breaking: the CUDA bandit learner picks the first maximum "
                                      "(TiebreakingStrategy.NO_TIEBREAKING)")
        if ex._enable_efficient_sampling:
            raise NotImplementedError(f"ThompsonSamplingExplorationLinearDisjoint(enable_efficient_sampling=True) on {learner}: "
                                      "the reference fails its own shape assertion there, so there is nothing to "
                                      "reproduce; use the default sampling")
        return "ts", 0.0
    raise NotImplementedError(f"act / get_scores with {type(ex).__name__}: the CUDA disjoint bandit learner scores with "
                              "DisjointUCBExploration or ThompsonSamplingExplorationLinearDisjoint")


def _refuse_representation(learner) -> None:
    if type(learner.action_representation_module) is not IdentityActionRepresentationModule:
        raise NotImplementedError(f"{type(learner.action_representation_module).__name__}: the disjoint bandit learners "
                                  "route rows by the raw action index and need the identity action representation")


class _Ridges:
    """The flat device arrays of K ridge regressions and the prl_dcb handle over them."""

    def __init__(self, mode: int) -> None:
        self.mode = mode
        self.flat: Optional[dict] = None
        self.handle = C.c_void_p(0)
        self.key = None
        self.batch = 0
        self.ws = self.lib = None
        self.params = None
        self.last_host: list = []
        self.feat: Optional[torch.Tensor] = None      # DisjointLinearBandit's action features [K][1]
        self.draws = PinnedDraws()

    def close(self) -> None:
        if self.handle.value:
            self.lib.prl_dcb_destroy(self.handle)
            self.handle = C.c_void_p(0)

    def arrays(self, dev: torch.device, models: list, d: int) -> dict:
        """The flat arrays on `dev`, each model's buffers made views of its slice (copied in first when a buffer is not
        that view: a fresh arm, a loaded or reassigned buffer, a move)."""
        K = len(models)
        f = self.flat
        if f is None or f["A"].device != dev:
            f = self.flat = dict(A=torch.empty(K, d, d, device=dev), b=torch.empty(K, d, device=dev),
                                 sw=torch.empty(K, device=dev), inv_A=torch.empty(K, d, d, device=dev),
                                 coefs=torch.empty(K, d, device=dev), last=torch.zeros(K, dtype=torch.float64, device=dev),
                                 lam=torch.empty(K, device=dev), gamma=torch.empty(K, device=dev),
                                 interval=torch.empty(K, dtype=torch.float64, device=dev))
            self.params, self.last_host = None, [None] * K
            self.close()
        for k, m in enumerate(models):
            for name, flat in zip(_BUFS, (f["A"], f["b"], f["sw"], f["inv_A"], f["coefs"])):
                view = flat[k:k + 1] if name == "_sum_weight" else flat[k]
                t = getattr(m, name)
                if t.data_ptr() != view.data_ptr() or t.shape != view.shape or t.dtype != torch.float32:
                    view.copy_(t.reshape(view.shape))
                    setattr(m, name, view)
        return f

    def set_params(self, lam: list, gamma: list, interval: list) -> None:
        p = (tuple(lam), tuple(gamma), tuple(interval))
        if p != self.params:
            f = self.flat
            f["lam"].copy_(torch.tensor(lam, dtype=torch.float32))
            f["gamma"].copy_(torch.tensor(gamma, dtype=torch.float32))
            f["interval"].copy_(torch.tensor(interval, dtype=torch.float64))
            self.params = p

    def bind(self, dev: torch.device, obs: int, adim: int, act_feat: Optional[torch.Tensor], batch: int, batch_size: int,
             max_rounds: int) -> "_Ridges":
        f = self.flat
        K = int(f["A"].shape[0])
        key = (obs, adim, max_rounds, _lib.ptr(act_feat)) + tuple(t.data_ptr() for t in f.values())
        if self.handle.value and key == self.key and batch <= self.batch:
            return self
        lib = _lib.init(dev.index)
        self.close()
        B = max(batch, batch_size if batch_size > 0 else batch, 1)
        cfg = _lib.DcbCfg(obs, K, adim, self.mode, B, max_rounds)
        nbytes = int(lib.prl_dcb_workspace_bytes(C.byref(cfg)))
        if nbytes < 0:
            raise ValueError(_lib.last_error())
        ws = torch.empty(nbytes, dtype=torch.uint8, device=dev)
        h = C.c_void_p(0)
        p = _lib.ptr
        with torch.cuda.device(dev):
            _lib.check(lib.prl_dcb_create(C.byref(h), C.byref(cfg), p(f["A"]), p(f["b"]), p(f["sw"]), p(f["inv_A"]),
                                          p(f["coefs"]), p(f["lam"]), p(f["gamma"]), p(f["interval"]), p(f["last"]),
                                          p(act_feat), p(ws)))
        self.handle, self.key, self.batch, self.ws, self.lib = h, key, B, ws, lib
        return self

    # ------------------------------------------------------------------ scoring
    def scores(self, dev, states: torch.Tensor, act_feat: Optional[torch.Tensor], kind: str, alpha: float, with_sigma: bool,
               mask=None, want_index: bool = False):
        """(n, K) scores: UCB (kind "ucb"; mu alone without sigma) or Thompson ("ts", arm-major as the reference lays
        them out), and the first maximum over the mask."""
        f = self.flat
        K, d = int(f["A"].shape[0]), int(f["A"].shape[1])
        n = int(states.shape[0])
        scores = torch.empty((n, K), dtype=torch.float32, device=dev)
        index = torch.empty(n, dtype=torch.int32, device=dev) if want_index else None
        m = None if mask is None else torch.as_tensor(mask).to(dev).reshape(n, K).ne(0).to(torch.uint8).contiguous()
        lib, h, p, st = self.lib, self.handle, _lib.ptr, _stream_ptr(dev)
        with torch.cuda.device(dev):
            if kind == "ucb":
                _lib.check(lib.prl_dcb_scores(h, n, p(states), p(act_feat), float(alpha), int(with_sigma), p(m), p(scores),
                                              p(index), st))
                return scores, index
            # MultivariateNormal(coefs_k, precision_matrix = A_k + lambda_k I).sample() per arm, in arm order: K draws of d
            eps = self.draws.put(torch.cat([torch.empty(d).normal_() for _ in range(K)]), dev)
            theta = torch.empty((K, d), dtype=torch.float32, device=dev)
            status = torch.empty(K, dtype=torch.int32, device=dev)
            _lib.check(lib.prl_dcb_ts_sample(h, p(eps), p(theta), p(status), st))
            _lib.check(lib.prl_dcb_ts_scores(h, n, p(states), p(act_feat), p(theta), p(m), p(scores), p(index), st))
        _ts_failed(status.max().reshape(1), False)
        return scores, index


def _learn_common(learner, replay_buffer) -> int:
    if not isinstance(replay_buffer, B200ReplayBuffer):
        raise TypeError(f"{type(learner).__name__} learns from a B200ReplayBuffer (GPU-resident ring)")
    if isinstance(replay_buffer, B200PrioritizedReplayBuffer):
        raise NotImplementedError("the disjoint bandits sample uniformly, as the reference: a B200PrioritizedReplayBuffer "
                                  "is not supported")
    if replay_buffer._shard is not None:
        raise NotImplementedError("a sharded replay buffer: the CUDA bandit learner samples local buffers only")
    _refuse_distributed()
    _check_history(learner)
    _refuse_representation(learner)
    if bool(replay_buffer.is_action_continuous):
        raise ValueError("the disjoint bandits learn from a replay buffer with discrete actions")
    return len(replay_buffer)


def _run_learn(learner, rg: _Ridges, replay_buffer, B: int, K: int, report: bool, trace: Optional[dict]):
    """training_rounds rounds in chunks of max_rounds_per_call; (out [3][R][B + K] or None, counts [R][K])."""
    dev = replay_buffer.device
    R, lib = learner._training_rounds, rg.lib
    out = torch.empty((3, R, B + K), dtype=torch.float32, device=dev) if report else None
    counts = torch.empty((R, K), dtype=torch.int32, device=dev)
    idx = torch.empty((R, B), dtype=torch.int32, device=dev) if trace is not None else None
    p, done = _lib.ptr, 0
    while done < R:
        r = min(learner.max_rounds_per_call, R - done)
        replay_buffer._rng_push()
        with torch.cuda.device(dev):
            _lib.check(lib.prl_dcb_set_graph(rg.handle, int(learner.use_cuda_graph)))
            _lib.check(lib.prl_dcb_learn(rg.handle, replay_buffer.handle, r, B,
                                         *((p(out[0, done]), p(out[1, done]), p(out[2, done])) if report else (None,) * 3),
                                         p(counts[done]), p(idx[done]) if idx is not None else None, _stream_ptr(dev)))
        replay_buffer._rng_pull()
        done += r
    learner._training_steps += R
    if trace is not None:
        trace["idx"] = idx.cpu()
        trace["launches"] = int(lib.prl_dcb_last_launches(rg.handle))
    return out, counts


class B200DisjointBanditContainer(_RefDisjointBanditContainer):
    def __init__(self, feature_dim: int, arm_bandits: list, exploration_module, training_rounds: int = 100, batch_size: int = 128,
                 *, max_rounds_per_call: int = 1024) -> None:
        for arm in arm_bandits:
            if not isinstance(arm, _RefLinearBandit):
                raise NotImplementedError(f"{type(arm).__name__} arm: the CUDA DisjointBanditContainer supports LinearBandit "
                                          "(or B200LinearBandit) arms only")
            _check_ridge(arm._feature_dim, arm.model.l2_reg_lambda, arm.model.force_pinv)
            if int(arm._feature_dim) != int(feature_dim):
                raise ValueError(f"arm feature_dim {arm._feature_dim} != the container's feature_dim {feature_dim}: each "
                                 "arm reads the state alone")
        if not 1 <= len(arm_bandits) <= MAX_ARMS:
            raise NotImplementedError(f"{len(arm_bandits)} arms: the CUDA disjoint learner supports 1 to {MAX_ARMS} arms")
        _check_ridge(feature_dim, 1.0, False)
        super().__init__(feature_dim=feature_dim, arm_bandits=arm_bandits, exploration_module=exploration_module,
                         training_rounds=training_rounds, batch_size=batch_size)
        object.__setattr__(self, "_dj", _Ridges(0))
        self.max_rounds_per_call = max(int(max_rounds_per_call), 1)
        self.use_cuda_graph = True       # False: plain stream launches (profilers)

    def __del__(self):
        try:
            self.__dict__["_dj"].close()
        except Exception:
            pass

    # ------------------------------------------------------------------ binding
    def _device_of(self, hint: Optional[torch.device] = None) -> torch.device:
        dev = self._arm_bandits[0].model._A.device
        if dev.type != "cuda":
            dev = hint if hint is not None else torch.device("cuda", torch.cuda.current_device())
        return dev

    def _ridges(self, dev: torch.device, batch: int) -> _Ridges:
        """Flat arrays gathered from the arms (and their last_sum_weight_when_discounted), the per-arm lambda, gamma and
        interval, and the handle."""
        rg, arms = self._dj, list(self._arm_bandits)
        f = rg.arrays(dev, [a.model for a in arms], self._feature_dim + 1)
        for k, arm in enumerate(arms):
            if isinstance(arm, B200LinearBandit):
                view = f["last"][k:k + 1]
                t = arm.__dict__["_last_discount"]
                if t.data_ptr() != view.data_ptr():
                    view.copy_(t.reshape(1))
                    object.__setattr__(arm, "_last_discount", view)
            else:
                v = float(arm.last_sum_weight_when_discounted)
                if rg.last_host[k] != v:
                    f["last"][k] = v
                    rg.last_host[k] = v
        rg.set_params([float(a.model.l2_reg_lambda) for a in arms], [float(a.model.gamma) for a in arms],
                      [float(a.apply_discounting_interval) for a in arms])
        return rg.bind(dev, self._feature_dim, 0, None, batch, self._batch_size, self.max_rounds_per_call)

    def _check_learner(self) -> None:
        _refuse_distributed()
        _check_history(self)
        _refuse_representation(self)

    def _after(self, counts: torch.Tensor) -> torch.Tensor:
        """One copy back: the per-round arm counts and, for reference LinearBandit arms, the device's discounting marks."""
        rg = self._dj
        last = rg.flat["last"]
        both = torch.cat([last.view(torch.int32), counts.reshape(-1)]).cpu()      # the doubles first: 8-byte aligned
        n = 2 * last.numel()
        lh = both[:n].view(torch.float64).tolist()
        for k, arm in enumerate(self._arm_bandits):
            if not isinstance(arm, B200LinearBandit):
                arm.last_sum_weight_when_discounted = lh[k]
                rg.last_host[k] = lh[k]
        return both[n:].reshape(counts.shape)

    def _report(self, out: torch.Tensor, counts: torch.Tensor, report: dict) -> None:
        """Round r's arm_{i}_{label, prediction, weight} from the partition-ordered rows of out[:, r]."""
        K = self._n_arms
        for r in range(counts.shape[0]):
            o = 0
            for i in range(K):
                n = max(int(counts[r, i]), 1)
                for j, name in enumerate(("prediction", "label", "weight")):
                    report.setdefault(f"arm_{i}_{name}", []).append(out[j, r, o:o + n].view(n, 1))
                o += n

    # ------------------------------------------------------------------ PolicyLearner.learn (policy_learner.py:162-195)
    def learn(self, replay_buffer: B200ReplayBuffer, trace: Optional[dict] = None) -> dict[str, Any]:
        n = _learn_common(self, replay_buffer)
        if n == 0:
            return {}
        if int(replay_buffer.n_actions) > self._n_arms:
            raise ValueError(f"the buffer holds {replay_buffer.n_actions} actions but the container has {self._n_arms} arms "
                             "(a stored action id names its arm)")
        if int(replay_buffer.obs_dim) != self._feature_dim:
            raise ValueError(f"buffer obs_dim {replay_buffer.obs_dim} != feature_dim {self._feature_dim}")
        B = n if (self._batch_size == -1 or n < self._batch_size) else self._batch_size
        rg = self._ridges(replay_buffer.device, B)
        out, counts = _run_learn(self, rg, replay_buffer, B, self._n_arms, True, trace)
        counts_h = self._after(counts)
        if trace is not None:
            trace["counts"] = counts_h
        report: dict = {}
        self._report(out, counts_h, report)
        return report

    # ------------------------------------------------------------------ learn_batch (disjoint_bandit.py:67-161)
    def learn_batch(self, batch) -> dict[str, Any]:
        self._check_learner()
        # _validate_batch: the reference asserts here, before any arm learns
        assert batch.action.dtype == torch.long, "action must be torch.long type (index of arm)"
        assert batch.action.min().item() >= 0, "action must be >= 0"
        assert batch.action.max().item() < self._n_arms, "action must be < number of arms"
        K = self._n_arms
        dev = self._device_of(batch.state.device if batch.state.is_cuda else None)
        f32 = lambda t: t.to(device=dev, dtype=torch.float32).contiguous()  # noqa: E731
        B = int(batch.state.shape[0])
        state3d = batch.state.dim() == 3
        if state3d:
            assert batch.state.shape[1] == K, "For 3D state, 2nd dimension must be equal to number of arms"
        state = f32(batch.state)
        if int(state.shape[-1]) != self._feature_dim:
            raise ValueError(f"state width {state.shape[-1]} != feature_dim {self._feature_dim}")
        arm = batch.action.reshape(B, -1)[:, 0].to(device=dev, dtype=torch.int32).contiguous()
        reward = f32(batch.reward.reshape(B))
        weight = None if batch.weight is None else f32(batch.weight.reshape(B))
        _refuse_negative_weights(weight)
        rg = self._ridges(dev, B)
        out = torch.empty((3, 1, B + K), dtype=torch.float32, device=dev)
        counts = torch.empty((1, K), dtype=torch.int32, device=dev)
        p = _lib.ptr
        with torch.cuda.device(dev):
            _lib.check(rg.lib.prl_dcb_set_graph(rg.handle, int(self.use_cuda_graph)))
            _lib.check(rg.lib.prl_dcb_learn_batch(rg.handle, B, p(state), int(state3d), p(arm), p(reward), p(weight),
                                                  p(out[0, 0]), p(out[1, 0]), p(out[2, 0]), p(counts), _stream_ptr(dev)))
        report: dict = {}
        self._report(out, self._after(counts), report)
        return {k: v[0] for k, v in report.items()}

    # ------------------------------------------------------------------ act / get_scores (disjoint_bandit.py:171-239)
    def _scores(self, subjective_state, space, kind: str, alpha: float, with_sigma: bool, mask=None, want_index=False):
        _refuse_distributed()
        K = self._n_arms
        if int(space.n) != K:
            raise ValueError(f"an action space of {space.n} actions for {K} arms")
        dev = self._device_of(subjective_state.device if torch.is_tensor(subjective_state) and subjective_state.is_cuda else None)
        states = torch.as_tensor(subjective_state).to(device=dev, dtype=torch.float32).reshape(-1, self._feature_dim).contiguous()
        rg = self._ridges(dev, 1)
        return rg.scores(dev, states, None, kind, alpha, with_sigma, mask, want_index)

    def act(self, subjective_state, available_action_space, action_availability_mask: Optional[torch.Tensor] = None,
            exploit: bool = False):
        kind, alpha = _disjoint_explorer(self.exploration_module, "DisjointBanditContainer")
        _, index = self._scores(subjective_state, available_action_space, kind, alpha, True, action_availability_mask, True)
        actions_batch = torch.stack(list(available_action_space.actions)).to(index.device)
        return torch.nn.functional.embedding(index.long(), actions_batch.reshape(int(available_action_space.n), -1))

    def get_scores(self, subjective_state, action_space_to_score, exploit: bool = False) -> torch.Tensor:
        if exploit:         # ensemble_forward: each arm's mu
            return self._scores(subjective_state, action_space_to_score, "ucb", 0.0, False)[0]
        kind, alpha = _disjoint_explorer(self.exploration_module, "DisjointBanditContainer")
        return self._scores(subjective_state, action_space_to_score, kind, alpha, True)[0]


class B200DisjointLinearBandit(_RefDisjointLinearBandit):
    def __init__(self, feature_dim: int, action_space, exploration_module, l2_reg_lambda: float = 1.0, training_rounds: int = 100,
                 batch_size: int = 128, state_features_only: bool = False, *, max_rounds_per_call: int = 1024) -> None:
        _check_ridge(feature_dim, l2_reg_lambda, False)
        acts = list(action_space.actions)
        if any(not torch.is_tensor(a) or a.numel() != 1 or a.reshape(-1)[0].item() != i for i, a in enumerate(acts)):
            raise NotImplementedError("DisjointLinearBandit routes a row to arm k when its action equals k: the CUDA learner "
                                      "needs the action space [tensor([0]), ..., tensor([n - 1])]")
        if not 1 <= len(acts) <= MAX_ARMS:
            raise NotImplementedError(f"{len(acts)} arms: the CUDA disjoint learner supports 1 to {MAX_ARMS} arms")
        super().__init__(feature_dim=feature_dim, action_space=action_space, exploration_module=exploration_module,
                         l2_reg_lambda=l2_reg_lambda, training_rounds=training_rounds, batch_size=batch_size,
                         state_features_only=state_features_only)
        object.__setattr__(self, "_dj", _Ridges(1))
        self.max_rounds_per_call = max(int(max_rounds_per_call), 1)
        self.use_cuda_graph = True

    def __del__(self):
        try:
            self.__dict__["_dj"].close()
        except Exception:
            pass

    def _adim(self) -> int:
        return 0 if self._state_features_only else 1

    def _ridges(self, dev: torch.device, batch: int) -> _Ridges:
        rg, models = self._dj, list(self._linear_regressions)
        f = rg.arrays(dev, models, self._feature_dim + 1)
        K = len(models)
        rg.set_params([float(m.l2_reg_lambda) for m in models], [1.0] * K, [0.0] * K)   # DisjointLinearBandit never discounts
        feat = None
        if not self._state_features_only:       # the constructor's action space, torch.Tensor(space[k]) = [k]
            feat = rg.feat
            if feat is None or feat.device != dev:
                feat = rg.feat = torch.arange(K, dtype=torch.float32, device=dev).reshape(K, 1)
        return rg.bind(dev, self._feature_dim - self._adim(), self._adim(), feat, batch, self._batch_size,
                       self.max_rounds_per_call)

    def _device_of(self, hint: Optional[torch.device] = None) -> torch.device:
        dev = self._linear_regressions[0]._A.device
        if dev.type != "cuda":
            dev = hint if hint is not None else torch.device("cuda", torch.cuda.current_device())
        return dev

    def learn(self, replay_buffer: B200ReplayBuffer, trace: Optional[dict] = None) -> dict[str, Any]:
        n = _learn_common(self, replay_buffer)
        if n == 0:
            return {}
        K = len(self._linear_regressions)
        if int(replay_buffer.n_actions) > K:
            raise ValueError(f"the buffer holds {replay_buffer.n_actions} actions but DisjointLinearBandit has {K} arms")
        if int(replay_buffer.obs_dim) != self._feature_dim - self._adim():
            raise ValueError(f"buffer obs_dim {replay_buffer.obs_dim} != {self._feature_dim - self._adim()} state features")
        B = n if (self._batch_size == -1 or n < self._batch_size) else self._batch_size
        rg = self._ridges(replay_buffer.device, B)
        _, counts = _run_learn(self, rg, replay_buffer, B, K, False, trace)
        if trace is not None:
            trace["counts"] = counts.cpu()
        return {}

    # ------------------------------------------------------------------ learn_batch (disjoint_linear_bandit.py:69-116)
    def learn_batch(self, batch) -> dict[str, Any]:
        _refuse_distributed()
        _check_history(self)
        _refuse_representation(self)
        K = len(self._linear_regressions)
        dev = self._device_of(batch.state.device if batch.state.is_cuda else None)
        f32 = lambda t: t.to(device=dev, dtype=torch.float32).contiguous()  # noqa: E731
        B = int(batch.state.shape[0])
        state = f32(batch.state.reshape(B, -1))
        if int(state.shape[1]) != self._feature_dim - self._adim():
            raise ValueError(f"state width {state.shape[1]} != {self._feature_dim - self._adim()} state features")
        # a row belongs to arm k when its action equals k; any other action (fractional, negative, >= K) matches no arm
        a = batch.action.reshape(B, -1)[:, 0].to(device=dev, dtype=torch.float64)
        arm = torch.where((a == a.floor()) & (a >= 0) & (a < K), a, torch.full_like(a, -1.0)).to(torch.int32).contiguous()
        reward = f32(batch.reward.reshape(B))
        weight = None if batch.weight is None else f32(batch.weight.reshape(B))
        _refuse_negative_weights(weight)
        rg = self._ridges(dev, B)
        with torch.cuda.device(dev):
            _lib.check(rg.lib.prl_dcb_set_graph(rg.handle, int(self.use_cuda_graph)))
            _lib.check(rg.lib.prl_dcb_learn_batch(rg.handle, B, _lib.ptr(state), 0, _lib.ptr(arm), _lib.ptr(reward),
                                                  _lib.ptr(weight), None, None, None, None, _stream_ptr(dev)))
        return {}

    def act(self, subjective_state, action_space, exploit: bool = False):
        kind, alpha = _disjoint_explorer(self.exploration_module, "DisjointLinearBandit")
        _refuse_distributed()
        _refuse_representation(self)
        K = len(self._linear_regressions)
        if int(action_space.n) != K:
            raise ValueError(f"an action space of {action_space.n} actions for {K} arms")
        dev = self._device_of(subjective_state.device if torch.is_tensor(subjective_state) and subjective_state.is_cuda else None)
        obs = self._feature_dim - self._adim()
        states = torch.as_tensor(subjective_state).to(device=dev, dtype=torch.float32).reshape(-1, obs).contiguous()
        feats = None
        if not self._state_features_only:       # concatenate_actions_to_state with the identity representation
            feats = torch.stack(list(action_space.actions)).to(device=dev, dtype=torch.float32).reshape(K, -1).contiguous()
            if int(feats.shape[1]) != 1:
                raise ValueError("DisjointLinearBandit's actions are one index each")
        rg = self._ridges(dev, 1)
        _, index = rg.scores(dev, states, feats, kind, alpha, True, None, True)
        actions_batch = torch.stack(list(action_space.actions)).to(index.device)
        return torch.nn.functional.embedding(index.long(), actions_batch.reshape(K, -1))

    def get_scores(self, subjective_state, action_space_to_score, exploit: bool = False) -> torch.Tensor:
        raise NotImplementedError("DisjointLinearBandit.get_scores is not yet implemented")
