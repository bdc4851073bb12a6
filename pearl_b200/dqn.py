"""B200DeepQLearning / B200DoubleDQN — drop-in policy learners whose `learn()` runs
in one persistent CUDA kernel (libpearlb200.so), replacing

    PolicyLearner.learn            pearl/policy_learners/policy_learner.py:162-195
    DeepTDLearning.learn_batch     .../sequential_decision_making/deep_td_learning.py:269-360
    DeepQLearning / DoubleDQN.get_next_state_values   deep_q_learning.py:130-167, double_dqn.py:29-57
    VanillaQValueNetwork.get_q_values                 q_value_networks.py:152-174
        (VanillaQValueMultiHeadNetwork, q_value_networks.py:185-241: multihead.py;
         CNNQValueNetwork / CNNQValueMultiHeadNetwork, q_value_networks.py:713-917: cnn_q.py)
    torch.optim.AdamW(amsgrad=True).step, update_target_network (common/utils.py:214-226)

Constructor arguments, attributes (`_Q`, `_Q_target`, `optimizer`, `_training_steps`,
`batch_size`, ...), `state_dict()` keys and the `learn()` report
(`{"loss": [mean |q - y| per round]}`) are those of the reference classes, which
these subclass whenever `pearl` is importable (see _compat.py).

Python keeps torch tensors only as containers: all parameters of `_Q` (and of
`_Q_target`) are views into ONE flat fp32 CUDA tensor in torch's own parameter
order, the AdamW state likewise, so `state_dict()` / `optimizer.state_dict()`
need no copies and the kernels see one contiguous parameter vector.
"""
from __future__ import annotations

import ctypes as C
from typing import Any

import torch

from . import _lib
from . import cnn_q, cql, dueling, multihead, sarsa
from ._batch import action_ids
from ._compat import _RefDeepQLearning, _RefDeepSARSA, _RefDoubleDQN, TransitionBatch
from .replay_buffer import B200ReplayBuffer, _stream_ptr


def _linears(qnet) -> list:
    mods = [m for m in qnet.modules() if isinstance(m, torch.nn.Linear)]
    others = [m for m in qnet.modules()
              if not isinstance(m, (torch.nn.Linear, torch.nn.ReLU, torch.nn.Sequential, type(qnet)))]
    if len(mods) != 3 or others:
        raise NotImplementedError(
            "pearl_b200 fuses VanillaQValueNetwork with exactly two hidden Linear+ReLU layers; "
            f"got {len(mods)} Linear layers and extra modules {[type(m).__name__ for m in others]}")
    return mods


class _B200DQNMixin:
    _double = False
    _sarsa = False          # DeepSARSA (sarsa.py)

    def __init__(self, *args: Any, max_rounds_per_call: int = 4096, rows_per_cta: int = 0,
                 engine: str = "auto", **kwargs: Any) -> None:
        """`engine`: "simt" = cooperative multi-SM fp32 kernel (lowest single-learner latency),
        "tc" = tensor-core one-SM-per-learner kernel (what B200LearnerGroup uses), "auto" = simt."""
        super().__init__(*args, **kwargs)
        if engine not in ("auto", "simt", "tc"):
            raise ValueError("engine must be 'auto', 'simt' or 'tc'")
        self._engine = engine
        self._conservative = bool(getattr(self, "_is_conservative", False))   # conservative (CQL) rounds (cql.py)
        arm = self.action_representation_module
        if type(arm).__name__ != "OneHotActionTensorRepresentationModule":
            raise NotImplementedError("the fused Q network assumes a one-hot action representation")
        self._n_actions = int(arm.max_number_actions)
        self._dueling = dueling.is_dueling(self._Q)           # DuelingQValueNetwork (dueling.py)
        self._multihead = multihead.is_multihead(self._Q)     # VanillaQValueMultiHeadNetwork (multihead.py)
        cnn = cnn_q.is_cnn(self._Q)                           # CNNQValueNetwork / CNNQValueMultiHeadNetwork (cnn_q.py)
        # the module of the learner this instance binds (its C prefix, refusals, cfg, learn_batch); None: the fused prl_dqn
        self._variant = cnn_q if cnn else sarsa if self._sarsa else dueling if self._dueling else \
            multihead if self._multihead else cql if self._conservative else None
        if self._sarsa and (self._dueling or self._conservative or self._multihead):
            sarsa.check_config(self, engine)            # refused before any network shape is parsed
        if cnn:
            cnn_q.check_config(self, engine)            # refused before the network shape is parsed
            self._cnn = cnn_q.shape_of(self._Q, self._n_actions)
            self._obs_dim = self._cnn["input"][0] * self._cnn["input"][1] * self._cnn["input"][2]
        elif self._dueling:
            self._obs_dim, self._duel_dims = dueling.shape_of(self._Q, self._n_actions)
        elif self._multihead:
            self._obs_dim, self._hidden = multihead.shape_of(self._Q, self._n_actions)
        else:
            lin = _linears(self._Q)
            self._obs_dim = lin[0].in_features - self._n_actions
            self._hidden = (lin[0].out_features, lin[1].out_features)
            if lin[1].in_features != self._hidden[0] or lin[2].in_features != self._hidden[1] or lin[2].out_features != 1:
                raise NotImplementedError("unexpected Q-network shape")
        self._max_rounds = int(max_rounds_per_call)
        self._rows_per_cta = int(rows_per_cta)
        if self._variant is not None:
            self._variant.check_config(self, engine)
            self.use_cuda_graph = True          # False: plain stream launches (profilers)
        self._handle = C.c_void_p(0)
        self._bound_ptr = None
        self._bound_batch = 0
        self._flat = {}

    # ------------------------------------------------------------------ binding
    def __del__(self):
        try:
            if getattr(self, "_handle", None) and self._handle.value:
                self._c("destroy")(self._handle)
                self._handle = C.c_void_p(0)
        except Exception:
            pass

    def _c(self, name: str):
        """C entry point `name` of the learner this instance binds: the variant's (prl_cql_*, ...), prl_dqn_* without one."""
        return getattr(self._libh, (self._variant.PREFIX if self._variant is not None else "prl_dqn_") + name)

    def _adam_hparams(self) -> dict:
        opt = self._optimizer
        if not isinstance(opt, torch.optim.AdamW) or len(opt.param_groups) < 1:
            raise NotImplementedError("the fused update implements torch.optim.AdamW(amsgrad=True)")
        g = opt.param_groups[0]
        if not g.get("amsgrad", False) or g.get("maximize", False):
            raise NotImplementedError("the fused update implements torch.optim.AdamW(amsgrad=True)")
        return dict(lr=float(g["lr"]), beta1=float(g["betas"][0]), beta2=float(g["betas"][1]),
                    eps=float(g["eps"]), weight_decay=float(g["weight_decay"]))

    def _flatten(self, module: torch.nn.Module, device) -> torch.Tensor:
        params = list(module.parameters())
        flat = torch.cat([p.detach().reshape(-1).to(device=device, dtype=torch.float32) for p in params])
        off = 0
        for p in params:
            n = p.numel()
            p.data = flat[off:off + n].view(p.shape)
            off += n
        return flat

    def _bind(self, need_batch: int) -> None:
        # `list(module.parameters())` walks the module tree (12 us): with a hundred learners per group.learn() that is milliseconds of host
        # time ahead of the launch.  The Parameter objects of a module only change if the module itself is replaced.
        if self.__dict__.get("_params_of") is not self._Q:   # via __dict__: as an nn.Module attribute `_Q` would be registered twice
            self.__dict__["_params_of"], self.__dict__["_params"] = self._Q, list(self._Q.parameters())
        params = self._params
        device = params[0].device
        if device.type != "cuda":
            raise RuntimeError(
                "B200 learner parameters are on %s: move the learner to a CUDA device "
                "(PearlAgent(device_id=0) does this); pearl_b200 has no CPU path" % device)
        if (self._handle.value and self._bound_ptr == params[0].data_ptr()
                and need_batch <= self._bound_batch):
            self._refresh_optimizer_binding(params)
            return
        # the configuration is checked before anything is released or allocated: a refused shape leaves the bound handle as it was
        self._libh = _lib.init(device.index if device.index is not None else torch.cuda.current_device())
        hp = self._adam_hparams()
        bound_batch = max(int(need_batch), int(self._batch_size) if self._batch_size > 0 else 0, 1)
        cfg = self._variant.make_cfg(self, hp, bound_batch) if self._variant is not None else _lib.DqnCfg(
            obs_dim=self._obs_dim, n_actions=self._n_actions, hidden1=self._hidden[0], hidden2=self._hidden[1],
            double_dqn=int(self._double), target_update_freq=int(self._target_update_freq),
            max_batch=bound_batch, max_rounds=self._max_rounds, rows_per_cta=self._rows_per_cta,
            lr=hp["lr"], beta1=hp["beta1"], beta2=hp["beta2"], eps=hp["eps"],
            weight_decay=hp["weight_decay"], gamma=float(self._discount_factor),
            tau=float(self._soft_update_tau))
        P_cfg = int(self._c("param_count")(C.byref(cfg)))
        if P_cfg < 0:
            raise ValueError(_lib.last_error())
        old_state = None
        if self._handle.value:
            st0 = self._optimizer.state.get(params[0], {})
            if "exp_avg" not in st0 or st0["exp_avg"].data_ptr() == self._flat["m"].data_ptr():
                # the optimizer still shows our flat vectors (no load_state_dict in between): carry them over
                old_state = {k: v.clone() for k, v in self._flat.items() if k in ("m", "v", "vmax")}
                old_step = int(self._c("adam_step")(self._handle))
            self._c("destroy")(self._handle)
            self._handle = C.c_void_p(0)
        w = self._flatten(self._Q, device)
        wt = self._flatten(self._Q_target, device)
        P = w.numel()
        opt_state = self._optimizer.state
        step = 0
        if old_state is not None:
            m, v, vmax, step = old_state["m"].to(device), old_state["v"].to(device), old_state["vmax"].to(device), old_step
        elif len(opt_state) and all(p in opt_state and "exp_avg" in opt_state[p] for p in params):
            cat = lambda key: torch.cat([opt_state[p][key].detach().reshape(-1).to(device, torch.float32) for p in params])
            m, v, vmax = cat("exp_avg"), cat("exp_avg_sq"), cat("max_exp_avg_sq")
            step = int(float(opt_state[params[0]]["step"]))
        else:
            m, v, vmax = (torch.zeros(P, dtype=torch.float32, device=device) for _ in range(3))
        self._bound_batch = bound_batch
        if P_cfg != P:
            raise RuntimeError("parameter count mismatch between the module and the fused kernel")
        ws_bytes = int(self._c("workspace_bytes")(C.byref(cfg)))
        ws = torch.empty(ws_bytes, dtype=torch.uint8, device=device)
        handle = C.c_void_p(0)
        with torch.cuda.device(device):
            _lib.check(self._c("create")(C.byref(handle), C.byref(cfg), _lib.ptr(w), _lib.ptr(wt),
                                         _lib.ptr(m), _lib.ptr(v), _lib.ptr(vmax), step, _lib.ptr(ws)))
        self._handle, self._cfg = handle, cfg
        if getattr(self, "_comm", None) is not None:
            _lib.check(self._libh.prl_dqn_set_comm(self._handle, self._comm.handle))
        self._flat = dict(w=w, wt=wt, m=m, v=v, vmax=vmax, ws=ws)
        self._expose_state(params, step)   # the flat AdamW state seen through the torch optimizer (views, no copies)
        self._bound_hp = hp
        self._bound_ptr = params[0].data_ptr()
        self._device = device

    def _refresh_optimizer_binding(self, params) -> None:
        """The kernels read the flat AdamW vectors and the hyper-parameters captured at bind time.  A checkpoint
        resume (`optimizer.load_state_dict`) replaces `optimizer.state[p]` with fresh tensors, and a scheduler or
        the user may change `param_groups[0]`: pick both up on every learn() (a few pointer / float compares)."""
        hp = self._adam_hparams()
        if hp != self._bound_hp:
            if {k: v for k, v in hp.items() if k != "lr"} != {k: v for k, v in self._bound_hp.items() if k != "lr"}:
                self._bound_ptr = None          # betas / eps / weight decay changed: full re-bind with the new config
                self._bind(self._bound_batch)
                return
            _lib.check(self._c("set_lr")(self._handle, hp["lr"]))
            self._bound_hp = hp
        st = self._optimizer.state
        m = self._flat["m"]
        p0 = params[0]
        if p0 in st and "exp_avg" in st[p0] and st[p0]["exp_avg"].data_ptr() == m.data_ptr():
            return
        if not all(p in st and "exp_avg" in st[p] for p in params):
            if len(st) == 0:                    # state dropped (fresh optimizer): restart the moments
                for k in ("m", "v", "vmax"):
                    self._flat[k].zero_()
                _lib.check(self._c("set_adam_step")(self._handle, 0))
                self._expose_state(params, 0)
            return
        dev = m.device
        cat = lambda key: torch.cat([st[p][key].detach().reshape(-1).to(dev, torch.float32) for p in params])
        has_max = all("max_exp_avg_sq" in st[p] for p in params)
        self._flat["m"].copy_(cat("exp_avg"))
        self._flat["v"].copy_(cat("exp_avg_sq"))
        self._flat["vmax"].copy_(cat("max_exp_avg_sq") if has_max else cat("exp_avg_sq"))
        step = int(float(st[p0]["step"]))
        _lib.check(self._c("set_adam_step")(self._handle, step))
        self._expose_state(params, step)

    def _expose_state(self, params, step: int) -> None:
        """Make `optimizer.state` a set of views into the flat AdamW vectors (no copies for state_dict())."""
        m, v, vmax = self._flat["m"], self._flat["v"], self._flat["vmax"]
        opt_state = self._optimizer.state
        off = 0
        self._step_tensors = []
        for p in params:
            n = p.numel()
            st = torch.tensor(float(step), dtype=torch.float32)
            self._step_tensors.append(st)
            opt_state[p] = dict(step=st, exp_avg=m[off:off + n].view(p.shape),
                                exp_avg_sq=v[off:off + n].view(p.shape),
                                max_exp_avg_sq=vmax[off:off + n].view(p.shape))
            off += n

    def _sync_step_tensors(self) -> None:
        step = float(self._c("adam_step")(self._handle))
        for st in self._step_tensors:
            st.fill_(step)

    @property
    def flat_parameters(self) -> torch.Tensor:
        """The online network's parameters as one flat CUDA tensor (torch order)."""
        self._bind(1)
        return self._flat["w"]

    @property
    def flat_target_parameters(self) -> torch.Tensor:
        self._bind(1)
        return self._flat["wt"]

    def adam_state(self) -> dict:
        self._bind(1)
        return dict(exp_avg=self._flat["m"], exp_avg_sq=self._flat["v"], max_exp_avg_sq=self._flat["vmax"],
                    step=int(self._c("adam_step")(self._handle)))

    def launch_info(self) -> dict:
        if self._variant is not None:
            return {k: int(self._c(fn)(self._handle)) for k, fn in self._variant.LAUNCH_INFO.items()}
        a, b, c = C.c_int32(0), C.c_int32(0), C.c_int32(0)
        self._libh.prl_dqn_last_launch_info(self._handle, C.byref(a), C.byref(b), C.byref(c))
        return dict(launches=a.value, ctas=b.value, rows_per_cta=c.value)

    def set_communicator(self, comm) -> None:
        """Data-parallel learning over `comm` (pearl_b200.dist.B200Communicator): every rank's
        `learn(B200ReplayBuffer)` then applies the mean gradient of all ranks' batches, exchanged
        inside the kernel.  All ranks must call learn() with the same number of rounds and start
        from identical parameters."""
        if self._variant is not None:
            raise NotImplementedError(f"{self._variant.NAME} runs on one GPU: set_communicator is not supported")
        self._bind(1)
        self._comm = comm
        _lib.check(self._libh.prl_dqn_set_comm(self._handle, comm.handle if comm is not None else None))

    def set_kernel_timing(self, enable: bool = True) -> None:
        if self._variant is not None:
            raise NotImplementedError(f"kernel timing belongs to the fused DQN kernel; time {self._variant.NAME} rounds with "
                                      "CUDA events")
        self._bind(1)
        _lib.check(self._libh.prl_dqn_set_timing(self._handle, int(enable)))

    def last_kernel_ms(self) -> float:
        ms = C.c_float(0)
        _lib.check(self._libh.prl_dqn_last_kernel_ms(self._handle, C.byref(ms)))
        return ms.value

    # ------------------------------------------------------------------ learn
    def learn(self, replay_buffer, trace: bool = False) -> dict:
        """`PolicyLearner.learn` (policy_learner.py:162-195): `training_rounds` gradient
        steps.  With a B200ReplayBuffer the whole call is sampler + one persistent kernel;
        `trace=True` additionally returns q, y and the sampled logical indices (tests)."""
        n = len(replay_buffer)
        if n == 0:
            return {}
        bs = n if (self._batch_size == -1 or n < self._batch_size) else self._batch_size
        rounds = int(self._training_rounds)
        if not isinstance(replay_buffer, B200ReplayBuffer):
            report: dict = {}
            for _ in range(rounds):  # foreign buffer: its own sample(), then the fused update
                self._training_steps += 1
                batch = replay_buffer.sample(bs)
                if isinstance(batch, TransitionBatch):
                    for k, v in self.learn_batch(self.preprocess_batch(batch)).items():
                        report.setdefault(k, []).append(v)
            return report
        if self._variant is not None:
            return self._learn_rounds(replay_buffer, bs, rounds, trace)
        self._bind(bs)
        dev = self._device
        if replay_buffer.device != dev:
            raise RuntimeError(f"replay buffer is on {replay_buffer.device}, learner on {dev}")
        from .per import B200PrioritizedReplayBuffer
        if isinstance(replay_buffer, B200PrioritizedReplayBuffer):
            return self._learn_prioritized(replay_buffer, bs, rounds, trace)
        mae = torch.empty(rounds, dtype=torch.float32, device=dev)
        q = y = idx = None
        if trace:
            q = torch.empty((rounds, bs), dtype=torch.float32, device=dev)
            y = torch.empty((rounds, bs), dtype=torch.float32, device=dev)
            idx = torch.empty((rounds, bs), dtype=torch.int32, device=dev)
        with torch.cuda.device(dev):
            stream = _stream_ptr(dev)
            replay_buffer._rng_push()
            done = 0
            use_tc = self._engine == "tc"
            if use_tc and not self._libh.prl_dqn_tc_supported(self._handle, bs):
                raise NotImplementedError("engine='tc' does not support this network / batch shape")
            while done < rounds:
                r = min(self._max_rounds, rounds - done)
                off = lambda t, w=1: C.c_void_p(0) if t is None else C.c_void_p(t.data_ptr() + 4 * done * w)
                if use_tc:
                    one = lambda p: (C.c_void_p * 1)(p)
                    _lib.check(self._libh.prl_dqn_learn_multi(
                        one(self._handle), one(replay_buffer.handle), 1, r, bs, (C.c_int64 * 1)(int(self._training_steps)),
                        one(off(mae)), one(off(q, bs)), one(off(y, bs)), one(off(idx, bs)), stream))
                else:
                    _lib.check(self._libh.prl_dqn_learn(self._handle, replay_buffer.handle, r, bs,
                                                        int(self._training_steps), off(mae), off(q, bs), off(y, bs),
                                                        off(idx, bs), stream))
                self._training_steps += r
                done += r
            replay_buffer._rng_pull()
        self._sync_step_tensors()
        report = {"loss": mae.cpu().tolist()}  # the one device->host read of the call
        if trace:
            report.update(q=q, y=y, idx=idx)
        return report

    def _learn_rounds(self, replay_buffer, bs: int, rounds: int, trace: bool) -> dict:
        """learn() of a variant learner over a B200ReplayBuffer: `rounds` x (sample -> round) through its prl_*_learn, which
        takes the variant's learn_args (alpha for CQL and multi-head) after the training-step count; DeepSARSA's needs
        the committed next actions of a B200SARSAReplayBuffer.  The ring holds no current action sets, so every round uses
        the full set, as B200ReplayBuffer.sample reports it."""
        from .per import B200PrioritizedReplayBuffer
        if isinstance(replay_buffer, B200PrioritizedReplayBuffer):
            raise NotImplementedError(f"{self._variant.NAME} samples uniformly: a B200PrioritizedReplayBuffer is not supported")
        self._bind(bs)
        dev = self._device
        if replay_buffer.device != dev:
            raise RuntimeError(f"replay buffer is on {replay_buffer.device}, learner on {dev}")
        extra = self._variant.learn_args(self)
        h = self._handle
        mae = torch.empty(rounds, dtype=torch.float32, device=dev)
        idx = torch.empty((rounds, bs), dtype=torch.int32, device=dev) if trace else None
        with torch.cuda.device(dev):
            stream = _stream_ptr(dev)
            _lib.check(self._c("set_graph")(h, int(self.use_cuda_graph)))
            replay_buffer._rng_push()
            done = 0
            while done < rounds:
                r = min(self._max_rounds, rounds - done)
                off = lambda t, w=1: C.c_void_p(0) if t is None else C.c_void_p(t.data_ptr() + 4 * done * w)  # noqa: E731
                _lib.check(self._c("learn")(h, replay_buffer.handle, r, bs, int(self._training_steps), *extra, off(mae),
                                            off(idx, bs), stream))
                self._training_steps += r
                done += r
            replay_buffer._rng_pull()
        self._sync_step_tensors()
        report = {"loss": mae.cpu().tolist()}
        if trace:
            report.update(idx=idx, **self.launch_info())
        return report

    def _learn_prioritized(self, rb, bs: int, rounds: int, trace: bool) -> dict:
        """learn() over a B200PrioritizedReplayBuffer: per round stratified sum-tree draw, importance-weighted
        MSE step, priority update from |q - y| (prl_dqn_learn_per)."""
        dev = self._device
        mae = torch.empty(rounds, dtype=torch.float32, device=dev)
        q = y = slots = w = None
        if trace:
            q = torch.empty((rounds, bs), dtype=torch.float32, device=dev)
            y = torch.empty((rounds, bs), dtype=torch.float32, device=dev)
            slots = torch.empty((rounds, bs), dtype=torch.int32, device=dev)
            w = torch.empty((rounds, bs), dtype=torch.float32, device=dev)
        with torch.cuda.device(dev):
            done = 0
            while done < rounds:
                r = min(self._max_rounds, rounds - done)
                off = lambda t, k=1: C.c_void_p(0) if t is None else C.c_void_p(t.data_ptr() + 4 * done * k)
                _lib.check(self._libh.prl_dqn_learn_per(self._handle, rb.handle, rb.per_handle, r, bs, int(self._training_steps),
                                                        off(mae), off(q, bs), off(y, bs), off(slots, bs), off(w, bs),
                                                        _stream_ptr(dev)))
                self._training_steps += r
                done += r
        self._sync_step_tensors()
        report = {"loss": mae.cpu().tolist()}
        if trace:
            report.update(q=q, y=y, slots=slots, weight=w)
        return report

    def preprocess_batch(self, batch):
        """The fused kernel consumes action ids directly; the one-hot expansion of
        policy_learner.py:197-218 is folded into the first layer (identity history only)."""
        hsm = getattr(self, "_history_summarization_module", None)
        if hsm is not None and type(hsm).__name__ != "IdentityHistorySummarizationModule":
            raise NotImplementedError("only the identity history summarization module is fused")
        return batch

    def learn_batch(self, batch) -> dict:
        """`DeepTDLearning.learn_batch` on a caller-supplied batch (raw ids, or the one-hot
        tensors the reference's preprocess_batch produces)."""
        if self._variant is not None:
            return self._variant.learn_batch(self, batch)
        B = len(batch)
        self._bind(B)
        dev = self._device
        f32 = lambda t: t.to(device=dev, dtype=torch.float32).contiguous()
        state, next_state = f32(batch.state), f32(batch.next_state)
        reward = f32(batch.reward.reshape(B))
        term = batch.terminated.reshape(B).to(device=dev, dtype=torch.uint8).contiguous()
        action = action_ids(batch.action.to(dev), self._n_actions, batch.action.dim() == 2).reshape(B).contiguous()
        avail = mask = None
        if batch.next_available_actions is not None:
            na = batch.next_available_actions.to(dev)
            avail = action_ids(na, self._n_actions, na.dim() == 3).reshape(B, self._n_actions).to(torch.float32).contiguous()
        if batch.next_unavailable_actions_mask is not None:
            mask = batch.next_unavailable_actions_mask.to(device=dev, dtype=torch.uint8).contiguous()
        mae = torch.empty(1, dtype=torch.float32, device=dev)
        upd = int((self._training_steps + 1) % self._target_update_freq == 0)
        with torch.cuda.device(dev):
            _lib.check(self._libh.prl_dqn_learn_batch(
                self._handle, B, _lib.ptr(state), _lib.ptr(action), _lib.ptr(reward), _lib.ptr(next_state),
                _lib.ptr(term), _lib.ptr(avail), _lib.ptr(mask), upd, _lib.ptr(mae), None, None,
                _stream_ptr(dev)))
        out = mae.item()  # also keeps the inputs alive until the kernel is done
        self._sync_step_tensors()
        return {"loss": out}

    # ------------------------------------------------------------------ act
    def q_values(self, states: torch.Tensor, target: bool = False) -> torch.Tensor:
        """Q(s, a) for every action id: [n, obs] -> [n, n_actions]."""
        own = getattr(self._variant, "q_values", None)
        if own is not None:
            return own(self, states, target)
        self._bind(1)
        dev = self._device
        s = states.to(device=dev, dtype=torch.float32).reshape(-1, self._obs_dim).contiguous()
        out = torch.empty((s.shape[0], self._n_actions), dtype=torch.float32, device=dev)
        with torch.cuda.device(dev):
            _lib.check(self._c("q_values")(self._handle, s.shape[0], _lib.ptr(s), int(target), _lib.ptr(out), _stream_ptr(dev)))
        torch.cuda.current_stream(dev).synchronize()
        return out

    def act(self, subjective_state, available_action_space, exploit: bool = False):
        """`DeepTDLearning.act` (deep_td_learning.py:200-254).  A variant with its own q_values (dueling: the advantage mean
        runs over the query) evaluates the available actions only, as get_q_values does with the available set as its
        query."""
        ids = available_action_space.actions_batch.reshape(available_action_space.n, -1)[:, 0].long()
        own = getattr(self._variant, "q_values", None)
        if self._variant is cnn_q:                     # a [1, C, H, W] state, as the reference's get_q_values asserts
            qs = cnn_q.act_values(self, subjective_state)
            q_avail = qs[ids.to(qs.device)]
        elif own is not None:
            q_avail = own(self, torch.as_tensor(subjective_state).reshape(1, -1), False, ids.view(1, -1))[0]
        else:
            qs = self.q_values(torch.as_tensor(subjective_state).reshape(1, -1))[0]
            q_avail = qs[ids.to(qs.device)]
        best = int(torch.argmax(q_avail))
        exploit_action = available_action_space.actions[best]
        if exploit or self.exploration_module is None:
            return exploit_action
        return self.exploration_module.act(subjective_state=subjective_state, action_space=available_action_space,
                                           exploit_action=exploit_action, values=q_avail)


class B200LearnerGroup:
    """`count` independent learners (seeds / agents) trained by ONE launch of the tensor-core kernel,
    one SM per learner: `group.learn()` == `[l.learn(b) for l, b in zip(learners, buffers)]`, but the
    learners run concurrently (the reference runs such replicas as separate processes,
    utils/scripts/benchmark.py:80-116).  All learners must share one configuration."""

    def __init__(self, learners, buffers) -> None:
        if len(learners) != len(buffers) or not learners:
            raise ValueError("need one replay buffer per learner")
        for l in learners:
            if getattr(l, "_variant", None) is not None:
                raise NotImplementedError(f"B200LearnerGroup runs the tensor-core DQN kernel, which has no {l._variant.NAME} update")
        self.learners, self.buffers = list(learners), list(buffers)

    def learn(self) -> list:
        n = len(self.learners)
        l0 = self.learners[0]
        rounds = int(l0._training_rounds)
        sizes = [len(b) for b in self.buffers]
        bs = [s if (l._batch_size == -1 or s < l._batch_size) else l._batch_size for l, s in zip(self.learners, sizes)]
        if min(sizes) == 0 or len(set(bs)) != 1:
            raise ValueError("all buffers of a group must be non-empty and give the same batch size")
        bs = bs[0]
        if n > 1 and any(b._rng_mode != "device" for b in self.buffers):
            # with rng="python" every buffer would be handed the SAME global `random` state: identical index streams in
            # all learners and a global stream advanced by one learner's consumption only
            raise ValueError('B200LearnerGroup needs buffers with rng="device" (one private MT19937 stream per learner, '
                             'like the separate processes the reference runs its replicas in)')
        for l in self.learners:
            l._bind(bs)
        dev = l0._device
        lib = l0._libh
        if not lib.prl_dqn_tc_supported(l0._handle, bs):
            raise NotImplementedError("the tensor-core group kernel does not support this network / batch shape")
        mae = torch.empty((n, rounds), dtype=torch.float32, device=dev)
        with torch.cuda.device(dev):
            stream = _stream_ptr(dev)
            for b in self.buffers:
                b._rng_push()
            done = 0
            while done < rounds:
                r = min(l0._max_rounds, rounds - done)
                arr = lambda xs: (C.c_void_p * n)(*xs)
                _lib.check(lib.prl_dqn_learn_multi(
                    arr([l._handle.value for l in self.learners]), arr([b.handle.value for b in self.buffers]), n, r, bs,
                    (C.c_int64 * n)(*[int(l._training_steps) for l in self.learners]),
                    arr([mae[i].data_ptr() + 4 * done for i in range(n)]), None, None, None, stream))
                for l in self.learners:
                    l._training_steps += r
                done += r
            for b in self.buffers:
                b._rng_pull()
        for l in self.learners:          # host-side bookkeeping while the GPU works
            l._sync_step_tensors()
        host = mae.cpu()                 # the one device->host read of the call
        return [{"loss": host[i].tolist()} for i in range(n)]

    def push_batch(self, state, action, reward, next_state, terminated, truncated) -> None:
        """One push for the whole group (a vectorised environment): HOST tensors with a leading learner axis,
        state / next_state [R, n, obs], action [R, n] ints, reward [R, n], terminated / truncated [R, n] bool.
        Equivalent to `buffers[i].push_batch(state[i], ...)` for every i, in one library call
        (`prl_buf_push_host_multi`: records packed by a few threads, one copy per buffer)."""
        R = len(self.buffers)
        b0 = self.buffers[0]
        state = torch.as_tensor(state)
        if state.is_cuda:
            raise ValueError("group push_batch takes host tensors; push device data per buffer")
        if state.dim() != 3 or state.shape[0] != R:
            raise ValueError(f"state must be [{R}, n, obs]")
        n = state.shape[1]
        if n == 0:
            return
        if any(not b._handle.value for b in self.buffers) or b0._is_action_continuous:
            for i, b in enumerate(self.buffers):     # first push allocates; continuous actions: per-buffer path
                b.push_batch(state[i], action[i], reward[i], next_state[i], terminated[i], truncated[i],
                             max_number_actions=self.learners[i]._n_actions)
            return
        prep = lambda x, dt, shape: torch.as_tensor(x).to(dtype=dt).reshape(shape).contiguous()
        st = prep(state, torch.float32, (R, n, -1))
        if st.shape[2] != b0.obs_dim:
            raise ValueError(f"state has {st.shape[2]} features, buffers store {b0.obs_dim}")
        ns = prep(next_state, torch.float32, (R, n, b0.obs_dim))
        ac = prep(action, torch.int32, (R, n))
        rw = prep(reward, torch.float32, (R, n))
        te, tr = prep(terminated, torch.uint8, (R, n)), prep(truncated, torch.uint8, (R, n))
        dev = b0._device
        with torch.cuda.device(dev):
            _lib.check(b0._lib.prl_buf_push_host_multi((C.c_void_p * R)(*[b.handle.value for b in self.buffers]), R, n, _lib.ptr(st),
                                                       _lib.ptr(ac), _lib.ptr(rw), _lib.ptr(ns), _lib.ptr(te), _lib.ptr(tr),
                                                       _stream_ptr(dev)))

    def set_kernel_timing(self, enable: bool = True) -> None:
        self.learners[0].set_kernel_timing(enable)

    def last_kernel_ms(self) -> float:
        return self.learners[0].last_kernel_ms()


class B200DeepQLearning(_B200DQNMixin, _RefDeepQLearning):
    """Drop-in for `pearl...deep_q_learning.DeepQLearning`."""
    _double = False


class B200DoubleDQN(_B200DQNMixin, _RefDoubleDQN):
    """Drop-in for `pearl...double_dqn.DoubleDQN`."""
    _double = True


class B200DeepSARSA(_B200DQNMixin, _RefDeepSARSA):
    """Drop-in for `pearl...deep_sarsa.DeepSARSA`: learn() over a B200SARSAReplayBuffer, learn_batch on a batch with
    `next_action` (sarsa.py, csrc/sarsa.cu)."""
    _sarsa = True
