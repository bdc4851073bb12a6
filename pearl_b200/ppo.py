"""PPO preprocessing on the GPU: generalized advantage estimation and truncated lambda returns
(`ProximalPolicyOptimization.preprocess_replay_buffer`, pearl/policy_learners/
sequential_decision_making/ppo.py:201-293) for a whole rollout in one kernel launch."""
from __future__ import annotations

import ctypes as C

import torch

from . import _lib
from ._core import FlatCore
from .replay_buffer import _stream_ptr


def gae_and_lambda_returns(values: torch.Tensor, last_next_value: float, reward: torch.Tensor,
                           terminated: torch.Tensor, truncated: torch.Tensor, discount_factor: float,
                           trace_decay_param: float):
    """values[i] = critic(state_i) in TIME order (0 = oldest), CUDA tensors.
    Returns (gae, lam_return), each [n] fp32, bit-identical to the reference's newest->oldest loop."""
    if not values.is_cuda:
        raise RuntimeError("pearl_b200 has no CPU path: the rollout must live on a CUDA device")
    dev = values.device
    lib = _lib.init(dev.index if dev.index is not None else torch.cuda.current_device())
    n = values.numel()
    v = values.reshape(n).to(torch.float32).contiguous()
    r = reward.reshape(n).to(device=dev, dtype=torch.float32).contiguous()
    te = terminated.reshape(n).to(device=dev, dtype=torch.uint8).contiguous()
    tr = truncated.reshape(n).to(device=dev, dtype=torch.uint8).contiguous()
    gae = torch.empty(n, dtype=torch.float32, device=dev)
    lam = torch.empty(n, dtype=torch.float32, device=dev)
    scratch = torch.empty(n + 1, dtype=torch.int32, device=dev)      # chain heads + their count (caching allocator: no driver call)
    with torch.cuda.device(dev):
        _lib.check(lib.prl_ppo_gae(n, _lib.ptr(v), float(last_next_value), _lib.ptr(r), _lib.ptr(te), _lib.ptr(tr),
                                   float(discount_factor), float(trace_decay_param), _lib.ptr(gae), _lib.ptr(lam),
                                   _lib.ptr(scratch), _stream_ptr(dev)))
    return gae, lam


class B200ProximalPolicyOptimization(FlatCore):
    """The learner side of Pearl's ProximalPolicyOptimization (pearl/policy_learners/sequential_decision_making/
    ppo.py:96-293) for discrete actions on an H100.  `learn(replay_buffer)` = `preprocess_replay_buffer` (state values,
    taken-action probabilities, GAE and lambda returns over the whole rollout) followed by `training_rounds` x
    (sample -> clipped-surrogate actor step -> state-value critic step), all in CUDA through `prl_ppo_*`
    (include/pearl_b200.h).  Same constructor argument names and reporting keys (`actor_loss`, `critic_loss`) as the
    reference.  No CPU fallback."""
    _ABI = "prl_ppo"
    _ONE_STEP = "PPO steps actor and critic once per round: one AdamW step count"

    def __init__(self, state_dim: int, action_space=None, actor_hidden_dims=None, critic_hidden_dims=None,
                 actor_learning_rate: float = 1e-4, critic_learning_rate: float = 1e-4, discount_factor: float = 0.99,
                 training_rounds: int = 100, batch_size: int = 128, epsilon: float = 0.0, trace_decay_param: float = 0.95,
                 entropy_bonus_scaling: float = 0.01, *, n_actions: int | None = None, device=None,
                 max_rounds_per_call: int = 1024, max_rollout: int = 1 << 17, seed: int | None = None) -> None:
        self._open(device, training_rounds, batch_size, max_rounds_per_call, seed)
        if n_actions is None:
            if action_space is None or not hasattr(action_space, "n"):
                raise ValueError("PPO needs a discrete action space (`action_space.n`) or n_actions")
            n_actions = int(action_space.n)
        actor_hidden_dims, critic_hidden_dims = list(actor_hidden_dims or []), list(critic_hidden_dims or [])
        if len(actor_hidden_dims) != 2 or len(critic_hidden_dims) != 2:
            raise NotImplementedError("the CUDA PPO learner is built for two hidden layers in the actor and in the critic")
        self._state_dim, self._n_actions = int(state_dim), int(n_actions)
        self._actor_hidden_dims, self._critic_hidden_dims = actor_hidden_dims, critic_hidden_dims
        self._actor_learning_rate, self._critic_learning_rate = float(actor_learning_rate), float(critic_learning_rate)
        self._discount_factor, self._trace_decay_param = float(discount_factor), float(trace_decay_param)
        self._epsilon, self._entropy_bonus_scaling = float(epsilon), float(entropy_bonus_scaling)
        self._max_rollout = int(max_rollout)
        cfg = self._cfg(1)
        pa, pc = int(self._lib.prl_ppo_actor_param_count(C.byref(cfg))), int(self._lib.prl_ppo_critic_param_count(C.byref(cfg)))
        dev, f32 = self._device, torch.float32
        self.actor_params = torch.empty(pa, dtype=f32, device=dev)
        self.critic_params = torch.empty(pc, dtype=f32, device=dev)
        self._init_like_reference()
        self._actor_state = [torch.zeros(pa, dtype=f32, device=dev) for _ in range(3)]
        self._critic_state = [torch.zeros(pc, dtype=f32, device=dev) for _ in range(3)]
        self.last_preprocess = None     # dict(values, action_probs, gae, lam_return) of the last learn()

    def _cfg(self, max_batch: int) -> _lib.PpoCfg:
        return _lib.PpoCfg(self._state_dim, self._n_actions, self._actor_hidden_dims[0], self._actor_hidden_dims[1],
                           self._critic_hidden_dims[0], self._critic_hidden_dims[1], max_batch, self._max_rounds, self._max_rollout,
                           self._actor_learning_rate, self._critic_learning_rate, 0.9, 0.999, 1e-8, 0.01, self._discount_factor,
                           self._trace_decay_param, self._epsilon, self._entropy_bonus_scaling)

    def _shapes(self, hidden, out):
        O, (h1, h2) = self._state_dim, hidden
        return [(h1, O), (h1,), (h2, h1), (h2,), (out, h2), (out,)]

    def _init_like_reference(self) -> None:
        """Actor: Xavier-uniform weights, biases 0.01 (actor_critic_base.py:154); critic: nn.Linear's default init
        (VanillaValueNetwork is not re-initialised)."""
        self._fill(self.actor_params, self._shapes(self._actor_hidden_dims, self._n_actions))
        self._fill(self.critic_params, self._shapes(self._critic_hidden_dims, 1), xavier=False)

    def load_parameters(self, actor, critic) -> None:
        """Flat fp32 vectors in `parameters()` order of the reference's VanillaActorNetwork / VanillaValueNetwork."""
        self._load((self.actor_params, actor), (self.critic_params, critic))

    def _create(self, h, cfg) -> int:
        p = _lib.ptr
        return self._lib.prl_ppo_create(
            C.byref(h), C.byref(cfg), p(self.actor_params), p(self._actor_state[0]), p(self._actor_state[1]), p(self._actor_state[2]),
            p(self.critic_params), p(self._critic_state[0]), p(self._critic_state[1]), p(self._critic_state[2]), self._adam_steps[0],
            p(self._workspace))

    def preprocess_replay_buffer(self, replay_buffer, process_group=None) -> dict:
        """`process_group`: the rollout is sharded over the ranks of that torch.distributed group by contiguous time
        chunks (rank r holds chunk r, rank world-1 the newest transitions).  The network passes are row-parallel; the
        GAE chains are stitched with `pearl_b200.dist.sharded_gae_fixup` (4 floats per rank and round) and come out
        bit-identical to the unsharded rollout.  The training rounds of `learn()` stay local to each shard."""
        n = len(replay_buffer)
        if n == 0:
            raise AssertionError("preprocess_replay_buffer needs a non-empty rollout")
        if n > self._max_rollout:
            raise ValueError(f"rollout of {n} transitions exceeds max_rollout={self._max_rollout}")
        B = self._batch(n)
        self._bind(B)
        dev = self._device
        out = {k: torch.empty(n, dtype=torch.float32, device=dev) for k in ("values", "action_probs", "gae", "lam_return")}
        cut = torch.empty(n, dtype=torch.uint8, device=dev) if process_group is not None else None
        with torch.cuda.device(dev):
            _lib.check(self._lib.prl_ppo_preprocess(self._handle, replay_buffer.handle, _lib.ptr(out["values"]),
                                                    _lib.ptr(out["action_probs"]), _lib.ptr(out["gae"]), _lib.ptr(out["lam_return"]),
                                                    _lib.ptr(cut), _stream_ptr(dev)))
            if process_group is not None:
                from .dist import sharded_gae_fixup

                def redo(next_value: float, incoming_gae: float) -> float:
                    _lib.check(self._lib.prl_ppo_gae_redo(self._handle, _lib.ptr(out["values"]), next_value, incoming_gae,
                                                          _lib.ptr(out["gae"]), _lib.ptr(out["lam_return"]), _stream_ptr(dev)))
                    return float(out["gae"][0].item())
                self.last_shard_rounds = sharded_gae_fixup(float(out["values"][0].item()), float(out["gae"][0].item()),
                                                           bool(cut.any().item()), redo, group=process_group, device=dev)
        self.last_preprocess = out
        return out

    def learn(self, replay_buffer, trace: dict | None = None, process_group=None) -> dict:
        if not self._accepts(replay_buffer, False, "the PPO learner supports discrete actions (as the reference's `_actor_loss` does)",
                             "rollout"):
            return {}
        pre = self.preprocess_replay_buffer(replay_buffer, process_group=process_group)
        B = self._batch(len(replay_buffer))

        def chunk(r, done, out, idx):
            return self._lib.prl_ppo_learn(self._handle, replay_buffer.handle, r, B, _lib.ptr(pre["gae"]), _lib.ptr(pre["lam_return"]),
                                           _lib.ptr(pre["action_probs"]), _lib.ptr(out[0]), _lib.ptr(out[1]), _lib.ptr(idx),
                                           _stream_ptr(self._device))
        return self._rounds(replay_buffer, B, trace, 2, {"actor_loss": 0, "critic_loss": 1}, chunk)
