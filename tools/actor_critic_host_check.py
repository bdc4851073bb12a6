"""Developer check (CPU, needs facebookresearch/Pearl at argv[1]): the host logic of
pearl_b200/actor_critic.py — how the reference-derived plugins bind the reference's modules and optimizers to the flat vectors
of a CUDA learner — exercised against a stand-in learner that only has the attributes the binding touches (no CUDA: the
stand-in's learn() just moves numbers).  Checked: the constructor arguments handed to the CUDA learner, parameters and AdamW
state as views (no copies), step counts, SAC's entropy block, import of a checkpoint loaded into a fresh and into an already
bound learner, refusal of optimizers the kernels do not implement."""
import ctypes as C
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.dont_write_bytecode = True
sys.path[:0] = [os.path.join(ROOT, "oracle", "stubs"), sys.argv[1], ROOT]

import torch  # noqa: E402

import pearl_b200  # noqa: E402
from pearl_b200 import actor_critic as ac  # noqa: E402
from pearl.action_representation_modules.one_hot_action_representation_module import OneHotActionTensorRepresentationModule  # noqa: E402
from pearl.utils.instantiations.spaces.box_action import BoxActionSpace  # noqa: E402
from pearl.utils.instantiations.spaces.discrete_action import DiscreteActionSpace  # noqa: E402

assert ac.HAVE_REFERENCE
CPU = torch.device("cpu")
ac._B200ActorCriticMixin._device_of_parameters = lambda self: CPU      # the real one refuses anything but CUDA (tested in test_abi_and_host)


def mlp_count(i, h1, h2, o):
    return h1 * i + h1 + h2 * h1 + h2 + o * h2 + o


class Stub:
    """What the binding touches of pearl_b200.sac / td3 / ppo learners."""
    made = []

    def __init__(self, **kw):
        self.kw, self._device, self._handle, self._lib = kw, CPU, C.c_void_p(0), None
        O, (h1, h2), (c1, c2) = kw["state_dim"], kw["actor_hidden_dims"], kw["critic_hidden_dims"]
        A = kw["n_actions"] if "n_actions" in kw else int(torch.as_tensor(kw["low"]).numel())
        if self.kind == "sac":
            pa, pc = mlp_count(O, h1, h2, A) + A * h2 + A, 2 * mlp_count(O + A, c1, c2, 1)
        elif self.kind == "ppo":
            pa, pc = mlp_count(O, h1, h2, A), mlp_count(O, c1, c2, 1)
        else:
            pa, pc = mlp_count(O, h1, h2, A), 2 * mlp_count(O + A, c1, c2, 1)
        z = lambda n: torch.zeros(n)  # noqa: E731
        self.actor_params, self.critic_params = z(pa), z(pc)
        self.actor_target_params, self.critic_target_params = z(pa), z(pc)
        self._actor_state, self._critic_state = [z(pa) for _ in range(3)], [z(pc) for _ in range(3)]
        self._log_entropy, self._entropy_coef = z(4), torch.ones(1)
        self._adam_step, self._adam_steps, self._training_steps = 0, (0, 0), 0
        self._training_rounds, self._batch_size = kw["training_rounds"], kw["batch_size"]
        self._actor_learning_rate, self._critic_learning_rate = float(kw["actor_learning_rate"]), float(kw["critic_learning_rate"])
        Stub.made.append(self)

    def learn(self, buf):           # "one call": every parameter + 1, moments + 0.5, one AdamW step per round
        R = self._training_rounds
        for t in (self.actor_params, self.critic_params):
            t += 1.0
        for t in self._actor_state + self._critic_state:
            t += 0.5
        self._log_entropy += 0.25
        self._entropy_coef.copy_(torch.exp(self._log_entropy[:1]))
        self._adam_step += R
        self._adam_steps = (self._adam_steps[0] + (R + 1) // 2, self._adam_steps[1] + R)
        self._training_steps += R
        return {"actor_loss": [0.0] * R, "critic_loss": [0.0] * R}


def stub(kind):
    return type("Stub_" + kind, (Stub,), {"kind": kind})


ac.SacCore, ac.PpoCore, ac.Td3Core, ac.DdpgCore = stub("sac"), stub("ppo"), stub("td3"), stub("ddpg")
ac._DeterministicMixin._core_cls = ac.Td3Core
pearl_b200.B200DeepDeterministicPolicyGradient._core_cls = ac.DdpgCore


class Buf:
    def __len__(self):
        return 100


box = BoxActionSpace(low=torch.tensor([-1.0, -2.0]), high=torch.tensor([1.0, 3.0]))
flat = lambda m: torch.cat([p.detach().reshape(-1) for p in m.parameters()])  # noqa: E731

# ---------------------------------------------------------------- SAC
kw = dict(state_dim=6, action_space=box, actor_hidden_dims=[16, 8], critic_hidden_dims=[12, 10], actor_learning_rate=3e-4,
          critic_learning_rate=7e-4, critic_soft_update_tau=0.01, discount_factor=0.97, training_rounds=4, batch_size=32, seed=5)
l = pearl_b200.B200ContinuousSoftActorCritic(**kw)
a0, c0 = flat(l._actor).clone(), flat(l._critic).clone()
rep = l.learn(Buf())
core = l._b200
for k, v in dict(state_dim=6, actor_hidden_dims=[16, 8], critic_hidden_dims=[12, 10], actor_learning_rate=3e-4, critic_learning_rate=7e-4,
                 critic_soft_update_tau=0.01, discount_factor=0.97, training_rounds=4, batch_size=32, entropy_autotune=True, seed=5,
                 max_rounds_per_call=1024).items():
    assert core.kw[k] == v, (k, core.kw[k], v)
assert torch.equal(torch.as_tensor(core.kw["low"]), box.low) and torch.equal(torch.as_tensor(core.kw["high"]), box.high)
assert rep["actor_loss"] == [0.0] * 4 and l._training_steps == 4
# parameters: copied in once, then views (the stand-in's +1 is visible through the modules)
assert next(l._actor.parameters()).data_ptr() == core.actor_params.data_ptr()
assert torch.equal(flat(l._actor), a0 + 1) and torch.equal(flat(l._critic), c0 + 1)
assert next(l._critic_target.parameters()).data_ptr() == core.critic_target_params.data_ptr()
# AdamW state through the torch optimizers, step counts
p0 = next(l._actor.parameters())
st = l._actor_optimizer.state[p0]
assert st["exp_avg"].data_ptr() == core._actor_state[0].data_ptr() and float(st["exp_avg"].reshape(-1)[0]) == 0.5 and float(st["step"]) == 4
assert all(float(s["step"]) == 4 for s in l._critic_optimizer.state.values())
# entropy block
assert l._log_entropy.data_ptr() == core._log_entropy.data_ptr() and float(l._log_entropy) == 0.25
assert l._entropy_coef.shape == (1,) and l._entropy_coef.data_ptr() == core._entropy_coef.data_ptr()
assert float(l._entropy_optimizer.state[l._log_entropy]["step"]) == 4
# second call: nothing is re-bound
l.learn(Buf())
assert l._b200 is core and len(Stub.made) == 1 and float(st["step"]) == 8 and l._training_steps == 8
try:
    l.learn_batch(None)
    raise SystemExit("learn_batch must not fall back to torch")
except NotImplementedError:
    pass

# checkpoint into a FRESH learner: parameters land in place, optimizer state is imported, AdamW continues at step 8
sd = l.state_dict()
l2 = pearl_b200.B200ContinuousSoftActorCritic(**kw)
l2.load_state_dict(sd)
l2._training_steps = l._training_steps
assert l.compare(l2) == "", l.compare(l2)
l2.learn(Buf())
core2 = l2._b200
assert core2 is not core and core2._adam_step == 8 + 4
assert torch.equal(core2._actor_state[0], core._actor_state[0] + 0.5) and torch.equal(core2.actor_params, core.actor_params + 1)
assert float(l2._log_entropy) == 0.5 + 0.25 and float(l2._actor_optimizer.state[next(l2._actor.parameters())]["step"]) == 12

# checkpoint into an ALREADY BOUND learner (resume in place): load_state_dict replaces optimizer.state with new tensors
l.learn(Buf())                                   # l is now at step 12, like l2
sd2 = l2.state_dict()
l.load_state_dict(sd2)
assert not ac._is_bound(l._actor_optimizer, l._actor, core._actor_state)          # torch swapped the state tensors
l.learn(Buf())
assert ac._is_bound(l._actor_optimizer, l._actor, core._actor_state) and core._adam_step == 12 + 4
assert torch.equal(core._actor_state[1], core2._actor_state[1] + 0.5)

# a learning-rate change (scheduler / user) reaches the CUDA learner: same vectors, same step count, new rate
restarts = []
orig_restart = type(l)._restart_core
type(l)._restart_core = lambda self, c, steps: (restarts.append(steps), orig_restart(self, c, steps))[1]
l.learn(Buf())
assert restarts == []                                        # nothing changed: the handle is kept
l._actor_optimizer.param_groups[0]["lr"] = 1e-5
at = core._adam_step
l.learn(Buf())
assert restarts == [(at, at)] and core._actor_learning_rate == 1e-5 and core._critic_learning_rate == 7e-4 and core._adam_step == at + 4
type(l)._restart_core = orig_restart

# fixed entropy coefficient
lf = pearl_b200.B200ContinuousSoftActorCritic(**dict(kw, entropy_autotune=False, entropy_coef=0.3))
lf.learn(Buf())
assert lf._b200.kw["entropy_autotune"] is False and abs(lf._b200.kw["entropy_coef"] - 0.3) < 1e-7

# an optimizer the kernels do not implement is refused, loudly
a_net = pearl_b200.B200ContinuousSoftActorCritic(**kw)._actor
bad = pearl_b200.B200ContinuousSoftActorCritic(**dict(kw, actor_network_instance=a_net, actor_optimizer=torch.optim.SGD(a_net.parameters(), lr=0.1)))
try:
    bad.learn(Buf())
    raise SystemExit("SGD must be refused")
except NotImplementedError as e:
    assert "AdamW" in str(e)

# ---------------------------------------------------------------- TD3 / DDPG: separate actor / critic step counts
t = pearl_b200.B200TD3(state_dim=6, action_space=box, actor_hidden_dims=[16, 8], critic_hidden_dims=[12, 10], training_rounds=5, batch_size=16,
                       actor_update_freq=2, actor_update_noise=0.1, actor_update_noise_clip=0.3, actor_soft_update_tau=0.02)
t.learn(Buf())
ct = t._b200
assert ct.kind == "td3" and ct.kw["actor_update_freq"] == 2 and ct.kw["actor_update_noise"] == 0.1 and ct.kw["actor_update_noise_clip"] == 0.3
assert ct.kw["actor_soft_update_tau"] == 0.02 and ct.kw["critic_soft_update_tau"] == 0.005
assert next(t._actor_target.parameters()).data_ptr() == ct.actor_target_params.data_ptr()
assert float(t._actor_optimizer.state[next(t._actor.parameters())]["step"]) == 3 and float(t._critic_optimizer.state[next(t._critic.parameters())]["step"]) == 5
t2 = pearl_b200.B200TD3(state_dim=6, action_space=box, actor_hidden_dims=[16, 8], critic_hidden_dims=[12, 10], training_rounds=5, batch_size=16)
t2.load_state_dict(t.state_dict())
t2.learn(Buf())
assert t2._b200._adam_steps == (3 + 3, 5 + 5)
d = pearl_b200.B200DeepDeterministicPolicyGradient(state_dim=6, action_space=box, actor_hidden_dims=[16, 8], critic_hidden_dims=[12, 10], batch_size=16)
d.learn(Buf())
assert d._b200.kind == "ddpg" and "actor_update_freq" not in d._b200.kw

# ---------------------------------------------------------------- PPO
ds = DiscreteActionSpace([torch.tensor([i]) for i in range(5)])
p = pearl_b200.B200ProximalPolicyOptimization(state_dim=7, action_space=ds, actor_hidden_dims=[16, 8], critic_hidden_dims=[12, 10], training_rounds=3,
                                              batch_size=8, epsilon=0.2, trace_decay_param=0.9, entropy_bonus_scaling=0.02,
                                              action_representation_module=OneHotActionTensorRepresentationModule(5))
p.learn(Buf())
cp = p._b200
assert cp.kw["n_actions"] == 5 and cp.kw["epsilon"] == 0.2 and cp.kw["trace_decay_param"] == 0.9 and cp.kw["entropy_bonus_scaling"] == 0.02
assert cp.kw["actor_learning_rate"] == 1e-4 and p.on_policy and next(p._critic.parameters()).data_ptr() == cp.critic_params.data_ptr()
# a network the CUDA learner is not built for
deep = pearl_b200.B200ProximalPolicyOptimization(state_dim=7, action_space=ds, actor_hidden_dims=[16, 8, 8], critic_hidden_dims=[12, 10], training_rounds=3,
                                                 batch_size=8, action_representation_module=OneHotActionTensorRepresentationModule(5))
try:
    deep.learn(Buf())
    raise SystemExit("three hidden layers must be refused")
except NotImplementedError:
    pass
print("ACTOR_CRITIC_HOST_OK")
