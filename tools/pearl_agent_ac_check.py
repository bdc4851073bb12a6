"""Developer check (needs facebookresearch/Pearl) for the actor-critic plugins: B200ContinuousSoftActorCritic, B200TD3,
B200DeepDeterministicPolicyGradient and B200ProximalPolicyOptimization as SUBCLASSES of the reference classes
(pearl_b200/actor_critic.py), (1) against the stand-alone CUDA learner they wrap, bit for bit, (2) under the reference's own
PearlAgent facade (pearl/pearl_agent.py:55-330: reset -> act -> observe -> learn), (3) through a checkpoint round trip of
`agent.state_dict()` (actor_critic_base.py:411-428) after which both agents continue identically.  The numerics of the CUDA
learners against recordings of the reference are tests/test_sac.py, test_td3.py, test_ppo_learn.py; this file is about the
plugin boundary.  Test infrastructure: needs facebookresearch/Pearl on sys.path (argv[1] = its root) plus the test-only
gymnasium / matplotlib stubs."""
import io
import os
import random
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.dont_write_bytecode = True
sys.path[:0] = [os.path.join(ROOT, "oracle", "stubs"), sys.argv[1], ROOT]

import torch  # noqa: E402

import pearl_b200  # noqa: E402
from pearl_b200 import actor_critic as ac  # noqa: E402
from pearl.action_representation_modules.one_hot_action_representation_module import OneHotActionTensorRepresentationModule  # noqa: E402
from pearl.api.action_result import ActionResult  # noqa: E402
from pearl.pearl_agent import PearlAgent  # noqa: E402
from pearl.policy_learners.sequential_decision_making.ddpg import DeepDeterministicPolicyGradient  # noqa: E402
from pearl.policy_learners.sequential_decision_making.ppo import ProximalPolicyOptimization  # noqa: E402
from pearl.policy_learners.sequential_decision_making.soft_actor_critic_continuous import ContinuousSoftActorCritic  # noqa: E402
from pearl.policy_learners.sequential_decision_making.td3 import TD3  # noqa: E402
from pearl.utils.instantiations.spaces.box_action import BoxActionSpace  # noqa: E402
from pearl.utils.instantiations.spaces.discrete_action import DiscreteActionSpace  # noqa: E402

assert pearl_b200.HAVE_PEARL and ac.HAVE_REFERENCE
OBS, ACT, NACT, CAP, B, ROUNDS, STEPS = 10, 3, 4, 400, 32, 3, 48
DEV = torch.device("cuda", 0)
KINDS = {
    "sac": (pearl_b200.B200ContinuousSoftActorCritic, ContinuousSoftActorCritic, ac.SacCore),
    "td3": (pearl_b200.B200TD3, TD3, ac.Td3Core),
    "ddpg": (pearl_b200.B200DeepDeterministicPolicyGradient, DeepDeterministicPolicyGradient, ac.DdpgCore),
    "ppo": (pearl_b200.B200ProximalPolicyOptimization, ProximalPolicyOptimization, ac.PpoCore),
}


def space_of(kind):
    if kind == "ppo":
        return DiscreteActionSpace([torch.tensor([i]) for i in range(NACT)], seed=5)
    return BoxActionSpace(low=torch.tensor([-1.0, -2.0, -0.5]), high=torch.tensor([1.0, 2.0, 1.5]), seed=5)


def make_learner(kind, seed=7):
    kw = dict(state_dim=OBS, action_space=space_of(kind), actor_hidden_dims=[64, 64], critic_hidden_dims=[64, 64],
              training_rounds=ROUNDS, batch_size=B, seed=seed)
    if kind == "ppo":
        kw.update(action_representation_module=OneHotActionTensorRepresentationModule(NACT), epsilon=0.2)
    return KINDS[kind][0](**kw)


def make_buffer(kind, n, seed):
    g = torch.Generator().manual_seed(seed)
    buf = pearl_b200.B200ReplayBuffer(CAP, rng="python")
    buf.is_action_continuous = kind != "ppo"
    st, ns, rw = torch.randn((n, OBS), generator=g), torch.randn((n, OBS), generator=g), torch.randn(n, generator=g)
    tm = torch.rand(n, generator=g) < 0.1
    if kind == "ppo":
        buf.push_batch(st, torch.randint(0, NACT, (n,), generator=g).to(torch.int32), rw, ns, tm, torch.zeros(n, dtype=torch.bool),
                       max_number_actions=NACT)
    else:
        buf.push_batch(st, torch.rand((n, ACT), generator=g) * 2 - 1, rw, ns, tm, torch.zeros(n, dtype=torch.bool))
    return buf


def flat(module):
    return torch.cat([p.detach().reshape(-1).float().cpu() for p in module.parameters()])


def wrapped_vs_core(kind):
    """The reference-backed plugin == the CUDA learner it wraps: same initial parameters, same replay contents, same index
    stream (CPython's global `random`, re-seeded) and the same noise seed -> identical reports and parameters, twice in a
    row (the second call continues AdamW from the first)."""
    cls, ref_cls, core_cls = KINDS[kind]
    assert issubclass(cls, ref_cls)
    learner = make_learner(kind).to(DEV)
    init = {n: flat(getattr(learner, n)) for n in ("_actor", "_critic") + (("_actor_target",) if kind in ("td3", "ddpg") else ())
            + (("_critic_target",) if kind != "ppo" else ())}
    sp = space_of(kind)
    kw = dict(state_dim=OBS, actor_hidden_dims=[64, 64], critic_hidden_dims=[64, 64], training_rounds=ROUNDS, batch_size=B, seed=7,
              device=DEV)
    if kind == "ppo":
        core = core_cls(n_actions=NACT, epsilon=0.2, **kw)
        core.load_parameters(init["_actor"], init["_critic"])
    else:
        core = core_cls(low=sp.low, high=sp.high, **kw)
        pc = init["_critic"].numel() // 2
        if kind == "sac":
            core.load_parameters(init["_actor"], init["_critic"][:pc], init["_critic"][pc:], init["_critic_target"][:pc], init["_critic_target"][pc:])
        else:
            core.load_parameters(init["_actor"], init["_critic"][:pc], init["_critic"][pc:], init["_actor_target"],
                                 init["_critic_target"][:pc], init["_critic_target"][pc:])
    buf = make_buffer(kind, 200, seed=31)
    for call in range(2):
        random.seed(100 + call); ra = learner.learn(buf)
        random.seed(100 + call); rb = core.learn(buf)
        assert ra.keys() == rb.keys(), (kind, "wrapped vs core: report keys", list(ra), list(rb))
        for k in ra:
            assert ra[k] == rb[k], (kind, f"wrapped vs core, call {call}: {k}", ra[k], rb[k])
        assert len(ra["actor_loss"]) == ROUNDS and all(x == x for v in ra.values() for x in v)
    assert torch.equal(flat(learner._actor), core.actor_params.cpu()), kind
    assert torch.equal(flat(learner._critic), core.critic_params.cpu()), kind
    if kind != "ppo":
        assert torch.equal(flat(learner._critic_target), core.critic_target_params.cpu()), kind
    if kind == "sac":
        assert float(learner._entropy_coef) == core.entropy_coef and learner._entropy_coef.shape == (1,)
        assert float(learner._log_entropy) == float(core._log_entropy[0])
    # the torch optimizers show the live AdamW state (views) and the step count
    p0 = next(learner._actor.parameters())
    st = learner._actor_optimizer.state[p0]
    assert st["exp_avg"].data_ptr() == learner._b200._actor_state[0].data_ptr() and float(st["exp_avg"].abs().sum()) > 0
    expect = 2 * ROUNDS if kind != "td3" else ROUNDS         # TD3 steps its actor every second round
    assert int(st["step"]) == expect, (kind, int(st["step"]))
    assert learner._training_steps == 2 * ROUNDS
    try:
        learner.learn_batch(None)
        raise AssertionError("learn_batch should not silently fall back to the torch path")
    except NotImplementedError:
        pass


def make_agent(kind, seed=7):
    return PearlAgent(policy_learner=make_learner(kind, seed), replay_buffer=pearl_b200.B200ReplayBuffer(CAP, rng="python"), device_id=0)


def drive(agent, kind, steps, seed):
    g = torch.Generator().manual_seed(seed)
    obs, rew, done = torch.randn((steps + 1, OBS), generator=g), torch.randn(steps, generator=g), torch.rand(steps, generator=g) < 0.08
    sp = space_of(kind)
    agent.reset(obs[0], sp)
    reports = []
    for t in range(steps):
        a = agent.act(exploit=False)
        a = torch.as_tensor(a)
        if kind == "ppo":
            assert 0 <= int(a.reshape(-1)[0]) < NACT
        else:
            assert a.numel() == ACT and bool(((a.cpu() >= sp.low - 1e-5) & (a.cpu() <= sp.high + 1e-5)).all()), a
        agent.observe(ActionResult(observation=obs[t + 1], reward=float(rew[t]), terminated=bool(done[t]), truncated=False))
        if kind != "ppo" or (t + 1) % 16 == 0:       # on-policy: learn on a 16-step rollout (PearlAgent clears the buffer after)
            rep = agent.learn()
            if rep:
                reports.append(rep)
        if bool(done[t]):
            agent.reset(obs[t + 1], sp)
    return reports


def under_pearl_agent(kind):
    random.seed(1); torch.manual_seed(1)
    agent = make_agent(kind)
    before = flat(agent.policy_learner._actor)
    reports = drive(agent, kind, STEPS, seed=3)
    assert reports and all(set(r) >= {"actor_loss", "critic_loss"} for r in reports)
    assert all(x == x and abs(x) < 1e6 for r in reports for v in r.values() for x in v), reports[-1]
    pl = agent.policy_learner
    assert not torch.equal(flat(pl._actor), before), "the actor did not move"
    assert next(pl._actor.parameters()).data_ptr() == pl._b200.actor_params.data_ptr()      # act() reads what the kernels write
    if kind == "ppo":
        assert len(agent.replay_buffer) == 0                                                   # pearl_agent.py:217-218
    # ---- checkpoint round trip through the agent's own state_dict
    blob = io.BytesIO()
    torch.save(agent.state_dict(), blob)
    blob.seek(0)
    other = make_agent(kind, seed=11)
    other.load_state_dict(torch.load(blob, weights_only=False))
    assert agent.compare(other) == "", agent.compare(other)[:600]
    # both continue identically: same replay contents, index stream and noise stream; AdamW continues from the restored step
    buf = make_buffer(kind, 150, seed=77)
    other.policy_learner._training_steps = pl._training_steps
    other.policy_learner._ensure_core()
    for a in (agent, other):
        a.policy_learner._b200._gen.manual_seed(1234)
    if kind == "sac":   # the reference does not checkpoint `_entropy_optimizer` (actor_critic_base.py:411-418): carry its AdamW state over
        other.policy_learner._b200._log_entropy[1:].copy_(pl._b200._log_entropy[1:])
    random.seed(9); r1 = pl.learn(buf)
    random.seed(9); r2 = other.policy_learner.learn(buf)
    for k in r1:
        # TD3 repeats `_last_actor_loss` in the rounds that skip the delayed actor update (td3.py:116-122); like the reference's
        # attribute it is not part of a checkpoint, so the first such round after a restore reports 0.0
        if not (kind == "td3" and k == "actor_loss"):
            assert r1[k] == r2[k], (kind, f"continuation after the checkpoint: {k}", r1[k], r2[k])
    assert agent.compare(other) == "", agent.compare(other)[:600]
    return len(reports)


for kind in KINDS:
    wrapped_vs_core(kind)
    n = under_pearl_agent(kind)
    print(f"{kind}: subclass of the reference class; wrapped learner == stand-alone CUDA learner (reports and parameters identical, "
          f"AdamW state seen through the torch optimizers); PearlAgent: {STEPS} env steps, {n} learn() reports; "
          f"checkpoint round trip: compare() == '' and identical continuation")
print("PEARL_AGENT_AC_OK")
