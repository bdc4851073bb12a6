"""The host code the flat-vector learner cores share (pearl_b200/_core.py), on the CPU: the reference initialisation of
every core against the per-learner loops it replaced, and the handle lifecycle and round loop against a stand-in C
library.  Cores are built with `__new__`, so nothing here needs a GPU."""
import contextlib
import ctypes as C
import math

import pytest
import torch

from pearl_b200._core import FlatCore, fill_like_reference
from pearl_b200.iql import B200ImplicitQLearning
from pearl_b200.ppo import B200ProximalPolicyOptimization
from pearl_b200.qrdqn import B200QuantileRegressionDeepQLearning
from pearl_b200.reinforce import B200REINFORCE
from pearl_b200.sac import B200ContinuousSoftActorCritic
from pearl_b200.sac_discrete import B200SoftActorCritic
from pearl_b200.td3 import B200TD3, B200TD3BC

# ---------------------------------------------------------------- the initialisation each learner had (the specification)


def _xavier_loop(gen, vec, shapes):
    """sac.py, sac_discrete.py, td3.py: one call per network, both critics filled one after the other."""
    off = 0
    for shp in shapes:
        if len(shp) == 2:
            n = shp[0] * shp[1]
            bound = (6.0 / (shp[0] + shp[1])) ** 0.5
            vec[off:off + n].uniform_(-bound, bound, generator=gen)
        else:
            n = shp[0]
            vec[off:off + n].fill_(0.01)
        off += n
    assert off == vec.numel()


def _iql_loop(gen, vec, shapes, xavier):
    off, fan_in = 0, 1
    for shp in shapes:
        n = shp[0] * (shp[1] if len(shp) == 2 else 1)
        if len(shp) == 2:
            fan_in = shp[1]
            bound = (6.0 / (shp[0] + shp[1])) ** 0.5 if xavier else fan_in ** -0.5
            vec[off:off + n].uniform_(-bound, bound, generator=gen)
        elif xavier:
            vec[off:off + n].fill_(0.01)
        else:
            vec[off:off + n].uniform_(-fan_in ** -0.5, fan_in ** -0.5, generator=gen)
        off += n
    assert off == vec.numel()


def _ppo_loop(gen, vec, shapes, xavier):
    """ppo.py and reinforce.py: the default-init bound spelled (1 / fan_in) ** 0.5."""
    off, fan_in = 0, 1
    for shp in shapes:
        n = shp[0] * (shp[1] if len(shp) == 2 else 1)
        if len(shp) == 2:
            fan_in = shp[1]
            bound = (6.0 / (shp[0] + shp[1])) ** 0.5 if xavier else (1.0 / fan_in) ** 0.5
            vec[off:off + n].uniform_(-bound, bound, generator=gen)
        elif xavier:
            vec[off:off + n].fill_(0.01)
        else:
            vec[off:off + n].uniform_(-(1.0 / fan_in) ** 0.5, (1.0 / fan_in) ** 0.5, generator=gen)
        off += n
    assert off == vec.numel()


def _qrdqn_loop(gen, vec, shapes):
    off, fan_in = 0, 1
    for shp in shapes:
        n = shp[0] * (shp[1] if len(shp) == 2 else 1)
        if len(shp) == 2:
            fan_in = shp[1]
        vec[off:off + n].uniform_(-fan_in ** -0.5, fan_in ** -0.5, generator=gen)
        off += n
    assert off == vec.numel()


def _rc_loop(gen, params, O, A, c1, c2):
    """rc_safety._CostStep: the twin cost critic."""
    off = 0
    for net in range(2):
        for shp in [(c1, O + A), (c1,), (c2, c1), (c2,), (1, c2), (1,)]:
            n = shp[0] * (shp[1] if len(shp) == 2 else 1)
            if len(shp) == 2:
                params[off:off + n].uniform_(-(6.0 / sum(shp)) ** 0.5, (6.0 / sum(shp)) ** 0.5, generator=gen)
            else:
                params[off:off + n].fill_(0.01)
            off += n


def _mlp(i, h1, h2, o):
    return [(h1, i), (h1,), (h2, h1), (h2,), (o, h2), (o,)]


def _zeros(shapes, copies=1):
    return torch.zeros(copies * sum(math.prod(s) for s in shapes))


def _gen(seed=1234):
    return torch.Generator().manual_seed(seed)


# The fan-ins 7, 15, 21, 28 and 60 are ones where (1 / fan_in) ** 0.5 and fan_in ** -0.5 differ as doubles; each reaches a
# default-initialised layer (PPO / REINFORCE critic, IQL value net, QR-DQN) in one of these shapes.
SHAPES = [(7, 3, (15, 21), (28, 60)), (28, 4, (60, 7), (15, 21))]


def test_the_bound_spellings_differ_at_the_covered_fan_ins():
    for fan_in in (7, 15, 21, 28, 60):
        assert (1.0 / fan_in) ** 0.5 != fan_in ** -0.5


def _learner(cls, **attrs):
    pl = cls.__new__(cls)
    for k, v in attrs.items():
        setattr(pl, k, v)
    pl._gen = _gen()
    return pl


@pytest.mark.parametrize("O, A, hidden, other", SHAPES)
def test_continuous_and_discrete_sac_and_td3_init(O, A, hidden, other):
    for cls in (B200ContinuousSoftActorCritic, B200SoftActorCritic, B200TD3, B200TD3BC):
        discrete = cls is B200SoftActorCritic
        actor = _mlp(O, *hidden, A) + ([(A, hidden[1]), (A,)] if cls is B200ContinuousSoftActorCritic else [])
        critic = _mlp(O + A, *other, 1)
        pl = _learner(cls, _state_dim=O, _actor_hidden_dims=list(hidden), _critic_hidden_dims=list(other),
                      actor_params=_zeros(actor), critic_params=_zeros(critic, 2), **{"_n_actions" if discrete else "_action_dim": A})
        pl._init_like_reference()
        g, a, c = _gen(), _zeros(actor), _zeros(critic, 2)
        _xavier_loop(g, a, actor)
        _xavier_loop(g, c[:c.numel() // 2], critic)
        _xavier_loop(g, c[c.numel() // 2:], critic)
        assert torch.equal(pl.actor_params, a) and torch.equal(pl.critic_params, c), cls.__name__
        assert torch.equal(pl._gen.get_state(), g.get_state()), cls.__name__


@pytest.mark.parametrize("O, A, hidden, other", SHAPES)
@pytest.mark.parametrize("discrete", [True, False])
def test_iql_init(O, A, hidden, other, discrete):
    actor, critic, value = _mlp(O, *hidden, A), _mlp(O + A, *other, 1), _mlp(O, *other[::-1], 1)
    pl = _learner(B200ImplicitQLearning, _state_dim=O, _n_actions=A if discrete else 0, _action_dim=0 if discrete else A,
                  _actor_hidden_dims=list(hidden), _critic_hidden_dims=list(other), _value_hidden_dims=list(other[::-1]),
                  actor_params=_zeros(actor), critic_params=_zeros(critic, 2), value_params=_zeros(value))
    pl._init_like_reference()
    g, a, c, v = _gen(), _zeros(actor), _zeros(critic, 2), _zeros(value)
    _iql_loop(g, a, actor, True)
    _iql_loop(g, c[:c.numel() // 2], critic, True)
    _iql_loop(g, c[c.numel() // 2:], critic, True)
    _iql_loop(g, v, value, False)
    assert torch.equal(pl.actor_params, a) and torch.equal(pl.critic_params, c) and torch.equal(pl.value_params, v)
    assert torch.equal(pl._gen.get_state(), g.get_state())


@pytest.mark.parametrize("O, A, hidden, other", SHAPES)
def test_ppo_and_reinforce_init(O, A, hidden, other):
    for cls in (B200ProximalPolicyOptimization, B200REINFORCE):
        actor, critic = _mlp(O, *hidden, A), _mlp(O, *other, 1)
        pl = _learner(cls, _state_dim=O, _n_actions=A, _actor_hidden_dims=list(hidden), _critic_hidden_dims=list(other),
                      actor_params=_zeros(actor), critic_params=_zeros(critic))
        pl._init_like_reference()
        g, a, c = _gen(), _zeros(actor), _zeros(critic)
        _ppo_loop(g, a, actor, True)
        _ppo_loop(g, c, critic, False)
        assert torch.equal(pl.actor_params, a) and torch.equal(pl.critic_params, c), cls.__name__
        assert torch.equal(pl._gen.get_state(), g.get_state()), cls.__name__


@pytest.mark.parametrize("O, A, hidden, other", SHAPES)
def test_qrdqn_init(O, A, hidden, other):
    shapes = _mlp(O + A, *hidden, other[0])
    pl = _learner(B200QuantileRegressionDeepQLearning, _state_dim=O, _n_actions=A, _hidden_dims=list(hidden),
                  _num_quantiles=other[0], params=_zeros(shapes))
    pl._init_like_reference()
    g, q = _gen(), _zeros(shapes)
    _qrdqn_loop(g, q, shapes)
    assert torch.equal(pl.params, q) and torch.equal(pl._gen.get_state(), g.get_state())


@pytest.mark.parametrize("O, A, hidden, other", SHAPES)
def test_cost_critic_init(O, A, hidden, other):
    shapes = _mlp(O + A, *hidden, 1)
    got, want = _zeros(shapes, 2), _zeros(shapes, 2)
    fill_like_reference(got, 2 * shapes, _gen())
    _rc_loop(_gen(), want, O, A, *hidden)
    assert torch.equal(got, want)


# ---------------------------------------------------------------- lifecycle and round loop against a stand-in library


class _Cfg(C.Structure):
    _fields_ = [("max_batch", C.c_int64)]


class _Lib:
    """prl_fake_*: a handle is an int holding its AdamW step counts; every call is logged."""

    def __init__(self):
        self.steps, self.log, self._next = {}, [], 100

    def create(self, h, steps):
        h.value, self._next = self._next, self._next + 1
        self.steps[h.value] = list(steps)
        self.log.append(("create", h.value, tuple(steps)))
        return 0

    def prl_fake_destroy(self, h):
        self.log.append(("destroy", h.value))
        del self.steps[h.value]
        return 0

    def prl_fake_adam_step(self, h):
        return self.steps[h.value][0]

    def prl_fake_actor_adam_step(self, h):
        return self.steps[h.value][0]

    def prl_fake_critic_adam_step(self, h):
        return self.steps[h.value][1]

    def prl_fake_workspace_bytes(self, cfg):
        return 64

    def prl_fake_set_graph(self, h, on):
        self.log.append(("set_graph", h.value, on))
        return 0

    def prl_fake_last_launches(self, h):
        return 7


class _OneCount(FlatCore):
    _ABI = "prl_fake"
    _ONE_STEP = "the stand-in steps its networks once per round: one AdamW step count"

    def _cfg(self, max_batch):
        return _Cfg(max_batch)

    def _create(self, h, cfg):
        return self._lib.create(h, self._adam_steps)


class _TwoCounts(_OneCount):
    _STEPS = ("_actor_adam_step", "_critic_adam_step")


class _Buffer:
    def __init__(self, log):
        self.log = log

    def _rng_push(self):
        self.log.append("push")

    def _rng_pull(self):
        self.log.append("pull")


@pytest.fixture
def core(monkeypatch):
    monkeypatch.setattr(torch.cuda, "device", lambda d: contextlib.nullcontext())

    def make(cls=_OneCount, rounds=5, max_rounds=2, batch=4):
        c = cls.__new__(cls)
        c._device, c._lib = torch.device("cpu"), _Lib()
        c._training_rounds, c._batch_size, c._max_rounds, c._training_steps = rounds, batch, max_rounds, 0
        c.use_cuda_graph, c._handle, c._bound_batch, c._adam_steps = True, C.c_void_p(0), 0, (0,) * len(cls._STEPS)
        return c
    return make


@pytest.mark.parametrize("cls, taken", [(_OneCount, [5]), (_TwoCounts, [3, 5])])
def test_rebind_to_a_larger_batch_carries_the_adam_steps(core, cls, taken):
    c = core(cls)
    c._bind(3)
    first = c._handle.value
    assert c._bound_batch == 4 and c._lib.log == [("create", first, (0,) * len(taken))]
    c._lib.steps[first] = list(taken)          # the handle trained
    c._bind(4)
    assert c._handle.value == first            # still big enough: kept
    c._bind(9)
    assert c._bound_batch == 9 and c._workspace.numel() == 64
    assert c._lib.log[1:] == [("destroy", first), ("create", c._handle.value, tuple(taken))]
    assert c.adam_steps() == tuple(taken)


def test_adam_steps_and_restart_with_one_count(core):
    c = core()
    c._bind(4)
    h = c._handle.value
    c._lib.steps[h] = [6]
    assert c.adam_steps() == (6,)
    c.restart()                                # drop the handle, keep its count
    assert not c._handle.value and c._lib.log[-1] == ("destroy", h) and c.adam_steps() == (6,)
    c.restart((9, 9, 9))                       # one count per optimizer, all equal (IQL's three)
    assert c.adam_steps() == (9,)
    with pytest.raises(NotImplementedError, match="one AdamW step count"):
        c.restart((9, 10))
    assert c.adam_steps() == (9,)
    c._bind(4)
    assert c._lib.log[-1] == ("create", c._handle.value, (9,))
    with pytest.raises(NotImplementedError, match="one AdamW step count"):
        c.restart((3, 4))
    assert c._handle.value                     # a refused restart leaves the handle alone


def test_adam_steps_and_restart_with_two_counts(core):
    c = core(_TwoCounts)
    c._bind(4)
    c._lib.steps[c._handle.value] = [2, 4]
    assert c.adam_steps() == (2, 4)
    c.restart((3, 8))
    assert not c._handle.value and c.adam_steps() == (3, 8)
    c._bind(4)
    assert c._lib.log[-1] == ("create", c._handle.value, (3, 8))


@pytest.mark.parametrize("traced", [True, False])
def test_round_loop_chunks(core, traced):
    c = core(rounds=5, max_rounds=2)
    c._training_steps = 10
    c._bind(4)
    h, log = c._handle.value, c._lib.log
    del log[:]

    def chunk(r, done, out, idx):
        log.append(("learn", r, done, c._training_steps, idx is None))
        out[0].fill_(float(done))
        out[1].fill_(-1.0)
        if idx is not None:
            idx.fill_(done)
        return 0
    trace = {} if traced else None
    report = c._rounds(_Buffer(log), 4, trace, 2, {"loss": 0}, chunk)
    per_chunk = lambda r, done: ["push", ("set_graph", h, 1), ("learn", r, done, 10 + done, not traced), "pull"]  # noqa: E731
    assert log == per_chunk(2, 0) + per_chunk(2, 2) + per_chunk(1, 4)
    assert report == {"loss": [0.0, 0.0, 2.0, 2.0, 4.0]} and c._training_steps == 15
    if traced:
        assert trace["launches"] == 7 and torch.equal(trace["idx"], torch.tensor([0, 0, 2, 2, 4], dtype=torch.int32)[:, None].expand(5, 4))


def test_round_loop_counts_the_chunks_that_completed(core):
    c = core(rounds=5, max_rounds=2)
    c._bind(4)

    def chunk(r, done, out, idx):
        if done == 2:
            raise RuntimeError("second chunk")
        return 0
    with pytest.raises(RuntimeError, match="second chunk"):
        c._rounds(_Buffer([]), 4, None, 1, {"loss": 0}, chunk)
    assert c._training_steps == 2
