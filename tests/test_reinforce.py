"""REINFORCE on the GPU (pearl_b200.B200REINFORCE, csrc/reinforce.cu) against
(a) the recordings of the reference's PearlAgent(REINFORCE, REINFORCEReplayBuffer).learn() (tests/golden/rf_*.npz): same
    indices and `random` state, R bit for bit (from the GPU's own bootstrap term when it is nonzero), losses, parameters and
    AdamW states elementwise 1e-4 (tests/_tol.py), with graph replay on and off and with a ring that wraps;
(b) oracle/reinforce_oracle.py at a stress shape (obs 128, 16 actions, [256, 256], batch 256, a 20k-transition rollout)
    under contraction engines 0, 1 and 2;
plus bit-identity (run to run, round chunking, graph replay), the launch count, a learning-rate change without a new
handle, an optimizer checkpoint restored with load_state_dict, and the rejected inputs."""
import copy
import importlib
import os
import random
import sys
import types

import numpy as np
import pytest
import torch

from conftest import GOLDEN
from oracle.pearl_oracle import _mlp, flat
from oracle.reinforce_oracle import OracleREINFORCE, fold_returns

pytestmark = pytest.mark.gpu

from _tol import close as _close, close_params as _close_params  # noqa: E402


def _buffer(n, A, state, action, reward, next_state, term, prefill=0, **kw):
    """A ring of capacity n; `prefill` other transitions are pushed first, so the rollout's oldest transition sits at
    physical slot `prefill` and the rollout wraps around the end of the ring."""
    import pearl_b200
    buf = pearl_b200.B200ReplayBuffer(n, **kw)
    t = torch.as_tensor
    obs = np.asarray(state).shape[1]
    if prefill:
        g = torch.Generator().manual_seed(prefill)
        buf.push_batch(torch.randn(prefill, obs, generator=g), torch.zeros(prefill, dtype=torch.int32), torch.randn(prefill, generator=g),
                       torch.randn(prefill, obs, generator=g), torch.zeros(prefill, dtype=torch.bool),
                       torch.zeros(prefill, dtype=torch.bool), max_number_actions=A)
    buf.push_batch(t(state), t(action).to(torch.int32), t(reward), t(next_state), t(term), torch.zeros(len(reward), dtype=torch.bool),
                   max_number_actions=A)
    assert len(buf) == n
    return buf


def _learner(obs, A, hidden, **kw):
    import pearl_b200
    return pearl_b200.B200REINFORCE(state_dim=obs, n_actions=A, actor_hidden_dims=list(hidden), critic_hidden_dims=list(hidden), **kw)


@pytest.mark.parametrize("case", ["rf_method", "rf_multi", "rf_lr"])
@pytest.mark.parametrize("graph,prefill", [(True, 0), (False, 0), (True, 37)])
def test_reinforce_matches_reference_recording(case, graph, prefill):
    fx = np.load(os.path.join(GOLDEN, f"{case}.npz"))
    A, R, B, lr = int(fx["n_actions"]), int(fx["rounds"]), int(fx["batch"]), fx["call_lr"]
    h = fx["hidden"].tolist()
    pl = _learner(int(fx["obs"]), A, h, training_rounds=R, batch_size=B, actor_learning_rate=float(lr[0][0]),
                  critic_learning_rate=float(lr[0][1]))
    pl.use_cuda_graph = graph
    pl.load_parameters(fx["init_actor"], fx["init_critic"])
    al, cl, idx, handles, off = [], [], [], [], 0
    for c, n in enumerate(fx["call_n"].tolist()):
        if c:   # a learning-rate change between calls goes through prl_reinforce_set_lr: same handle, same graph
            pl.set_learning_rates(float(lr[c][0]), float(lr[c][1]))
        sl = slice(off, off + n)
        buf = _buffer(n, A, fx["state"][sl], fx["action"][sl], fx["reward"][sl], fx["next_state"][sl], fx["terminated"][sl], prefill)
        random.setstate((3, tuple(int(x) for x in fx["rng_before"][c]), None))
        trace = {}
        rep = pl.learn(buf, trace=trace)
        assert random.getstate() == (3, tuple(int(x) for x in fx["rng_after"][c]), None)
        handles.append(pl._handle.value)
        al += rep["actor_loss"]
        cl += rep["critic_loss"]
        idx += trace["idx"].tolist()
        got_R = np.float32(pl.last_return)
        if fx["terminated"][off + n - 1]:
            assert pl.last_bootstrap == 0.0
            assert got_R.tobytes() == fx["ret"][c:c + 1].tobytes(), (got_R, fx["ret"][c])
        else:
            _close([pl.last_bootstrap], fx["bootstrap"][c:c + 1], "bootstrap", rtol=1e-5, atol=1e-6)
            want = fold_returns(np.float32(pl.last_bootstrap), fx["reward"][sl]).numpy()
            assert got_R.tobytes() == want.tobytes(), (got_R, want)
        off += n
    assert len(set(handles)) == 1, "a learning-rate change re-created the C handle"
    assert idx == fx["idx"].tolist()
    _close(al, fx["actor_loss"], "actor_loss")
    _close(cl, fx["critic_loss"], "critic_loss")
    _close(pl.actor_params.cpu().numpy(), fx["actor_after"], "actor")
    _close(pl.critic_params.cpu().numpy(), fx["critic_after"], "critic")
    # the moments accumulate gradients of scale B |R - v| (hundreds here): elements that cancel to near zero carry the
    # fp32 summation noise of that scale, so the absolute floor is relative to the largest element
    for i, key in enumerate(("exp_avg", "exp_avg_sq", "max_exp_avg_sq")):
        for which, got in (("actor", pl._actor_state[i]), ("critic", pl._critic_state[i])):
            want = fx[f"{which}_{key}"]
            _close(got.cpu().numpy(), want, f"{which} {key}", atol=1e-5 * float(np.abs(want).max()))


def _data(n, obs, A, seed, p_term=0.02):
    rng = np.random.Generator(np.random.PCG64(seed))
    q8 = lambda x: (np.rint(x * 256) / 256).astype(np.float32)  # noqa: E731
    term = rng.random(n) < p_term
    term[-1] = False
    return dict(state=q8(rng.standard_normal((n, obs))), next_state=q8(rng.standard_normal((n, obs))),
                reward=q8(rng.standard_normal(n) * 0.1), action=rng.integers(0, A, size=n).astype(np.int32), term=term)


def _sync_from_oracle(pl, orc):
    pl.load_parameters(flat(orc.actor), flat(orc.critic))
    for i, key in enumerate(("exp_avg", "exp_avg_sq", "max_exp_avg_sq")):
        pl._actor_state[i].copy_(orc.adam_state("actor", key))
        pl._critic_state[i].copy_(orc.adam_state("critic", key))


@pytest.mark.parametrize("engine", [0, 1, 2])
def test_reinforce_stress_shape_against_oracle(engine):
    """obs 128, 16 actions, [256, 256], batch 256, a 20 000-transition rollout, 4 learn() calls of one round each.  Each
    call starts from the oracle's state (AdamW's first steps move an element by lr * sign(gradient) whatever its size, so
    an element whose gradient is zero to within summation noise may step the other way: DESIGN.md §4).  The oracle's
    bootstrap must match the GPU's at 1e-5 and the oracle folds R from the GPU's bootstrap, bit for bit."""
    from pearl_b200 import _lib
    torch.manual_seed(5)
    threads = torch.get_num_threads()
    torch.set_num_threads(8)
    n, obs, A, B, lr = 20000, 128, 16, 256, 3e-4
    d = _data(n, obs, A, seed=71)
    buf = _buffer(n, A, d["state"], d["action"], d["reward"], d["next_state"], d["term"])
    orc = OracleREINFORCE(obs, A, (256, 256), (256, 256), actor_lr=lr, critic_lr=lr)
    lib = _lib.load()
    prev = lib.prl_get_contraction_engine()
    _lib.check(lib.prl_set_contraction_engine(engine))
    try:
        pl = _learner(obs, A, (256, 256), training_rounds=1, batch_size=B, actor_learning_rate=lr, critic_learning_rate=lr)
        pl.load_parameters(flat(orc.actor), flat(orc.critic))
        random.seed(23)
        for r in range(4):
            trace = {}
            rep = pl.learn(buf, trace=trace)
            boot = orc.bootstrap(d["next_state"][-1], d["term"][-1])
            _close([pl.last_bootstrap], boot.numpy(), f"round {r} bootstrap", rtol=1e-5, atol=1e-6)
            ret = fold_returns(np.float32(pl.last_bootstrap), d["reward"])
            assert np.float32(pl.last_return).tobytes() == ret.numpy().tobytes()
            i = trace["idx"][0].numpy()
            out = orc.learn_batch(torch.from_numpy(d["state"][i]), torch.from_numpy(d["action"][i]), ret)
            _close(rep["actor_loss"], [out["actor_loss"]], f"round {r} actor_loss")
            _close(rep["critic_loss"], [out["critic_loss"]], f"round {r} critic_loss")
            _close_params(pl.actor_params.cpu().numpy(), flat(orc.actor).numpy(), "actor", lr, 1)
            _close_params(pl.critic_params.cpu().numpy(), flat(orc.critic).numpy(), "critic", lr, 1)
            _sync_from_oracle(pl, orc)
    finally:
        _lib.check(lib.prl_set_contraction_engine(prev))
        torch.set_num_threads(threads)


def test_reinforce_is_bit_reproducible_and_launch_count_is_fixed():
    """One call of R rounds == R one-round calls (max_rounds_per_call=1); CUDA-graph replay == plain launches; two runs
    agree, bit for bit.  Every round is 21 launches: gather, 2 x 3 forward contractions, the loss kernel, 2 x (4
    backward contractions + the fifth or the head kernel), 2 x AdamW, the round counter."""
    n, obs, A, B, R = 1500, 24, 6, 128, 9
    d = _data(n, obs, A, seed=29, p_term=0.05)

    def run(per_call, graph):
        buf = _buffer(n, A, d["state"], d["action"], d["reward"], d["next_state"], d["term"], prefill=100)
        pl = _learner(obs, A, (64, 64), training_rounds=R, batch_size=B, actor_learning_rate=1e-3, critic_learning_rate=1e-3,
                      max_rounds_per_call=per_call, seed=3)
        pl.use_cuda_graph = graph
        random.seed(31)
        trace = {}
        rep = pl.learn(buf, trace=trace)
        assert trace["launches"] == 21 * (R - per_call * ((R - 1) // per_call))      # the last call's rounds
        return rep, [pl.actor_params.cpu(), pl.critic_params.cpu(), pl._actor_state[1].cpu(), pl._critic_state[2].cpu(),
                     torch.tensor([pl.last_return, pl.last_bootstrap])]

    base_rep, base = run(R, True)
    for per_call, graph in [(1, True), (R, False), (R, True), (4, False)]:
        rep, vecs = run(per_call, graph)
        assert rep == base_rep, (per_call, graph)
        for a, b in zip(vecs, base):
            assert torch.equal(a, b), (per_call, graph)


def _fake_reference(monkeypatch):
    """Stand-in for pearl's REINFORCE module: the attributes the plugin reads, built as ActorCriticBase builds them."""
    def named(net, cls):
        net.__class__ = type(cls, (torch.nn.Sequential,), {})
        return net

    class REINFORCE:
        def __init__(self, state_dim, action_space=None, actor_hidden_dims=None, critic_hidden_dims=None, use_critic=False,
                     actor_learning_rate=1e-4, critic_learning_rate=1e-4, discount_factor=0.99, training_rounds=8, batch_size=64):
            A = action_space.n
            self._actor = named(_mlp([state_dim] + list(actor_hidden_dims) + [A]), "VanillaActorNetwork").cuda()
            self._critic = named(_mlp([state_dim] + list(critic_hidden_dims) + [1]), "VanillaValueNetwork").cuda()
            self._use_critic = use_critic
            self._actor_optimizer = torch.optim.AdamW(self._actor.parameters(), lr=actor_learning_rate, amsgrad=True)
            self._critic_optimizer = torch.optim.AdamW(self._critic.parameters(), lr=critic_learning_rate, amsgrad=True)
            self._history_summarization_module = type("IdentityHistorySummarizationModule", (torch.nn.Module,), {})()
            self._action_representation_module = type("OneHotActionTensorRepresentationModule", (torch.nn.Module,), {})()
            self.safety_module = None
            self._discount_factor, self._training_rounds, self._batch_size = discount_factor, training_rounds, batch_size
            self._training_steps = 0
    base = "pearl.policy_learners.sequential_decision_making"
    for p in ["pearl", "pearl.policy_learners", base]:
        monkeypatch.setitem(sys.modules, p, types.ModuleType(p))
    m = types.ModuleType(base + ".reinforce")
    m.REINFORCE = REINFORCE
    monkeypatch.setitem(sys.modules, base + ".reinforce", m)


def test_plugin_learning_rate_change_and_optimizer_load_state_dict(monkeypatch):
    """The plugin over a stand-in of the reference class: a change of param_groups' lr reaches the CUDA learner without a
    new handle; an optimizer (and network) checkpoint restored with load_state_dict is picked up by the next learn(), which
    then repeats the checkpoint's next call bit for bit."""
    import pearl_b200.actor_critic as ac
    n, obs, A, B = 500, 8, 3, 64
    d = _data(n, obs, A, seed=41, p_term=0.05)
    buf = _buffer(n, A, d["state"], d["action"], d["reward"], d["next_state"], d["term"])
    _fake_reference(monkeypatch)
    try:
        importlib.reload(ac)
        assert ac.HAVE_REFERENCE_REINFORCE
        torch.manual_seed(3)
        pl = ac.B200REINFORCE(state_dim=obs, action_space=types.SimpleNamespace(n=A), actor_hidden_dims=[32, 32],
                              critic_hidden_dims=[32, 32], use_critic=True, training_rounds=3, batch_size=B,
                              actor_learning_rate=1e-3, critic_learning_rate=1e-3)
        random.seed(1)
        pl.learn(buf)
        handle = pl._b200._handle.value
        pl._actor_optimizer.param_groups[0]["lr"] = 5e-4
        pl._critic_optimizer.param_groups[0]["lr"] = 2e-3
        pl.learn(buf)
        assert pl._b200._handle.value == handle, "a learning-rate change re-created the C handle"
        assert (pl._b200._actor_learning_rate, pl._b200._critic_learning_rate) == (5e-4, 2e-3)
        ck = [copy.deepcopy(x.state_dict()) for x in (pl._actor, pl._critic, pl._actor_optimizer, pl._critic_optimizer)]
        random.seed(9)
        rep = pl.learn(buf)
        want = [pl._b200.actor_params.clone(), pl._b200.critic_params.clone(), pl._b200._actor_state[2].clone()]
        pl.learn(buf)
        for x, s in zip((pl._actor, pl._critic, pl._actor_optimizer, pl._critic_optimizer), ck):
            x.load_state_dict(s)
        random.seed(9)
        assert pl.learn(buf) == rep
        got = [pl._b200.actor_params, pl._b200.critic_params, pl._b200._actor_state[2]]
        for a, b in zip(got, want):
            assert torch.equal(a, b)
        assert float(pl._actor_optimizer.state[next(pl._actor.parameters())]["step"]) == 9       # the checkpoint's 6 steps + 3
        with pytest.raises(NotImplementedError):
            pl.learn_batch(None)
    finally:
        monkeypatch.undo()
        importlib.reload(ac)


def test_reinforce_rejects_bad_inputs():
    import pearl_b200
    from pearl_b200 import _lib
    n, obs, A, B = 64, 6, 4, 16
    d = _data(n, obs, A, seed=43)
    pl = _learner(obs, A, (16, 16), training_rounds=2, batch_size=B)
    assert pl.learn(pearl_b200.B200ReplayBuffer(16)) == {}                  # empty buffer: nothing to do
    with pytest.raises(NotImplementedError):
        pearl_b200.B200REINFORCE(state_dim=obs, n_actions=A, actor_hidden_dims=[16, 16, 16], critic_hidden_dims=[16, 16])
    with pytest.raises(NotImplementedError):
        pearl_b200.B200REINFORCE(state_dim=obs, n_actions=A, actor_hidden_dims=[16, 16], critic_hidden_dims=[16, 16], use_critic=False)
    with pytest.raises(ValueError):                                         # n_actions outside 1..255
        _learner(obs, 256, (16, 16))
    cont = pearl_b200.B200ReplayBuffer(n)                                   # continuous actions
    cont.is_action_continuous = True
    t = torch.from_numpy
    cont.push_batch(t(d["state"]), torch.zeros(n, 2), t(d["reward"]), t(d["next_state"]), t(d["term"]), torch.zeros(n, dtype=torch.bool))
    with pytest.raises(ValueError):
        pl.learn(cont)
    params0 = [pl.actor_params.clone(), pl.critic_params.clone()]
    other = _buffer(n, A + 1, d["state"], d["action"], d["reward"], d["next_state"], d["term"])   # mismatched n_actions
    with pytest.raises(ValueError, match="matching"):
        pl.learn(other)
    # a shard of a multi-GPU buffer: rejected before the sampler or any learner kernel runs
    sharded = pearl_b200.B200ReplayBuffer(n, rng="device")
    sharded.push_batch_sharded(0, 2, t(d["state"]), t(d["action"]), t(d["reward"]), t(d["next_state"]), t(d["term"]),
                               torch.zeros(n, dtype=torch.bool), max_number_actions=A)
    sharded.seed(5)
    rng0 = sharded.get_rng_state()
    with pytest.raises(ValueError, match="shard"):
        pl.learn(sharded)
    torch.cuda.synchronize()
    assert np.array_equal(sharded.get_rng_state(), rng0), "the sampler ran"
    assert torch.equal(pl.actor_params, params0[0]) and torch.equal(pl.critic_params, params0[1]), "a learner kernel ran"
    # rounds / batch above the configured maxima, through the C ABI
    buf = _buffer(n, A, d["state"], d["action"], d["reward"], d["next_state"], d["term"])
    pl.learn(buf)
    lib, dev = pl._lib, torch.device("cuda")
    out = torch.zeros(4096, device=dev)
    for rounds, batch in ((pl._max_rounds + 1, B), (1, pl._bound_batch + 1), (0, B), (1, 0)):
        assert lib.prl_reinforce_learn(pl._handle, buf.handle, rounds, batch, _lib.ptr(pl._returns), _lib.ptr(out), _lib.ptr(out),
                                       None, None) == _lib.PRL_EINVAL
    assert torch.equal(out, torch.zeros_like(out))
