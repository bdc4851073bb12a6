"""Discrete SAC on the GPU (pearl_b200.B200SoftActorCritic, csrc/sac_discrete.cu) against
(a) the recordings of the reference's PearlAgent(SoftActorCritic, BasicReplayBuffer).learn() (tests/golden/sacd_*.npz:
    same indices from CPython's `random.sample`), elementwise 1e-4 (tests/_tol.py);
(b) oracle/sac_discrete_oracle.py at a stress shape (obs 128, 16 actions, [256, 256], batch 256: the B*A = 4096-row
    critic products are where the automatic contraction engine switches to the tensor-core tiles), step by step from a
    re-synchronised state, under the SIMT engine and the tensor-core engine;
(c) the oracle with a saturated policy (probabilities exactly 0) and a 40-round entropy chain started at log alpha = -7;
plus bit-identity (round chunking, graph replay, run to run) and the rejected inputs."""
import os
import random

import numpy as np
import pytest
import torch

from conftest import GOLDEN
from oracle.pearl_oracle import flat
from oracle.sac_discrete_oracle import OracleSACDiscrete

pytestmark = pytest.mark.gpu

from _tol import close as _close, close_params as _close_params  # noqa: E402


def _buffer(n, A, state, action, reward, next_state, term, ids=None, cnt=None, **kw):
    import pearl_b200
    buf = pearl_b200.B200ReplayBuffer(n, **kw)
    t = torch.as_tensor
    buf.push_batch(t(state), t(action).to(torch.int32), t(reward), t(next_state), t(term), torch.zeros(n, dtype=torch.bool),
                   next_available_ids=None if ids is None else t(ids).to(torch.uint8),
                   next_available_count=None if cnt is None else t(cnt).to(torch.int32), max_number_actions=A)
    return buf


def _learner(obs, A, hidden, **kw):
    import pearl_b200
    return pearl_b200.B200SoftActorCritic(state_dim=obs, n_actions=A, actor_hidden_dims=list(hidden), critic_hidden_dims=list(hidden), **kw)


@pytest.mark.parametrize("case", ["sacd_full", "sacd_dynamic", "sacd_reset"])
def test_sac_discrete_matches_reference_recording(case):
    fx = np.load(os.path.join(GOLDEN, f"{case}.npz"))
    n, A, R, B, calls = int(fx["n"]), int(fx["n_actions"]), int(fx["rounds"]), int(fx["batch"]), int(fx["calls"])
    dyn = bool(fx["dynamic"])
    buf = _buffer(n, A, fx["state"], fx["action"], fx["reward"], fx["next_state"], fx["terminated"],
                  fx["next_ids"] if dyn else None, fx["next_count"] if dyn else None)
    pl = _learner(int(fx["obs"]), A, fx["hidden"].tolist(), training_rounds=R, batch_size=B, actor_learning_rate=float(fx["actor_lr"]),
                  critic_learning_rate=float(fx["critic_lr"]), critic_soft_update_tau=float(fx["tau"]), discount_factor=float(fx["gamma"]),
                  entropy_coef=float(fx["entropy_coef"]), entropy_autotune=bool(fx["autotune"]))
    pl.load_parameters(fx["init_actor"], fx["init_q1"], fx["init_q2"], fx["init_q1t"], fx["init_q2t"])
    before = (3, tuple(int(x) for x in fx["rng_before"]), None)
    random.setstate(before)
    al, cl, el, idx, handles = [], [], [], [], []
    for c in range(calls):
        if c:   # agent.reset(): the actor's ExponentialLR stepped; the change goes through prl_sacd_set_lr
            pl.set_learning_rates(float(fx["call_actor_lr"][c]), float(fx["critic_lr"]))
        trace = {}
        rep = pl.learn(buf, trace=trace)
        handles.append(pl._handle.value)
        al += rep["actor_loss"]
        cl += rep["critic_loss"]
        el += rep.get("entropy_coef", [])
        idx += trace["idx"].tolist()
    assert len(set(handles)) == 1, "a learning-rate change re-created the C handle"
    assert idx == fx["idx"].tolist()                                   # bit-exact sampling
    after = random.getstate()
    random.setstate(before)
    for _ in range(R * calls):
        random.sample(range(n), B)
    assert random.getstate() == after                                  # the python RNG advanced as R random.sample calls
    _close(al, fx["actor_loss"], "actor_loss")
    _close(cl, fx["critic_loss"], "critic_loss")
    pc = pl.critic_params.numel() // 2
    _close(pl.actor_params.cpu().numpy(), fx["actor_after"], "actor")
    _close(pl.critic_params[:pc].cpu().numpy(), fx["q1_after"], "q1")
    _close(pl.critic_params[pc:].cpu().numpy(), fx["q2_after"], "q2")
    _close(pl.critic_target_params[:pc].cpu().numpy(), fx["q1t_after"], "q1 target")
    _close(pl.critic_target_params[pc:].cpu().numpy(), fx["q2t_after"], "q2 target")
    if bool(fx["autotune"]):
        _close(el, fx["entropy_loss"], "entropy loss")
        _close(pl._log_entropy[:1].cpu().numpy(), fx["log_alpha_after"], "log_alpha")
        _close(pl._log_entropy[1:2].cpu().numpy(), fx["alpha_exp_avg"], "log_alpha exp_avg")
        _close(pl._log_entropy[2:3].cpu().numpy(), fx["alpha_exp_avg_sq"], "log_alpha exp_avg_sq")
        _close([pl.entropy_coef], fx["alpha_after"], "entropy coefficient")
    else:
        assert pl.entropy_coef == pytest.approx(float(fx["entropy_coef"]))


def _data(n, obs, A, seed, p_term=0.1):
    rng = np.random.Generator(np.random.PCG64(seed))
    q8 = lambda x: (np.rint(x * 256) / 256).astype(np.float32)  # noqa: E731
    ids = np.zeros((n, A), dtype=np.uint8)
    cnt = rng.integers(1, A + 1, size=n).astype(np.int32)
    for i in range(n):
        ids[i, :cnt[i]] = np.sort(rng.choice(A, size=cnt[i], replace=False))
    return dict(state=q8(rng.standard_normal((n, obs))), next_state=q8(rng.standard_normal((n, obs))),
                reward=q8(rng.standard_normal(n)), action=rng.integers(0, A, size=n).astype(np.int32),
                term=rng.random(n) < p_term, ids=ids, cnt=cnt)


def _adam_flat(opt, params, key):
    return torch.cat([opt.state[p][key].reshape(-1) for p in params])


def _sync_from_oracle(pl, orc, entropy=True):
    """Parameters and AdamW moments of both networks from the oracle; with `entropy`, also log alpha and its Adam state."""
    pl.load_parameters(flat(orc.actor), flat(orc.q[0]), flat(orc.q[1]), flat(orc.qt[0]), flat(orc.qt[1]))
    ap = list(orc.actor.parameters())
    cp = list(orc.q[0].parameters()) + list(orc.q[1].parameters())
    for i, key in enumerate(("exp_avg", "exp_avg_sq", "max_exp_avg_sq")):
        pl._actor_state[i].copy_(_adam_flat(orc.opt_actor, ap, key))
        pl._critic_state[i].copy_(_adam_flat(orc.opt_critic, cp, key))
    if not entropy:
        return
    st = orc.opt_alpha.state[orc.log_alpha]
    pl._log_entropy.copy_(torch.stack([orc.log_alpha.detach()[0], st["exp_avg"][0], st["exp_avg_sq"][0]]))
    pl._entropy_coef.copy_(orc.alpha.reshape(1))


@pytest.mark.parametrize("engine", [0, 2])
def test_sac_discrete_stress_shape_against_oracle(engine):
    """obs 128, 16 actions, [256, 256], batch 256, dynamic next-action sets, 20 rounds.  Each round starts from the oracle's
    state (parameters, AdamW and Adam moments): AdamW's first steps move an element by lr * sign(gradient) whatever its
    magnitude, so an element whose gradient is zero to within fp32 summation noise may step the other way (DESIGN.md §4);
    each round must agree elementwise to 1e-4 up to the counted outliers of `close_params`."""
    from pearl_b200 import _lib
    torch.manual_seed(7)
    threads = torch.get_num_threads()
    torch.set_num_threads(8)
    n, obs, A, B, R, lr = 3000, 128, 16, 256, 20, 3e-4
    d = _data(n, obs, A, seed=11)
    buf = _buffer(n, A, d["state"], d["action"], d["reward"], d["next_state"], d["term"], d["ids"], d["cnt"])
    orc = OracleSACDiscrete(obs, A, (256, 256), (256, 256), actor_lr=lr, critic_lr=lr, gamma=0.99, tau=0.005, autotune=True)
    for m in [orc.actor] + orc.q:
        for mod in m.modules():
            if isinstance(mod, torch.nn.Linear):
                torch.nn.init.xavier_uniform_(mod.weight)
                mod.bias.data.fill_(0.01)
    for i in range(2):
        orc.qt[i].load_state_dict(orc.q[i].state_dict())
    lib = _lib.load()
    prev = lib.prl_get_contraction_engine()
    _lib.check(lib.prl_set_contraction_engine(engine))
    try:
        pl = _learner(obs, A, (256, 256), training_rounds=1, batch_size=B, actor_learning_rate=lr, critic_learning_rate=lr,
                      critic_soft_update_tau=0.005, discount_factor=0.99)
        pl.load_parameters(flat(orc.actor), flat(orc.q[0]), flat(orc.q[1]))
        random.seed(19)
        pc = pl.critic_params.numel() // 2
        mask = lambda i: torch.arange(A).unsqueeze(0) >= torch.from_numpy(d["cnt"][i]).unsqueeze(1)  # noqa: E731
        for r in range(R):
            trace = {}
            rep = pl.learn(buf, trace=trace)
            i = trace["idx"][0].numpy()
            t = lambda k: torch.from_numpy(d[k][i])  # noqa: E731
            out = orc.learn_batch(dict(state=t("state"), action=t("action"), reward=t("reward"), next_state=t("next_state"),
                                       terminated=t("term"), next_ids=t("ids").long(), next_mask=mask(i)))
            _close(rep["actor_loss"], [out["actor_loss"]], f"round {r} actor_loss")
            _close(rep["critic_loss"], [out["critic_loss"]], f"round {r} critic_loss")
            _close(rep["entropy_coef"], [out["entropy_coef"]], f"round {r} entropy loss")
            _close_params(pl.actor_params.cpu().numpy(), flat(orc.actor).numpy(), "actor", lr, 1)
            _close_params(pl.critic_params[:pc].cpu().numpy(), flat(orc.q[0]).numpy(), "q1", lr, 1)
            _close_params(pl.critic_params[pc:].cpu().numpy(), flat(orc.q[1]).numpy(), "q2", lr, 1)
            _close_params(pl.critic_target_params[:pc].cpu().numpy(), flat(orc.qt[0]).numpy(), "q1 target", lr, 1)
            _close_params(pl.critic_target_params[pc:].cpu().numpy(), flat(orc.qt[1]).numpy(), "q2 target", lr, 1)
            _close(pl._log_entropy[:1].cpu().numpy(), orc.log_alpha.detach().numpy(), "log_alpha")
            _sync_from_oracle(pl, orc)
    finally:
        _lib.check(lib.prl_set_contraction_engine(prev))
        torch.set_num_threads(threads)


def test_sac_discrete_saturated_policy_and_entropy_chain():
    """Two regimes the recordings do not reach.
    * A saturated policy: the actor head's bias puts three of six actions ~300 below the rest, so their softmax
      probabilities are exactly 0 in fp32.  Only the + 1e-8 inside log(pi + 1e-8) keeps the actor loss, its gradient, the
      critic target and the entropy finite there (0 * log 0 is NaN), as in the reference.
    * The entropy step's own arithmetic: log alpha starts at -7 and the entropy Adam (critic lr 1e-2) runs 40 rounds
      without being re-synchronised.  The gradient exp(log alpha) (H - target) is then ~1e-3, so Adam's eps = 1e-4 is a
      large part of the denominator, and AdamW's decoupled decay of log alpha (or amsgrad) would move it by far more than
      1e-4 over the run.
    The networks are re-synchronised with the oracle every round (as in the stress test); log alpha is not."""
    torch.manual_seed(13)
    n, obs, A, B, R, clr, la0 = 2000, 8, 6, 128, 40, 1e-2, -7.0
    d = _data(n, obs, A, seed=17)
    buf = _buffer(n, A, d["state"], d["action"], d["reward"], d["next_state"], d["term"], d["ids"], d["cnt"])
    orc = OracleSACDiscrete(obs, A, (32, 32), (32, 32), actor_lr=1e-3, critic_lr=clr, gamma=0.99, tau=0.005, autotune=True)
    with torch.no_grad():
        head = orc.actor.net[-1][0]
        head.weight.mul_(4.0)
        head.bias.copy_(torch.tensor([0.0, 0.0, 0.0, -300.0, -300.0, -300.0]))
        orc.log_alpha.fill_(la0)
    orc.alpha = torch.exp(orc.log_alpha).detach()
    for i in range(2):
        orc.qt[i].load_state_dict(orc.q[i].state_dict())
    pl = _learner(obs, A, (32, 32), training_rounds=1, batch_size=B, actor_learning_rate=1e-3, critic_learning_rate=clr,
                  critic_soft_update_tau=0.005, discount_factor=0.99)
    pl.load_parameters(flat(orc.actor), flat(orc.q[0]), flat(orc.q[1]))
    pl._log_entropy.copy_(torch.tensor([la0, 0.0, 0.0]))
    pl._entropy_coef.copy_(orc.alpha.reshape(1))
    random.seed(37)
    pc = pl.critic_params.numel() // 2
    mask = lambda i: torch.arange(A).unsqueeze(0) >= torch.from_numpy(d["cnt"][i]).unsqueeze(1)  # noqa: E731
    for r in range(R):
        trace = {}
        rep = pl.learn(buf, trace=trace)
        i = trace["idx"][0].numpy()
        t = lambda k: torch.from_numpy(d[k][i])  # noqa: E731
        if r == 0:
            assert int((orc.actor(t("state")) == 0).sum()) >= B, "the policy is not saturated"
        out = orc.learn_batch(dict(state=t("state"), action=t("action"), reward=t("reward"), next_state=t("next_state"),
                                   terminated=t("term"), next_ids=t("ids").long(), next_mask=mask(i)))
        got = [rep["actor_loss"][0], rep["critic_loss"][0], rep["entropy_coef"][0]]
        assert np.isfinite(got).all() and torch.isfinite(pl.actor_params).all() and torch.isfinite(pl._log_entropy).all(), \
            f"round {r}: non-finite values {got}"
        _close(got, [out["actor_loss"], out["critic_loss"], out["entropy_coef"]], f"round {r} actor / critic / entropy loss")
        _close_params(pl.actor_params.cpu().numpy(), flat(orc.actor).numpy(), "actor", 1e-3, 1)
        _close_params(pl.critic_params[:pc].cpu().numpy(), flat(orc.q[0]).numpy(), "q1", clr, 1)
        _close_params(pl.critic_params[pc:].cpu().numpy(), flat(orc.q[1]).numpy(), "q2", clr, 1)
        st = orc.opt_alpha.state[orc.log_alpha]
        _close(pl._log_entropy.cpu().numpy(), [float(orc.log_alpha), float(st["exp_avg"]), float(st["exp_avg_sq"])],
               f"round {r} [log alpha, exp_avg, exp_avg_sq]", atol=1e-12)
        _sync_from_oracle(pl, orc, entropy=False)


def test_sac_discrete_is_bit_reproducible():
    """One call of R rounds == R one-round calls (max_rounds_per_call=1); CUDA-graph replay == plain launches; two runs
    agree.  Bit for bit: the launch sequence and every summation order are fixed."""
    n, obs, A, B, R = 1500, 24, 6, 128, 9
    d = _data(n, obs, A, seed=23)

    def run(per_call, graph):
        buf = _buffer(n, A, d["state"], d["action"], d["reward"], d["next_state"], d["term"], d["ids"], d["cnt"])
        pl = _learner(obs, A, (64, 64), training_rounds=R, batch_size=B, actor_learning_rate=1e-3, critic_learning_rate=1e-3,
                      max_rounds_per_call=per_call, seed=3)
        pl.use_cuda_graph = graph
        random.seed(29)
        rep = pl.learn(buf)
        return rep, [pl.actor_params.cpu(), pl.critic_params.cpu(), pl.critic_target_params.cpu(), pl._log_entropy.cpu(),
                     pl._actor_state[1].cpu(), pl._critic_state[2].cpu()]

    base_rep, base = run(R, True)
    for per_call, graph in [(1, True), (R, False), (R, True)]:
        rep, vecs = run(per_call, graph)
        assert rep == base_rep, (per_call, graph)
        for a, b in zip(vecs, base):
            assert torch.equal(a, b), (per_call, graph)


def test_sac_discrete_launch_count_is_fixed():
    n, obs, A, B = 600, 8, 4, 64
    d = _data(n, obs, A, seed=31)
    buf = _buffer(n, A, d["state"], d["action"], d["reward"], d["next_state"], d["term"])
    pl = _learner(obs, A, (32, 32), training_rounds=5, batch_size=B)
    trace = {}
    pl.learn(buf, trace=trace)
    assert trace["launches"] == 5 * 33          # 21 contractions + 12 small kernels per round (DESIGN.md §3.4)


def test_sac_discrete_rejects_bad_inputs():
    import pearl_b200
    n, obs, A, B = 64, 6, 4, 16
    d = _data(n, obs, A, seed=41)
    pl = _learner(obs, A, (16, 16), training_rounds=2, batch_size=B)
    assert pl.learn(pearl_b200.B200ReplayBuffer(16)) == {}                  # empty buffer: nothing to do
    with pytest.raises(NotImplementedError):                                # three hidden layers
        pearl_b200.B200SoftActorCritic(state_dim=obs, n_actions=A, actor_hidden_dims=[16, 16, 16], critic_hidden_dims=[16, 16])
    cont = pearl_b200.B200ReplayBuffer(n)                                   # continuous actions
    cont.is_action_continuous = True
    cont.push_batch(torch.from_numpy(d["state"]), torch.zeros(n, 2), torch.from_numpy(d["reward"]), torch.from_numpy(d["next_state"]),
                    torch.from_numpy(d["term"]), torch.zeros(n, dtype=torch.bool))
    with pytest.raises(ValueError):
        pl.learn(cont)
    # a shard of a multi-GPU buffer samples global slots: rejected before the sampler or any learner kernel runs
    sharded = pearl_b200.B200ReplayBuffer(n, rng="device")
    t = torch.from_numpy
    sharded.push_batch_sharded(0, 2, t(d["state"]), t(d["action"]), t(d["reward"]), t(d["next_state"]), t(d["term"]),
                               torch.zeros(n, dtype=torch.bool), max_number_actions=A)
    sharded.seed(5)
    rng0 = sharded.get_rng_state()
    params0 = [pl.actor_params.clone(), pl.critic_params.clone()]
    with pytest.raises(ValueError, match="shard"):
        pl.learn(sharded)
    torch.cuda.synchronize()
    assert np.array_equal(sharded.get_rng_state(), rng0), "the sampler ran"
    assert torch.equal(pl.actor_params, params0[0]) and torch.equal(pl.critic_params, params0[1]), "a learner kernel ran"
