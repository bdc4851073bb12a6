#!/usr/bin/env python
"""Generate tests/golden/cb_nb_*.npz by RUNNING THE REFERENCE's NeuralBandit (CPU, same stubs and import path as
oracle/gen_golden.py).

    PYTHONDONTWRITEBYTECODE=1 python oracle/gen_neural_bandit_golden.py

Cases:
  cb_nb_squarecb  the reference's CB benchmark config (return_neural_squarecb_config: hidden [64, 16], lr 0.01, batch 128,
                  10 rounds, 5-bit binary action code, gamma = 10 sqrt(T (obs + bits)) with T = 10000) as an agent loop:
                  act -> push -> learn() per step over a BasicReplayBuffer.  A second run (keys `g5_*`) uses gamma = 5,
                  where most choices are not the greedy one
  cb_nb_fastcb    FastCB with one-hot codes; reward bounds under which some states clamp several values to the
                  upper bound (a tie the first index wins) and some have every value at or below the lower bound (the
                  uniform branch)
  cb_nb_batch     learn_batch with weights of both signs (their sum away from 0), MSE and MAE, with an lr change and a
                  load_state_dict round trip of the learner and of its optimizer
  cb_nb_scores    state_features_only=True: get_scores of 1-D and 2-D states, NoExploration act with and without masks

Recorded: the initial flat parameters, the pushes, the sampled logical indices, CPython's `random` state and torch's CPU
generator state before the first act and after the run, the per-round loss and predictions, and after every call the
flat parameters and the AdamW state; for every act the probability vector the explorer hands to `Categorical`, the
normalised one, the exponential draws of the sample and the chosen index; the state_dict keys.  The generator checks
that each sample is the first maximum of pn / E over draws replayed from the generator (and that they advance it exactly
as the sample did), and asserts a relative margin of MARGIN between the best and second-best pn / E of every choice,
between the two largest values wherever a greedy maximum decides, between every value and a clamping bound, and
|p - y| away from 0 on MAE rows.
"""
from __future__ import annotations

import os
import random
import sys

import numpy as np

sys.dont_write_bytecode = True
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from oracle.gen_golden import GOLDEN, state_words  # noqa: E402  (sets up the reference import path and stubs)

import torch  # noqa: E402
from pearl.action_representation_modules.binary_action_representation_module import (  # noqa: E402
    BinaryActionTensorRepresentationModule,
)
from pearl.action_representation_modules.one_hot_action_representation_module import (  # noqa: E402
    OneHotActionTensorRepresentationModule,
)
from pearl.policy_learners.contextual_bandits.neural_bandit import NeuralBandit  # noqa: E402
from pearl.policy_learners.exploration_modules.common.no_exploration import NoExploration  # noqa: E402
from pearl.policy_learners.exploration_modules.contextual_bandits import squarecb_exploration as sq  # noqa: E402
from pearl.replay_buffers.basic_replay_buffer import BasicReplayBuffer  # noqa: E402
from pearl.replay_buffers.transition import TransitionBatch  # noqa: E402
from pearl.utils.instantiations.spaces.discrete_action import DiscreteActionSpace  # noqa: E402

MARGIN = 1e-4
MAE_GAP = 1e-3
T_BENCH = 10000


class CategoricalSpy:
    """Stands in for squarecb_exploration's `Categorical`: records p, the normalised probs, the draws and the sample, and
    checks the sample against argmax(pn / E) with E replayed from the generator."""
    log: list = []

    def __init__(self, probs):
        self.p = probs.detach().clone()
        self.d = torch.distributions.Categorical(probs)

    def sample(self):
        before = torch.get_rng_state()
        a = self.d.sample()
        after = torch.get_rng_state()
        torch.set_rng_state(before)
        E = torch.empty(self.p.numel()).exponential_()
        assert torch.equal(torch.get_rng_state(), after), "the sample does not advance the generator by A exponential draws"
        pn = self.d.probs.detach()
        q = (pn / E).double()
        assert int(torch.argmax(pn / E)) == int(a), "the sample is not the first maximum of pn / E"
        top = torch.topk(q, min(2, q.numel())).values
        assert q.numel() == 1 or float(top[0] - top[1]) > MARGIN * float(top[0]), "pn / E margin too small"
        CategoricalSpy.log.append(dict(p=self.p.numpy().copy(), pn=pn.numpy().copy(), E=E.numpy().copy(), a=int(a)))
        return a


sq.Categorical = CategoricalSpy


def flat(pl):
    return torch.cat([p.detach().reshape(-1) for p in pl.model.parameters()]).numpy().copy()


def adam(pl):
    params = list(pl.model.parameters())
    st = pl.optimizer.state
    if not all(p in st for p in params):
        z = np.zeros(sum(p.numel() for p in params), np.float32)
        return dict(m=z, v=z, vmax=z, step=0.0)
    cat = lambda k: torch.cat([st[p][k].reshape(-1) for p in params]).numpy().copy()  # noqa: E731
    return dict(m=cat("exp_avg"), v=cat("exp_avg_sq"), vmax=cat("max_exp_avg_sq"), step=float(st[params[0]]["step"]))


def snapshot(pl):
    return dict(params=flat(pl), **{f"adam_{k}": np.asarray(v) for k, v in adam(pl).items()})


def stack(snaps, prefix="call_"):
    return {f"{prefix}{k}": np.stack([np.asarray(s[k]) for s in snaps]) for k in snaps[0]}


def greedy_ok(values, ex):
    """The values the explorer sees decide its greedy maximum and its clamping by clear margins."""
    v = values.double().reshape(-1)
    clamp = ex.clamp_values
    if clamp:
        for bnd in (ex.reward_lb, ex.reward_ub):
            assert bool(((v - bnd).abs() > MARGIN * (1 + abs(bnd))).all()), "a value sits at a clamping bound"
        v = v.clamp(ex.reward_lb, ex.reward_ub)
    top = torch.topk(v, min(2, v.numel())).values
    at_bound = clamp and float(top[0]) in (float(np.float32(ex.reward_lb)), float(np.float32(ex.reward_ub)))
    assert at_bound or v.numel() == 1 or float(top[0] - top[1]) > MARGIN * (1 + abs(float(top[0]))), "greedy margin too small"
    return at_bound


def save(name, out, what):
    path = os.path.join(GOLDEN, f"{name}.npz")
    np.savez_compressed(path, **out)
    print(f"{name}.npz: {os.path.getsize(path) // 1024} KB, {what}")


def run_agent(*, obs, n_act, rep, hidden, lr, batch, rounds, prefill, steps, explorer, loss, seed, scale=1.0, act_scale=None):
    torch.manual_seed(seed)
    random.seed(seed)
    torch.set_num_threads(1)
    rng = np.random.default_rng(seed)
    module = OneHotActionTensorRepresentationModule(n_act) if rep == "one_hot" else BinaryActionTensorRepresentationModule(rep)
    act_dim = module.representation_dim
    space = DiscreteActionSpace([torch.tensor([i]) for i in range(n_act)])
    feats = module(torch.arange(n_act).view(-1, 1)).numpy().reshape(n_act, act_dim)
    pl = NeuralBandit(feature_dim=obs + act_dim, hidden_dims=list(hidden), exploration_module=explorer,
                      action_representation_module=module, training_rounds=rounds, batch_size=batch, learning_rate=lr,
                      loss_type=loss)
    init = flat(pl)
    buf = BasicReplayBuffer(100000)
    theta, beta = rng.standard_normal(obs).astype(np.float32) * 0.5, rng.standard_normal(act_dim).astype(np.float32)
    idxs, preds, losses, snaps = [], [], [], []
    orig_sample = buf.sample

    def sample_spy(k):
        pos = {id(t): j for j, t in enumerate(buf.memory)}
        s0 = random.getstate()
        idxs.append([pos[id(t)] for t in random.sample(buf.memory, k)])
        random.setstate(s0)
        return orig_sample(k)
    buf.sample = sample_spy
    P = dict(state=[], action=[], reward=[])

    def push(s, a):
        r = np.float32(np.round((np.tanh(s @ theta) + feats[a] @ beta * 0.5 + 0.1 * rng.standard_normal()) * 256) / 256)
        buf.push(state=torch.from_numpy(s), action=torch.tensor([a]), reward=float(r), terminated=True, truncated=False,
                 curr_available_actions=None, next_state=None, next_available_actions=None, max_number_actions=n_act)
        P["state"].append(s); P["action"].append(a); P["reward"].append(r)

    def learn():
        rep_ = pl.learn(buf)
        p = [x.detach().numpy().ravel() for x in rep_["prediction"]]
        if loss == "mae":
            y = [x.numpy().ravel() for x in rep_["label"]]
            assert min(np.abs(a - b).min() for a, b in zip(p, y)) > MAE_GAP, "an MAE row sits at |p - y| = 0"
        preds.extend(p)
        losses.extend(float(x) for x in rep_["loss"])
        snaps.append(snapshot(pl))

    for _ in range(prefill):
        push(np.round(rng.standard_normal(obs) * scale * 64).astype(np.float32) / 64, int(rng.integers(n_act)))
    rs = random.getstate()
    learn()
    torch_before = torch.get_rng_state().numpy().copy()
    CategoricalSpy.log = []
    chosen, states, values, at_bound = [], [], [], []
    for k in range(steps):
        sc = scale if act_scale is None else act_scale[k % len(act_scale)]
        s = np.round(rng.standard_normal(obs) * sc * 64).astype(np.float32) / 64
        with torch.no_grad():
            v = pl.get_scores(torch.from_numpy(s), space).reshape(-1)
        at_bound.append(greedy_ok(v, explorer))
        a = pl.act(torch.from_numpy(s), space)
        assert a.dtype == torch.int32 and a.dim() == 0 and a.device.type == "cpu"
        chosen.append(int(a)); states.append(s); values.append(v.numpy().copy())
        push(s, int(a))
        learn()
    log = CategoricalSpy.log
    assert [e["a"] for e in log] == chosen
    out = dict(seed=seed, obs=obs, n_actions=n_act, rep=rep if isinstance(rep, str) else f"binary{rep}", act_dim=act_dim,
               hidden=np.asarray(hidden, np.int32), lr=lr, batch=batch, rounds=rounds, prefill=prefill, loss=loss,
               gamma=float(explorer._gamma), reward_lb=float(explorer.reward_lb), reward_ub=float(explorer.reward_ub),
               clamp=bool(explorer.clamp_values), fastcb=isinstance(explorer, sq.FastCBExploration), init=init,
               push_state=np.stack(P["state"]), push_action=np.asarray(P["action"], np.int32),
               push_reward=np.asarray(P["reward"], np.float32), act_state=np.stack(states), act_chosen=np.asarray(chosen, np.int32),
               act_values=np.stack(values), act_p=np.stack([e["p"] for e in log]), act_pn=np.stack([e["pn"] for e in log]),
               act_E=np.stack([e["E"] for e in log]), act_at_bound=np.asarray(at_bound),
               rng_before=state_words(rs), rng_after=state_words(random.getstate()),
               torch_before=torch_before, torch_after=torch.get_rng_state().numpy().copy(),
               idx=np.asarray([j for r in idxs for j in r], dtype=np.int32), idx_len=np.asarray([len(r) for r in idxs], np.int32),
               pred=np.concatenate(preds).astype(np.float32), losses=np.asarray(losses, np.float32),
               keys=np.asarray(list(pl.state_dict().keys())), **stack(snaps))
    return out


def gen_squarecb(name):
    obs, bits = 16, 5
    gamma = torch.sqrt(torch.tensor(T_BENCH) * (obs + bits)).item() * 10.0      # return_neural_squarecb_config
    kw = dict(obs=obs, n_act=26, rep=bits, hidden=(64, 16), lr=0.01, batch=128, rounds=10, prefill=150, steps=8, loss="mse",
              scale=0.5)
    out = run_agent(explorer=sq.SquareCBExploration(gamma=gamma), seed=95, **kw)
    g5 = run_agent(explorer=sq.SquareCBExploration(gamma=5.0), seed=96, **kw)
    greedy = lambda o: int((o["act_chosen"] == o["act_values"].argmax(1)).sum())  # noqa: E731
    assert greedy(g5) < len(g5["act_chosen"]), "gamma 5 never leaves the greedy action"
    out.update({f"g5_{k}": v for k, v in g5.items()})
    save(name, out, f"gamma {gamma:.1f}: {greedy(out)} of {len(out['act_chosen'])} greedy; gamma 5: {greedy(g5)} greedy")


def gen_fastcb(name):
    out = run_agent(explorer=sq.FastCBExploration(gamma=50.0, reward_lb=-0.25, reward_ub=0.25), obs=8, n_act=6, rep="one_hot",
                    hidden=(16, 8), lr=0.01, batch=64, rounds=4, prefill=80, steps=12, loss="mse", seed=97,
                    act_scale=(0.5, 3.0, 3.0))
    ub, lb = np.float32(out["reward_ub"]), np.float32(out["reward_lb"])
    clamped = np.clip(out["act_values"], lb, ub)
    ties = int(((clamped == ub).sum(1) >= 2).sum())
    uniform = int((clamped.max(1) <= lb).sum())
    assert ties and uniform, (ties, uniform)
    save(name, out, f"{ties} states with clamped ties at the upper bound, {uniform} in the uniform branch")


def gen_batch(name, *, obs, act_dim, hidden, batch, calls, seed):
    """Two learners on dense batches, MSE and MAE, with weights of both signs."""
    torch.manual_seed(seed)
    torch.set_num_threads(1)
    rng = np.random.default_rng(seed)
    out = dict(seed=seed, obs=obs, act_dim=act_dim, hidden=np.asarray(hidden, np.int32), batch=batch, calls=calls,
               lr0=0.005, lr1=0.02, lr_change_at=2, reload_at=3)
    for loss in ("mse", "mae"):
        pl = NeuralBandit(feature_dim=obs + act_dim, hidden_dims=list(hidden), exploration_module=NoExploration(),
                          batch_size=batch, learning_rate=0.005, loss_type=loss)
        out[f"{loss}_init"] = flat(pl)
        B = dict(state=[], action=[], reward=[], weight=[])
        preds, losses, snaps = [], [], []
        for c in range(calls):
            if c == out["lr_change_at"]:
                for g in pl.optimizer.param_groups:
                    g["lr"] = out["lr1"]
            if c == out["reload_at"]:
                pl.load_state_dict({k: v.clone() for k, v in pl.state_dict().items()})
                pl.optimizer.load_state_dict(pl.optimizer.state_dict())
            s = rng.standard_normal((batch, obs)).astype(np.float32)
            a = rng.uniform(-1, 1, (batch, act_dim)).astype(np.float32)
            r = (s.sum(1) * 0.3 + a @ np.linspace(-1, 1, act_dim).astype(np.float32) + 0.1 * rng.standard_normal(batch))
            r = r.astype(np.float32)
            w = (rng.uniform(0.25, 2.0, batch) * np.where(rng.random(batch) < 0.2, -1.0, 1.0)).astype(np.float32)
            assert w.sum() > 0.25 * np.abs(w).sum()
            rep_ = pl.learn_batch(TransitionBatch(state=torch.from_numpy(s), action=torch.from_numpy(a), reward=torch.from_numpy(r),
                                                  weight=torch.from_numpy(w)))
            p = rep_["prediction"].detach().numpy().ravel()
            if loss == "mae":
                assert np.abs(p - r).min() > MAE_GAP, "an MAE row sits at |p - y| = 0"
            preds.append(p); losses.append(float(rep_["loss"]))
            snaps.append(snapshot(pl))
            B["state"].append(s); B["action"].append(a); B["reward"].append(r); B["weight"].append(w)
        out.update({f"{loss}_b_{k}": np.stack(v) for k, v in B.items()})
        out.update({f"{loss}_pred": np.stack(preds), f"{loss}_loss": np.asarray(losses, np.float32)})
        out.update(stack(snaps, f"{loss}_call_"))
    save(name, out, f"{calls} calls x 2 losses")


def gen_scores(name, *, obs, n_act, hidden, n_states, seed):
    """A state-features-only learner fitted by learn_batch, then scored over a batch of states."""
    torch.manual_seed(seed)
    torch.set_num_threads(1)
    rng = np.random.default_rng(seed)
    space = DiscreteActionSpace([torch.tensor([i]) for i in range(n_act)])
    pl = NeuralBandit(feature_dim=obs, hidden_dims=list(hidden), exploration_module=NoExploration(), batch_size=256,
                      learning_rate=0.01, state_features_only=True,
                      action_representation_module=OneHotActionTensorRepresentationModule(n_act))
    s = rng.standard_normal((256, obs)).astype(np.float32)
    r = (s[:, 0] + 0.1 * rng.standard_normal(256)).astype(np.float32)
    for _ in range(3):
        pl.learn_batch(TransitionBatch(state=torch.from_numpy(s), action=torch.zeros(256, n_act), reward=torch.from_numpy(r)))
    states = torch.from_numpy(rng.standard_normal((n_states, obs)).astype(np.float32))
    mask = torch.from_numpy(rng.random((n_states, n_act)) < 0.6)
    mask[:, 0] = False
    mask[:, 3] = True
    with torch.no_grad():
        scores = pl.get_scores(states, space)
        one = pl.get_scores(states[0], space)
        act_all = pl.act(states, space).reshape(-1)
    assert tuple(one.shape) == (1, n_act) and tuple(scores.shape) == (n_states, n_act)
    # every action of a state scores the same: the first available one is chosen.  The reference's masked act fails in
    # `embedding` (float indices) under this torch version, so masked choices follow its first-maximum rule.
    first_max = lambda sc: torch.argmax(torch.where(mask, sc, torch.tensor(-float("inf"))), dim=1)  # noqa: E731
    act_mask = first_max(scores)
    assert (act_all == 0).all()
    out = dict(seed=seed, obs=obs, n_actions=n_act, hidden=np.asarray(hidden, np.int32), params=flat(pl), states=states.numpy(),
               mask=mask.numpy(), scores=scores.numpy(), scores_one=one.numpy(), act_mask=act_mask.numpy().astype(np.int32),
               act_all=act_all.numpy().astype(np.int32), keys=np.asarray(list(pl.state_dict().keys())))
    save(name, out, f"{n_states} states")


if __name__ == "__main__":
    gen_squarecb("cb_nb_squarecb")
    gen_fastcb("cb_nb_fastcb")
    gen_batch("cb_nb_batch", obs=8, act_dim=4, hidden=(32, 8), batch=64, calls=5, seed=98)
    gen_scores("cb_nb_scores", obs=12, n_act=7, hidden=(24, 12), n_states=64, seed=99)
