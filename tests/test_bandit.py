"""GPU checks of B200LinearBandit (csrc/bandit.cu) against the reference's recordings (tests/golden/cb_*.npz), the eager
oracle (oracle/bandit_oracle.py) and itself: bit-identity run to run, graph vs eager and across round chunking, the launch
count, checkpoint views, act with masks and the refusals.  Tolerances as in test_bandit_oracle.py: sums elementwise,
solved quantities normwise."""
from __future__ import annotations

import os
import random
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from oracle import bandit_oracle as bo  # noqa: E402
from test_bandit_oracle import act_features, close_normwise, close_state, load  # noqa: E402

pytestmark = pytest.mark.gpu

DEV = "cuda:0"


class Space:
    def __init__(self, n):
        self.n = n
        self.actions = [torch.tensor([i]) for i in range(n)]
        self.actions_batch = torch.arange(n).view(n, 1)


def module_of(fx):
    import pearl_b200 as P
    if str(fx["rep"]) == "one_hot":
        return P.OneHotActionTensorRepresentationModule(int(fx["n_actions"]))
    return P.BinaryActionTensorRepresentationModule(int(fx["act_dim"]))


def make(fx, **kw):
    import pearl_b200 as P
    return P.B200LinearBandit(feature_dim=int(fx["obs"]) + int(fx["act_dim"]), exploration_module=P.UCBExploration(float(fx["alpha"])),
                              l2_reg_lambda=float(fx["l2_reg_lambda"]), gamma=float(fx["gamma"]),
                              apply_discounting_interval=float(fx["interval"]), training_rounds=int(fx["rounds"]),
                              batch_size=int(fx["batch"]), action_representation_module=module_of(fx), **kw)


def state_of(lb):
    m = lb.model
    return dict(A=m._A.cpu().numpy(), b=m._b.cpu().numpy(), sum_weight=m._sum_weight.cpu().numpy(), inv_A=m._inv_A.cpu().numpy(),
                coefs=m._coefs.cpu().numpy())


def run_method(fx, capacity=100000, graph=True, act=True, **kw):
    """The recorded agent loop on the GPU: prefill, learn, then act -> push -> learn per step."""
    import pearl_b200 as P
    torch.cuda.set_device(0)
    lb = make(fx, **kw)
    lb.use_cuda_graph = graph
    buf = P.B200ReplayBuffer(capacity, rng="python")
    A, pre = int(fx["n_actions"]), int(fx["prefill"])
    space = Space(A)
    random.setstate((3, tuple(int(x) for x in fx["rng_before"]), None))

    def push(i):
        buf.push(torch.from_numpy(fx["push_state"][i]), int(fx["push_action"][i]), float(fx["push_reward"][i]), True, False,
                 next_state=None, max_number_actions=A)

    for i in range(pre):
        push(i)
    preds, calls, chosen, idx = [], [], [], []
    for c in range(len(fx["call_A"])):
        if c:
            if act:
                chosen.append(int(lb.act(torch.from_numpy(fx["act_state"][c - 1]), space).reshape(-1)[0]))
            push(pre + c - 1)
        tr = {}
        rep = lb.learn(buf, trace=tr)
        idx.append(tr["idx"])
        preds += [p.cpu().numpy().ravel() for p in rep["prediction"]]
        calls.append(dict(state_of(lb), last=lb.last_sum_weight_when_discounted, launches=tr["launches"]))
    return lb, buf, np.concatenate(preds), calls, chosen, idx


@pytest.mark.parametrize("graph", [True, False])
@pytest.mark.parametrize("name", ["cb_lin_method", "cb_lin_binary"])
def test_agent_loop_matches_the_recording(name, graph):
    fx = load(name)
    lb, buf, preds, calls, chosen, idx = run_method(fx, graph=graph)
    flat = np.concatenate([i.numpy().ravel() for i in idx])
    assert np.array_equal(flat, fx["idx"]), "sampled indices differ from the reference"
    assert np.array_equal(np.asarray(random.getstate()[1], np.uint64).astype(np.uint32), fx["rng_after"])
    assert chosen == fx["act_chosen"].tolist()
    o = 0
    for r, n in enumerate(fx["idx_len"]):
        close_normwise(preds[o:o + n], fx["pred"][o:o + n], f"prediction of round {r}")
        o += n
    for c, s in enumerate(calls):
        close_state(s, fx, c, name)
        assert s["last"] == fx["call_last"][c]
        assert s["launches"] == 5 * int(fx["rounds"])


def test_wrapping_ring_matches_the_oracle():
    fx = load("cb_lin_method")
    cap = 100
    lb, buf, preds, calls, _, idx = run_method(fx, capacity=cap, act=False)
    feats = act_features(fx)
    X = np.concatenate([fx["push_state"], feats[fx["push_action"]]], axis=1)
    r = bo.Ridge(X.shape[1] + 1, float(fx["l2_reg_lambda"]), float(fx["gamma"]), float(fx["interval"]))
    pre, o, got = int(fx["prefill"]), 0, []
    for c, ic in enumerate(idx):
        n_pushed = pre + c
        first = max(0, n_pushed - cap)           # logical index 0 = the oldest transition still stored
        for row in ic.numpy():
            got.append(r.round(torch.from_numpy(X[first + row]), torch.from_numpy(fx["push_reward"][first + row])).numpy().ravel())
        close_state({k: v for k, v in calls[c].items() if k not in ("last", "launches")},
                    {f"call_{k}": [getattr(r, k).numpy()] * (c + 1) for k in ("A", "b", "sum_weight", "inv_A", "coefs")}, c, "wrap")
    close_normwise(preds, np.concatenate(got))


def test_learn_batch_matches_the_recording():
    import pearl_b200 as P
    fx = load("cb_lin_batch")
    torch.cuda.set_device(0)
    lb = P.B200LinearBandit(feature_dim=int(fx["obs"]) + int(fx["act_dim"]), l2_reg_lambda=float(fx["l2_reg_lambda"]),
                            gamma=float(fx["gamma"]), apply_discounting_interval=float(fx["interval"]), batch_size=int(fx["batch"]),
                            initial_coefs=torch.from_numpy(fx["initial_coefs"])).to(DEV)
    for c in range(len(fx["pred"])):
        w = torch.from_numpy(fx["b_weight"][c]).to(DEV) if fx["b_has_weight"][c] else None
        rep = lb.learn_batch(P.TransitionBatch(state=torch.from_numpy(fx["b_state"][c]).to(DEV),
                                               action=torch.from_numpy(fx["b_action"][c]).to(DEV),
                                               reward=torch.from_numpy(fx["b_reward"][c]).to(DEV), weight=w))
        close_normwise(rep["prediction"].cpu().numpy().ravel(), fx["pred"][c])
        close_state(state_of(lb), fx, c, "learn_batch")
        assert lb.last_sum_weight_when_discounted == fx["call_last"][c]
        assert rep["weight"].shape == rep["label"].shape


def scored_learner(fx, alpha):
    import pearl_b200 as P
    torch.cuda.set_device(0)
    A = int(fx["n_actions"])
    lb = P.B200LinearBandit(feature_dim=int(fx["obs"]) + A, exploration_module=P.UCBExploration(alpha),
                            action_representation_module=P.OneHotActionTensorRepresentationModule(A)).to(DEV)
    lb.load_state_dict({f"model.{k}": torch.from_numpy(np.asarray(fx[k[1:]])) for k in ("_A", "_b", "_sum_weight", "_inv_A", "_coefs")})
    return lb, Space(A)


def test_scores_and_act_match_the_recording():
    fx = load("cb_lin_scores")
    lb, space = scored_learner(fx, float(fx["alpha"]))
    states = torch.from_numpy(fx["states"]).to(DEV)
    close_normwise(lb.get_scores(states, space).cpu().numpy(), fx["ucb"])
    close_normwise(lb.get_scores(states, space, exploit=True).cpu().numpy(), fx["exploit"])
    mask = torch.from_numpy(fx["mask"]).to(DEV)
    assert lb.act(states, space, action_availability_mask=mask).reshape(-1).cpu().tolist() == fx["act_mask"].tolist()
    assert lb.act(states, space).reshape(-1).cpu().tolist() == fx["act_all"].tolist()
    assert lb.get_scores(states[0], space).shape == (1, int(fx["n_actions"]))
    lb0, _ = scored_learner(fx, 0.0)
    close_normwise(lb0.get_scores(states, space).cpu().numpy(), fx["ucb0"])
    assert lb0.act(states, space, action_availability_mask=mask).reshape(-1).cpu().tolist() == fx["act0"].tolist()


def test_checkpoint_views_and_load_pick_up():
    fx = load("cb_lin_method")
    lb, buf, _, _, _, _ = run_method(fx, act=False)
    sd = {k: v.clone() for k, v in lb.state_dict().items()}
    assert sd["model._A"].device.type == "cuda"
    assert sd["model._A"].data_ptr() != lb.model._A.data_ptr()
    lb2, _, _, _, _, _ = run_method(fx, act=False)
    lb2.load_state_dict(sd)
    random.seed(3)
    lb.learn(buf)
    random.seed(3)
    lb2.learn(buf)
    for k in sd:
        assert torch.equal(lb.state_dict()[k], lb2.state_dict()[k]), k


def stress(seed=0, obs=119, A=8, B=256, rounds=6):
    g = torch.Generator().manual_seed(seed)
    s = torch.randn(4096, obs, generator=g)
    a = torch.randint(0, A, (4096,), generator=g)
    r = s[:, 0] + 0.1 * a + 0.1 * torch.randn(4096, generator=g)
    return s, a, r, dict(obs=obs, A=A, B=B, rounds=rounds)


def run_stress(graph=True, max_rounds=1024, calls=3, seed=0):
    import pearl_b200 as P
    torch.cuda.set_device(0)
    s, a, r, c = stress(seed)
    lb = P.B200LinearBandit(feature_dim=c["obs"] + c["A"], exploration_module=P.UCBExploration(1.0), gamma=0.9,
                            apply_discounting_interval=2000.0, training_rounds=c["rounds"], batch_size=c["B"],
                            action_representation_module=P.OneHotActionTensorRepresentationModule(c["A"]),
                            max_rounds_per_call=max_rounds)
    lb.use_cuda_graph = graph
    buf = P.B200ReplayBuffer(10000, rng="device")
    buf.push_batch(s, a, r, None, torch.ones(4096, dtype=torch.bool), torch.zeros(4096, dtype=torch.bool), max_number_actions=c["A"])
    buf.seed(seed)
    out, idx = [], []
    for _ in range(calls):
        tr = {}
        rep = lb.learn(buf, trace=tr)
        out.append(torch.stack(rep["prediction"]).cpu())
        idx.append(tr["idx"])
    return lb, torch.cat(out), torch.cat(idx), (s, a, r, c)


def test_stress_shape_matches_the_oracle():
    lb, preds, idx, (s, a, r, c) = run_stress()
    X = torch.cat([s, torch.eye(c["A"])[a]], dim=1)
    o = bo.Ridge(X.shape[1] + 1, 1.0, 0.9, 2000.0)
    want = torch.stack([o.round(X[row.long()], r[row.long()]) for row in idx])
    for k in range(len(idx)):
        close_normwise(preds[k].numpy(), want[k].numpy(), f"round {k}")
    for k in ("A", "b", "sum_weight"):
        np.testing.assert_allclose(getattr(lb.model, f"_{k}").cpu().numpy(), getattr(o, k).numpy(), rtol=1e-4, atol=2e-6 * 256)
    assert lb.last_sum_weight_when_discounted == o.last and o.last > 0
    inv64, coefs64, cond = bo.fp64_yardstick(lb.model._A.cpu(), lb.model._b.cpu(), 1.0)
    bound = 4 * 128 * (2.0 ** -24 + cond * 2.0 ** -53)        # as test_gpu_bandit_shapes.py explains
    assert np.abs(lb.model._inv_A.cpu().double() - inv64).max() <= bound * inv64.abs().max()
    assert np.abs(lb.model._coefs.cpu().double() - coefs64).max() <= bound * coefs64.abs().max()


def test_bit_identity_run_to_run_graph_eager_and_chunking():
    ref, p0, i0, _ = run_stress()
    for kw in (dict(), dict(graph=False), dict(max_rounds=1), dict(max_rounds=4)):
        lb, p, i, _ = run_stress(**kw)
        assert torch.equal(i, i0), kw
        assert torch.equal(p, p0), kw
        for k, v in ref.state_dict().items():
            assert torch.equal(lb.state_dict()[k], v), (kw, k)
        assert lb.last_sum_weight_when_discounted == ref.last_sum_weight_when_discounted


def test_refusals():
    import pearl_b200 as P
    fx = load("cb_lin_scores")
    lb, space = scored_learner(fx, 1.0)
    st = torch.from_numpy(fx["states"]).to(DEV)
    lb.exploration_module.randomized_tiebreaking = P._compat.TiebreakingStrategy.PER_ROW_TIEBREAKING
    with pytest.raises(NotImplementedError, match="tie-breaking"):
        lb.act(st, space)
    lb.exploration_module = object()
    with pytest.raises(NotImplementedError, match="UCBExploration"):
        lb.get_scores(st, space)
    lb.get_scores(st, space, exploit=True)                    # values only: no exploration module needed
    ident = P.B200LinearBandit(feature_dim=13)
    buf = P.B200ReplayBuffer(100)
    buf.push(torch.zeros(12), 0, 1.0, True, False, max_number_actions=4)
    with pytest.raises(NotImplementedError, match="one-hot or binary"):
        ident.learn(buf)
    per = P.B200PrioritizedReplayBuffer(100)
    with pytest.raises(NotImplementedError, match="Prioritized"):
        lb.learn(per)
    lb2, _ = scored_learner(fx, 1.0)
    x = torch.zeros(4, 19, device=DEV)
    with pytest.raises(NotImplementedError, match="negative weights"):
        lb2.learn_batch(P.TransitionBatch(state=x[:, :12], action=x[:, 12:], reward=torch.zeros(4, device=DEV),
                                          weight=torch.tensor([1.0, -0.5, 1.0, 1.0], device=DEV)))
    lb.set_history_summarization_module(torch.nn.Linear(2, 2))
    with pytest.raises(NotImplementedError, match="history summarization"):
        lb.learn_batch(P.TransitionBatch(state=st[:4], action=torch.zeros(4, 7, device=DEV), reward=torch.zeros(4, device=DEV)))
