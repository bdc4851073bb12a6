"""GPU checks of B200NeuralBandit (csrc/neural_bandit.cu) against the reference's recordings (tests/golden/cb_nb_*.npz) and
itself: the SquareCB and FastCB agent loops with graphs on and off (the same actions, and torch's CPU generator and
CPython's `random` in the recorded states afterwards), learn_batch with weights of both signs, an lr change and a
checkpoint round trip, scores and greedy act with masks, bit-identity run to run, graph vs eager and across round
chunking, the launch and capture counts, the action-choice kernel against a float64 restatement, and the refusals.
Parameters are held with tests/_tol.py's close_params and the AdamW moments with close_adam_state."""
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

from _tol import close_params  # noqa: E402
from test_bandit_oracle import close_normwise, load  # noqa: E402
from test_neural_linear_bandit import close_adam_state  # noqa: E402
from test_neural_bandit_oracle import AGENTS, agent  # noqa: E402

pytestmark = pytest.mark.gpu

DEV = "cuda:0"


class Space:
    def __init__(self, n):
        self.n = n
        self.actions = [torch.tensor([i]) for i in range(n)]
        self.actions_batch = torch.arange(n).view(n, 1)


def load_flat(nb, vec):
    off = 0
    with torch.no_grad():
        for p in nb.model.parameters():
            n = p.numel()
            p.copy_(torch.from_numpy(np.asarray(vec[off:off + n])).view(p.shape))
            off += n
    assert off == len(vec)


def flat_of(nb):
    return torch.cat([p.detach().reshape(-1) for p in nb.model.parameters()]).cpu().numpy()


def adam_of(nb):
    st = nb.optimizer.state
    used = [p for p in nb.model.parameters() if p in st]
    return {k: torch.cat([st[p][k].reshape(-1) for p in used]).cpu().numpy()
            for k in ("exp_avg", "exp_avg_sq", "max_exp_avg_sq")}, float(st[used[0]]["step"])


def check_call(nb, g, c, what, lr, steps, prefix="call_"):
    close_params(flat_of(nb), g[prefix + "params"][c], f"{what}: parameters after call {c}", lr, steps)
    st, step = adam_of(nb)
    assert step == float(g[prefix + "adam_step"][c]), (what, c, step)
    for k, r in (("exp_avg", "adam_m"), ("exp_avg_sq", "adam_v"), ("max_exp_avg_sq", "adam_vmax")):
        close_adam_state(st[k], g[prefix + r][c], f"{what}: {k} after call {c}")


def explorer_of(fx):
    import pearl_b200 as P
    if bool(fx["fastcb"]):
        return P.FastCBExploration(gamma=float(fx["gamma"]), reward_lb=float(fx["reward_lb"]), reward_ub=float(fx["reward_ub"]))
    return P.SquareCBExploration(gamma=float(fx["gamma"]), reward_lb=float(fx["reward_lb"]), reward_ub=float(fx["reward_ub"]),
                                 clamp_values=bool(fx["clamp"]))


def make_agent(fx, **kw):
    import pearl_b200 as P
    A = int(fx["n_actions"])
    mod = P.OneHotActionTensorRepresentationModule(A) if str(fx["rep"]) == "one_hot" else \
        P.BinaryActionTensorRepresentationModule(int(fx["act_dim"]))
    nb = P.B200NeuralBandit(feature_dim=int(fx["obs"]) + int(fx["act_dim"]), hidden_dims=[int(x) for x in fx["hidden"]],
                            exploration_module=explorer_of(fx), action_representation_module=mod,
                            training_rounds=int(fx["rounds"]), batch_size=int(fx["batch"]), learning_rate=float(fx["lr"]),
                            loss_type=str(fx["loss"]), **kw)
    load_flat(nb, fx["init"])
    return nb


def run_agent(fx, graph=True, act=True, calls=None, **kw):
    import pearl_b200 as P
    torch.cuda.set_device(0)
    nb = make_agent(fx, **kw)
    nb.use_cuda_graph = graph
    buf = P.B200ReplayBuffer(100000, rng="python")
    A, pre = int(fx["n_actions"]), int(fx["prefill"])
    space = Space(A)
    random.setstate((3, tuple(int(x) for x in fx["rng_before"]), None))

    def push(i):
        buf.push(torch.from_numpy(fx["push_state"][i]), int(fx["push_action"][i]), float(fx["push_reward"][i]), True, False,
                 next_state=None, max_number_actions=A)

    for i in range(pre):
        push(i)
    out = dict(pred=[], loss=[], chosen=[], prob=[], idx=[], launches=[])
    for c in range(len(fx["call_params"]) if calls is None else calls):
        if c:
            if act:
                if c == 1:
                    torch.set_rng_state(torch.from_numpy(fx["torch_before"]))
                a = nb.act(torch.from_numpy(fx["act_state"][c - 1]), space)
                assert a.dtype == torch.int32 and a.dim() == 0 and a.device.type == "cpu"
                out["chosen"].append(int(a))
                out["prob"].append(nb._nb["prob"][:A].cpu().numpy())
            push(pre + c - 1)
        tr = {}
        rep = nb.learn(buf, trace=tr)
        out["idx"].append(tr["idx"])
        out["launches"].append(tr["launches"])
        out["pred"] += [p.cpu().numpy().ravel() for p in rep["prediction"]]
        out["loss"] += [float(x) for x in rep["loss"]]
        yield nb, c, out


@pytest.mark.parametrize("graph", [True, False])
@pytest.mark.parametrize("name,prefix", AGENTS)
def test_agent_loop_matches_the_recording(name, prefix, graph):
    fx = agent(name, prefix)
    R = int(fx["rounds"])
    for nb, c, out in run_agent(fx, graph=graph):
        check_call(nb, fx, c, name + prefix, float(fx["lr"]), R * (c + 1))
        assert out["launches"][-1] % R == 0
    assert out["chosen"] == fx["act_chosen"].tolist()
    assert np.array_equal(torch.get_rng_state().numpy(), fx["torch_after"]), "torch's CPU generator left the reference's stream"
    assert np.array_equal(np.asarray(random.getstate()[1], np.uint64).astype(np.uint32), fx["rng_after"])
    flat = np.concatenate([i.numpy().ravel() for i in out["idx"]])
    assert np.array_equal(flat, fx["idx"]), "sampled indices differ from the reference"
    for k, p in enumerate(out["prob"]):
        np.testing.assert_allclose(p, fx["act_pn"][k], rtol=1e-4, atol=1e-7, err_msg=f"probabilities of act {k}")
    o = 0
    for r, n in enumerate(fx["idx_len"]):
        close_normwise(out["pred"][r], fx["pred"][o:o + n], f"prediction of round {r}")
        o += n
    np.testing.assert_allclose(out["loss"], fx["losses"], rtol=1e-4, atol=1e-6)


@pytest.mark.parametrize("graph", [True, False])
@pytest.mark.parametrize("loss", ["mse", "mae"])
def test_learn_batch_matches_the_recording(loss, graph):
    import pearl_b200 as P
    fx = load("cb_nb_batch")
    torch.cuda.set_device(0)
    nb = P.B200NeuralBandit(feature_dim=int(fx["obs"]) + int(fx["act_dim"]), hidden_dims=[int(x) for x in fx["hidden"]],
                            exploration_module=P.NoExploration(), batch_size=int(fx["batch"]), learning_rate=float(fx["lr0"]),
                            loss_type=loss)
    nb.use_cuda_graph = graph
    load_flat(nb, fx[f"{loss}_init"])
    for c in range(int(fx["calls"])):
        if c == int(fx["lr_change_at"]):
            for g in nb.optimizer.param_groups:
                g["lr"] = float(fx["lr1"])
        if c == int(fx["reload_at"]):
            nb.load_state_dict({k: v.clone() for k, v in nb.state_dict().items()})
            nb.optimizer.load_state_dict(nb.optimizer.state_dict())
        b = lambda k: torch.from_numpy(fx[f"{loss}_b_{k}"][c]).to(DEV)  # noqa: E731
        before = (nb._nb["handle"].value, int(nb._nb["lib"].prl_nb_graph_captures(nb._nb["handle"]))) if c else None
        rep = nb.learn_batch(P.TransitionBatch(state=b("state"), action=b("action"), reward=b("reward"), weight=b("weight")))
        if c in (int(fx["lr_change_at"]), int(fx["reload_at"])):     # the new lr and the reloaded state reach the captured round
            assert (nb._nb["handle"].value, int(nb._nb["lib"].prl_nb_graph_captures(nb._nb["handle"]))) == before
        close_normwise(rep["prediction"].cpu().numpy().ravel(), fx[f"{loss}_pred"][c], f"{loss} prediction of call {c}")
        np.testing.assert_allclose(float(rep["loss"]), fx[f"{loss}_loss"][c], rtol=1e-4, atol=1e-6)
        check_call(nb, fx, c, f"learn_batch {loss}", float(fx["lr1"]), c + 1, prefix=f"{loss}_call_")


def test_a_zero_weight_sum_gives_torchs_nan_and_takes_the_step():
    import pearl_b200 as P
    torch.cuda.set_device(0)
    nb = P.B200NeuralBandit(feature_dim=4, hidden_dims=[8, 4], exploration_module=P.NoExploration(), state_features_only=True)
    x = torch.randn(16, 4, device=DEV)
    rep = nb.learn_batch(P.TransitionBatch(state=x, action=x[:, :0], reward=torch.randn(16, device=DEV),
                                           weight=torch.zeros(16, device=DEV)))
    assert np.isnan(float(rep["loss"]))
    assert nb._nb["lib"].prl_nb_adam_step(nb._nb["handle"]) == 1


def test_scores_and_greedy_act_match_the_recording():
    import pearl_b200 as P
    fx = load("cb_nb_scores")
    torch.cuda.set_device(0)
    A = int(fx["n_actions"])
    nb = P.B200NeuralBandit(feature_dim=int(fx["obs"]), hidden_dims=[int(x) for x in fx["hidden"]],
                            exploration_module=P.NoExploration(), state_features_only=True,
                            action_representation_module=P.OneHotActionTensorRepresentationModule(A)).to(DEV)
    load_flat(nb, fx["params"])
    space = Space(A)
    states = torch.from_numpy(fx["states"]).to(DEV)
    close_normwise(nb.get_scores(states, space).cpu().numpy(), fx["scores"])
    one = nb.get_scores(states[0], space)
    assert one.shape == (1, A)
    close_normwise(one.cpu().numpy(), fx["scores_one"])
    mask = torch.from_numpy(fx["mask"]).to(DEV)
    assert nb.act(states, space).reshape(-1).cpu().tolist() == fx["act_all"].tolist()
    assert nb.act(states, space, action_availability_mask=mask).reshape(-1).cpu().tolist() == fx["act_mask"].tolist()
    with pytest.raises(AssertionError):
        nb.get_scores(states, space, exploit=True)
    assert sorted(nb.state_dict().keys()) == sorted(fx["keys"].tolist())


def test_scores_in_chunks_match_one_pass():
    import pearl_b200 as P
    fx = agent("cb_nb_squarecb", "")
    torch.cuda.set_device(0)
    nb = make_agent(fx).to(DEV)
    space = Space(int(fx["n_actions"]))
    g = torch.Generator().manual_seed(5)
    states = torch.randn(P.neural_bandit.SCORE_ROWS // 13 + 7, int(fx["obs"]), generator=g).to(DEV)
    whole = nb.get_scores(states, space)
    parts = torch.cat([nb.get_scores(states[i:i + 50], space) for i in range(0, states.shape[0], 50)])
    close_normwise(parts.cpu().numpy(), whole.cpu().numpy(), "chunked scores")
    nb.exploration_module = P.NoExploration()
    greedy = nb.act(states, space).reshape(-1)
    assert torch.equal(greedy.cpu(), whole.argmax(1).cpu().to(greedy.dtype))


def run_stress(graph=True, max_rounds=1024, calls=3):
    fx = agent("cb_nb_fastcb", "")
    out = None
    for nb, c, out in run_agent(fx, graph=graph, act=False, calls=calls, max_rounds_per_call=max_rounds):
        pass
    return nb, torch.tensor(np.stack(out["pred"])), out


def test_bit_identity_run_to_run_graph_eager_and_chunking():
    ref, p0, o0 = run_stress()
    for kw in (dict(), dict(graph=False), dict(max_rounds=1), dict(max_rounds=3)):
        nb, p, o = run_stress(**kw)
        assert torch.equal(p, p0), kw
        assert o["loss"] == o0["loss"], kw
        for k, v in ref.state_dict().items():
            assert torch.equal(nb.state_dict()[k], v), (kw, k)
        for a, b in zip(adam_of(nb)[0].values(), adam_of(ref)[0].values()):
            assert np.array_equal(a, b), kw


def test_launch_and_capture_counts():
    import pearl_b200 as P
    torch.cuda.set_device(0)
    nb = P.B200NeuralBandit(feature_dim=8, hidden_dims=[16, 8], exploration_module=P.NoExploration(), batch_size=32,
                            state_features_only=True)
    x = torch.randn(32, 8, device=DEV)
    b = P.TransitionBatch(state=x, action=x[:, :0], reward=torch.randn(32, device=DEV), weight=torch.ones(32, device=DEV))
    nb.learn_batch(b)
    # load, 3 forward contractions, head, 4 backward contractions + k_head_bwd, AdamW, the round counter
    assert int(nb._nb["lib"].prl_nb_last_launches(nb._nb["handle"])) == 1 + 3 + 1 + 5 + 1 + 1
    for lr in (0.01, 0.02):
        nb.optimizer.param_groups[0]["lr"] = lr
        nb.learn_batch(b)
    assert int(nb._nb["lib"].prl_nb_graph_captures(nb._nb["handle"])) == 1
    buf = P.B200ReplayBuffer(1000, rng="device")
    s = torch.randn(200, 8)
    buf.push_batch(s, torch.randint(0, 4, (200,)), s[:, 0], None, torch.ones(200, dtype=torch.bool),
                   torch.zeros(200, dtype=torch.bool), max_number_actions=4)
    buf.seed(3)
    nb.learn(buf)           # learn folds action ids: a handle for the buffer's layout, which learn_batch then shares
    h = nb._nb["handle"].value
    for _ in range(2):
        nb.learn_batch(b)
        nb.learn(buf)
    assert nb._nb["handle"].value == h and int(nb._nb["lib"].prl_nb_graph_captures(h)) == 2
    assert int(nb._nb["lib"].prl_nb_adam_step(h)) == 3 + 3 * 100 + 2


def explore64(v, E, kind, gamma, lb, ub, clamp):
    """float64 restatement of k_nb_explore on fp32 inputs (gamma, lb, ub rounded to fp32 first): (pn, the choice, the
    choice)."""
    f = lambda x: float(np.float32(x))  # noqa: E731
    v = v.astype(np.float64)
    g, lb, ub = f(gamma), f(lb), f(ub)
    if clamp or kind == 2:
        v = np.clip(v, lb, ub)
    im = int(np.argmax(v))
    mx, A = v[im], v.size
    gap = mx - v
    if kind == 1:
        p = 1.0 / (A + g * gap)
    elif mx <= lb:
        p = np.full(A, 1.0 / A)
    else:
        p = (mx - lb) / (A * (mx - lb) + g * gap)
    p[im] = 0.0
    p[im] = 1.0 - p.sum()
    pn = p / p.sum()
    return pn, im, int(np.argmax(pn / E.astype(np.float64)))


def test_explore_kernel_against_float64():
    from pearl_b200 import _lib
    lib = _lib.init(0)
    torch.cuda.set_device(0)
    g = np.random.default_rng(11)
    checked = decided = 0
    for case in range(400):
        A = [1, 2, 3, 7, 26, 255, 256, 257, 1000, 4096][case % 10]
        kind = 1 + (case // 10) % 2
        clamp = bool((case // 20) % 2)
        style = (case // 40) % 5
        v = g.standard_normal(A).astype(np.float32) * [1.0, 0.05, 3.0, 1.0, 1.0][style]
        if style == 3:
            v[g.integers(0, A, size=max(1, A // 4))] = v.max()      # ties at the maximum
        if style == 4:
            v = np.minimum(v, -2.0).astype(np.float32)               # every value below lb: FastCB's uniform branch
        gamma = float([5.0, 4582.6, 0.3, 100.0][case % 4])
        lb, ub = -0.5, 0.75
        E = g.exponential(size=A).astype(np.float32)
        vd, Ed = torch.from_numpy(v).to(DEV), torch.from_numpy(E).to(DEV)
        prob, idx = torch.empty(A, device=DEV), torch.empty(1, dtype=torch.int32, device=DEV)
        _lib.check(lib.prl_nb_explore(A, _lib.ptr(vd), kind, gamma, lb, ub, int(clamp), _lib.ptr(Ed), _lib.ptr(prob), _lib.ptr(idx),
                                      None))
        pn, im, a = explore64(v, E, kind, gamma, lb, ub, clamp)
        got = prob.cpu().numpy()
        # the fp32 chain: four roundings per element, and two sums of A terms (A / 256 in sequence per thread, then a
        # tree of 8 levels); p[max] = 1 - the others' sum carries that sum's absolute error
        u, depth = 2.0 ** -24, -(-A // 256) + 8
        tol = 2 * ((4 + depth) * u * pn + (depth + 2) * u * (np.arange(A) == im))
        assert (np.abs(got - pn) <= tol).all(), (case, A, kind, float((np.abs(got - pn) / tol).max()))
        # the choice is the first maximum of fp32(pn) / E over the kernel's own probabilities
        q32 = got / E
        assert int(idx.item()) == int(np.argmax(q32)), (case, A, kind)
        # and the float64 rule's choice wherever the probabilities' tolerance cannot reorder the two best
        r = tol / np.maximum(pn, 1e-300)
        q = pn / E.astype(np.float64)
        top = np.argsort(q)[::-1][:2]
        if A == 1 or q[top[0]] - q[top[1]] > (r[top[0]] + r[top[1]] + 1e-6) * q[top[0]]:
            assert int(idx.item()) == a, (case, A, kind, clamp, style)
            decided += 1
        checked += 1
    print(f"    {decided} of {checked} choices held to the float64 rule")
    assert checked == 400 and decided > 200


def test_call_time_refusals():
    import pearl_b200 as P
    torch.cuda.set_device(0)
    nb = P.B200NeuralBandit(feature_dim=6, hidden_dims=[8, 4], exploration_module=P.SquareCBExploration(gamma=5.0),
                            state_features_only=True)
    x = torch.zeros(3, 6, device=DEV)
    rng = torch.get_rng_state()
    with pytest.raises(NotImplementedError, match="more than one state"):
        nb.act(x, Space(3))
    assert torch.equal(torch.get_rng_state(), rng)          # a refused act draws nothing
    nb.exploration_module = P.UCBExploration(1.0)
    with pytest.raises(NotImplementedError, match="SquareCBExploration"):
        nb.act(x[0], Space(3))
    nb.exploration_module = P.NoExploration(randomized_tiebreaking=True)
    with pytest.raises(NotImplementedError, match="tie-breaking"):
        nb.act(x, Space(3))
    with pytest.raises(NotImplementedError, match="Prioritized"):
        nb.learn(P.B200PrioritizedReplayBuffer(100))
    nb.loss_type = P.LossType.CROSS_ENTROPY
    with pytest.raises(NotImplementedError, match="MSE and MAE"):
        nb.learn_batch(P.TransitionBatch(state=x, action=x[:, :0], reward=torch.zeros(3, device=DEV)))
    nb.loss_type = P.LossType.MSE
    nb._optimizer = torch.optim.Adam(nb.model.parameters())
    with pytest.raises(NotImplementedError, match="AdamW"):
        nb.learn_batch(P.TransitionBatch(state=x, action=x[:, :0], reward=torch.zeros(3, device=DEV)))
