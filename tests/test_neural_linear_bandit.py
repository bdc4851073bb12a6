"""GPU checks of B200NeuralLinearBandit (csrc/neural_linear.cu) against the reference's recordings
(tests/golden/cb_nl_*.npz) and itself: the agent loop with graphs on and off, learn_batch with weights (MAE and cross
entropy, an all-zero-weight call, an lr change and a load_state_dict round trip), scores and act with masks, bit-identity
run to run, graph vs eager and across round chunking, the launch count of both round variants, checkpoint views and the
refusals.  Ridge sums are held elementwise to 1e-4 and inv_A and the predictions normwise, as test_bandit.py does; the
coefs by their backward error in the reference's system (coefs_backward_error); parameters with tests/_tol.py's
close_params, and all three AdamW moments with close_adam_state."""
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


def load_flat(nl, vec):
    off = 0
    with torch.no_grad():
        for p in nl.model.parameters():
            n = p.numel()
            p.copy_(torch.from_numpy(np.asarray(vec[off:off + n])).view(p.shape))
            off += n
    assert off == len(vec)


def flat_of(nl):
    return torch.cat([p.detach().reshape(-1) for p in nl.model.parameters()]).cpu().numpy()


def adam_of(nl):
    st = nl.optimizer.state
    used = [p for p in nl.model.parameters() if p in st]
    return {k: torch.cat([st[p][k].reshape(-1) for p in used]).cpu().numpy()
            for k in ("exp_avg", "exp_avg_sq", "max_exp_avg_sq")}, float(st[used[0]]["step"]), len(used)


def ridge_of(nl):
    m = nl.model._linear_regression_layer
    return dict(A=m._A.cpu().numpy(), b=m._b.cpu().numpy(), sum_weight=m._sum_weight.cpu().numpy(), inv_A=m._inv_A.cpu().numpy(),
                coefs=m._coefs.cpu().numpy())


def check_call(nl, fx, c, what, lr, rounds, prefix="call_"):
    g = {k[len(prefix):]: fx[k] for k in fx.files if k.startswith(prefix)}
    got = ridge_of(nl)
    for k in ("A", "b", "sum_weight"):
        np.testing.assert_allclose(got[k], g[k][c], rtol=1e-4, atol=1e-5 * max(1.0, np.abs(g[k][c]).max()), err_msg=f"{what}: {k} after call {c}")
    close_normwise(got["inv_A"], g["inv_A"][c], f"{what}: inv_A after call {c}")
    coefs_backward_error(got["coefs"], g["A"][c], g["b"][c], float(fx["l2_reg_lambda"]), f"{what}: coefs after call {c}")
    close_params(flat_of(nl), g["params"][c], f"{what}: parameters after call {c}", lr, rounds)
    st, step, n = adam_of(nl)
    assert n == int(g["adam_n_state"][c]) and step == float(g["adam_step"][c]), (what, c, n, step)
    for k, r in (("exp_avg", "adam_m"), ("exp_avg_sq", "adam_v"), ("max_exp_avg_sq", "adam_vmax")):
        close_adam_state(st[k], g[r][c], f"{what}: {k} after call {c}")
    # unit weights sum exactly; the recorded learn_batch weights are fractional, and their fixed-order sum may differ
    # from torch's in the last place
    np.testing.assert_allclose(nl.last_sum_weight_when_discounted, float(g["last"][c]), rtol=1e-6 if prefix != "call_" else 0)


def close_adam_state(got, want, what):
    """AdamW moments elementwise to 1e-4, with an absolute floor of 1e-4 of the vector's largest magnitude: a moment is a
    running average of gradients, and an element whose gradients cancel to near zero keeps only the absolute error of
    the sums that made it."""
    got, want = np.asarray(got, np.float64), np.asarray(want, np.float64)
    err, bound = np.abs(got - want), 1e-4 * np.abs(want) + 1e-4 * np.abs(want).max()
    assert (err <= bound).all(), f"{what}: {int((err > bound).sum())} of {got.size} elements beyond 1e-4 (worst {(err / bound).max():.3g} x bound)"


def coefs_backward_error(c_got, A_ref, b_ref, lam, what):
    """The network's output rows, and so A and b, agree with the reference's to about 1e-4 elementwise, and coefs =
    inv(A + lambda I) b magnifies such input differences by up to cond(A + lambda I) (<= 1e4 in the recordings).  So the
    coefs are held by their backward error: they solve the reference's own system to within 1e-4 of its scale."""
    M = A_ref.astype(np.float64) + lam * np.eye(A_ref.shape[0])
    r = M @ np.asarray(c_got, np.float64) - b_ref.astype(np.float64)
    scale = np.abs(M).sum(1).max() * np.abs(c_got).max() + np.abs(b_ref).max()
    assert np.abs(r).max() <= 1e-4 * scale, f"{what}: residual {np.abs(r).max():.3e} > 1e-4 x {scale:.3e}"


def make_agent(fx, **kw):
    import pearl_b200 as P
    h = [int(x) for x in fx["hidden"]]
    nl = P.B200NeuralLinearBandit(feature_dim=int(fx["obs"]) + int(fx["act_dim"]), hidden_dims=h,
                                  exploration_module=P.UCBExploration(float(fx["alpha"])), action_representation_module=module_of(fx),
                                  training_rounds=int(fx["rounds"]), batch_size=int(fx["batch"]), learning_rate=float(fx["lr"]),
                                  l2_reg_lambda_linear=float(fx["l2_reg_lambda"]), gamma=float(fx["gamma"]),
                                  apply_discounting_interval=float(fx["interval"]), state_features_only=False,
                                  use_skip_connections=bool(fx["skip"]), nn_e2e=bool(fx["e2e"]), **kw)
    load_flat(nl, fx["init"])
    return nl


def run_agent(fx, graph=True, act=True, calls=None, **kw):
    import pearl_b200 as P
    torch.cuda.set_device(0)
    nl = make_agent(fx, **kw)
    nl.use_cuda_graph = graph
    buf = P.B200ReplayBuffer(100000, rng="python")
    A, pre = int(fx["n_actions"]), int(fx["prefill"])
    space = Space(A)
    random.setstate((3, tuple(int(x) for x in fx["rng_before"]), None))

    def push(i):
        buf.push(torch.from_numpy(fx["push_state"][i]), int(fx["push_action"][i]), float(fx["push_reward"][i]), True, False,
                 next_state=None, max_number_actions=A)

    for i in range(pre):
        push(i)
    out = dict(pred=[], loss=[], mu=[], chosen=[], idx=[], launches=[], snaps=[])
    for c in range(len(fx["call_A"]) if calls is None else calls):
        if c:
            if act:
                out["chosen"].append(int(nl.act(torch.from_numpy(fx["act_state"][c - 1]), space).reshape(-1)[0]))
            push(pre + c - 1)
        tr = {}
        rep = nl.learn(buf, trace=tr)
        out["idx"].append(tr["idx"])
        out["launches"].append(tr["launches"])
        out["pred"] += [p.cpu().numpy().ravel() for p in rep["prediction"]]
        out["loss"] += [float(x) for x in rep["loss"]]
        out["mu"] += [float(x) for x in rep["mu_scores"]]
        yield nl, c, out


@pytest.mark.parametrize("graph", [True, False])
@pytest.mark.parametrize("name", ["cb_nl_agent", "cb_nl_onehot"])
def test_agent_loop_matches_the_recording(name, graph):
    fx = load(name)
    R = int(fx["rounds"])
    for nl, c, out in run_agent(fx, graph=graph):
        check_call(nl, fx, c, name, float(fx["lr"]), R * (c + 1))
        assert out["launches"][-1] % R == 0
    flat = np.concatenate([i.numpy().ravel() for i in out["idx"]])
    assert np.array_equal(flat, fx["idx"]), "sampled indices differ from the reference"
    assert np.array_equal(np.asarray(random.getstate()[1], np.uint64).astype(np.uint32), fx["rng_after"])
    assert out["chosen"] == fx["act_chosen"].tolist()
    o = 0
    for r, n in enumerate(fx["idx_len"]):
        close_normwise(out["pred"][r], fx["pred"][o:o + n], f"prediction of round {r}")
        o += n
    np.testing.assert_allclose(out["loss"], fx["loss"], rtol=1e-4, atol=1e-6)
    np.testing.assert_allclose(out["mu"], fx["mu"], rtol=1e-4, atol=1e-6)


@pytest.mark.parametrize("graph", [True, False])
@pytest.mark.parametrize("tag", ["mae", "ce"])
def test_learn_batch_matches_the_recording(tag, graph):
    import pearl_b200 as P
    fx = load("cb_nl_batch")
    torch.cuda.set_device(0)
    loss, act = ("mae", "linear") if tag == "mae" else ("cross_entropy", "sigmoid")
    nl = P.B200NeuralLinearBandit(feature_dim=int(fx["obs"]) + int(fx["act_dim"]), hidden_dims=[int(x) for x in fx["hidden"]],
                                  batch_size=int(fx["batch"]), learning_rate=float(fx["lr0"]),
                                  l2_reg_lambda_linear=float(fx["l2_reg_lambda"]), gamma=float(fx["gamma"]),
                                  apply_discounting_interval=float(fx["interval"]), state_features_only=False, loss_type=loss,
                                  output_activation_name=act)
    nl.use_cuda_graph = graph
    load_flat(nl, fx[f"{tag}_init"])
    steps = 0
    for c in range(int(fx["calls"])):
        if c == int(fx["lr_change_at"]):
            for g in nl.optimizer.param_groups:
                g["lr"] = float(fx["lr1"])
        if c == int(fx["reload_at"]):
            nl.load_state_dict({k: v.clone() for k, v in nl.state_dict().items()})
        b = lambda k: torch.from_numpy(fx[f"{tag}_b_{k}"][c]).to(DEV)  # noqa: E731
        before = (nl._nl["handle"].value, int(nl._nl["lib"].prl_nlb_graph_captures(nl._nl["handle"]))) if c else None
        rep = nl.learn_batch(P.TransitionBatch(state=b("state"), action=b("action"), reward=b("reward"), weight=b("weight")))
        if c == int(fx["lr_change_at"]):      # the new lr (and the reloaded state) reach the captured round as it is
            assert (nl._nl["handle"].value, int(nl._nl["lib"].prl_nlb_graph_captures(nl._nl["handle"]))) == before
        close_normwise(rep["prediction"].cpu().numpy().ravel(), fx[f"{tag}_pred"][c], f"{tag} prediction of call {c}")
        np.testing.assert_allclose(float(rep["loss"]), fx[f"{tag}_loss"][c], rtol=1e-4, atol=1e-6)
        np.testing.assert_allclose(float(rep["mu_scores"]), fx[f"{tag}_mu"][c], rtol=1e-4, atol=1e-6)
        steps += c != int(fx["zero_at"])
        check_call(nl, fx, c, f"learn_batch {tag}", float(fx["lr1"]), max(steps, 1), prefix=f"{tag}_call_")
        if c == int(fx["zero_at"]):
            assert float(rep["loss"]) == 0.0
            assert nl._nl["lib"].prl_nlb_adam_step(nl._nl["handle"]) == c     # no optimizer step


def scored(fx):
    import pearl_b200 as P
    torch.cuda.set_device(0)
    A = int(fx["n_actions"])
    nl = P.B200NeuralLinearBandit(feature_dim=int(fx["obs"]), hidden_dims=[int(x) for x in fx["hidden"]],
                                  exploration_module=P.UCBExploration(float(fx["alpha"])),
                                  action_representation_module=P.OneHotActionTensorRepresentationModule(A),
                                  output_activation_name="sigmoid").to(DEV)
    load_flat(nl, fx["params"])
    lin = nl.model._linear_regression_layer
    for k in ("A", "b", "sum_weight", "inv_A", "coefs"):
        getattr(lin, f"_{k}").copy_(torch.from_numpy(np.asarray(fx[k])))
    return nl, Space(A)


def test_scores_and_act_match_the_recording():
    fx = load("cb_nl_scores")
    nl, space = scored(fx)
    states = torch.from_numpy(fx["states"]).to(DEV)
    close_normwise(nl.get_scores(states, space).cpu().numpy(), fx["ucb"])
    nl.separate_uncertainty = True
    close_normwise(nl.get_scores(states, space).cpu().numpy(), fx["ucb_sep"])
    nl.separate_uncertainty = False
    mask = torch.from_numpy(fx["mask"]).to(DEV)
    assert nl.act(states, space).reshape(-1).cpu().tolist() == fx["act_all"].tolist()
    assert nl.act(states, space, action_availability_mask=mask).reshape(-1).cpu().tolist() == fx["act_mask"].tolist()
    assert nl.get_scores(states[0], space).shape == (1, int(fx["n_actions"]))
    with pytest.raises(AssertionError):
        nl.get_scores(states, space, exploit=True)
    assert sorted(nl.state_dict().keys()) == sorted(fx["keys"].tolist())


def test_scores_in_chunks_match_one_pass():
    """More rows than one scoring chunk of the workspace: the chunks give the rows one pass would (to rounding: the
    contraction kernels chosen depend on the row count)."""
    import pearl_b200 as P
    fx = load("cb_nl_agent")
    torch.cuda.set_device(0)
    nl = make_agent(fx).to(DEV)
    space = Space(int(fx["n_actions"]))
    g = torch.Generator().manual_seed(5)
    states = torch.randn(P.neural_linear.SCORE_ROWS // 13 + 7, int(fx["obs"]), generator=g).to(DEV)
    whole = nl.get_scores(states, space)
    parts = torch.cat([nl.get_scores(states[i:i + 50], space) for i in range(0, states.shape[0], 50)])
    close_normwise(parts.cpu().numpy(), whole.cpu().numpy(), "chunked scores")


def run_stress(graph=True, max_rounds=1024, calls=3):
    fx = load("cb_nl_onehot")
    out = None
    for nl, c, out in run_agent(fx, graph=graph, act=False, calls=calls, max_rounds_per_call=max_rounds):
        pass
    return nl, torch.tensor(np.stack(out["pred"])), out


def test_bit_identity_run_to_run_graph_eager_and_chunking():
    ref, p0, o0 = run_stress()
    for kw in (dict(), dict(graph=False), dict(max_rounds=1), dict(max_rounds=3)):
        nl, p, o = run_stress(**kw)
        assert torch.equal(p, p0), kw
        assert o["loss"] == o0["loss"], kw
        for k, v in ref.state_dict().items():
            assert torch.equal(nl.state_dict()[k], v), (kw, k)
        for a, b in zip(adam_of(nl)[0].values(), adam_of(ref)[0].values()):
            assert np.array_equal(a, b), kw
        assert nl.last_sum_weight_when_discounted == ref.last_sum_weight_when_discounted


def test_launch_counts_of_both_variants():
    import pearl_b200 as P
    torch.cuda.set_device(0)
    for skip, h, e2e in ((False, [16, 8], True), (True, [8, 8], False)):
        nl = P.B200NeuralLinearBandit(feature_dim=8, hidden_dims=h, use_skip_connections=skip, nn_e2e=e2e, batch_size=32)
        x = torch.randn(32, 8, device=DEV)
        b = P.TransitionBatch(state=x, action=torch.zeros(32, 0, device=DEV), reward=torch.randn(32, device=DEV),
                              weight=torch.ones(32, device=DEV))
        nl.learn_batch(b)
        full = int(nl._nl["lib"].prl_nlb_last_launches(nl._nl["handle"]))
        b.weight = torch.zeros(32, device=DEV)
        nl.learn_batch(b)
        zero = int(nl._nl["lib"].prl_nlb_last_launches(nl._nl["handle"]))
        # load, 3 forward contractions (+ residual adds), rows, loss, ridge x 3; variant 0 adds grad, the backward and AdamW
        adds = (1 if skip and h[0] == h[1] else 0) + (1 if skip else 0) + (1 if skip and h[0] == 8 else 0)
        assert zero == 1 + 3 + adds + 2 + 3, (skip, zero)
        back = 5 + (2 if skip else 0) + (1 if e2e else 0)
        assert full == zero + 1 + back + 1, (skip, full, zero)
        assert nl.optimizer.state[next(nl.model.parameters())]["step"] == 1
        # both variants stay captured: alternating them replays, it does not capture again
        captures = int(nl._nl["lib"].prl_nlb_graph_captures(nl._nl["handle"]))
        for zero in (False, True, False):
            b.weight = torch.zeros(32, device=DEV) if zero else torch.ones(32, device=DEV)
            nl.learn_batch(b)
        assert int(nl._nl["lib"].prl_nlb_graph_captures(nl._nl["handle"])) == captures == 2


def test_learn_and_learn_batch_share_one_handle():
    """learn() folds action ids (a one-hot or binary representation); learn_batch and scoring read only the widths, so
    an agent that mixes them keeps one handle and its captured rounds."""
    import pearl_b200 as P
    torch.cuda.set_device(0)
    nl = P.B200NeuralLinearBandit(feature_dim=6 + 4, hidden_dims=[16, 8], state_features_only=False, training_rounds=2,
                                  batch_size=32, exploration_module=P.UCBExploration(1.0),
                                  action_representation_module=P.OneHotActionTensorRepresentationModule(4))
    buf = P.B200ReplayBuffer(1000, rng="device")
    g = torch.Generator().manual_seed(2)
    s = torch.randn(200, 6, generator=g)
    buf.push_batch(s, torch.randint(0, 4, (200,), generator=g), s[:, 0], None, torch.ones(200, dtype=torch.bool),
                   torch.zeros(200, dtype=torch.bool), max_number_actions=4)
    buf.seed(2)
    nl.learn(buf)
    h = nl._nl["handle"].value
    batch = P.TransitionBatch(state=s[:32].to(DEV), action=torch.eye(4)[torch.arange(32) % 4].to(DEV), reward=s[:32, 1].to(DEV))
    for _ in range(2):
        nl.learn_batch(batch)
        nl.act(s[:3].to(DEV), Space(4))
        nl.learn(buf)
    assert nl._nl["handle"].value == h
    assert int(nl._nl["lib"].prl_nlb_graph_captures(h)) == 2       # the buffer round and the dense round
    assert int(nl._nl["lib"].prl_nlb_adam_step(h)) == 2 * 3 + 2


def test_checkpoint_views_and_refusals():
    import pearl_b200 as P
    fx = load("cb_nl_onehot")
    for nl, c, out in run_agent(fx, act=False, calls=2):
        pass
    p0 = next(nl.model.parameters())
    assert p0.data_ptr() == nl._nl["flat"].data_ptr()
    st = nl.optimizer.state[p0]
    assert st["exp_avg"].data_ptr() == nl._nl["state"][0].data_ptr()
    assert nl.model.linear_layer_e2e.weight not in nl.optimizer.state       # no gradient without e2e
    sd = {k: v.clone() for k, v in nl.state_dict().items()}
    nl.load_state_dict({k: torch.zeros_like(v) if "weight" in k else v for k, v in sd.items()})
    assert float(nl._nl["flat"].abs().sum()) < float(torch.cat([v.reshape(-1) for v in sd.values()]).abs().sum())
    for bad, match in ((dict(hidden_dims=[8]), "two hidden"), (dict(hidden_dims=[8, 128]), "127"),
                       (dict(dropout_ratio=0.1), "dropout"), (dict(use_layer_norm=True), "norm"),
                       (dict(use_batch_norm=True), "norm"), (dict(hidden_activation="tanh"), "relu"),
                       (dict(last_activation="relu"), "last_activation"), (dict(output_activation_name="tanh"), "linear and sigmoid"),
                       (dict(force_pinv=True), "force_pinv"), (dict(l2_reg_lambda_linear=0.0), "lambda")):
        kw = dict(feature_dim=8, hidden_dims=[8, 8])
        kw.update(bad)
        with pytest.raises(NotImplementedError, match=match):
            P.B200NeuralLinearBandit(**kw)
    nl2 = P.B200NeuralLinearBandit(feature_dim=8, hidden_dims=[8, 4])
    x = torch.zeros(4, 8, device=DEV)
    with pytest.raises(NotImplementedError, match="negative weights"):
        nl2.learn_batch(P.TransitionBatch(state=x, action=x[:, :0], reward=torch.zeros(4, device=DEV),
                                          weight=torch.tensor([1.0, -0.5, 1.0, 1.0], device=DEV)))
    with pytest.raises(NotImplementedError, match="Prioritized"):
        nl2.learn(P.B200PrioritizedReplayBuffer(100))
    nl2.exploration_module = object()
    with pytest.raises(NotImplementedError, match="UCBExploration"):
        nl2.act(x, Space(3))
    nl2.exploration_module = P.UCBExploration(1.0)
    nl2.exploration_module.randomized_tiebreaking = P._compat.TiebreakingStrategy.PER_ROW_TIEBREAKING
    with pytest.raises(NotImplementedError, match="tie-breaking"):
        nl2.act(x, Space(3))


def test_state_features_only_learn_over_a_buffer_and_act():
    """The reference's default: the network sees the state alone, so every action of a state scores the same and act
    picks the first available one."""
    import pearl_b200 as P
    torch.cuda.set_device(0)
    nl = P.B200NeuralLinearBandit(feature_dim=6, hidden_dims=[16, 8], exploration_module=P.UCBExploration(1.0),
                                  action_representation_module=P.OneHotActionTensorRepresentationModule(4), training_rounds=3,
                                  batch_size=32)
    buf = P.B200ReplayBuffer(1000, rng="device")
    g = torch.Generator().manual_seed(1)
    s = torch.randn(200, 6, generator=g)
    buf.push_batch(s, torch.randint(0, 4, (200,), generator=g), s[:, 0], None, torch.ones(200, dtype=torch.bool),
                   torch.zeros(200, dtype=torch.bool), max_number_actions=4)
    buf.seed(1)
    rep = nl.learn(buf)
    assert len(rep["loss"]) == 3 and all(np.isfinite(float(v)) for v in rep["loss"])
    sc = nl.get_scores(s[:5].to(DEV), Space(4))
    assert torch.equal(sc, sc[:, :1].expand_as(sc))
    mask = torch.tensor([[0, 1, 1, 1]] * 5, device=DEV)
    assert nl.act(s[:5].to(DEV), Space(4), action_availability_mask=mask).reshape(-1).tolist() == [1] * 5
