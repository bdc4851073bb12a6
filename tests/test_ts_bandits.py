"""GPU checks of Thompson sampling (ThompsonSamplingExplorationLinear) on B200LinearBandit and B200NeuralLinearBandit
against the reference's recordings (tests/golden/cb_ts_*.npz, oracle/gen_ts_golden.py): the agent loops with graphs on and
off (identical actions, sampled indices, and torch and CPython generator states), scores and act over many states with
and without masks, bit-identity run to run, and the error paths and refusals.

Tolerances: theta is held to THETA_TOL = 1e-4 (1 + |theta_ref|) elementwise against the reference's theta sampled from
the same draws; the recorded ridge buffers are reproduced to 1e-4 elementwise (test_bandit.py's bound), and the fp32
reference is itself within 1.4e-6 of the float64 sample (asserted by the generator at THETA_TOL / 4).  The generator
asserts that every recorded choice's margin exceeds 4 x the largest score change a theta within THETA_TOL can cause.
Scores are held normwise (test_bandit_oracle.close_normwise); the efficient mode's per-score draws make them
z sigma + mu with mu and sigma from the GPU's ridge, within the same bound."""
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

from test_bandit_oracle import close_normwise, load  # noqa: E402
from test_neural_linear_bandit import Space, load_flat  # noqa: E402

pytestmark = pytest.mark.gpu

DEV = "cuda:0"
THETA_TOL = 1e-4


def ts(efficient=False):
    import pearl_b200 as P
    return P.ThompsonSamplingExplorationLinear(enable_efficient_sampling=efficient)


def theta_of(ridge, draws):
    """The CUDA sampler on the learner's ridge buffers for the recorded draws (no generator involved)."""
    import pearl_b200 as P
    lib = P._lib.init(0)
    d = draws.size
    eps = torch.from_numpy(draws).to(DEV)
    theta = torch.empty(d, device=DEV)
    status = torch.empty(1, dtype=torch.int32, device=DEV)
    P._lib.check(lib.prl_cb_ts_sample(d, float(ridge.l2_reg_lambda), P._lib.ptr(ridge._A), P._lib.ptr(ridge._coefs),
                                      P._lib.ptr(eps), P._lib.ptr(theta), P._lib.ptr(status), None))
    assert int(status.item()) == 0
    return theta.cpu().numpy()


def close_theta(got, want, what):
    err = np.abs(got.astype(np.float64) - want).max() / (1 + np.abs(want).max())
    assert err <= THETA_TOL, f"{what}: theta {err:.3g} from the reference's (bound {THETA_TOL})"
    return err


def split(fx, key, lens_key):
    o, out = 0, []
    for n in fx[lens_key]:
        out.append(fx[key][o:o + n])
        o += n
    return out


def run_loop(fx, kind, p="", graph=True):
    """The recorded agent loop: act -> push -> learn().  Yields (learner, call index, chosen so far)."""
    import pearl_b200 as P
    torch.cuda.set_device(0)
    A, act_dim = int(fx["n_act"]), int(fx["act_dim"])
    if kind == "nl":
        h = [int(x) for x in fx["hidden"]]
        pl = P.B200NeuralLinearBandit(feature_dim=int(fx["obs"]) + act_dim, hidden_dims=h, exploration_module=ts(),
                                      action_representation_module=P.BinaryActionTensorRepresentationModule(act_dim),
                                      training_rounds=int(fx["rounds"]), batch_size=int(fx["batch"]), learning_rate=float(fx["lr"]),
                                      l2_reg_lambda_linear=float(fx["lam"]), gamma=float(fx["gamma"]),
                                      apply_discounting_interval=float(fx["interval"]), state_features_only=False)
        load_flat(pl, fx["init"])
        ridge = lambda: pl.model._linear_regression_layer  # noqa: E731
    else:
        pl = P.B200LinearBandit(feature_dim=int(fx["obs"]) + act_dim, exploration_module=ts(p == "eff_"),
                                l2_reg_lambda=float(fx["lam"]), gamma=float(fx["gamma"]),
                                apply_discounting_interval=float(fx["interval"]), training_rounds=int(fx["rounds"]),
                                batch_size=int(fx["batch"]), action_representation_module=P.OneHotActionTensorRepresentationModule(A))
        ridge = lambda: pl.model  # noqa: E731
    pl.use_cuda_graph = graph
    buf = P.B200ReplayBuffer(100000, rng="python")
    pre = int(fx["prefill"])
    space = Space(A)
    random.setstate((3, tuple(int(x) for x in fx[f"{p}rng_before"]), None))

    def push(i):
        buf.push(torch.from_numpy(fx[f"{p}push_state"][i]), int(fx[f"{p}push_action"][i]), float(fx[f"{p}push_reward"][i]), True,
                 False, next_state=None, max_number_actions=A)

    for i in range(pre):
        push(i)
    chosen, idx = [], []
    draws = split(fx, f"{p}draws", f"{p}draws_len")
    for c in range(len(fx[f"{p}call_A"])):
        if c:
            if c == 1:
                torch.set_rng_state(torch.from_numpy(fx[f"{p}torch_start"]))
            assert np.array_equal(torch.get_rng_state().numpy(), fx[f"{p}torch_before"][c - 1])
            if p != "eff_":
                close_theta(theta_of(ridge(), draws[c - 1]), fx[f"{p}theta"][c - 1], f"act {c - 1}")
            chosen.append(int(pl.act(torch.from_numpy(fx[f"{p}act_state"][c - 1]), space).reshape(-1)[0]))
            assert np.array_equal(torch.get_rng_state().numpy(), fx[f"{p}torch_after"][c - 1])
            push(pre + c - 1)
        tr = {}
        pl.learn(buf, trace=tr)
        idx.append(tr["idx"].numpy().ravel())
        yield pl, ridge(), c, chosen, idx


def check_ridge(ridge, fx, p, c):
    for k in ("A", "b", "sum_weight"):
        want = fx[f"{p}call_{k}"][c]
        np.testing.assert_allclose(getattr(ridge, f"_{k}").cpu().numpy(), want, rtol=1e-4, atol=1e-5 * max(1.0, np.abs(want).max()),
                                   err_msg=f"{k} after call {c}")


@pytest.mark.parametrize("graph", [True, False])
@pytest.mark.parametrize("case", ["neural", "linear_def", "linear_eff"])
def test_agent_loop_matches_the_recording(case, graph):
    fx = load("cb_ts_neural" if case == "neural" else "cb_ts_linear")
    kind, p = {"neural": ("nl", ""), "linear_def": ("lin", "def_"), "linear_eff": ("lin", "eff_")}[case]
    for pl, ridge, c, chosen, idx in run_loop(fx, kind, p, graph):
        check_ridge(ridge, fx, p, c)
    assert chosen == fx[f"{p}act_chosen"].tolist(), "Thompson choices differ from the reference"
    assert np.array_equal(np.concatenate(idx), fx[f"{p}idx"]), "sampled indices differ from the reference"
    assert np.array_equal(np.asarray(random.getstate()[1], np.uint64).astype(np.uint32), fx[f"{p}rng_after"])
    assert np.array_equal(torch.get_rng_state().numpy(), fx[f"{p}torch_end"])


def scores_learners(fx):
    import pearl_b200 as P
    torch.cuda.set_device(0)
    A, obs = int(fx["n_actions"]), int(fx["obs"])
    nl = P.B200NeuralLinearBandit(feature_dim=obs + A, hidden_dims=[int(x) for x in fx["hidden"]], exploration_module=ts(),
                                  action_representation_module=P.OneHotActionTensorRepresentationModule(A),
                                  output_activation_name="sigmoid", state_features_only=False,
                                  l2_reg_lambda_linear=float(fx["nl_l2_reg_lambda"])).to(DEV)
    load_flat(nl, fx["nl_params"])
    for k in ("A", "b", "sum_weight", "inv_A", "coefs"):
        getattr(nl.model._linear_regression_layer, f"_{k}").copy_(torch.from_numpy(np.asarray(fx[f"nl_{k}"])))
    lins = {}
    for p, eff in (("lin_def_", False), ("lin_eff_", True)):
        lb = P.B200LinearBandit(feature_dim=obs + A, exploration_module=ts(eff), l2_reg_lambda=float(fx[f"{p}l2_reg_lambda"]),
                                action_representation_module=P.OneHotActionTensorRepresentationModule(A)).to(DEV)
        for k in ("A", "b", "sum_weight", "inv_A", "coefs"):
            getattr(lb.model, f"_{k}").copy_(torch.from_numpy(np.asarray(fx[f"{p}{k}"])))
        lins[p] = lb
    return nl, lins, Space(A)


def test_scores_and_act_match_the_recording():
    fx = load("cb_ts_scores")
    nl, lins, space = scores_learners(fx)
    states = torch.from_numpy(fx["states"]).to(DEV)
    mask = torch.from_numpy(fx["mask"]).to(DEV)
    tb, ta = fx["nl_torch_before"], fx["nl_torch_after"]
    torch.set_rng_state(torch.from_numpy(tb[0]))
    close_normwise(nl.get_scores(states, space).cpu().numpy(), fx["nl_scores_act"], "get_scores")
    assert np.array_equal(torch.get_rng_state().numpy(), ta[0])
    nl.separate_uncertainty = True
    close_normwise(nl.get_scores(states, space).cpu().numpy(), fx["nl_scores_sep"], "get_scores, separate_uncertainty")
    assert np.array_equal(torch.get_rng_state().numpy(), ta[1])
    nl.separate_uncertainty = False
    assert nl.act(states, space).reshape(-1).cpu().tolist() == fx["nl_act_all"].tolist()
    assert np.array_equal(torch.get_rng_state().numpy(), ta[2])
    torch.set_rng_state(torch.from_numpy(tb[3]))
    assert nl.act(states, space, action_availability_mask=mask).reshape(-1).cpu().tolist() == fx["nl_act_mask"].tolist()
    assert np.array_equal(torch.get_rng_state().numpy(), ta[3])
    assert sorted(nl.state_dict().keys()) == sorted(fx["nl_keys"].tolist())
    for p, lb in lins.items():
        torch.set_rng_state(torch.from_numpy(fx[f"{p}torch_start"]))
        close_normwise(lb.get_scores(states, space).cpu().numpy(), fx[f"{p}get_scores"], f"{p}get_scores")
        assert lb.act(states, space).reshape(-1).cpu().tolist() == fx[f"{p}act"].tolist(), p
        assert np.array_equal(torch.get_rng_state().numpy(), fx[f"{p}torch_after"][-1]), p
        ex = lb.get_scores(states, space, exploit=True)      # bypasses the explorer: no draws
        assert np.array_equal(torch.get_rng_state().numpy(), fx[f"{p}torch_after"][-1]), p
        assert ex.shape == (states.shape[0], space.n)


def test_bit_identity_run_to_run():
    fx = load("cb_ts_neural")
    runs = []
    for graph in (True, True, False):
        scores = []
        nl = None
        for nl, ridge, c, chosen, idx in run_loop(fx, "nl", "", graph):
            pass
        torch.manual_seed(3)
        for _ in range(3):
            scores.append(nl.get_scores(torch.from_numpy(fx["act_state"]).to(DEV), Space(int(fx["n_act"]))))
        runs.append((torch.stack(scores).cpu(), {k: v.clone().cpu() for k, v in nl.state_dict().items()}))
    for s, sd in runs[1:]:
        assert torch.equal(s, runs[0][0])
        for k, v in sd.items():
            assert torch.equal(v, runs[0][1][k]), k


def test_error_paths_and_refusals():
    import pearl_b200 as P
    from pearl_b200 import _compat
    torch.cuda.set_device(0)
    space = Space(3)
    x = torch.randn(2, 4, device=DEV)
    lb = P.B200LinearBandit(feature_dim=7, exploration_module=ts(),
                            action_representation_module=P.OneHotActionTensorRepresentationModule(3)).to(DEV)
    lb.model._A.copy_(-4 * torch.eye(8))          # A + lambda I = -3 I: not positive definite
    with pytest.raises(ValueError, match="positive definite"):
        lb.act(x, space)
    lb.model._A.zero_()
    lb.act(x, space)                               # the status is written afresh on every call
    lb.exploration_module = ts(True)
    lb.model._inv_A.copy_(-torch.eye(8))           # a negative form: sigma is NaN
    with pytest.raises(RuntimeError, match="std >= 0.0"):
        lb.act(x, space)
    lb.model._inv_A.copy_(torch.eye(8))
    assert lb.get_scores(x, space).shape == (2, 3)
    nl = P.B200NeuralLinearBandit(feature_dim=4, hidden_dims=[8, 4], exploration_module=ts(True))
    with pytest.raises(NotImplementedError, match="reference fails"):
        nl.act(x, space)
    for learner in (lb, nl):
        learner.exploration_module = _compat.ThompsonSamplingExplorationLinearDisjoint()
        with pytest.raises(NotImplementedError, match="UCBExploration"):
            learner.act(x, space)
        learner.exploration_module = ts()
        learner.exploration_module.randomized_tiebreaking = _compat.TiebreakingStrategy.PER_ROW_TIEBREAKING
        with pytest.raises(NotImplementedError, match="tie-breaking"):
            learner.get_scores(x, space)
