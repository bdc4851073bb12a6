"""CPU checks of the Thompson sampling recordings (tests/golden/cb_ts_*.npz) against oracle/ts_oracle.py: the draws
replay from torch's generator state as recorded, the eager restatement reproduces every recorded theta and score, and the
stand-in explorer and the refusals that need no GPU."""
from __future__ import annotations

import os
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from oracle import ts_oracle  # noqa: E402
from test_bandit_oracle import load  # noqa: E402


def split(fx, key, lens_key):
    o, out = 0, []
    for n in fx[lens_key]:
        out.append(fx[key][o:o + n])
        o += n
    return out


CASES = [("cb_ts_neural", ""), ("cb_ts_linear", "def_"), ("cb_ts_linear", "eff_"), ("cb_ts_scores", "nl_"),
         ("cb_ts_scores", "lin_def_"), ("cb_ts_scores", "lin_eff_")]


@pytest.mark.parametrize("name,p", CASES)
def test_draws_replay_from_the_recorded_generator_states(name, p):
    fx = load(name)
    for k, d in enumerate(split(fx, f"{p}draws", f"{p}draws_len")):
        torch.set_rng_state(torch.from_numpy(fx[f"{p}torch_before"][k]))
        assert torch.equal(torch.empty(d.size).normal_(), torch.from_numpy(d))
        assert np.array_equal(torch.get_rng_state().numpy(), fx[f"{p}torch_after"][k])


@pytest.mark.parametrize("name,p", [c for c in CASES if not c[1].endswith("eff_")])
def test_restatement_reproduces_every_recorded_theta(name, p):
    fx = load(name)
    draws = split(fx, f"{p}draws", f"{p}draws_len")
    for k, eps in enumerate(draws):
        if name == "cb_ts_scores":
            A, coefs, lam = fx[f"{p}A"], fx[f"{p}coefs"], float(fx[f"{p}l2_reg_lambda"])
        else:            # act k follows learn call k
            A, coefs, lam = fx[f"{p}call_A"][k], fx[f"{p}call_coefs"][k], float(fx["l2_reg_lambda"])
        theta = ts_oracle.sample_theta(torch.from_numpy(A), lam, torch.from_numpy(coefs), torch.from_numpy(eps))
        want = fx[f"{p}theta"][k]
        assert np.abs(theta.numpy() - want).max() <= 1e-6 * (1 + np.abs(want).max()), k


@pytest.mark.parametrize("p", ["def_", "eff_"])
def test_restatement_reproduces_the_linear_scores_and_choices(p):
    fx = load("cb_ts_linear")
    S = int(fx["n_act"])
    feats = torch.eye(S)
    draws = split(fx, f"{p}draws", f"{p}draws_len")
    scores = fx[f"{p}scores"].reshape(-1, S)
    for k, s in enumerate(fx[f"{p}act_state"]):
        x = torch.cat([torch.from_numpy(s)[None].expand(S, -1), feats], 1)
        if p == "def_":
            got = ts_oracle.theta_scores(x, torch.from_numpy(fx[f"{p}theta"][k]))
        else:
            got = ts_oracle.efficient_scores(torch.from_numpy(fx[f"{p}call_inv_A"][k]), torch.from_numpy(fx[f"{p}call_coefs"][k]), x,
                                             torch.from_numpy(draws[k]))
        np.testing.assert_allclose(got.numpy(), scores[k], rtol=1e-5, atol=1e-6)
        assert int(np.argmax(scores[k])) == int(fx[f"{p}act_chosen"][k])


def test_efficient_restatement_raises_on_a_nan_sigma():
    with pytest.raises(RuntimeError, match="std >= 0.0"):
        ts_oracle.efficient_scores(-torch.eye(3), torch.zeros(3), torch.ones(1, 2), torch.zeros(1))


def test_stand_in_attributes_and_refusals():
    import pearl_b200 as P
    from pearl_b200 import _compat
    ex = P.ThompsonSamplingExplorationLinear()
    assert ex._enable_efficient_sampling is False and ex.randomized_tiebreaking is False
    assert P.ThompsonSamplingExplorationLinear(enable_efficient_sampling=True)._enable_efficient_sampling is True

    class Space:
        n = 3
        actions = [torch.tensor([i]) for i in range(3)]

    x = torch.zeros(2, 4)
    nl = P.B200NeuralLinearBandit(feature_dim=4, hidden_dims=[8, 4],
                                  exploration_module=P.ThompsonSamplingExplorationLinear(enable_efficient_sampling=True))
    with pytest.raises(NotImplementedError, match="reference fails"):
        nl.act(x, Space())
    with pytest.raises(NotImplementedError, match="reference fails"):
        nl.get_scores(x, Space())
    lb = P.B200LinearBandit(feature_dim=7, action_representation_module=P.OneHotActionTensorRepresentationModule(3))
    for learner in (lb, nl):
        learner.exploration_module = _compat.ThompsonSamplingExplorationLinearDisjoint()
        with pytest.raises(NotImplementedError, match="UCBExploration"):
            learner.act(x, Space())
        learner.exploration_module = P.ThompsonSamplingExplorationLinear()
        for strategy in (_compat.TiebreakingStrategy.PER_ROW_TIEBREAKING, _compat.TiebreakingStrategy.BATCH_TIEBREAKING):
            learner.exploration_module.randomized_tiebreaking = strategy
            with pytest.raises(NotImplementedError, match="tie-breaking"):
                learner.act(x, Space())
