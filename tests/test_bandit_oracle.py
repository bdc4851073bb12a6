"""CPU checks of the LinearBandit oracle (oracle/bandit_oracle.py) against the reference's recordings
(tests/golden/cb_*.npz, oracle/gen_bandit_golden.py), of the stand-in's state_dict keys, and of the refusals the plugin
makes before any device work."""
from __future__ import annotations

import os
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from oracle import bandit_oracle as bo  # noqa: E402
from _tol import RTOL  # noqa: E402

ATOL = 2e-6
# A, b and sum_weight are sums and are held elementwise.  inv_A, coefs and the predictions come out of a linear solve,
# whose rounding error is bounded normwise (about cond(A + lambda I) * 2^-24 * ||x||), not per element: a small
# coefficient next to large ones carries the absolute error of the large ones.  They are held to 1e-4 of the largest
# magnitude of the quantity (per call for inv_A and coefs, per round for the predictions).
SOLVED = ("inv_A", "coefs")


def close_normwise(got, want, what=""):
    got, want = np.asarray(got, np.float64), np.asarray(want, np.float64)
    np.testing.assert_allclose(got, want, rtol=RTOL, atol=RTOL * np.abs(want).max() + ATOL, err_msg=what)


def close_state(got: dict, fx, c, what):
    for k in ("A", "b", "sum_weight", "inv_A", "coefs"):
        if k in SOLVED:
            close_normwise(got[k], fx[f"call_{k}"][c], f"{what}: {k} after call {c}")
        else:
            np.testing.assert_allclose(got[k], fx[f"call_{k}"][c], rtol=RTOL, atol=ATOL, err_msg=f"{what}: {k} after call {c}")

GOLDEN = os.path.join(ROOT, "tests", "golden")


def load(name):
    return np.load(os.path.join(GOLDEN, f"{name}.npz"))


def act_features(fx) -> np.ndarray:
    A, rep = int(fx["n_actions"]), str(fx["rep"])
    if rep == "one_hot":
        return np.eye(A, dtype=np.float32)
    bits = int(fx["act_dim"])
    return ((np.arange(A)[:, None] >> np.arange(bits)[None, :]) & 1).astype(np.float32)


def replay_method(fx):
    """The oracle over the recorded sampling: call c sees the prefill plus c pushes; each round's rows are the recorded
    logical indices (the reference's buffer never evicts, so logical = push order)."""
    feats = act_features(fx)
    X = np.concatenate([fx["push_state"], feats[fx["push_action"]]], axis=1)
    Y = fx["push_reward"]
    r = bo.Ridge(X.shape[1] + 1, float(fx["l2_reg_lambda"]), float(fx["gamma"]), float(fx["interval"]))
    idx, lens = fx["idx"], fx["idx_len"]
    o, preds, calls = 0, [], []
    rounds = int(fx["rounds"])
    for c in range(len(fx["call_A"])):
        n_avail = int(fx["prefill"]) + c
        for k in range(rounds):
            rr = c * rounds + k
            sel = idx[o:o + lens[rr]]
            assert sel.max() < n_avail
            o += lens[rr]
            preds.append(r.round(torch.from_numpy(X[sel]), torch.from_numpy(Y[sel])).numpy().ravel())
        calls.append(dict(A=r.A.clone(), b=r.b.clone(), sum_weight=r.sum_weight.clone(), inv_A=r.inv_A.clone(),
                          coefs=r.coefs.clone(), last=r.last))
    return np.concatenate(preds), calls


@pytest.mark.parametrize("name", ["cb_lin_method", "cb_lin_binary"])
def test_oracle_reproduces_the_agent_loop(name):
    fx = load(name)
    preds, calls = replay_method(fx)
    o = 0
    for r, n in enumerate(fx["idx_len"]):
        close_normwise(preds[o:o + n], fx["pred"][o:o + n], f"prediction of round {r}")
        o += n
    for c, s in enumerate(calls):
        close_state({k: v.numpy() for k, v in s.items() if k != "last"}, fx, c, name)
        assert s["last"] == fx["call_last"][c]
    assert (fx["call_cond"] <= 1e4).all()


def test_oracle_reproduces_learn_batch():
    fx = load("cb_lin_batch")
    r = bo.Ridge(int(fx["obs"]) + int(fx["act_dim"]) + 1, float(fx["l2_reg_lambda"]), float(fx["gamma"]), float(fx["interval"]),
                 coefs=fx["initial_coefs"])
    for c in range(len(fx["pred"])):
        x = torch.from_numpy(np.concatenate([fx["b_state"][c], fx["b_action"][c]], axis=1))
        w = torch.from_numpy(fx["b_weight"][c]) if fx["b_has_weight"][c] else None
        p = r.round(x, torch.from_numpy(fx["b_reward"][c]), w)
        close_normwise(p.numpy().ravel(), fx["pred"][c])
        close_state({k: getattr(r, k).numpy() for k in ("A", "b", "sum_weight", "inv_A", "coefs")}, fx, c, "learn_batch")
        assert r.last == fx["call_last"][c]
    assert not fx["b_weight"][1].any(), "the recording has an all-zero-weight batch"


def test_oracle_reproduces_scores():
    fx = load("cb_lin_scores")
    A = int(fx["n_actions"])
    x = bo.features(torch.from_numpy(fx["states"]), torch.eye(A))
    inv, coefs = torch.from_numpy(fx["inv_A"]), torch.from_numpy(fx["coefs"])
    ucb = bo.scores(inv, coefs, x, float(fx["alpha"]))
    np.testing.assert_allclose(ucb.numpy(), fx["ucb"], rtol=RTOL, atol=ATOL)
    np.testing.assert_allclose(bo.scores(inv, coefs, x, 0.0).numpy(), fx["ucb0"], rtol=RTOL, atol=ATOL)
    np.testing.assert_allclose(bo.scores(inv, coefs, x, 0.0, with_sigma=False).numpy(), fx["exploit"], rtol=RTOL, atol=ATOL)
    mask = torch.from_numpy(fx["mask"])
    assert np.array_equal(bo.first_max(ucb, mask).numpy(), fx["act_mask"])
    assert np.array_equal(bo.first_max(ucb).numpy(), fx["act_all"])


def test_fp64_yardstick_is_the_inverse_of_the_fp32_matrix():
    g = torch.Generator().manual_seed(5)
    x = torch.randn(200, 9, generator=g)
    r = bo.Ridge(10, 0.3)
    r.round(x, torch.randn(200, generator=g))
    inv, coefs, cond = bo.fp64_yardstick(r.A, r.b, 0.3)
    M = (r.A + 0.3 * torch.eye(10)).double()
    assert torch.allclose(inv @ M, torch.eye(10, dtype=torch.float64), atol=1e-10)
    assert 1.0 <= cond < 1e3


def test_stand_in_state_dict_keys_match_the_reference():
    from pearl_b200 import B200LinearBandit, OneHotActionTensorRepresentationModule, UCBExploration
    fx = load("cb_lin_method")
    lb = B200LinearBandit(feature_dim=26, exploration_module=UCBExploration(1.0),
                          action_representation_module=OneHotActionTensorRepresentationModule(10))
    assert list(lb.state_dict().keys()) == [str(k) for k in fx["keys"]]
    assert lb.last_sum_weight_when_discounted == 0.0
    lb.last_sum_weight_when_discounted = 3.5
    assert lb.last_sum_weight_when_discounted == 3.5


@pytest.mark.parametrize("kw,needle", [(dict(force_pinv=True), "force_pinv"), (dict(l2_reg_lambda=0.0), "l2_reg_lambda"),
                                       (dict(l2_reg_lambda=-1.0), "l2_reg_lambda"), (dict(feature_dim=128), "at most 127")])
def test_construction_refusals(kw, needle):
    from pearl_b200 import B200LinearBandit
    with pytest.raises(NotImplementedError, match=needle):
        B200LinearBandit(**{"feature_dim": 26, **kw})


def test_widest_supported_ridge_is_accepted():
    from pearl_b200 import B200LinearBandit
    assert B200LinearBandit(feature_dim=127).model._A.shape == (128, 128)
