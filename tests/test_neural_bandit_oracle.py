"""CPU checks for NeuralBandit: the eager oracle (oracle/neural_bandit_oracle.py) against the reference's recordings
(tests/golden/cb_nb_*.npz), the float64 step (oracle/neural_bandit_fp64.py) against float64 autograd, the SquareCB /
FastCB action rule against every recorded probability vector and choice, the stand-in's state_dict keys against the
reference's, and the constructor refusals of B200NeuralBandit."""
from __future__ import annotations

import os
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from oracle import neural_bandit_oracle as no  # noqa: E402
from test_bandit_oracle import close_normwise, load  # noqa: E402
from _tol import close_params  # noqa: E402

# the agent recordings: (fixture, key prefix)
AGENTS = [("cb_nb_squarecb", ""), ("cb_nb_squarecb", "g5_"), ("cb_nb_fastcb", "")]


def agent(name, prefix):
    fx = load(name)
    return {k[len(prefix):]: fx[k] for k in fx.files if k.startswith(prefix) and (prefix or not k.startswith("g5_"))}


def features(fx):
    A, bits = int(fx["n_actions"]), int(fx["act_dim"])
    return np.eye(A, dtype=np.float32) if str(fx["rep"]) == "one_hot" else \
        ((np.arange(A)[:, None] >> np.arange(bits)[None, :]) & 1).astype(np.float32)


@pytest.mark.parametrize("loss", ["mse", "mae"])
def test_oracle_reproduces_learn_batch(loss):
    fx = load("cb_nb_batch")
    f, (h1, h2) = int(fx["obs"]) + int(fx["act_dim"]), [int(x) for x in fx["hidden"]]
    o = no.NeuralBandit(fx[f"{loss}_init"], f, h1, h2, lr=float(fx["lr0"]), loss=loss)
    for c in range(int(fx["calls"])):
        if c == int(fx["lr_change_at"]):
            for g in o.opt.param_groups:
                g["lr"] = float(fx["lr1"])
        b = lambda k: torch.from_numpy(fx[f"{loss}_b_{k}"][c])  # noqa: E731
        pred, lo = o.round(torch.cat([b("state"), b("action")], 1), b("reward"), b("weight"))
        close_normwise(pred.numpy().ravel(), fx[f"{loss}_pred"][c], f"{loss} prediction of call {c}")
        np.testing.assert_allclose(float(lo), fx[f"{loss}_loss"][c], rtol=1e-4, atol=1e-6)
        close_params(o.flat().numpy(), fx[f"{loss}_call_params"][c], f"{loss} parameters after call {c}", float(fx["lr1"]), c + 1)


@pytest.mark.parametrize("name,prefix", AGENTS)
def test_oracle_reproduces_the_first_learn_call(name, prefix):
    """The first learn() of an agent recording: its rounds replayed on the recorded sampled rows."""
    fx = agent(name, prefix)
    X = torch.from_numpy(np.concatenate([fx["push_state"], features(fx)[fx["push_action"]]], axis=1))
    Y = torch.from_numpy(fx["push_reward"])
    f, (h1, h2) = X.shape[1], [int(x) for x in fx["hidden"]]
    o = no.NeuralBandit(fx["init"], f, h1, h2, lr=float(fx["lr"]), loss=str(fx["loss"]))
    off = 0
    for r in range(int(fx["rounds"])):
        n = int(fx["idx_len"][r])
        rows = torch.from_numpy(fx["idx"][off:off + n].astype(np.int64))
        pred, loss = o.round(X[rows], Y[rows])
        close_normwise(pred.numpy().ravel(), fx["pred"][off:off + n], f"prediction of round {r}")
        np.testing.assert_allclose(float(loss), fx["losses"][r], rtol=1e-4, atol=1e-6)
        off += n
    close_params(o.flat().numpy(), fx["call_params"][0], "parameters after call 0", float(fx["lr"]), int(fx["rounds"]))


@pytest.mark.parametrize("name,prefix", AGENTS)
def test_act_rule_reproduces_every_recorded_choice(name, prefix):
    fx = agent(name, prefix)
    for k, v in enumerate(fx["act_values"]):
        p, pn, a = no.explore(torch.from_numpy(v), fastcb=bool(fx["fastcb"]), gamma=float(fx["gamma"]), lb=float(fx["reward_lb"]),
                              ub=float(fx["reward_ub"]), clamp=bool(fx["clamp"]), E=torch.from_numpy(fx["act_E"][k]))
        np.testing.assert_allclose(p.numpy(), fx["act_p"][k], rtol=2e-6, atol=1e-9, err_msg=f"p of act {k}")
        np.testing.assert_allclose(pn.numpy(), fx["act_pn"][k], rtol=2e-6, atol=1e-9, err_msg=f"pn of act {k}")
        assert a == int(fx["act_chosen"][k]), k


def test_recordings_cover_clamping_ties_the_uniform_branch_and_exploration():
    fx = load("cb_nb_fastcb")
    ub, lb = np.float32(fx["reward_ub"]), np.float32(fx["reward_lb"])
    c = np.clip(fx["act_values"], lb, ub)
    assert ((c == ub).sum(1) >= 2).any() and (c.max(1) <= lb).any()
    uni = fx["act_p"][(c.max(1) <= lb)]
    assert np.allclose(uni, 1.0 / c.shape[1])
    g5 = agent("cb_nb_squarecb", "g5_")
    assert (g5["act_chosen"] != g5["act_values"].argmax(1)).any()


@pytest.mark.parametrize("loss", ["mse", "mae"])
def test_fp64_step_matches_float64_autograd(loss):
    from oracle import neural_bandit_fp64 as f64
    g = torch.Generator().manual_seed(7)
    f, h1, h2, B = 6, 9, 5, 40
    p = [t.double() for t in no.unflatten(torch.randn(sum(int(torch.tensor(s).prod()) for s in no.shapes(f, h1, h2)),
                                                      generator=g) * 0.5, f, h1, h2)]
    X = torch.randn(B, f, generator=g, dtype=torch.float64)
    y = torch.randn(B, generator=g, dtype=torch.float64)
    w = (torch.rand(B, generator=g, dtype=torch.float64) + 0.25) * torch.where(torch.rand(B, generator=g) < 0.2, -1.0, 1.0).double()
    got = f64.step(p, X, y, w, loss=loss)
    q = [t.clone().requires_grad_() for t in p]
    fn = {"mse": torch.nn.functional.mse_loss, "mae": torch.nn.functional.l1_loss}[loss]
    L = (fn(no.value(q, X).view(y.shape), y, reduction="none") * w).sum() / w.sum()
    L.backward()
    torch.testing.assert_close(got["loss"], L.detach(), rtol=1e-12, atol=0)
    scale = f64.step(p, X, y, w, loss=loss, absolute=True)
    for k, t in zip(f64.BLOCKS, q):
        torch.testing.assert_close(got[k].reshape(t.shape), t.grad, rtol=1e-10, atol=1e-13, msg=k)
        assert bool((got[k].abs() <= scale[k] * (1 + 1e-12)).all()), k


@pytest.mark.parametrize("name", ["cb_nb_squarecb", "cb_nb_fastcb", "cb_nb_scores"])
def test_stand_in_state_dict_keys_are_the_references(name):
    from pearl_b200._compat import _RefNeuralBandit, NoExploration
    fx = load(name)
    f = int(fx["obs"]) + (0 if name == "cb_nb_scores" else int(fx["act_dim"]))
    keys = list(_RefNeuralBandit(f, [int(x) for x in fx["hidden"]], NoExploration()).state_dict().keys())
    assert keys == fx["keys"].tolist()


@pytest.mark.parametrize("bad,match", [(dict(hidden_dims=[8]), "two hidden"), (dict(hidden_dims=[8, 8, 8]), "two hidden"),
                                       (dict(output_dim=2), "output_dim"), (dict(loss_type="cross_entropy"), "CROSS_ENTROPY")])
def test_constructor_refusals(bad, match):
    import pearl_b200 as P
    kw = dict(feature_dim=8, hidden_dims=[8, 8], exploration_module=P.NoExploration())
    kw.update(bad)
    with pytest.raises(NotImplementedError, match=match):
        P.B200NeuralBandit(**kw)
    if "loss_type" in bad:
        kw["loss_type"] = P.LossType.CROSS_ENTROPY
        with pytest.raises(NotImplementedError, match=match):
            P.B200NeuralBandit(**kw)


def test_defaults_are_the_references():
    import pearl_b200 as P
    nb = P.B200NeuralBandit(feature_dim=8, hidden_dims=[8, 4], exploration_module=P.SquareCBExploration(gamma=5.0))
    assert (nb._training_rounds, nb._batch_size, nb.optimizer.param_groups[0]["lr"]) == (100, 128, 0.001)
    assert nb.optimizer.param_groups[0]["amsgrad"] and not nb._state_features_only
    fc = P.FastCBExploration(gamma=3.0, reward_lb=-1.0)
    assert fc.clamp_values and (fc._gamma, fc.reward_lb, fc.reward_ub) == (3.0, -1.0, 1.0)
