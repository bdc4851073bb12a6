"""CPU checks for NeuralLinearBandit: the eager oracle (oracle/neural_linear_oracle.py) against the reference's
recordings (tests/golden/cb_nl_*.npz), the stand-in's state_dict keys against the reference's, and the constructor
refusals of B200NeuralLinearBandit."""
from __future__ import annotations

import os
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from oracle import neural_linear_oracle as no  # noqa: E402
from test_bandit_oracle import close_normwise, load  # noqa: E402
from _tol import close_params  # noqa: E402


@pytest.mark.parametrize("tag", ["mae", "ce"])
def test_oracle_reproduces_learn_batch(tag):
    fx = load("cb_nl_batch")
    f, (h1, h2) = int(fx["obs"]) + int(fx["act_dim"]), [int(x) for x in fx["hidden"]]
    o = no.NeuralLinear(fx[f"{tag}_init"], f, h1, h2, lr=float(fx["lr0"]), loss="mae" if tag == "mae" else "cross_entropy",
                        sigmoid=tag == "ce", lam=float(fx["l2_reg_lambda"]), gamma=float(fx["gamma"]),
                        interval=float(fx["interval"]))
    steps = 0
    for c in range(int(fx["calls"])):
        if c == int(fx["lr_change_at"]):
            for g in o.opt.param_groups:
                g["lr"] = float(fx["lr1"])
        b = lambda k: torch.from_numpy(fx[f"{tag}_b_{k}"][c])  # noqa: E731
        pred, loss = o.round(torch.cat([b("state"), b("action")], 1), b("reward"), b("weight"))
        steps += c != int(fx["zero_at"])
        close_normwise(pred.numpy().ravel(), fx[f"{tag}_pred"][c], f"{tag} prediction of call {c}")
        np.testing.assert_allclose(float(loss), fx[f"{tag}_loss"][c], rtol=1e-4, atol=1e-6)
        close_params(o.flat().numpy(), fx[f"{tag}_call_params"][c], f"{tag} parameters after call {c}", float(fx["lr1"]), max(steps, 1))
        np.testing.assert_allclose(o.ridge.A.numpy(), fx[f"{tag}_call_A"][c], rtol=1e-4, atol=1e-4)


@pytest.mark.parametrize("name", ["cb_nl_agent", "cb_nl_onehot"])
def test_oracle_reproduces_the_first_learn_call(name):
    """The first learn() of an agent recording: its rounds replayed on the recorded sampled rows."""
    fx = load(name)
    A, bits = int(fx["n_actions"]), int(fx["act_dim"])
    feats = np.eye(A, dtype=np.float32) if str(fx["rep"]) == "one_hot" else \
        ((np.arange(A)[:, None] >> np.arange(bits)[None, :]) & 1).astype(np.float32)
    X = torch.from_numpy(np.concatenate([fx["push_state"], feats[fx["push_action"]]], axis=1))
    Y = torch.from_numpy(fx["push_reward"])
    f, (h1, h2) = X.shape[1], [int(x) for x in fx["hidden"]]
    o = no.NeuralLinear(fx["init"], f, h1, h2, lr=float(fx["lr"]), skip=bool(fx["skip"]), e2e=bool(fx["e2e"]),
                        lam=float(fx["l2_reg_lambda"]), gamma=float(fx["gamma"]), interval=float(fx["interval"]))
    off = 0
    for r in range(int(fx["rounds"])):
        n = int(fx["idx_len"][r])
        rows = torch.from_numpy(fx["idx"][off:off + n].astype(np.int64))
        pred, loss = o.round(X[rows], Y[rows])
        close_normwise(pred.numpy().ravel(), fx["pred"][off:off + n], f"prediction of round {r}")
        np.testing.assert_allclose(float(loss), fx["loss"][r], rtol=1e-4, atol=1e-6)
        off += n
    close_params(o.flat().numpy(), fx["call_params"][0], "parameters after call 0", float(fx["lr"]), int(fx["rounds"]))


def test_without_e2e_the_e2e_weight_has_no_adamw_state():
    fx = load("cb_nl_onehot")
    assert not bool(fx["e2e"]) and set(fx["call_adam_n_state"].tolist()) == {6}
    assert set(load("cb_nl_agent")["call_adam_n_state"].tolist()) == {7}


@pytest.mark.parametrize("name,kw", [("cb_nl_agent", dict(feature_dim=21, hidden_dims=[64, 16])),
                                     ("cb_nl_onehot", dict(feature_dim=16, hidden_dims=[16, 16], use_skip_connections=True)),
                                     ("cb_nl_scores", dict(feature_dim=12, hidden_dims=[24, 12]))])
def test_stand_in_state_dict_keys_are_the_references(name, kw):
    from pearl_b200._compat import _RefNeuralLinearBandit
    assert list(_RefNeuralLinearBandit(**kw).state_dict().keys()) == load(name)["keys"].tolist()


@pytest.mark.parametrize("bad,match", [(dict(hidden_dims=[8]), "two hidden"), (dict(hidden_dims=[8, 8, 8]), "two hidden"),
                                       (dict(hidden_dims=[8, 128]), "127"), (dict(dropout_ratio=0.1), "dropout"),
                                       (dict(use_batch_norm=True), "norm"), (dict(use_layer_norm=True), "norm"),
                                       (dict(hidden_activation="tanh"), "relu"), (dict(last_activation="relu"), "last_activation"),
                                       (dict(output_activation_name="softplus"), "linear and sigmoid"),
                                       (dict(force_pinv=True), "force_pinv"), (dict(l2_reg_lambda_linear=0.0), "lambda")])
def test_constructor_refusals(bad, match):
    import pearl_b200 as P
    kw = dict(feature_dim=8, hidden_dims=[8, 8])
    kw.update(bad)
    with pytest.raises(NotImplementedError, match=match):
        P.B200NeuralLinearBandit(**kw)


@pytest.mark.parametrize("skip", [False, True])
@pytest.mark.parametrize("e2e", [True, False])
@pytest.mark.parametrize("loss", ["mse", "mae", "cross_entropy"])
def test_fp64_step_matches_float64_autograd(loss, e2e, skip):
    from oracle import neural_linear_fp64 as f64
    g = torch.Generator().manual_seed(7)
    f, h1, h2, B = 6, 6, 6, 40                  # equal widths: every layer residual when skip
    p = [t.double() for t in no.unflatten(torch.randn(sum(int(torch.tensor(s).prod()) for s in no.shapes(f, h1, h2)),
                                                      generator=g) * 0.5, f, h1, h2)]
    X = torch.randn(B, f, generator=g, dtype=torch.float64)
    y = torch.rand(B, generator=g, dtype=torch.float64) if loss == "cross_entropy" else torch.randn(B, generator=g, dtype=torch.float64)
    w = torch.rand(B, generator=g, dtype=torch.float64) + 0.25
    coefs = torch.randn(h2 + 1, generator=g, dtype=torch.float64)
    sigmoid = loss == "cross_entropy"
    got = f64.step(p, X, y, w, coefs, e2e=e2e, loss=loss, sigmoid=sigmoid, skip=skip)
    q = [t.clone().requires_grad_() for t in p]
    n = no.nn_output(q, X, skip)
    mu = (n @ q[6].t()).reshape(-1) if e2e else coefs[0] + n @ coefs[1:]
    pr = torch.sigmoid(mu) if sigmoid else mu
    fn = {"mse": torch.nn.functional.mse_loss, "mae": torch.nn.functional.l1_loss,
          "cross_entropy": torch.nn.functional.binary_cross_entropy}[loss]
    L = (fn(pr, y, reduction="none") * w).sum() / w.sum()
    L.backward()
    torch.testing.assert_close(got["loss"], L.detach(), rtol=1e-12, atol=0)
    for k, t in zip(f64.BLOCKS, q):
        if k == "dwe" and not e2e:
            assert t.grad is None
            continue
        torch.testing.assert_close(got[k].reshape(t.shape), t.grad, rtol=1e-10, atol=1e-13, msg=k)
    scale = f64.step(p, X, y, w, coefs, e2e=e2e, loss=loss, sigmoid=sigmoid, skip=skip, absolute=True)
    for k in f64.BLOCKS:
        if k in got:
            assert bool((got[k].abs() <= scale[k] * (1 + 1e-12)).all()), k
