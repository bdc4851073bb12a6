"""DeepSARSA (csrc/sarsa.cu) across its shape space against the float64 step of oracle/sarsa_fp64.py.

Per case, one learn() from a B200SARSAReplayBuffer under contraction engines 0 (SIMT tiles), 1 (the library default:
3xTF32 wgmma tiles from 4096 output rows on) and 2 (wgmma always), without (freq 1000) and with (freq 1) the soft target
update before the step: the reported loss and every gradient block (read from exp_avg after one step from zero moments)
within C x scale of the fp64 step, where scale is the sum of |a||b| over every product that contributed (the error
model of oracle/dqn_fp64.py); the target bit for bit.  Rows whose online pre-activations lie within MARGIN of their scale
of a ReLU kink are left out (dqn_fp64.make_data), so rounding cannot flip a ReLU derivative.  The target net's kinks need
no margin: y is continuous in them.

The grid spans obs 1-257, 1-255 actions, hidden widths 1-640 and batches 1-4096.  C = 4e-7, the bound of the other
DQN-family shape tests.  Measured on an H100 80GB HBM3 (700 W power limit), the largest err / scale over the grid, every
engine and both update frequencies is 1.38e-7 (dW1s at obs 3, 2 actions, [5, 3], batch 2, engine 2); each case prints
its own (MAXERR)."""
from collections import namedtuple

import numpy as np
import pytest
import torch

from oracle.pearl_oracle import load_flat

pytestmark = pytest.mark.gpu

C = 4e-7
MARGIN = 1e-6
GAMMA, TAU = 0.99, 0.3
ENGINES = (0, 1, 2)

Case = namedtuple("Case", "obs A H1 H2 B")
GRID = [Case(1, 1, 1, 1, 1), Case(3, 2, 5, 3, 2), Case(4, 2, 64, 64, 32), Case(127, 16, 65, 63, 255), Case(128, 17, 129, 257, 256),
        Case(257, 33, 300, 300, 1024), Case(8, 255, 64, 64, 4096), Case(16, 64, 640, 640, 512), Case(33, 3, 512, 512, 4096),
        Case(2, 255, 1, 640, 5)]


def _cid(c):
    return f"obs{c.obs}-A{c.A}-h{c.H1}x{c.H2}-B{c.B}"


class _Space:
    def __init__(self, A):
        self.n = A
        self.actions = [torch.tensor([i]) for i in range(A)]
        self.actions_batch = torch.arange(A).view(A, 1)


class _Engine:
    def __init__(self, engine):
        from pearl_b200 import _lib
        self.lib, self.engine = _lib.load(), engine

    def __enter__(self):
        from pearl_b200 import _lib
        self.prev = self.lib.prl_get_contraction_engine()
        _lib.check(self.lib.prl_set_contraction_engine(self.engine))

    def __exit__(self, *exc):
        from pearl_b200 import _lib
        _lib.check(self.lib.prl_set_contraction_engine(self.prev))


def _learner(c, seed, freq):
    import pearl_b200
    torch.manual_seed(seed)
    pl = pearl_b200.B200DeepSARSA(state_dim=c.obs, action_space=_Space(c.A), hidden_dims=[c.H1, c.H2], training_rounds=1,
                                  batch_size=c.B, target_update_freq=freq, soft_update_tau=TAU, discount_factor=GAMMA,
                                  action_representation_module=pearl_b200.OneHotActionTensorRepresentationModule(c.A)).to("cuda:0")
    g = torch.Generator().manual_seed(seed + 1)
    w = torch.cat([p.detach().reshape(-1).cpu() for p in pl._Q.parameters()])
    load_flat(pl._Q_target, w + 0.05 * torch.randn(w.shape, generator=g))     # a target that differs from the online net
    return pl


def _soft_update_f32(w, t):
    tau, omtau = torch.tensor(TAU, dtype=torch.float32), torch.tensor(1.0 - TAU, dtype=torch.float32)
    return (tau.to(w.device) * w) + (omtau.to(w.device) * t)


@pytest.mark.parametrize("case", GRID, ids=[_cid(c) for c in GRID])
def test_one_round_gradient_matches_fp64(case):
    import pearl_b200
    from oracle.dqn_fp64 import BLOCKS, block_view, check, make_data
    from oracle.sarsa_fp64 import sarsa_step
    c, hidden = case, (case.H1, case.H2)
    seed = 1000 + 7 * c.obs + 13 * c.A + c.B
    data = None
    for engine in ENGINES:
        with _Engine(engine):
            for freq in (1000, 1):
                pl = _learner(c, seed, freq)
                w0, wt0 = pl.flat_parameters.clone(), pl.flat_target_parameters.clone()
                if data is None:
                    data = make_data(w0.detach(), c.obs, c.A, c.B, seed, False, MARGIN, hidden)
                    n = data["state"].shape[0]
                    data["next_action"] = torch.from_numpy(np.random.default_rng(seed).integers(0, c.A, n))
                n = data["state"].shape[0]
                buf = pearl_b200.B200SARSAReplayBuffer(n, rng="device")
                buf.push_batch(data["state"], data["action"], data["reward"], data["next_state"], data["terminated"],
                               data["truncated"], max_number_actions=c.A, next_action=data["next_action"])
                buf.seed(seed)
                rep = pl.learn(buf, trace=True)
                wt = pl.flat_target_parameters.clone()
                if freq == 1:
                    assert torch.equal(wt, _soft_update_f32(w0, wt0)), "soft target update"
                else:
                    assert torch.equal(wt, wt0), "the target moved without a scheduled update"
                idx = rep["idx"][0].long().cpu()
                batch = {k: v[idx] for k, v in data.items()}
                val, sc = sarsa_step(w0.double(), wt.double(), batch, c.obs, c.A, GAMMA, hidden)
                worst = {}
                check("loss", torch.tensor(rep["loss"][0]), val["mae"], sc["mae"], worst, C)
                st = pl.adam_state()
                assert st["step"] == 1
                g = st["exp_avg"] / torch.tensor(1.0 - pl._adam_hparams()["beta1"], dtype=torch.float32, device=w0.device)
                for name in BLOCKS:
                    gb = block_view(g, name, c.obs, c.A, hidden)
                    check(name, gb, val[name].reshape(gb.shape), sc[name].reshape(gb.shape), worst, C)
                print(f"    MAXERR {_cid(c)} engine={engine} freq={freq} " + " ".join(f"{k}={e:.2e}" for k, e in worst.items()))
                del pl, buf
