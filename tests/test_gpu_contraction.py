"""The actor-critic learners' contraction (pearl_b200/csrc/gemm.cuh, gemm_tc.cu) against fp64 products: the three kinds the
learners use (nn.Linear forward, backward-data, backward-weight + bias gradient), on the tensor-core tiles (wgmma, 3xTF32) and on the
SIMT tiles, with every feature of the operand descriptor: two concatenated sources (state || action), stacked networks
(twin critics), ones column, ReLU / mask / accumulate epilogues, ragged sizes.

Tolerance: |err| <= 4e-6 * sum|a||b| per output (the natural scale of a dot product; a plain-TF32 product would be ~1e-3).
The learners' end-to-end parity gate (1e-4 relative against the reference's recordings) is in test_sac / test_ppo_learn /
test_td3; this file pins the building block."""
import ctypes as C

import pytest
import torch

pytestmark = pytest.mark.gpu

ENGINES = [0, 64, 32, 164, 132]   # SIMT tiles; wgmma with both operands in shared memory; wgmma with A in registers


def _p(t):
    return C.c_void_p(t.data_ptr()) if t is not None else None


def _run(op, engine, M, N, K, a, b, a2=None, split=0, bias=None, mask=None, relu=0, accumulate=0, c=None, c_tail=None, nets=1):
    from pearl_b200 import _lib
    lib = _lib.init(0)
    _lib.check(lib.prl_test_contraction(op, engine, M, N, K, _p(a), _p(b), _p(a2), split, _p(bias), _p(mask), relu, accumulate,
                                        _p(c), _p(c_tail), nets, None))
    torch.cuda.synchronize()


def _rel(got, want, scale):
    return ((got.double() - want).abs() / scale.clamp_min(1e-30)).max().item()


@pytest.mark.parametrize("engine", ENGINES)
@pytest.mark.parametrize("M,N,K,split,nets,relu", [
    (512, 256, 376, 0, 1, 1),        # SAC actor layer 1
    (512, 256, 393, 376, 2, 1),      # SAC twin critics: state || action, ragged K
    (512, 17, 256, 0, 1, 0),         # action head
    (512, 1, 256, 0, 2, 0),          # scalar heads of the twin critics
    (256, 64, 210, 0, 1, 1),         # PPO layer 1
    (8192, 64, 210, 0, 1, 1),        # PPO preprocessing pass
    (100, 40, 33, 20, 1, 0),         # ragged everything
    (1, 64, 128, 0, 1, 1),           # act(): one row
])
def test_forward(engine, M, N, K, split, nets, relu):
    g = torch.Generator(device="cuda").manual_seed(M * 7 + N * 3 + K)
    x = torch.randn((nets, M, K), generator=g, device="cuda")
    W = torch.randn((nets, N, K), generator=g, device="cuda") / K ** 0.5
    bias = torch.randn((nets, N), generator=g, device="cuda")
    want = torch.einsum("zmk,znk->zmn", x.double(), W.double()) + bias.double()[:, None, :]
    scale = torch.einsum("zmk,znk->zmn", x.abs().double(), W.abs().double()) + bias.abs().double()[:, None, :]
    if relu:
        want = want.clamp_min(0)
    if split:
        a, a2 = x[:, :, :split].contiguous(), x[:, :, split:].contiguous()
    else:
        a, a2 = x, None
    c = torch.full((nets, M, N), float("nan"), device="cuda")
    _run(0, engine, M, N, K, a, W, a2=a2, split=split, bias=bias, relu=relu, c=c, nets=nets)
    err = _rel(c, want, scale)
    print(f"    fwd engine={engine} {M}x{N}x{K}: {err:.2e}")
    assert err < 4e-6


@pytest.mark.parametrize("engine", ENGINES)
@pytest.mark.parametrize("M,N,K,nets,use_mask,accumulate", [
    (512, 256, 256, 1, True, False),
    (512, 256, 393, 2, False, False),    # gradient w.r.t. the critic input (actor loss)
    (256, 64, 64, 1, True, True),
    (100, 17, 50, 1, True, True),
])
def test_backward_data(engine, M, N, K, nets, use_mask, accumulate):
    g = torch.Generator(device="cuda").manual_seed(M + N * 5 + K * 11)
    dy = torch.randn((nets, M, N), generator=g, device="cuda")
    W = torch.randn((nets, N, K), generator=g, device="cuda") / N ** 0.5
    mask = torch.randn((nets, M, K), generator=g, device="cuda") if use_mask else None
    c0 = torch.randn((nets, M, K), generator=g, device="cuda")
    want = torch.einsum("zmn,znk->zmk", dy.double(), W.double())
    scale = torch.einsum("zmn,znk->zmk", dy.abs().double(), W.abs().double())
    if accumulate:
        want, scale = want + c0.double(), scale + c0.abs().double()
    if use_mask:
        want = torch.where(mask > 0, want, torch.zeros_like(want))
    c = c0.clone() if accumulate else torch.full((nets, M, K), float("nan"), device="cuda")
    _run(1, engine, M, N, K, dy, W, mask=mask, accumulate=int(accumulate), c=c, nets=nets)
    err = _rel(c, want, scale)
    print(f"    bwd-x engine={engine} {M}x{N}x{K}: {err:.2e}")
    assert err < 4e-6


@pytest.mark.parametrize("engine", ENGINES)
@pytest.mark.parametrize("M,N,K,split,nets", [
    (512, 256, 376, 0, 1),
    (512, 256, 393, 376, 2),
    (512, 1, 256, 0, 2),
    (256, 64, 210, 0, 1),
    (100, 40, 33, 20, 1),
])
def test_backward_weight(engine, M, N, K, split, nets):
    g = torch.Generator(device="cuda").manual_seed(M * 13 + N + K * 2)
    dy = torch.randn((nets, M, N), generator=g, device="cuda")
    x = torch.randn((nets, M, K), generator=g, device="cuda")
    want = torch.einsum("zmn,zmk->znk", dy.double(), x.double())
    scale = torch.einsum("zmn,zmk->znk", dy.abs().double(), x.abs().double())
    want_b, scale_b = dy.double().sum(1), dy.abs().double().sum(1)
    if split:
        b, a2 = x[:, :, :split].contiguous(), x[:, :, split:].contiguous()
    else:
        b, a2 = x, None
    c = torch.full((nets, N, K), float("nan"), device="cuda")
    ct = torch.full((nets, N), float("nan"), device="cuda")
    _run(2, engine, M, N, K, dy, b, a2=a2, split=split, c=c, c_tail=ct, nets=nets)
    err, err_b = _rel(c, want, scale), _rel(ct, want_b, scale_b)
    print(f"    bwd-w engine={engine} {M}x{N}x{K}: {err:.2e} bias {err_b:.2e}")
    assert err < 4e-6 and err_b < 4e-6


def test_engine_switch_is_validated():
    from pearl_b200 import _lib
    lib = _lib.init(0)
    assert lib.prl_get_contraction_engine() == 1          # tensor cores are the default
    assert lib.prl_set_contraction_engine(7) != 0
    _lib.check(lib.prl_set_contraction_engine(0))
    assert lib.prl_get_contraction_engine() == 0
    _lib.check(lib.prl_set_contraction_engine(1))
