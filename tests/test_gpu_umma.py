"""wgmma building block (pearl_b200/csrc/umma.cuh) against an fp64 product."""
import ctypes as C

import pytest
import torch

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("n,k", [(64, 64), (64, 128), (128, 64), (16, 8), (256, 32)])
def test_umma_3xtf32_matches_fp64(n, k):
    from pearl_b200 import _lib
    lib = _lib.init(0)
    g = torch.Generator(device="cuda").manual_seed(n * 1000 + k)
    a = torch.randn((128, k), generator=g, device="cuda")
    b = torch.randn((n, k), generator=g, device="cuda")
    want = (a.double() @ b.double().T)
    scale = (a.abs().double() @ b.abs().double().T)  # sum |a||b|: the natural error scale of a dot product
    for passes, tol in ((3, 4e-6), (1, 2e-3)):
        d = torch.full((128, n), float("nan"), device="cuda")
        _lib.check(lib.prl_test_umma_gemm(C.c_void_p(a.data_ptr()), C.c_void_p(b.data_ptr()), C.c_void_p(d.data_ptr()),
                                          n, k, passes, None))
        torch.cuda.synchronize()
        err = ((d.double() - want).abs() / scale).max().item()
        print(f"    N={n} K={k} passes={passes}: max |err| / sum|a||b| = {err:.3e}")
        assert err < tol
        if passes == 1:
            assert err > 1e-5  # really TF32 (a fp32 product would be ~1e-7)


@pytest.mark.parametrize("m,n,k,lbo", [(128, 64, 64, 144), (64, 64, 64, 128), (64, 64, 64, 144), (64, 128, 64, 144),
                                         (64, 32, 64, 144), (128, 64, 128, 128), (64, 8, 128, 144)])
def test_umma_m64_and_padded_chunk_pitch(m, n, k, lbo):
    """M = 64 / 128, N down to 8 and operand tiles with a 144-byte chunk pitch (the layout the
    backward pass uses for transposed tiles so that scattered column writes are bank-conflict free)."""
    from pearl_b200 import _lib
    lib = _lib.init(0)
    g = torch.Generator(device="cuda").manual_seed(7)
    A = torch.randn((m, k), generator=g, device="cuda")
    B = torch.randn((n, k), generator=g, device="cuda")
    raw = torch.full((m, n), float("nan"), device="cuda")
    _lib.check(lib.prl_test_umma_gemm2(C.c_void_p(A.data_ptr()), C.c_void_p(B.data_ptr()), C.c_void_p(raw.data_ptr()),
                                       m, n, k, lbo, None))
    torch.cuda.synchronize()
    want = A.double() @ B.double().T
    scale = A.abs().double() @ B.abs().double().T
    err = ((raw.double() - want).abs() / scale).max().item()
    print(f"    M={m} N={n} K={k} lbo={lbo}: err {err:.3e}")
    assert err < 4e-6


@pytest.mark.parametrize("n,k", [(64, 64), (64, 32), (128, 64), (32, 8)])
def test_umma_a_operand_in_registers(n, k):
    """RS form: every thread loads its own A fragments into registers (no shared-memory traffic for A)."""
    from pearl_b200 import _lib
    lib = _lib.init(0)
    g = torch.Generator(device="cuda").manual_seed(11)
    A = torch.randn((128, k), generator=g, device="cuda")
    B = torch.randn((n, k), generator=g, device="cuda")
    d = torch.full((128, n), float("nan"), device="cuda")
    _lib.check(lib.prl_test_umma_gemm_ts(C.c_void_p(A.data_ptr()), C.c_void_p(B.data_ptr()), C.c_void_p(d.data_ptr()), n, k, 1, None))
    torch.cuda.synchronize()
    want = A.double() @ B.double().T
    scale = A.abs().double() @ B.abs().double().T
    err = ((d.double() - want).abs() / scale).max().item()
    print(f"    RS N={n} K={k}: err {err:.3e}")
    assert err < 4e-6
