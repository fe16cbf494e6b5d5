"""GPU: the wgmma ("bf16x3 pair") operators in isolation against plain fp32 PyTorch references of the same op,
through the C-ABI self-test entry points.  Tolerance: the split scheme carries ~16 mantissa bits per operand, so
errors are ~1e-5 of the output scale (measured 7e-6 on the whole network); gate at 5e-5 relative to max|ref|."""
import ctypes as C

import numpy as np
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def lib(lib_built):
    assert torch.cuda.is_available()
    from audio_separator.separator.b200 import _lib

    return _lib


def rel_err(got, ref):
    return (got.double() - ref.double()).abs().max().item() / max(1e-30, ref.double().abs().max().item())


@pytest.mark.timeout(120)
@pytest.mark.parametrize("M,N,K,rpc,ch,res", [(256, 128, 64, 32, 8, False), (512, 96, 768, 32, 8, True), (300, 48, 48, 30, 10, True), (1024, 384, 3072, 256, 4, False), (384, 768, 96, 32, 12, True), (128, 16, 16, 16, 8, False), (2304, 96, 24, 8, 288, True)])
def test_umma_gemm_vs_torch(lib, M, N, K, rpc, ch, res):
    g = torch.Generator(device="cuda").manual_seed(M + N + K)
    a = torch.randn(M, K, device="cuda", generator=g) * 2
    w = torch.randn(N, K, device="cuda", generator=g) / K**0.5
    r = torch.randn(M, N, device="cuda", generator=g) if res else None
    scale = torch.rand(ch, device="cuda", generator=g) + 0.5
    shift = torch.randn(ch, device="cuda", generator=g) * 0.1
    out = torch.full((M, N), float("nan"), device="cuda")
    rc = lib.lib.b200sep_selftest_umma_gemm(a.data_ptr(), w.data_ptr(), r.data_ptr() if res else None, out.data_ptr(), M, N, K, rpc, ch, scale.data_ptr(), shift.data_ptr(), 1, None)
    lib.check(rc, "selftest_umma_gemm")
    c = (torch.arange(M, device="cuda") // rpc) % ch
    ref = torch.relu((a.double() @ w.double().T) * scale[c, None].double() + shift[c, None].double())
    if res:
        ref = ref + r.double()
    assert torch.isfinite(out).all()
    assert rel_err(out, ref) <= 5e-5


@pytest.mark.timeout(120)
@pytest.mark.parametrize("B,Cin,Cout,T,Fq", [(1, 16, 16, 4, 128), (2, 48, 48, 8, 256), (1, 96, 96, 6, 192), (1, 32, 64, 5, 96), (2, 144, 144, 4, 64), (1, 288, 288, 8, 96), (1, 48, 48, 16, 3072), (1, 640, 640, 3, 64), (1, 256, 256, 4, 128), (1, 768, 768, 2, 32)])  # the last three: MDX23C widths (n_c 80 / 64 / 48, smaller channel steps)
def test_umma_conv3x3_vs_torch(lib, B, Cin, Cout, T, Fq):
    g = torch.Generator(device="cuda").manual_seed(B * 1000 + Cin + Cout + T + Fq)
    x = torch.randn(B, Cin, T, Fq, device="cuda", generator=g)
    w = (torch.randn(Cout, Cin, 3, 3, device="cuda", generator=g) / (3 * Cin**0.5)).cpu().contiguous()
    scale = torch.rand(Cout, device="cuda", generator=g) + 0.5
    shift = torch.randn(Cout, device="cuda", generator=g) * 0.1
    out = torch.full((B, Cout, T, Fq), float("nan"), device="cuda")
    rc = lib.lib.b200sep_selftest_umma_conv3x3(x.data_ptr(), w.data_ptr(), out.data_ptr(), B, Cin, Cout, T, Fq, scale.data_ptr(), shift.data_ptr(), 1, None)
    lib.check(rc, "selftest_umma_conv3x3")
    ref = torch.relu(F.conv2d(x.double(), w.cuda().double(), padding=1) * scale.double()[None, :, None, None] + shift.double()[None, :, None, None])
    assert torch.isfinite(out).all()
    assert rel_err(out, ref) <= 5e-5


@pytest.mark.timeout(120)
@pytest.mark.parametrize("B,Cin,Cout,T,Fq,up,skip", [(1, 32, 16, 4, 128, 1, True), (2, 96, 48, 8, 256, 1, True), (1, 288, 240, 8, 96, 1, False), (1, 96, 48, 6, 1536, 1, True),
                                                     (1, 16, 32, 4, 128, 0, False), (2, 48, 96, 8, 256, 0, False), (1, 240, 288, 16, 192, 0, False), (1, 48, 96, 6, 3072, 0, False)])
def test_umma_updown_vs_torch(lib, B, Cin, Cout, T, Fq, up, skip):
    g = torch.Generator(device="cuda").manual_seed(B * 1000 + Cin + Cout + T + Fq + up)
    x = torch.randn(B, Cin, T, Fq, device="cuda", generator=g)
    wshape = (Cin, Cout, 2, 2) if up else (Cout, Cin, 2, 2)
    w = (torch.randn(*wshape, device="cuda", generator=g) / (2 * Cin**0.5)).cpu().contiguous()
    scale = torch.rand(Cout, device="cuda", generator=g) + 0.5
    shift = torch.randn(Cout, device="cuda", generator=g) * 0.1
    oshape = (B, Cout, 2 * T, 2 * Fq) if up else (B, Cout, T // 2, Fq // 2)
    sk = torch.randn(*oshape, device="cuda", generator=g) if skip else None
    out = torch.full(oshape, float("nan"), device="cuda")
    rc = lib.lib.b200sep_selftest_umma_updown(x.data_ptr(), w.data_ptr(), sk.data_ptr() if skip else None, out.data_ptr(), B, Cin, Cout, T, Fq, scale.data_ptr(), shift.data_ptr(), 1, up, None)
    lib.check(rc, "selftest_umma_updown")
    wd = w.cuda().double()
    y = F.conv_transpose2d(x.double(), wd, stride=2) if up else F.conv2d(x.double(), wd, stride=2)
    ref = torch.relu(y * scale.double()[None, :, None, None] + shift.double()[None, :, None, None])
    if skip:
        ref = ref * sk.double()
    assert torch.isfinite(out).all()
    assert rel_err(out, ref) <= 5e-5
