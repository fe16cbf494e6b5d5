"""GPU: the 3x3 tensor-core convolution (umma_conv3_kernel) with each compile-time epilogue variant it is instantiated for, against a float64
conv2d + BatchNorm + activation (+ residual) (* multiplier).  Same tolerance as test_umma_gpu.py: 5e-5 relative to max|ref|."""
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

# (act, residual, multiplier, BN scale/shift): MDX-Net's BN + ReLU; MDX23C's TFC convolutions (no BN in the epilogue, + shortcut, * first-conv output)
VARIANTS = {
    "relu": (1, False, False, True),
    "plain": (0, False, False, False),
    "res": (0, True, False, False),
    "res_mul": (0, True, True, False),
}

# (B, Cin, Cout, T, F): n_c = 16 / 32 / 48 / 64 / 80; resident weights (48 -> 48) and streamed ones (96 -> 96, 144 -> 144); F not a multiple of 112;
# one tile (B = T = 1, F <= 112); tile counts that leave the persistent CTAs 1, 2 or 3 tiles each, or a mix
SHAPES = [
    (1, 16, 16, 3, 200),
    (1, 32, 32, 4, 336),
    (1, 48, 48, 1, 96),
    (2, 48, 48, 66, 224),
    (1, 48, 48, 132, 336),
    (1, 48, 48, 50, 1000),
    (1, 96, 96, 7, 248),
    (2, 144, 144, 5, 112),
    (1, 64, 64, 6, 120),
    (1, 80, 80, 3, 232),
    (1, 640, 640, 2, 64),
]


@pytest.fixture(scope="module")
def lib(lib_built):
    assert torch.cuda.is_available()
    from audio_separator.separator.b200 import _lib

    return _lib


def rel_err(got, ref):
    return (got.double() - ref.double()).abs().max().item() / max(1e-30, ref.double().abs().max().item())


def run_conv3(lib, x, w, res, mul, scale, shift, act):
    B, Cin, T, Fq = x.shape
    Cout = w.shape[0]
    out = torch.full((B, Cout, T, Fq), float("nan"), device="cuda")
    ptr = lambda t: t.data_ptr() if t is not None else None
    rc = lib.lib.b200sep_selftest_umma_conv3x3_ex(ptr(x), w.data_ptr(), ptr(res), ptr(mul), out.data_ptr(), B, Cin, Cout, T, Fq, ptr(scale), ptr(shift), act, None)
    return rc, out


@pytest.mark.timeout(300)
@pytest.mark.parametrize("variant", sorted(VARIANTS))
@pytest.mark.parametrize("B,Cin,Cout,T,Fq", SHAPES)
def test_conv3_epilogue_vs_torch(lib, variant, B, Cin, Cout, T, Fq):
    act, has_res, has_mul, has_bn = VARIANTS[variant]
    g = torch.Generator(device="cuda").manual_seed(B * 1000 + Cin + Cout + T + Fq + act)
    x = torch.randn(B, Cin, T, Fq, device="cuda", generator=g)
    w = (torch.randn(Cout, Cin, 3, 3, device="cuda", generator=g) / (3 * Cin**0.5)).cpu().contiguous()
    scale = torch.rand(Cout, device="cuda", generator=g) + 0.5 if has_bn else None
    shift = torch.randn(Cout, device="cuda", generator=g) * 0.1 if has_bn else None
    res = torch.randn(B, Cout, T, Fq, device="cuda", generator=g) if has_res else None
    mul = torch.randn(B, Cout, T, Fq, device="cuda", generator=g) if has_mul else None
    rc, out = run_conv3(lib, x, w, res, mul, scale, shift, act)
    lib.check(rc, "selftest_umma_conv3x3_ex")
    ref = F.conv2d(x.double(), w.cuda().double(), padding=1)
    if has_bn:
        ref = ref * scale.double()[None, :, None, None] + shift.double()[None, :, None, None]
    if act == 1:
        ref = torch.relu(ref)
    if has_res:
        ref = ref + res.double()
    if has_mul:
        ref = ref * mul.double()
    assert torch.isfinite(out).all()
    assert rel_err(out, ref) <= 5e-5


@pytest.mark.timeout(60)
@pytest.mark.parametrize("act,has_res,has_mul", [(2, False, False), (1, True, False), (0, False, True)])
def test_conv3_epilogue_without_instance_is_an_error(lib, act, has_res, has_mul):
    x = torch.randn(1, 16, 2, 64, device="cuda")
    w = torch.randn(16, 16, 3, 3) / 12
    t = torch.randn(1, 16, 2, 64, device="cuda")
    rc, _ = run_conv3(lib, x, w, t if has_res else None, t if has_mul else None, None, None, act)
    assert rc != 0
