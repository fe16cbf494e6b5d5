"""GPU: the ping-pong schedule of umma_conv3_kernel (each consumer warpgroup owns whole tiles) at MDX-Net's TFC layer sizes and at tile counts
that leave a CTA's second warpgroup with no tile or one fewer than the first, against a float64 conv2d + BatchNorm + ReLU.  Same tolerance as
test_conv3_epilogue_gpu.py: 5e-5 relative to max|ref|.  Two runs of a shape are bitwise equal."""
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

# MDX-Net (Inst_HQ_3 geometry) TFC 3x3 layers, batch 8: C channels at T x F; 48 -> 48 keeps its weights resident, the rest stream them
MDX_LAYERS = [(48, 256, 3072), (96, 128, 1536), (144, 64, 768), (192, 32, 384), (240, 16, 192), (288, 8, 96)]
# one 112-pixel tile per output row: 1, 2, 131, 133, 263 and 265 tiles over 132 persistent CTAs
TILE_COUNTS = [1, 2, 131, 133, 263, 265]


@pytest.fixture(scope="module")
def lib(lib_built):
    assert torch.cuda.is_available()
    from audio_separator.separator.b200 import _lib

    return _lib


def run_conv3(lib, x, w, scale, shift):
    B, Cin, T, Fq = x.shape
    out = torch.full((B, w.shape[0], T, Fq), float("nan"), device="cuda")
    rc = lib.lib.b200sep_selftest_umma_conv3x3_ex(x.data_ptr(), w.data_ptr(), None, None, out.data_ptr(), B, Cin, w.shape[0], T, Fq, scale.data_ptr(),
                                                  shift.data_ptr(), 1, None)
    lib.check(rc, "selftest_umma_conv3x3_ex")
    return out


def check_shape(lib, B, C, T, Fq, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    x = torch.randn(B, C, T, Fq, device="cuda", generator=g)
    w = (torch.randn(C, C, 3, 3, device="cuda", generator=g) / (3 * C**0.5)).cpu().contiguous()
    scale = torch.rand(C, device="cuda", generator=g) + 0.5
    shift = torch.randn(C, device="cuda", generator=g) * 0.1
    out = run_conv3(lib, x, w, scale, shift)
    again = run_conv3(lib, x, w, scale, shift)
    assert torch.equal(out, again)
    ref = torch.relu(F.conv2d(x.double(), w.cuda().double(), padding=1) * scale.double()[None, :, None, None] + shift.double()[None, :, None, None])
    err = (out.double() - ref).abs().max().item() / ref.abs().max().item()
    assert torch.isfinite(out).all()
    assert err <= 5e-5


@pytest.mark.timeout(600)
@pytest.mark.parametrize("C,T,Fq", MDX_LAYERS)
def test_conv3_pingpong_mdx_layer(lib, C, T, Fq):
    check_shape(lib, 8, C, T, Fq, seed=C)


@pytest.mark.timeout(120)
@pytest.mark.parametrize("tiles", TILE_COUNTS)
def test_conv3_pingpong_tile_counts(lib, tiles):
    check_shape(lib, 1, 48, tiles, 112, seed=tiles)
