"""The fp32-in/fp32-out tensor-core GEMM / implicit-GEMM convolution (csrc/tc_f32.cu: in-kernel bf16 hi/lo split, three wgmma
products, fp32 accumulation in registers) against fp64 ATen on the CPU.  Shapes are chosen to take the tensor-core route
(tc_gemm_usable / tc_conv_usable) and to hit its edges: ragged M / N / K tiles, unaligned leading dimensions, batched strided
operands (the attention pattern), output channel slices, every activation."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def dm(lib_built):
    assert torch.cuda.is_available()
    from audio_separator.separator.b200 import demucs

    return demucs


def rel_err(got, ref):
    return float((got.double() - ref).abs().max() / max(1.0, float(ref.abs().max())))


@pytest.mark.parametrize("M,N,K", [(300, 200, 100), (128, 128, 64), (1000, 513, 72), (129, 260, 2048), (2688, 512, 512), (77, 40, 36)])
def test_tc_linear(dm, M, N, K):
    g = torch.Generator().manual_seed(M + N + K)
    x, w, b = torch.randn((M, K), generator=g), torch.randn((N, K), generator=g) / K**0.5, torch.randn(N, generator=g)
    res, rs = torch.randn((M, N), generator=g), torch.rand(N, generator=g)
    ref = res.double() + rs.double() * F.gelu(F.linear(x.double(), w.double(), b.double()))
    got = dm.linear(x.cuda(), w.cuda(), b.cuda(), act=dm.ACT_GELU, res=res.cuda(), res_scale=rs.cuda()).cpu()
    assert rel_err(got, ref) <= 3e-5
    got2 = dm.linear(x.cuda(), w.cuda(), None).cpu()
    assert rel_err(got2, x.double() @ w.double().t()) <= 3e-5


def test_tc_attention_pattern(dm):
    """scores = Q K^T / sqrt(hd) per head via strides into (L, D) tensors; V^T = Wv X^T with a per-row bias; O = P V into head columns."""
    from audio_separator.separator.b200.demucs import _gemm_raw

    g = torch.Generator().manual_seed(3)
    Lq, Lk, H, hd = 333, 270, 4, 64
    D = H * hd
    q, k = torch.randn((Lq, D), generator=g).cuda(), torch.randn((Lk, D), generator=g).cuda()
    sc = torch.empty((H, Lq, Lk), device="cuda")
    _gemm_raw(q.data_ptr(), k.data_ptr(), sc.data_ptr(), Lq, Lk, hd, D, D, Lk, H, hd, hd, Lq * Lk, alpha=0.125)
    ref = torch.einsum("qhd,khd->hqk", q.cpu().double().view(Lq, H, hd), k.cpu().double().view(Lk, H, hd)) * 0.125
    assert rel_err(sc.cpu(), ref) <= 3e-5
    wv, bv, x = torch.randn((D, D), generator=g).cuda() / 16, torch.randn(D, generator=g).cuda(), torch.randn((2, Lk, D), generator=g).cuda()
    vt = torch.empty((2, D, Lk), device="cuda")
    _gemm_raw(wv.data_ptr(), x.data_ptr(), vt.data_ptr(), D, Lk, D, D, D, Lk, 2, 0, Lk * D, D * Lk, bias_m=bv.data_ptr())
    refv = (x.cpu().double() @ wv.cpu().double().t() + bv.cpu().double()).transpose(1, 2)
    assert rel_err(vt.cpu(), refv) <= 3e-5
    p = torch.softmax(sc, -1).contiguous()
    o = torch.zeros((Lq, D), device="cuda")
    _gemm_raw(p.data_ptr(), vt.data_ptr(), o.data_ptr(), Lq, hd, Lk, Lk, Lk, D, H, Lq * Lk, hd * Lk, hd)
    refo = torch.einsum("hqk,hdk->qhd", p.cpu().double(), vt[0].cpu().double().view(H, hd, Lk)).reshape(Lq, D)
    assert rel_err(o.cpu(), refo) <= 3e-5


@pytest.mark.parametrize(
    "geom",
    [
        dict(cin=16, cout=32, k=(3, 3), s=(1, 1), p=(1, 1), dw=1, hw=(40, 70), act=1),
        dict(cin=24, cout=40, k=(3, 3), s=(2, 2), p=(1, 1), dw=1, hw=(42, 66), act=3),
        dict(cin=48, cout=300, k=(1, 1), s=(1, 1), p=(0, 0), dw=1, hw=(8, 300), act=0),
        dict(cin=8, cout=48, k=(8, 1), s=(4, 1), p=(2, 0), dw=1, hw=(256, 37), act=2),
        dict(cin=6, cout=20, k=(1, 8), s=(1, 4), p=(0, 2), dw=1, hw=(1, 9000), act=2),
        dict(cin=48, cout=16, k=(1, 3), s=(1, 1), p=(0, 2), dw=2, hw=(5, 600), act=0),
        dict(cin=130, cout=64, k=(1, 1), s=(1, 1), p=(0, 0), dw=1, hw=(64, 64), act=4),
    ],
)
def test_tc_conv2d(dm, geom):
    g = torch.Generator().manual_seed(geom["cin"] * 7 + geom["cout"])
    x = torch.randn((2, geom["cin"]) + geom["hw"], generator=g)
    fan = geom["cin"] * geom["k"][0] * geom["k"][1]
    w = torch.randn((geom["cout"], geom["cin"]) + geom["k"], generator=g) / fan**0.5
    b = torch.randn(geom["cout"], generator=g)
    act = {0: lambda t: t, 1: F.relu, 2: F.gelu, 3: lambda t: F.leaky_relu(t, 0.01), 4: torch.sigmoid}[geom["act"]]
    ref = act(F.conv2d(x.double(), w.double(), b.double(), stride=geom["s"], padding=geom["p"], dilation=(1, geom["dw"])))
    wb = torch.from_numpy(dm.block_conv_weight(w.numpy())).cuda()
    got = dm.conv2d(x.cuda(), wb, b.cuda(), geom["cout"], geom["k"], geom["s"], geom["p"], geom["dw"], act=geom["act"]).cpu()
    assert got.shape == ref.shape
    assert rel_err(got, ref) <= 3e-5, rel_err(got, ref)


def test_tc_conv2d_slice_and_add(dm):
    g = torch.Generator().manual_seed(11)
    x = torch.randn((3, 20, 30, 50), generator=g)
    w = torch.randn((33, 20, 3, 3), generator=g) / 13
    b = torch.randn(33, generator=g)
    ref = F.conv2d(x.double(), w.double(), b.double(), padding=1)
    add = torch.randn(ref.shape, generator=g)
    out = torch.full((3, 50, 30, 50), 7.0).cuda()
    wb = torch.from_numpy(dm.block_conv_weight(w.numpy())).cuda()
    dm.conv2d(x.cuda(), wb, b.cuda(), 33, (3, 3), p=(1, 1), act=dm.ACT_RELU, add=add.cuda(), add_before_act=True, out=out, out_c_off=10)
    o = out.cpu()
    assert rel_err(o[:, 10:43], F.relu(ref + add.double())) <= 3e-5
    assert (o[:, :10] == 7).all() and (o[:, 43:] == 7).all()
    got = dm.conv2d(x.cuda(), wb, b.cuda(), 33, (3, 3), p=(1, 1), act=dm.ACT_RELU, add=add.cuda(), add_before_act=False).cpu()
    assert rel_err(got, F.relu(ref) + add.double()) <= 3e-5


# ------------------------------------------------------------------------------------------------ fused attention (head dimension 64)
@pytest.mark.parametrize("packed", [1, 0])
@pytest.mark.parametrize(
    "B,H,Lq,Lk,v_kn",
    [(2, 3, 200, 1344, 0), (1, 2, 130, 130, 1), (1, 8, 2688, 2688, 0), (2, 2, 1344, 2688, 0), (3, 1, 1101, 1101, 1), (1, 1, 5, 7, 0), (1, 2, 128, 256, 1)],
)
def test_fused_attention_vs_fp64(lib_built, B, H, Lq, Lk, v_kn, packed):
    """b200sep_attention_f32 (scores in registers, running softmax, P as the register operand of P V) against softmax(q k^T / 8) v in float64; ragged query / key tiles,
    both V layouts (transposed with keys contiguous: HTDemucs; plain (keys, d): Roformer)."""
    from audio_separator.separator.b200._lib import check, lib
    from audio_separator.separator.b200.engine import _ptr, _stream

    g = torch.Generator().manual_seed(B * 1000 + Lq + Lk)
    D = H * 64
    q = torch.randn((B, Lq, D), generator=g) * 1.5
    k = torch.randn((B, Lk, D), generator=g) * 1.5
    v = torch.randn((B, Lk, D), generator=g)
    qh, kh, vh = (t.double().view(B, -1, H, 64).transpose(1, 2) for t in (q, k, v))
    ref = (torch.softmax(qh @ kh.transpose(-1, -2) / 8.0, dim=-1) @ vh).transpose(1, 2).reshape(B, Lq, D)
    qd, kd = q.cuda(), k.cuda()
    out = torch.full((B, Lq, D), float("nan"), device="cuda")
    # packed: Q / K / V^T pre-split into tile images in `work` and fetched by bulk copies; otherwise every CTA converts the tiles it reads
    work = torch.empty((lib.b200sep_attention_work_floats(B, H, Lq, Lk),), device="cuda") if packed else None
    wp = _ptr(work) if packed else None
    if v_kn:
        vd = v.cuda()
        check(lib.b200sep_attention_f32(_ptr(qd), _ptr(kd), _ptr(vd), _ptr(out), B, H, Lq, Lk, 64, Lq * D, D, Lk * D, D, Lk * D, D, Lq * D, D, 0.125, 1, wp, _stream()), "attention_f32")
    else:
        vd = v.transpose(1, 2).contiguous().cuda()  # (B, D, Lk)
        check(lib.b200sep_attention_f32(_ptr(qd), _ptr(kd), _ptr(vd), _ptr(out), B, H, Lq, Lk, 64, Lq * D, D, Lk * D, D, D * Lk, Lk, Lq * D, D, 0.125, 0, wp, _stream()), "attention_f32")
    torch.cuda.synchronize()
    err = (out.cpu().double() - ref).abs().max().item()
    assert err <= 3e-5 * max(1.0, ref.abs().max().item()), err
