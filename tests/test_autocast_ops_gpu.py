"""The fp16 mode (MATH_FP16, what use_autocast=True selects) of the fp32-operator tensor-core kernels against float64 products of fp16-rounded
operands: gemm_f32_math, conv2d_f32_math (plain, dilated, channel-slice, transposed) and attention_f32_math.  The bound is fp32-accumulation
sized, relative to sum |a||b| of each output (the rounding to fp16 itself is in the reference, so it is not part of the tolerance).  Also:
MATH_BF16X3 through the new entries is bit-identical to the old entries, packed images are half the size in fp16 mode, and an image packed
for one mode is rejected by a call of the other."""
import pytest
import torch
import torch.nn.functional as F

from fp16_operands import r16

pytestmark = pytest.mark.gpu

RTOL = 1e-5  # fp32 accumulation of up to a few thousand products, relative to sum |a||b|


@pytest.fixture(scope="module")
def L(lib_built):
    assert torch.cuda.is_available()
    from audio_separator.separator.b200 import _lib, ops

    return _lib, ops


def p(t):
    return t.data_ptr() if t is not None else None


def assert_fp16_close(got, ref, mag, exact):
    """got (fp16 mode) against ref (fp64 of fp16-rounded operands) within RTOL * mag; and visibly apart from the unrounded product `exact`
    (the fp16 mode really ran)."""
    got = got.double().cpu()
    err = (got - ref).abs()
    tol = RTOL * mag + 1e-6 * ref.abs() + 1e-6
    assert (err <= tol).all(), float((err / tol).max())
    assert float((got - exact).abs().max()) > 20 * float(err.max()), (float((got - exact).abs().max()), float(err.max()))


ACTS = {0: lambda t: t, 1: F.relu, 2: F.gelu, 3: lambda t: F.leaky_relu(t, 0.01), 4: torch.sigmoid, 5: torch.tanh}


# ------------------------------------------------------------------------------------------------------------------------------- GEMM
@pytest.mark.parametrize("packed", [0, 1])
@pytest.mark.parametrize(
    "M,N,K,batch,act,epi",
    [(300, 200, 100, 1, 2, "res_scale"), (128, 128, 64, 1, 0, "none"), (1000, 513, 72, 1, 5, "bias"), (129, 260, 2048, 1, 1, "res"),
     (2688, 512, 512, 1, 0, "bias"), (333, 270, 64, 4, 0, "none"), (77, 40, 36, 6, 4, "bias")],
)
def test_gemm_fp16(L, M, N, K, batch, act, epi, packed):
    _lib, ops = L
    g = torch.Generator().manual_seed(M * 7 + N + K)
    a = torch.randn((batch, M, K), generator=g)
    w = torch.randn((N, K), generator=g) / K**0.5 if batch == 1 or packed else torch.randn((batch, N, K), generator=g) / K**0.5
    bias = torch.randn(N, generator=g) if epi in ("bias", "res_scale") else None
    res = torch.randn((batch, M, N), generator=g) if epi in ("res", "res_scale") else None
    rs = torch.rand(N, generator=g) if epi == "res_scale" else None
    alpha = 0.7
    sB = 0 if w.dim() == 2 else N * K
    ad, wd, cd = a.cuda(), w.cuda(), torch.empty((batch, M, N), device="cuda")
    bd, resd, rsd = (t.cuda() if t is not None else None for t in (bias, res, rs))
    pk = ops._packed_linear(wd, _lib.MATH_FP16) if packed and sB == 0 else None
    _lib.check(_lib.lib.b200sep_gemm_f32_math(p(ad), p(wd), p(cd), M, N, K, K, K, N, batch, M * K, sB, M * N, alpha, p(bd), None, act, p(resd), p(rsd), p(pk),
                                              _lib.MATH_FP16, 0), "gemm_f32_math")

    def epilogue(prod):
        v = prod * alpha + (bias.double() if bias is not None else 0.0)
        v = ACTS[act](v)
        if res is None:
            return v
        return res.double() + (rs.double() * v if rs is not None else v)

    wb = w if w.dim() == 3 else w[None]
    ref = epilogue(r16(a) @ r16(wb).transpose(1, 2))
    mag = (a.double().abs() @ wb.double().abs().transpose(1, 2)) * alpha * (rs.double() if rs is not None else 1.0)
    assert_fp16_close(cd, ref, mag, epilogue(a.double() @ wb.double().transpose(1, 2)))


def test_math0_entries_match_old_entries(L):
    """MATH_BF16X3 through the *_math entries gives the same bits as the entries without the suffix (GEMM with and without a packed image, conv,
    attention), and the packed images are equal."""
    _lib, ops = L
    lib = _lib.lib
    g = torch.Generator().manual_seed(5)
    M, N, K = 700, 300, 200
    a, w, b = torch.randn((M, K), generator=g).cuda(), (torch.randn((N, K), generator=g) / 15).cuda(), torch.randn(N, generator=g).cuda()
    n = lib.b200sep_tc_packed_floats(N, K)
    assert lib.b200sep_tc_packed_floats_math(N, K, 0) == n and 2 * lib.b200sep_tc_packed_floats_math(N, K, 1) == n
    pk_old, pk_new = torch.empty(n, device="cuda"), torch.empty(n, device="cuda")
    _lib.check(lib.b200sep_tc_pack_linear_weights(p(w), N, K, K, p(pk_old), 0))
    _lib.check(lib.b200sep_tc_pack_linear_weights_math(p(w), N, K, K, p(pk_new), 0, 0))
    torch.cuda.synchronize()
    assert torch.equal(pk_old, pk_new)
    for pk in (None, pk_old):
        c_old, c_new = torch.empty((M, N), device="cuda"), torch.empty((M, N), device="cuda")
        _lib.check(lib.b200sep_gemm_f32(p(a), p(w), p(c_old), M, N, K, K, K, N, 1, 0, 0, 0, 1.0, p(b), None, 2, None, None, p(pk), 0))
        _lib.check(lib.b200sep_gemm_f32_math(p(a), p(w), p(c_new), M, N, K, K, K, N, 1, 0, 0, 0, 1.0, p(b), None, 2, None, None, p(pk), 0, 0))
        assert torch.equal(c_old, c_new)
    x = torch.randn((2, 24, 40, 60), generator=g).cuda()
    wc = torch.from_numpy(ops.block_conv_weight((torch.randn((48, 24, 3, 3), generator=g) / 15).numpy())).cuda()
    y_old, y_new = torch.empty((2, 48, 40, 60), device="cuda"), torch.empty((2, 48, 40, 60), device="cuda")
    args = (2, 24, 40, 60, 48, 40, 60, 3, 3, 1, 1, 1, 1, 1, 1, 1, 0, 0, 1, 0, 0, 0, 0)
    _lib.check(lib.b200sep_conv2d_f32(p(x), p(wc), None, None, p(y_old), *args, None, 0))
    _lib.check(lib.b200sep_conv2d_f32_math(p(x), p(wc), None, None, p(y_new), *args, None, 0, 0))
    assert torch.equal(y_old, y_new)
    B, H, Lq, Lk = 2, 2, 300, 260
    D = H * 64
    q, k, v = (torch.randn((B, Ln, D), generator=g).cuda() for Ln in (Lq, Lk, Lk))
    assert lib.b200sep_attention_work_floats_math(B, H, Lq, Lk, 0) == lib.b200sep_attention_work_floats(B, H, Lq, Lk)
    assert 2 * lib.b200sep_attention_work_floats_math(B, H, Lq, Lk, 1) == lib.b200sep_attention_work_floats(B, H, Lq, Lk)
    o_old, o_new = torch.empty((B, Lq, D), device="cuda"), torch.empty((B, Lq, D), device="cuda")
    st = (Lq * D, D, Lk * D, D, Lk * D, D, Lq * D, D, 0.125, 1)
    _lib.check(lib.b200sep_attention_f32(p(q), p(k), p(v), p(o_old), B, H, Lq, Lk, 64, *st, None, 0))
    _lib.check(lib.b200sep_attention_f32_math(p(q), p(k), p(v), p(o_new), B, H, Lq, Lk, 64, *st, None, 0, 0))
    assert torch.equal(o_old, o_new)


def test_packed_image_of_the_other_mode_is_rejected(L):
    _lib, ops = L
    lib = _lib.lib
    g = torch.Generator().manual_seed(6)
    M, N, K = 512, 256, 128
    a, w = torch.randn((M, K), generator=g).cuda(), torch.randn((N, K), generator=g).cuda()
    c = torch.empty((M, N), device="cuda")
    pk16 = torch.empty(lib.b200sep_tc_packed_floats_math(N, K, 1), device="cuda")
    _lib.check(lib.b200sep_tc_pack_linear_weights_math(p(w), N, K, K, p(pk16), 1, 0))
    with pytest.raises(_lib.B200SepError, match="other math mode"):
        _lib.check(lib.b200sep_gemm_f32_math(p(a), p(w), p(c), M, N, K, K, K, N, 1, 0, 0, 0, 1.0, None, None, 0, None, None, p(pk16), 0, 0))
    with pytest.raises(_lib.B200SepError, match="other math mode"):
        _lib.check(lib.b200sep_gemm_f32(p(a), p(w), p(c), M, N, K, K, K, N, 1, 0, 0, 0, 1.0, None, None, 0, None, None, p(pk16), 0))
    pk3 = torch.empty(lib.b200sep_tc_packed_floats(N, K), device="cuda")
    _lib.check(lib.b200sep_tc_pack_linear_weights(p(w), N, K, K, p(pk3), 0))
    with pytest.raises(_lib.B200SepError, match="other math mode"):
        _lib.check(lib.b200sep_gemm_f32_math(p(a), p(w), p(c), M, N, K, K, K, N, 1, 0, 0, 0, 1.0, None, None, 0, None, None, p(pk3), 1, 0))
    wc = torch.from_numpy(ops.block_conv_weight(torch.randn((32, 16, 3, 3), generator=g).numpy())).cuda()
    pkc = ops._packed_conv(wc, 16, 9, 32, 0)
    x, y = torch.randn((1, 16, 30, 40), generator=g).cuda(), torch.empty((1, 32, 30, 40), device="cuda")
    with pytest.raises(_lib.B200SepError, match="other math mode"):
        _lib.check(lib.b200sep_conv2d_f32_math(p(x), p(wc), None, None, p(y), 1, 16, 30, 40, 32, 30, 40, 3, 3, 1, 1, 1, 1, 1, 1, 0, 0, 0, 1, 0, 0, 0, 0, p(pkc), 1, 0))
    with pytest.raises(_lib.B200SepError, match="unknown math mode"):
        _lib.check(lib.b200sep_gemm_f32_math(p(a), p(w), p(c), M, N, K, K, K, N, 1, 0, 0, 0, 1.0, None, None, 0, None, None, None, 2, 0))
    torch.cuda.synchronize()


# ------------------------------------------------------------------------------------------------------------------------------- convolution
@pytest.mark.parametrize("packed", [0, 1])
@pytest.mark.parametrize(
    "geom",
    [
        dict(cin=16, cout=32, k=(3, 3), s=(1, 1), p=(1, 1), d=(1, 1), hw=(40, 70), act=1),
        dict(cin=24, cout=40, k=(3, 3), s=(2, 2), p=(1, 1), d=(1, 1), hw=(42, 66), act=3),
        dict(cin=48, cout=300, k=(1, 1), s=(1, 1), p=(0, 0), d=(1, 1), hw=(8, 300), act=0),
        dict(cin=8, cout=48, k=(8, 1), s=(4, 1), p=(2, 0), d=(1, 1), hw=(256, 37), act=2),
        dict(cin=37, cout=64, k=(3, 3), s=(1, 1), p=(8, 4), d=(8, 4), hw=(64, 96), act=1),  # VR 5.1 ASPP geometry: dilation (8, 4), K not a multiple of 64
        dict(cin=20, cout=17, k=(1, 3), s=(1, 1), p=(0, 2), d=(1, 2), hw=(1, 900), act=4),
    ],
)
def test_conv2d_fp16(L, geom, packed):
    _lib, ops = L
    g = torch.Generator().manual_seed(geom["cin"] * 7 + geom["cout"])
    x = torch.randn((2, geom["cin"]) + geom["hw"], generator=g)
    fan = geom["cin"] * geom["k"][0] * geom["k"][1]
    w = torch.randn((geom["cout"], geom["cin"]) + geom["k"], generator=g) / fan**0.5
    b = torch.randn(geom["cout"], generator=g)
    act = ACTS[geom["act"]]
    conv = lambda xx, ww: F.conv2d(xx, ww, stride=geom["s"], padding=geom["p"], dilation=geom["d"])  # noqa: E731
    wb = torch.from_numpy(ops.block_conv_weight(w.numpy())).cuda()
    if packed:
        got = ops.conv2d(x.cuda(), wb, b.cuda(), geom["cout"], geom["k"], geom["s"], geom["p"], geom["d"][1], act=geom["act"], dh=geom["d"][0], math=_lib.MATH_FP16)
    else:  # no packed image: the producer warps round the weights themselves
        (kh, kw), (sh, sw), (ph, pw), (dh, dw) = geom["k"], geom["s"], geom["p"], geom["d"]
        H, W = geom["hw"]
        Ho, Wo = (H + 2 * ph - dh * (kh - 1) - 1) // sh + 1, (W + 2 * pw - dw * (kw - 1) - 1) // sw + 1
        got = torch.empty((2, geom["cout"], Ho, Wo), device="cuda")
        xd, bd = x.cuda(), b.cuda()
        _lib.check(_lib.lib.b200sep_conv2d_f32_math(p(xd), p(wb), p(bd), None, p(got), 2, geom["cin"], H, W, geom["cout"], Ho, Wo, kh, kw, sh, sw, ph, pw, dh, dw,
                                                    geom["act"], 0, 0, 1, 0, 0, 0, 0, None, _lib.MATH_FP16, 0), "conv2d_f32_math")
    ref = act(conv(r16(x), r16(w)) + b.double()[:, None, None])
    assert_fp16_close(got, ref, conv(x.double().abs(), w.double().abs()), act(conv(x.double(), w.double()) + b.double()[:, None, None]))


def test_conv2d_fp16_slice_and_add(L):
    _lib, ops = L
    g = torch.Generator().manual_seed(11)
    x = torch.randn((3, 20, 30, 50), generator=g)
    w = torch.randn((33, 20, 3, 3), generator=g) / 13
    b = torch.randn(33, generator=g)
    add = torch.randn((3, 33, 30, 50), generator=g)
    wb = torch.from_numpy(ops.block_conv_weight(w.numpy())).cuda()
    out = torch.full((3, 50, 30, 50), 7.0).cuda()
    ops.conv2d(x.cuda(), wb, b.cuda(), 33, (3, 3), p=(1, 1), act=ops.ACT_RELU, add=add.cuda(), add_before_act=True, out=out, out_c_off=10, math=_lib.MATH_FP16)
    conv = lambda xx, ww: F.conv2d(xx, ww, padding=1)  # noqa: E731
    mag = conv(x.double().abs(), w.double().abs())
    o = out.cpu()
    assert_fp16_close(o[:, 10:43], F.relu(conv(r16(x), r16(w)) + b.double()[:, None, None] + add.double()), mag,
                      F.relu(conv(x.double(), w.double()) + b.double()[:, None, None] + add.double()))
    assert (o[:, :10] == 7).all() and (o[:, 43:] == 7).all()
    got = ops.conv2d(x.cuda(), wb, b.cuda(), 33, (3, 3), p=(1, 1), act=ops.ACT_RELU, add=add.cuda(), math=_lib.MATH_FP16)
    assert_fp16_close(got, F.relu(conv(r16(x), r16(w)) + b.double()[:, None, None]) + add.double(), mag,
                      F.relu(conv(x.double(), w.double()) + b.double()[:, None, None]) + add.double())


@pytest.mark.parametrize("axis", [1, 2])
def test_conv_transpose_fp16(L, axis):
    """nn.ConvTranspose (HTDemucs decoders) as the 2-tap up_axis convolution on the tensor cores, fp16 operands."""
    _lib, ops = L
    g = torch.Generator().manual_seed(20 + axis)
    cin, cout, stride = 64, 48, 4
    if axis == 1:
        x = torch.randn((2, cin, 40, 24), generator=g)
        w = torch.randn((cin, cout, 8, 1), generator=g) / 16
        b = torch.randn(cout, generator=g)
        out_len = 40 * stride
        ct = lambda xx, ww: F.conv_transpose2d(xx, ww, stride=(stride, 1))[..., 2 : 2 + out_len, :]  # noqa: E731
        got = ops.conv_transpose(x.cuda(), torch.from_numpy(ops.block_convtr_weight(w.numpy().reshape(cin, cout, 8), stride)).cuda(), b.cuda(), cout, 1, stride, 2,
                                out_len, ops.ACT_GELU, math=_lib.MATH_FP16)
        act = F.gelu
        bias = b.double()[:, None, None]
    else:
        x = torch.randn((2, cin, 1, 300), generator=g)
        w = torch.randn((cin, cout, 8), generator=g) / 16
        b = torch.randn(cout, generator=g)
        out_len = 1190
        ct = lambda xx, ww: F.conv_transpose1d(xx[:, :, 0], ww, stride=stride)[..., 2 : 2 + out_len][:, :, None]  # noqa: E731
        got = ops.conv_transpose(x.cuda(), torch.from_numpy(ops.block_convtr_weight(w.numpy(), stride)).cuda(), b.cuda(), cout, 2, stride, 2, out_len,
                                math=_lib.MATH_FP16)
        act = lambda t: t  # noqa: E731
        bias = b.double()[:, None, None]
    ref = act(ct(r16(x), r16(w)) + bias)
    assert got.shape == ref.shape
    assert_fp16_close(got, ref, ct(x.double().abs(), w.double().abs()), act(ct(x.double(), w.double()) + bias))


# ------------------------------------------------------------------------------------------------------------------------------- attention
@pytest.mark.parametrize("with_work", [1, 0])
@pytest.mark.parametrize("B,H,Lq,Lk,v_kn", [(2, 3, 200, 1344, 0), (1, 2, 130, 130, 1), (2, 2, 1344, 900, 0), (3, 1, 1101, 1101, 1), (1, 1, 5, 7, 0), (1, 2, 128, 256, 1)])
def test_attention_fp16(L, B, H, Lq, Lk, v_kn, with_work):
    """softmax(alpha Q K^T) V with fp16 Q / K / V and fp16 P (fp32 softmax): against float64 of the rounded operands.  P is rounded before the
    row normalisation in the kernel and after it here, so the bound carries one fp16 rounding of P (2^-11 relative) on top of accumulation."""
    _lib, _ = L
    lib = _lib.lib
    g = torch.Generator().manual_seed(B * 1000 + Lq + Lk)
    D = H * 64
    q, k, v = torch.randn((B, Lq, D), generator=g), torch.randn((B, Lk, D), generator=g), torch.randn((B, Lk, D), generator=g)
    alpha = 0.125
    qd, kd = q.cuda(), k.cuda()
    vd = v.cuda() if v_kn else v.transpose(1, 2).contiguous().cuda()
    o = torch.empty((B, Lq, D), device="cuda")
    work = torch.empty(lib.b200sep_attention_work_floats_math(B, H, Lq, Lk, 1), device="cuda") if with_work else None
    vt_bs, vt_rs = (Lk * D, D) if v_kn else (D * Lk, Lk)
    _lib.check(lib.b200sep_attention_f32_math(p(qd), p(kd), p(vd), p(o), B, H, Lq, Lk, 64, Lq * D, D, Lk * D, D, vt_bs, vt_rs, Lq * D, D, alpha, v_kn, p(work),
                                              _lib.MATH_FP16, 0), "attention_f32_math")
    heads = lambda t: t.view(t.shape[0], t.shape[1], H, 64).transpose(1, 2)  # noqa: E731
    qh, kh, vh = heads(r16(q)), heads(r16(k)), heads(r16(v))
    P = torch.softmax(qh @ kh.transpose(-1, -2) * alpha, dim=-1)
    ref = (r16(P) @ vh).transpose(1, 2).reshape(B, Lq, D)
    smax = float((heads(q.double().abs()) @ heads(k.double().abs()).transpose(-1, -2)).max() * alpha)
    pv = (P @ vh.abs()).transpose(1, 2).reshape(B, Lq, D)
    err = (o.cpu().double() - ref).abs()
    tol = (2.0**-11 + RTOL * smax) * pv + 1e-6
    assert (err <= tol).all(), float((err / tol).max())
    exact = (torch.softmax(heads(q.double()) @ heads(k.double()).transpose(-1, -2) * alpha, -1) @ heads(v.double())).transpose(1, 2).reshape(B, Lq, D)
    assert float((o.cpu().double() - exact).abs().max()) > 1e-5  # fp16 operands, not the ~1e-7 of the bf16x3 mode


# ------------------------------------------------------------------------------------------------------------------------------- shape rule
def test_shape_rule_matches_the_library(L):
    """tests/fp16_operands.py restates which launches the library sends to the tensor cores.  On either side of every threshold of that rule the
    fp16 mode must change the result exactly when the restated rule says tensor core (the SIMT kernels are fp32 in both modes, bit for bit)."""
    from fp16_operands import tc_conv_usable, tc_gemm_usable

    _lib, ops = L
    lib = _lib.lib
    g = torch.Generator().manual_seed(9)
    gemms = [(512, 32, 32), (512, 31, 32), (512, 32, 31), (512, 32, 64), (511, 32, 64), (128, 128, 40), (127, 129, 40)]
    for M, N, K in gemms:
        a, w = torch.randn((M, K), generator=g).cuda(), torch.randn((N, K), generator=g).cuda()
        out = {}
        for m in (0, 1):
            out[m] = torch.empty((M, N), device="cuda")
            _lib.check(lib.b200sep_gemm_f32_math(p(a), p(w), p(out[m]), M, N, K, K, K, N, 1, 0, 0, 0, 1.0, None, None, 0, None, None, None, m, 0))
        torch.cuda.synchronize()
        assert torch.equal(out[0], out[1]) != tc_gemm_usable(M, N, K), (M, N, K)
    convs = [(32, 16, 1, 1, 16, 32), (31, 16, 1, 1, 16, 32), (32, 15, 1, 1, 16, 32), (32, 16, 1, 1, 511, 1), (4, 16, 3, 3, 8, 64), (3, 16, 3, 3, 8, 64)]
    for cin, cout, kh, kw, H, W in convs:
        x = torch.randn((1, cin, H, W), generator=g).cuda()
        wb = torch.from_numpy(ops.block_conv_weight(torch.randn((cout, cin, kh, kw), generator=g).numpy())).cuda()
        out = {}
        for m in (0, 1):
            out[m] = torch.empty((1, cout, H, W), device="cuda")
            _lib.check(lib.b200sep_conv2d_f32_math(p(x), p(wb), None, None, p(out[m]), 1, cin, H, W, cout, H, W, kh, kw, 1, 1, kh // 2, kw // 2, 1, 1, 0, 0, 0, 1, 0, 0, 0, 0,
                                                   None, m, 0))
        torch.cuda.synchronize()
        assert torch.equal(out[0], out[1]) != tc_conv_usable(cin, cout, kh, kw, H, W, 1), (cin, cout, kh, kw, H, W)
