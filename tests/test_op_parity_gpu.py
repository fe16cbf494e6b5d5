"""Operator-level parity of the SIMT kernels that the network goldens only reach indirectly: every check calls one C-ABI entry point by name
and compares it with a plain float64 definition of the same operation (torch / NumPy, or the NumPy restatements in oracle/), at the
shapes that select each dispatch variant and at the numeric edges where a kernel goes wrong.

Gates: selection and data movement (copies, permutes, gathers, framing, min / median / select, PCM, range-vs-full) are bit-exact;
normalisations hold |got - ref| <= 1e-5 * max(1, |ref|) per element; the remaining arithmetic holds 2e-6 of max |ref|.  Output buffers are
filled with NaN or a sentinel first, so an element a kernel never writes fails, and padding a kernel must not touch is checked to still hold it."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

import vr_oracle as V

pytestmark = pytest.mark.gpu

SENTINEL = 12345.0
ERR_ARG = -1


@pytest.fixture(scope="module")
def L(lib_built):
    assert torch.cuda.is_available()
    from audio_separator.separator.b200 import _lib

    return _lib


def gen(seed):
    return torch.Generator().manual_seed(seed)


def cu(t):
    return t.contiguous().cuda()


_ALIVE = []  # tensors whose pointers were handed to the library: a temporary like p(cu(x)) must outlive the launch that reads it


def p(t):
    if t is None:
        return None
    _ALIVE.append(t)
    return t.data_ptr()


def run(L, rc, what):
    L.check(rc, what)
    torch.cuda.synchronize()
    _ALIVE.clear()


def assert_norm(got, ref, what=""):
    """normalisations: |got - ref| <= 1e-5 * max(1, |ref|) for every element (NaN fails)"""
    got = got.detach().cpu().double()
    err = ((got - ref).abs() / ref.abs().clamp_min(1.0)).max().item()
    assert err <= 1e-5, f"{what}: max scaled error {err:.3e}"


def assert_arith(got, ref, what="", tol=2e-6):
    """other arithmetic: max |got - ref| <= tol * max |ref| (NaN fails)"""
    got = got.detach().cpu().double()
    err = (got - ref).abs().max().item()
    scale = max(ref.abs().max().item(), 1e-30)
    assert err <= tol * scale, f"{what}: max error {err:.3e} = {err / scale:.3e} of max|ref| {scale:.3e}"


def act_ref(y, act):
    return {0: y, 1: F.relu(y), 2: F.gelu(y)}[act]


# ================================================================================================================ reductions and normalisations
def gn1_ref(x, gamma, beta, Fr, channel_last, act):
    xd = x.double()
    if channel_last:  # (B, L, C) tokens
        y = F.group_norm(xd.transpose(1, 2), 1, gamma.double(), beta.double(), eps=1e-5).transpose(1, 2)
    else:  # (B, C, Fr, L): one sample per (b, fr) row
        B, C, _, Lq = x.shape
        y = F.group_norm(xd.permute(0, 2, 1, 3).reshape(B * Fr, C, Lq), 1, gamma.double(), beta.double(), eps=1e-5)
        y = y.reshape(B, Fr, C, Lq).permute(0, 2, 1, 3)
    return act_ref(y, act)


def gn1_call(L, x, gamma, beta, y, B, C, Fr, Lq, act, channel_last):
    work = torch.empty(L.lib.b200sep_groupnorm1_work_floats(B, C, Fr, Lq), device="cuda")
    run(L, L.lib.b200sep_groupnorm1_f32(p(x), p(gamma), p(beta), p(y), B, C, Fr, Lq, act, channel_last, p(work), None), "groupnorm1_f32")


# (B, C, Fr, L, channel_last): sample sizes C*L around the one-CTA / several-CTA switch (65536 elements per CTA), a ragged 2^20 + 3, and one
# time-branch sample of the full-size HTDemucs (96 x 85995, 125 CTAs)
GN1_CASES = [(2, 5, 1, 13107, 0), (1, 1, 1, 131071, 0), (1, 64, 2, 2048, 0), (1, 7, 1, 149797, 1), (1, 96, 1, 85995, 0)]


@pytest.mark.parametrize("B,C,Fr,Lq,cl", GN1_CASES)
def test_groupnorm1_partition_sizes(L, B, C, Fr, Lq, cl):
    g = gen(C * 7 + Lq)
    shape = (B, Lq, C) if cl else (B, C, Fr, Lq)
    x = torch.randn(shape, generator=g) * 2 + 0.5
    ga, be = torch.rand(C, generator=g) + 0.5, torch.randn(C, generator=g)
    xd, gd, bd = cu(x), cu(ga), cu(be)
    for act in (0, 1, 2):
        ref = gn1_ref(x, ga, be, Fr, cl, act)
        y = torch.full_like(xd, float("nan"))
        gn1_call(L, xd, gd, bd, y, B, C, Fr, Lq, act, cl)
        assert_norm(y, ref, f"act {act}")
        xi = xd.clone()  # in place, as the networks use it: the same bits
        gn1_call(L, xi, gd, bd, xi, B, C, Fr, Lq, act, cl)
        assert torch.equal(xi, y)


@pytest.mark.parametrize("kind", ["constant", "mean1e3", "outlier30", "outlier300"])
def test_groupnorm1_numeric_edges(L, kind):
    """2^18-element samples (4 CTAs).  The partial sums are taken relative to the sample's first element; an outlier there must not cost accuracy."""
    B, C, Lq = 2, 4, 65536
    g = gen(11)
    x = torch.randn(B, C, 1, Lq, generator=g)
    if kind == "constant":
        x = torch.full_like(x, 0.37)
    elif kind == "mean1e3":
        x = x + 1e3
    else:
        x[:, 0, 0, 0] = 30.0 if kind == "outlier30" else 300.0
    ga, be = torch.rand(C, generator=g) + 0.5, torch.randn(C, generator=g)
    y = torch.full((B, C, 1, Lq), float("nan"), device="cuda")
    gn1_call(L, cu(x), cu(ga), cu(be), y, B, C, 1, Lq, 0, 0)
    if kind == "constant":  # zero variance: x - mean is exactly 0, so the output is beta bit for bit
        assert torch.equal(y.cpu(), be[None, :, None, None].expand_as(x))
    else:
        assert_norm(y, gn1_ref(x, ga, be, 1, 0, 0), kind)


def test_groupnorm_groups_multi_cta(L):
    B, C, G, X = 2, 16, 4, 40000  # 160000 elements per group: 2 CTAs
    g = gen(12)
    x = torch.randn(B, C, X, generator=g) * 1.5 - 0.3
    x[:, 4, 0] = 25.0  # the first element of group 1 is an outlier
    ga, be = torch.rand(C, generator=g) + 0.5, torch.randn(C, generator=g)
    for act in (0, 2):
        y = torch.full((B, C, X), float("nan"), device="cuda")
        work = torch.empty(L.lib.b200sep_groupnorm_work_floats(B, C, G, X), device="cuda")
        run(L, L.lib.b200sep_groupnorm_f32(p(cu(x)), p(cu(ga)), p(cu(be)), p(y), B, C, G, X, act, p(work), None), "groupnorm_f32")
        assert_norm(y, act_ref(F.group_norm(x.double(), G, ga.double(), be.double(), eps=1e-5), act), f"act {act}")


@pytest.mark.parametrize("C", [1, 31, 32, 33, 512, 1536])
@pytest.mark.parametrize("offset", [0.0, 100.0])
def test_layernorm(L, C, offset):
    """a row mean of 100 at std 1: fp32 sums of the raw values and an fp32-rounded mean would cost 1e-5 to 2e-5 here"""
    g = gen(C)
    x = torch.randn(37, C, generator=g) + offset
    ga, be = torch.rand(C, generator=g) + 0.5, torch.randn(C, generator=g)
    y = torch.full((37, C), float("nan"), device="cuda")
    run(L, L.lib.b200sep_layernorm_f32(p(cu(x)), p(cu(ga)), p(cu(be)), p(y), 37, C, None), "layernorm_f32")
    assert_norm(y, F.layer_norm(x.double(), (C,), ga.double(), be.double(), eps=1e-5))


@pytest.mark.parametrize("C", [1, 37, 512])
def test_rmsnorm_slices_and_zero_row(L, C):
    g = gen(C + 1)
    rows, ld_in, ld_out = 50, C + 5, C + 3
    xf = torch.randn(rows, ld_in, generator=g) * 3
    xf[3, :C] = 0.0  # F.normalize clamps the norm at 1e-12: an all-zero row gives 0, not NaN
    ga = torch.rand(C, generator=g) + 0.5
    y = torch.full((rows, ld_out), SENTINEL, device="cuda")
    y[:, :C] = float("nan")
    run(L, L.lib.b200sep_rmsnorm_f32(p(cu(xf)), p(cu(ga)), p(y), rows, C, ld_in, ld_out, None), "rmsnorm_f32")
    xd = xf[:, :C].double()
    ref = xd / xd.norm(dim=-1, keepdim=True).clamp_min(1e-12) * C**0.5 * ga.double()
    assert_norm(y[:, :C], ref)
    assert torch.equal(y[3, :C].cpu(), torch.zeros(C))
    assert (y[:, C:] == SENTINEL).all()


@pytest.mark.parametrize("n", [1, 64, 65, 256, 257, 832, 833, 2048, 2049, 4097])
def test_softmax_rows_dispatch(L, n):
    """warp-per-row kernels for n <= 64 / 256 / 832, then one CTA per row (registers up to 2048 columns, strided above)"""
    g = gen(n)
    rows, ld = 13, n + 3
    x = torch.randn(rows, ld, generator=g) * 5
    x[1, 2::3] = -float("inf")  # masked entries (column 0 stays finite, so no row is all -inf)
    x[2, :n] = 0.7  # equal values: 1/n each
    x[3] *= 1e3  # exp underflows for everything but the maximum
    x[:, n:] = SENTINEL
    ref = torch.softmax(x[:, :n].double(), dim=-1)
    xd = cu(x)
    run(L, L.lib.b200sep_softmax_rows_f32(p(xd), rows, n, ld, None), "softmax_rows_f32")
    for r in range(rows):
        assert_arith(xd[r, :n], ref[r], f"row {r}")
    assert (xd[:, n:] == SENTINEL).all()


@pytest.mark.parametrize("n", [32767, 32768, 32769, 100003])
def test_meanstd_and_batch(L, n):
    """kMsBlocks x 256 = 32768 is the grid stride of the partial pass; the batched form must give the single-sample bits"""
    g = gen(n)
    for batch in (1, 3):
        stride = n + 17
        x = torch.randn(batch, stride, generator=g) * 3 + 0.7
        xd = cu(x)
        out = torch.full((batch, 4), float("nan"), device="cuda")
        work = torch.empty(L.lib.b200sep_meanstd_work_floats(batch), device="cuda")
        run(L, L.lib.b200sep_meanstd_batch_f32(p(xd), n, batch, stride, p(out), 4, p(work), None), "meanstd_batch_f32")
        for z in range(batch):
            one = torch.full((2,), float("nan"), device="cuda")
            run(L, L.lib.b200sep_meanstd_f32(p(xd[z]), n, p(one), None), "meanstd_f32")
            assert torch.equal(out[z, :2], one)
            v = x[z, :n].double()
            assert_norm(one, torch.stack([v.mean(), v.std()]))
        assert out[:, 2:].isnan().all()


def test_absmax_and_normalize(L):
    res = torch.full((1,), float("nan"), device="cuda")
    x = torch.full((4,), 3.0, device="cuda")
    run(L, L.lib.b200sep_absmax(p(x), 0, p(res), None), "absmax")
    assert res.item() == 0.0
    run(L, L.lib.b200sep_absmax(p(cu(torch.tensor([-0.625]))), 1, p(res), None), "absmax")
    assert res.item() == 0.625
    g = gen(3)
    x = torch.rand(1025, generator=g) - 0.5
    x[-1] = -0.75  # a negative extremum at the last index
    xd = cu(x)
    run(L, L.lib.b200sep_absmax(p(xd), 1025, p(res), None), "absmax")
    assert res.item() == 0.75
    # spec_utils.normalize: scale down above max_peak, up below min_peak (min_peak >= 0), else leave alone
    # (min_peak < 0 disables the scale-up, but the peak is never negative, so that guard cannot change a result and has no case here)
    for max_peak, min_peak, s in [(0.5, 0.0, 0.5 / 0.75), (0.9, 0.8, 0.8 / 0.75), (0.9, 0.1, 1.0), (0.75, 0.75, 1.0)]:
        y = torch.full_like(xd, float("nan"))
        run(L, L.lib.b200sep_normalize(p(xd), 1025, p(res), max_peak, min_peak, p(y), None), "normalize")
        assert_arith(y, x.double() * s, f"max_peak {max_peak} min_peak {min_peak}")


def pcm_ref(x, bits, via_int16):
    """the writers' integers (test_abi_and_host.py): pydub's int16 widened by a shift, or libsndfile's lrint(x * (2^(bits-1) - 1)) (PCM_32: x * 2^31, saturated)"""
    if via_int16:
        return (x * np.float32(32767)).astype(np.int16).astype(np.int64) << (bits - 16)
    if bits == 32:
        return np.clip(np.rint(x.astype(np.float64) * 2147483648.0), -(2**31), 2**31 - 1).astype(np.int64)
    return np.rint(x * np.float32((1 << (bits - 1)) - 1)).astype(np.int64)


def half_ties(scale, count):
    """float32 x whose float32 product with `scale` is exactly k + 0.5, for even and odd k (round half to even must pick k or k + 1)"""
    out = []
    for k in range(1, 400000, 997):
        x = np.float32((k + 0.5) / scale)
        for cand in (x, np.nextafter(x, np.float32(0)), np.nextafter(x, np.float32(1))):
            if np.float32(cand * np.float32(scale)) == k + 0.5:
                out.append(cand)
                break
        if len(out) >= count:
            break
    assert len(out) >= 8 and len({int(np.floor(v * np.float32(scale))) % 2 for v in out}) == 2
    return np.array(out, np.float32)


@pytest.mark.parametrize("bits", [16, 24, 32])
@pytest.mark.parametrize("via_int16", [0, 1])
def test_pcm_bytes(L, bits, via_int16):
    g = np.random.default_rng(bits + via_int16)
    if bits == 32:
        ties = (2 * np.arange(1, 40, dtype=np.float64) + 1) / 2**32  # x * 2^31 = k + 0.5 exactly in double
        ties = ties.astype(np.float32)
    else:
        ties = half_ties((1 << (bits - 1)) - 1, 40)
    x = np.concatenate([[1.0, -1.0, 0.0, -0.0, 0.5, -0.5], ties, -ties, g.uniform(-1, 1, 1000)]).astype(np.float32)
    width = bits // 8
    y = torch.full((x.size * width + 5,), 0xA5, dtype=torch.uint8, device="cuda")
    run(L, L.lib.b200sep_to_pcm_bytes(p(cu(torch.from_numpy(x))), x.size, bits, via_int16, p(y), None), "to_pcm_bytes")
    want = pcm_ref(x, bits, via_int16)
    if bits == 32 and not via_int16:
        assert want[0] == 2**31 - 1 and want[1] == -(2**31)  # +1.0 saturates
    wb = ((want[:, None] >> (8 * np.arange(width))) & 0xFF).astype(np.uint8).reshape(-1)
    got = y.cpu().numpy()
    assert np.array_equal(got[: x.size * width], wb)
    assert (got[x.size * width :] == 0xA5).all()


def test_to_pcm16(L):
    g = np.random.default_rng(5)
    ties = half_ties(32767, 40)
    x = np.concatenate([[1.0, -1.0, 0.0], ties, -ties, g.uniform(-1, 1, 1000)]).astype(np.float32)
    y = torch.full((x.size,), 0x5A5A, dtype=torch.int16, device="cuda")
    run(L, L.lib.b200sep_to_pcm16(p(cu(torch.from_numpy(x))), x.size, p(y), None), "to_pcm16")
    assert np.array_equal(y.cpu().numpy(), (x * np.float32(32767)).astype(np.int16))  # truncation toward zero


# ================================================================================================================ layout and element-wise kernels
PERMS3 = [(0, 1, 2), (0, 2, 1), (1, 0, 2), (1, 2, 0), (2, 0, 1), (2, 1, 0)]


@pytest.mark.parametrize("perm", PERMS3)
def test_permute4_vector_and_scalar_paths(L, perm):
    g = gen(sum(perm) * 10 + perm[0])
    for d3, offset in ((8, 0), (6, 0), (8, 1)):  # float4 path; d3 % 4 != 0; a pointer one float off 16-byte alignment
        d = (3, 5, 7, d3)
        x = torch.randn(d, generator=g)
        buf = torch.zeros(x.numel() + 4, device="cuda")
        buf[offset : offset + x.numel()] = cu(x).reshape(-1)
        out = torch.full((x.numel() + 4,), float("nan"), device="cuda")
        run(L, L.lib.b200sep_permute4_f32(p(buf[offset:]), p(out[offset:]), *d, *perm, 3, None), "permute4_f32")
        want = x.permute(*perm, 3).contiguous().reshape(-1)
        assert torch.equal(out[offset : offset + x.numel()].cpu(), want)
    # a permutation that moves the innermost dimension (scalar path only)
    x = torch.randn(2, 3, 4, 8, generator=g)
    out = torch.full((192,), float("nan"), device="cuda")
    run(L, L.lib.b200sep_permute4_f32(p(cu(x)), p(out), 2, 3, 4, 8, 3, *perm, None), "permute4_f32")
    assert torch.equal(out.cpu(), x.permute(3, *perm).contiguous().reshape(-1))


def test_gate_merge_heads(L):
    g = gen(21)
    B, n, H = 2, 37, 4
    outs = {}
    for dh, offset in ((64, 0), (6, 0), (64, 1)):  # float4 path; dh % 4 != 0; an unaligned output (scalar path)
        o = torch.randn(B, H, n, dh, generator=g) if dh not in outs else outs[dh][0]
        gates = torch.randn(B * n, H, generator=g) * 3 if dh not in outs else outs[dh][1]
        y = torch.full((B * n * H * dh + 4,), float("nan"), device="cuda")
        run(L, L.lib.b200sep_gate_merge_heads_f32(p(cu(o)), p(cu(gates)), p(y[offset:]), B, n, H, dh, None), "gate_merge_heads_f32")
        got = y[offset : offset + B * n * H * dh].reshape(B * n, H * dh)
        ref = (o.double().permute(0, 2, 1, 3).reshape(B * n, H, dh) * torch.sigmoid(gates.double())[:, :, None]).reshape(B * n, H * dh)
        assert_arith(got, ref, f"dh {dh} offset {offset}")
        if dh in outs:
            assert torch.equal(got, outs[dh][2])  # both paths compute the same bits
        else:
            outs[dh] = (o, gates, got.clone())


def test_rope_split_heads(L):
    """positions up to 1100: the angle is the float32 product pos * freq (rotary-embedding-torch), its sine and cosine taken in fp64 here"""
    g = gen(22)
    B, n, H, dh = 2, 1101, 3, 64
    qkv = torch.randn(B, n, 3, H, dh, generator=g)
    freqs = (1.0 / 10000 ** (torch.arange(0, dh, 2).float() / dh)).float()
    q, k, v = (torch.full((B, H, n, dh), float("nan"), device="cuda") for _ in range(3))
    run(L, L.lib.b200sep_rope_split_heads_f32(p(cu(qkv)), p(cu(freqs)), p(q), p(k), p(v), B, n, H, dh, None), "rope_split_heads_f32")
    ang = (torch.arange(n).float()[:, None] * freqs[None, :]).double()  # (n, dh/2), the fp32 product
    cs, sn = ang.cos()[None, None], ang.sin()[None, None]

    def rot(t):  # (B, n, H, dh) -> (B, H, n, dh) with interleaved pairs rotated
        t = t.double().permute(0, 2, 1, 3)
        a, b = t[..., 0::2], t[..., 1::2]
        return torch.stack([a * cs - b * sn, b * cs + a * sn], dim=-1).reshape(t.shape)

    assert_arith(q, rot(qkv[:, :, 0]), "q")
    assert_arith(k, rot(qkv[:, :, 1]), "k")
    assert torch.equal(v.cpu(), qkv[:, :, 2].permute(0, 2, 1, 3).contiguous())


def test_glu_and_glu_rows(L):
    g = gen(23)
    a = torch.randn(2, 12, 5, 33, generator=g) * 3
    res, sc = torch.randn(2, 6, 5, 33, generator=g), torch.rand(6, generator=g)
    y = torch.full((2, 6, 5, 33), float("nan"), device="cuda")
    run(L, L.lib.b200sep_glu_f32(p(cu(a)), None, None, p(y), 2, 6, 5 * 33, None), "glu_f32")
    assert_arith(y, F.glu(a.double(), 1))
    run(L, L.lib.b200sep_glu_f32(p(cu(a)), p(cu(res)), p(cu(sc)), p(y), 2, 6, 5 * 33, None), "glu_f32")
    assert_arith(y, res.double() + sc.double()[None, :, None, None] * F.glu(a.double(), 1))
    rows, C = 37, 45
    ld_in, ld_out = 2 * C + 7, C + 5
    a = torch.randn(rows, ld_in, generator=g) * 3
    y = torch.full((rows, ld_out), SENTINEL, device="cuda")
    y[:, :C] = float("nan")
    run(L, L.lib.b200sep_glu_rows_f32(p(cu(a)), p(y), rows, C, ld_in, ld_out, None), "glu_rows_f32")
    assert_arith(y[:, :C], F.glu(a[:, : 2 * C].double(), -1))
    assert (y[:, C:] == SENTINEL).all()


def test_copy4_broadcast_into_channel_slice(L):
    g = gen(24)
    src = torch.randn(5, 9, generator=g)
    dst = torch.full((3, 12, 4, 9), SENTINEL, device="cuda")
    # src (5, 9) broadcast over d0 = 3 and d2 = 4 (zero strides) into channels [4, 9) of dst
    run(L, L.lib.b200sep_copy4_f32(p(cu(src)), p(dst[:, 4:]), 3, 5, 4, 9, 0, 9, 0, 1, 12 * 36, 36, 9, 1, None), "copy4_f32")
    want = torch.full((3, 12, 4, 9), SENTINEL)
    want[:, 4:9] = src[None, :, None, :]
    assert torch.equal(dst.cpu(), want)


@pytest.mark.parametrize("H,W", [(1, 17), (13, 1), (1, 1), (5, 7)])
def test_mean_h_and_upsample2x_edges(L, H, W):
    g = gen(H * 31 + W)
    x = torch.randn(2, 3, H, W, generator=g)
    y = torch.full((6, W), float("nan"), device="cuda")
    run(L, L.lib.b200sep_mean_h_f32(p(cu(x)), p(y), 6, H, W, None), "mean_h_f32")
    assert_arith(y, x.double().reshape(6, H, W).mean(1))
    up = torch.full((2, 7, 2 * H, 2 * W), SENTINEL, device="cuda")
    run(L, L.lib.b200sep_upsample2x_bilinear_f32(p(cu(x)), p(up), 2, 3, H, W, 7, 2, None), "upsample2x_bilinear_f32")
    ref = F.interpolate(x.double(), scale_factor=2, mode="bilinear", align_corners=True)
    assert_arith(up[:, 2:5], ref)
    assert (up[:, :2] == SENTINEL).all() and (up[:, 5:] == SENTINEL).all()


def test_add_rowvec_and_ew(L):
    g = gen(25)
    x = torch.randn(3, 10, 77, generator=g)
    v = torch.randn(10, generator=g)
    xd = cu(x)
    run(L, L.lib.b200sep_add_rowvec_f32(p(xd), p(cu(v)), 3, 10, 77, None), "add_rowvec_f32")
    assert torch.equal(xd.cpu(), x + v[None, :, None])
    n = 10007
    a, b = torch.randn(n, generator=g) * 3, torch.randn(n, generator=g)
    st = torch.tensor([0.7, 2.5])
    ad, bd, sd = cu(a), cu(b), cu(st)
    cases = [(0, bd, 1.5, -0.25, 1.5 * a.double() - 0.25 * b.double()), (0, None, 1.5, -0.25, 1.5 * a.double() - 0.25),
             (1, bd, 1.0, 0.0, a.double() * b.double()), (2, sd, 1.0, 0.0, (a.double() - 0.7) / (1e-5 + 2.5)), (3, sd, 1.0, 0.0, a.double() * 2.5 + 0.7)]
    for op, bb, alpha, beta, ref in cases:
        out = torch.full((n,), float("nan"), device="cuda")
        run(L, L.lib.b200sep_ew_f32(p(ad), p(bb), p(out), n, alpha, beta, op, None), "ew_f32")
        assert_arith(out, ref, f"op {op}")


def test_tc_pack_conv_weights_plain_is_bf16x3(L):
    """the entry without the _math suffix packs the BF16X3 image: the same bytes as tc_pack_conv_weights_math(..., BF16X3)"""
    g = gen(26)
    cin, taps, cout = 20, 9, 50
    wb = torch.zeros(cin, taps, -(-cout // 48) * 48)
    wb[:, :, :cout] = torch.randn(cin, taps, cout, generator=g)
    wd = cu(wb)
    nfl = L.lib.b200sep_tc_packed_floats(cout, -(-cin // 8) * 8 * taps)
    assert nfl > 0
    a = torch.full((nfl,), SENTINEL, device="cuda")
    b = torch.full((nfl,), SENTINEL, device="cuda")
    run(L, L.lib.b200sep_tc_pack_conv_weights(p(wd), cin, taps, cout, p(a), None), "tc_pack_conv_weights")
    run(L, L.lib.b200sep_tc_pack_conv_weights_math(p(wd), cin, taps, cout, p(b), L.MATH_BF16X3, None), "tc_pack_conv_weights_math")
    assert torch.equal(a.view(torch.int32), b.view(torch.int32))
    assert not (a == SENTINEL).all()


# ================================================================================================================ VR mask path
def planes_to_complex(s):
    s = s.double().numpy()
    return np.stack([s[0] + 1j * s[1], s[2] + 1j * s[3]])


def test_vr_magnitude_pad(L):
    g = gen(31)
    bins, frames, frames_out, pad_l = 33, 50, 70, 7
    spec = torch.randn(4, bins, frames, generator=g)
    mag = torch.full((2, bins, frames_out), float("nan"), device="cuda")
    run(L, L.lib.b200sep_vr_magnitude_pad(p(cu(spec)), p(mag), bins, frames, frames_out, pad_l, None), "vr_magnitude_pad")
    assert_arith(mag[:, :, pad_l : pad_l + frames], torch.from_numpy(np.abs(planes_to_complex(spec))))
    # the padding is the caller's zero fill: the kernel never writes it
    assert mag[:, :, :pad_l].isnan().all() and mag[:, :, pad_l + frames :].isnan().all()


EXPS = (1.1, 1.35, 0.8, 1.0)  # left below / from split_bin, right below / from split_bin (1.0 skips the power)


def mask_pow_ref(mask, split_bin, e=EXPS):
    m = mask.double().clone()
    m[0, :split_bin] **= e[0]
    m[0, split_bin:] **= e[1]
    m[1, :split_bin] **= e[2]
    m[1, split_bin:] **= e[3]
    return m


@pytest.mark.parametrize("special", [False, True])
def test_vr_apply_mask(L, special):
    g = gen(32 + special)
    bins, frames, stride = 37, 41, 48
    mask = torch.rand(2, bins, stride, generator=g)
    spec = torch.randn(4, bins, frames, generator=g)
    if special:  # non-finite spectrogram entries come out as 0 (np.nan_to_num), in one component or both
        spec[0, 3, 5], spec[1, 4, 6], spec[2, 7, 8], spec[3, 9, 10] = float("inf"), -float("inf"), float("nan"), float("inf")
        spec[0, 11, 12] = spec[1, 11, 12] = float("inf")
        mask[0, 3, 5] = 0.0  # 0 * inf
    X = planes_to_complex(spec)
    for split_bin in (0, bins // 3, bins):
        m = mask_pow_ref(mask, split_bin)[:, :, :frames].numpy()
        with np.errstate(invalid="ignore", over="ignore"):  # the reference's product: mask * |X| * exp(i angle X) (vr_separator.py:329-343)
            want_y = np.nan_to_num(m * np.abs(X) * np.exp(1j * np.angle(X)), nan=0, posinf=0, neginf=0)
            want_v = np.nan_to_num((1 - m) * np.abs(X) * np.exp(1j * np.angle(X)), nan=0, posinf=0, neginf=0)
        y = torch.full((4, bins, frames), float("nan"), device="cuda")
        v = torch.full((4, bins, frames), float("nan"), device="cuda")
        run(L, L.lib.b200sep_vr_apply_mask(p(cu(mask)), stride, p(cu(spec)), bins, frames, split_bin, *EXPS, p(y), p(v), None), "vr_apply_mask")
        for got, want in ((y, want_y), (v, want_v)):
            ref = torch.from_numpy(np.stack([want.real[0], want.imag[0], want.real[1], want.imag[1]]))
            assert_arith(got, ref, f"split_bin {split_bin}")


def test_vr_mask_pow_frame_min_merge(L):
    g = gen(33)
    bins, frames, stride = 37, 300, 310  # frames not a multiple of the 128-thread CTAs or 256
    mask = torch.rand(2, bins, stride, generator=g) * 0.9 + 0.05
    mask[:, :, frames:] = SENTINEL
    for split_bin in (0, 12, bins):
        md = cu(mask)
        run(L, L.lib.b200sep_vr_mask_pow(p(md), stride, bins, frames, split_bin, *EXPS, None), "vr_mask_pow")
        assert_arith(md[:, :, :frames], mask_pow_ref(mask[:, :, :frames], split_bin))
        assert (md[:, :, frames:] == SENTINEL).all()
    mask[1, 20, 299] = 0.001  # the minimum at the last frame
    md = cu(mask)
    fm = torch.full((frames + 3,), float("nan"), device="cuda")
    run(L, L.lib.b200sep_vr_frame_min(p(md), stride, 2 * bins, frames, p(fm), None), "vr_frame_min")
    assert torch.equal(fm[:frames].cpu(), mask[:, :, :frames].reshape(2 * bins, frames).min(0).values)  # y_mask.min(axis=(0, 1))
    assert fm[frames:].isnan().all()
    w = torch.rand(frames, generator=g)
    run(L, L.lib.b200sep_vr_mask_merge(p(md), p(cu(w)), stride, 2 * bins, frames, None), "vr_mask_merge")
    m = mask[:, :, :frames].double()
    assert_arith(md[:, :, :frames], m + w.double() * (1 - m))  # y_mask += weight * (1 - y_mask)
    assert (md[:, :, frames:] == SENTINEL).all()


def test_vr_mirror_high_end(L):
    g = gen(34)
    bins, frames, high_rows, high_frames, band_bins, h, max_bin, pfs = 100, 20, 12, 24, 80, 10, 70, 60
    spec_m = torch.randn(4, bins, frames, generator=g)
    high = torch.randn(4, high_rows, high_frames, generator=g) * 1.5  # about half the entries exceed the mirror's magnitude
    high[0:2, 2, 3] = 0.0  # |input| = 0: kept
    spec_m[0:2, pfs - 11 - 4, 5] = 0.0  # |mirror| = 0: the input is replaced by 0
    band = torch.full((4, band_bins, frames), SENTINEL, device="cuda")
    run(L, L.lib.b200sep_vr_mirror_high_end(p(cu(spec_m)), bins, p(cu(high)), high_rows, high_frames, p(band), band_bins, frames, h, max_bin, pfs, None),
        "vr_mirror_high_end")
    want = V.mirroring(planes_to_complex(spec_m), planes_to_complex(high)[:, :h, :frames], {"pre_filter_start": pfs})
    ref = torch.from_numpy(np.stack([want.real[0], want.imag[0], want.real[1], want.imag[1]]))
    assert_arith(band[:, max_bin - h : max_bin], ref)
    kept = np.abs(planes_to_complex(high)[:, :h, :frames]) <= np.abs(want) * (1 + 1e-6)
    assert kept.any() and (~kept).any()  # both branches taken
    assert (band[:, : max_bin - h] == SENTINEL).all() and (band[:, max_bin:] == SENTINEL).all()


def test_bin_gain_filter_masks(L):
    g = gen(35)
    bins, frames = 64, 30
    x = torch.randn(4, bins, frames, generator=g)
    for gain in (V.lp_filter_mask(bins, 20, 40)[:, 0], V.hp_filter_mask(bins, 40, 20)[:, 0]):
        gf = torch.from_numpy(gain.astype(np.float32))
        xd = cu(x)
        run(L, L.lib.b200sep_bin_gain_f32(p(xd), p(cu(gf)), 4, bins, frames, None), "bin_gain_f32")
        assert torch.equal(xd.cpu(), x * gf[None, :, None])


# ================================================================================================================ overlap-adds and framing
def covering(q_begin, q_end, shift, chunk_len, step, n_chunks):
    """global indices [lo, hi] of the chunks placed every `step` that cover positions [q_begin + shift, q_end + shift)"""
    p0, p1 = q_begin + shift, q_end - 1 + shift
    lo = 0 if p0 - chunk_len + 1 <= 0 else (p0 - chunk_len + step) // step
    return lo, min(p1 // step, n_chunks - 1)


@pytest.mark.parametrize("interleave", [0, 1])
@pytest.mark.parametrize("use_window", [0, 1])
def test_demix_overlap_add_ranges_equal_full(L, interleave, use_window):
    g = gen(41)
    n_chunks, chunk_len, step, trim, n_out = 6, 1000, 700, 150, 4000
    total_len = (n_chunks - 1) * step + 900  # the last chunk is clipped
    chunks = cu(torch.randn(n_chunks, 2, chunk_len, generator=g))
    mix = cu(torch.randn(2, n_out, generator=g))
    shape = (n_out, 2) if interleave else (2, n_out)
    full_p, full_s = torch.full(shape, float("nan"), device="cuda"), torch.full(shape, float("nan"), device="cuda")
    run(L, L.lib.b200sep_demix_overlap_add(p(chunks), n_chunks, chunk_len, step, total_len, trim, n_out, use_window, 1.25, p(mix), 0.97, interleave, p(full_p), p(full_s), None),
        "demix_overlap_add")
    got_p, got_s = torch.full(shape, float("nan"), device="cuda"), torch.full(shape, float("nan"), device="cuda")
    for qb, qe in ((0, 900), (900, 2300), (2300, 3100), (3100, n_out)):
        lo, hi = covering(qb, qe, trim, chunk_len, step, n_chunks)
        loc = chunks[lo : hi + 1].contiguous()
        if interleave:  # a rank holds only its rows of the stems and its samples of the mix
            sp, ss = torch.full((qe - qb, 2), float("nan"), device="cuda"), torch.full((qe - qb, 2), float("nan"), device="cuda")
            msl = mix[:, qb:qe].contiguous()
            run(L, L.lib.b200sep_demix_overlap_add_range_ex(p(loc), lo, hi + 1 - lo, n_chunks, chunk_len, step, total_len, trim, n_out, qb, qe, use_window, 1.25, p(msl), qe - qb,
                                                             qb, 0.97, 1, p(sp), p(ss), qb, None), "demix_overlap_add_range_ex")
            got_p[qb:qe], got_s[qb:qe] = sp, ss
        else:  # planar output is written into full-length rows
            run(L, L.lib.b200sep_demix_overlap_add_range_ex(p(loc), lo, hi + 1 - lo, n_chunks, chunk_len, step, total_len, trim, n_out, qb, qe, use_window, 1.25, p(mix), n_out,
                                                             0, 0.97, 0, p(got_p), p(got_s), 0, None), "demix_overlap_add_range_ex")
        if lo < hi:  # a buffer missing a covering chunk is refused on the host
            rc = L.lib.b200sep_demix_overlap_add_range(p(loc[1:]), lo + 1, hi - lo, n_chunks, chunk_len, step, total_len, trim, n_out, qb, qe, use_window, 1.25, p(mix), 0.97,
                                                       interleave, p(got_p), p(got_s), None)
            assert rc == ERR_ARG
    torch.cuda.synchronize()
    assert torch.equal(got_p, full_p) and torch.equal(got_s, full_s)


def test_rect_overlap_add_vs_numpy_and_ranges(L):
    g = gen(42)
    n_chunks, C, chunk_len, hop, front, divisor = 7, 2, 1100, 400, 250, 3.0
    n_out = (n_chunks - 1) * hop + chunk_len - front - 90
    x = torch.randn(n_chunks, C, chunk_len, generator=g)
    # mdxc_separator.py:395-402: result[..., i*hop : i*hop + chunk] += chunk_i; result[..., front : front + n_out] / overlap
    acc = np.zeros((C, (n_chunks - 1) * hop + chunk_len))
    for i in range(n_chunks):
        acc[:, i * hop : i * hop + chunk_len] += x[i].double().numpy()
    ref = torch.from_numpy(acc[:, front : front + n_out] / divisor)
    xd = cu(x)
    full = torch.full((C, n_out), float("nan"), device="cuda")
    run(L, L.lib.b200sep_rect_overlap_add(p(xd), n_chunks, C, chunk_len, hop, front, n_out, divisor, p(full), None), "rect_overlap_add")
    assert_arith(full, ref)
    bounds = (0, 333, 1500, 2222, n_out)
    for qb, qe in zip(bounds[:-1], bounds[1:]):
        lo, hi = covering(qb, qe, front, chunk_len, hop, n_chunks)
        sl = torch.full((C, qe - qb + 2), SENTINEL, device="cuda")
        run(L, L.lib.b200sep_rect_overlap_add_range(p(xd[lo : hi + 1]), lo, hi + 1 - lo, n_chunks, C, chunk_len, hop, front, n_out, qb, qe, divisor, p(sl), qe - qb + 2, qb, None),
            "rect_overlap_add_range")
        assert torch.equal(sl[:, : qe - qb], full[:, qb:qe])
        assert (sl[:, qe - qb :] == SENTINEL).all()


def test_triangle_overlap_add_ranges_equal_full(L):
    g = gen(43)
    n_segs, C, seg_len, stride = 5, 2, 1000, 600
    length = (n_segs - 1) * stride + 700
    segs = cu(torch.randn(n_segs, C, seg_len, generator=g))
    cs = cu(torch.tensor([0.75, 1.5]))
    full = torch.full((C, length), float("nan"), device="cuda")
    run(L, L.lib.b200sep_triangle_overlap_add(p(segs), n_segs, C, seg_len, stride, length, 0, length, 0.5, p(cs), 0, p(full), None), "triangle_overlap_add")
    # apply.py:215-250: each segment's valid part times the triangle weight cat(arange(1, s/2 + 1), arange(s - s/2, 0, -1)) / max, over the summed weights
    wt = torch.cat([torch.arange(1, seg_len // 2 + 1), torch.arange(seg_len - seg_len // 2, 0, -1)]).double()
    wt = wt / wt.max()
    acc, wsum = torch.zeros(C, length, dtype=torch.float64), torch.zeros(length, dtype=torch.float64)
    for i in range(n_segs):
        o = i * stride
        v = min(seg_len, length - o)
        acc[:, o : o + v] += segs[i, :, :v].cpu().double() * wt[:v]
        wsum[o : o + v] += wt[:v]
    assert_arith(full, acc / wsum * 0.5 * torch.tensor([0.75, 1.5], dtype=torch.float64)[:, None])
    got = torch.full((C, length), float("nan"), device="cuda")
    bounds = (0, 450, 1234, 2000, length)
    for qb, qe in zip(bounds[:-1], bounds[1:]):
        lo, hi = covering(qb, qe, 0, seg_len, stride, n_segs)
        run(L, L.lib.b200sep_triangle_overlap_add_range(p(segs[lo : hi + 1]), lo, hi + 1 - lo, n_segs, C, seg_len, stride, length, qb, qe - qb, 0.5, p(cs), 0, p(got), length, qb,
                                                        None), "triangle_overlap_add_range")
    assert torch.equal(got, full)


def test_overlap_add_starts_zero_ended_window(L):
    """np.hanning is 0 at both ends: where it is the only covering weight, the 1e-10 clamp turns 0 / 0 into 0"""
    g = gen(44)
    n, C, ln, n_out = 5, 2, 800, 2400
    starts = [0, 300, 700, 1500, 1600]  # uneven
    x = torch.randn(n, C, ln, generator=g)
    win = torch.from_numpy(np.hanning(ln).astype(np.float32))
    out = torch.full((C, n_out), float("nan"), device="cuda")
    run(L, L.lib.b200sep_overlap_add_starts(p(cu(x)), p(cu(torch.tensor(starts, dtype=torch.int64))), p(cu(win)), n, C, ln, n_out, p(out), None), "overlap_add_starts")
    acc, cnt = np.zeros((C, n_out)), np.zeros(n_out)
    for i, s in enumerate(starts):
        acc[:, s : s + ln] += x[i].double().numpy() * win.double().numpy()
        cnt[s : s + ln] += win.double().numpy()
    ref = torch.from_numpy(acc / np.maximum(cnt, 1e-10))
    assert_arith(out, ref)
    assert out[:, 0].abs().max().item() == 0.0 and out[:, -1].abs().max().item() == 0.0


def blstm_frames_ref(x, width, stride):
    """demucs.py:38-45 with demucs utils.unfold: nf = ceil(T / stride) frames, zero-padded to (nf - 1) * stride + width -> (width, B * nf, C)"""
    B, C, T = x.shape
    nf = 1 if T <= width else -(-T // stride)
    xp = F.pad(x, (0, (nf - 1) * stride + width - T))
    fr = xp.unfold(-1, width, stride)  # (B, C, nf, width)
    return fr.permute(0, 2, 1, 3).reshape(B * nf, C, width).permute(2, 0, 1).contiguous(), nf


def blstm_unframe_ref(frames, B, C, T, nf, width, stride, skip):
    """demucs.py:52-64: the trimmed concatenation of the frames, cut to T, plus the skip connection"""
    if nf == 1:
        y = frames.permute(1, 2, 0)[..., :T]
    else:
        fr = frames.permute(1, 2, 0).reshape(B, nf, C, width)
        limit = stride // 2
        out = []
        for k in range(nf):
            if k == 0:
                out.append(fr[:, k, :, :-limit])
            elif k == nf - 1:
                out.append(fr[:, k, :, limit:])
            else:
                out.append(fr[:, k, :, limit:-limit])
        y = torch.cat(out, -1)[..., :T]
    return y + skip if skip is not None else y


@pytest.mark.parametrize("T,width,stride", [(1003, 200, 100), (1000, 200, 100), (777, 777, 388)])
def test_lstm_frames_gather_scatter(L, T, width, stride):
    g = gen(T + width)
    B, C = 2, 5
    x = torch.randn(B, C, T, generator=g)
    want, nf = blstm_frames_ref(x, width, stride)
    frames = torch.full((width, B * nf, C), float("nan"), device="cuda")
    run(L, L.lib.b200sep_lstm_frames_gather_f32(p(cu(x)), p(frames), B, C, T, nf, width, stride, None), "lstm_frames_gather_f32")
    assert torch.equal(frames.cpu(), want)
    fr = torch.randn(width, B * nf, C, generator=g)
    skip = torch.randn(B, C, T, generator=g)
    for sk in (None, skip):
        y = torch.full((B, C, T), float("nan"), device="cuda")
        run(L, L.lib.b200sep_lstm_frames_scatter_f32(p(cu(fr)), p(None if sk is None else cu(sk)), p(y), B, C, T, nf, width, stride, None), "lstm_frames_scatter_f32")
        assert torch.equal(y.cpu(), blstm_unframe_ref(fr, B, C, T, nf, width, stride, sk))


# ================================================================================================================ ensembling
@pytest.mark.parametrize("M", [1, 2, 5, 16])
def test_ensemble_f32(L, M):
    g = np.random.default_rng(M)
    n = 1031
    x = g.standard_normal((M, n)).astype(np.float32)
    if M > 1:  # magnitude ties of opposite sign at the extremum: the first model wins
        x[:, :8] = 2.0
        x[0, :4], x[1:, :4] = -0.5, 0.5
        x[0, 4:8], x[1:, 4:8] = -3.0, 3.0
    w = (g.uniform(0.2, 2.0, M)).astype(np.float32)  # not normalised
    xd, wd = cu(torch.from_numpy(x)), cu(torch.from_numpy(w))
    outs = {}
    for algo in range(4):
        out = torch.full((n,), float("nan"), device="cuda")
        run(L, L.lib.b200sep_ensemble_f32(p(xd), M, n, p(wd), algo, p(out), None), "ensemble_f32")
        outs[algo] = out.cpu().numpy()
    ref_avg = (x.astype(np.float64) * w[:, None]).sum(0) / w.astype(np.float64).sum()
    assert_arith(torch.from_numpy(outs[0]), torch.from_numpy(ref_avg), "weighted mean")
    assert np.array_equal(outs[1], np.median(x, axis=0))
    cols = np.arange(n)
    assert np.array_equal(outs[2], x[np.argmin(np.abs(x), axis=0), cols])
    assert np.array_equal(outs[3], x[np.argmax(np.abs(x), axis=0), cols])
    if M > 1:
        assert (outs[2][:4] == -0.5).all() and (outs[3][4:8] == -3.0).all()


def test_ensemble_f32_rejects_17_models(L):
    x = torch.zeros(17, 4, device="cuda")
    w = torch.ones(17, device="cuda")
    out = torch.zeros(4, device="cuda")
    assert L.lib.b200sep_ensemble_f32(p(x), 17, 4, p(w), 0, p(out), None) == ERR_ARG


def test_ensemble_spec_abs_ties(L):
    g = np.random.default_rng(7)
    M, P = 4, 300
    x = g.standard_normal((M, 4, P)).astype(np.float32)
    # equal moduli (5) on the axes, every model, for the first 20 entries of both channels: min and max both tie
    axes = np.array([[5.0, 0.0], [0.0, 5.0], [-5.0, 0.0], [0.0, -5.0]], np.float32)
    for m in range(M):
        for c in range(2):
            x[m, 2 * c, :20], x[m, 2 * c + 1, :20] = axes[m]
    z = x[:, 0::2].astype(np.float64) + 1j * x[:, 1::2].astype(np.float64)  # (M, 2, P)
    a = np.abs(z)
    xd = cu(torch.from_numpy(x))
    for take_max in (0, 1):
        for last_wins in (0, 1):
            out = torch.full((4, P), float("nan"), device="cuda")
            run(L, L.lib.b200sep_ensemble_spec_abs(p(xd), M, P, take_max, last_wins, p(out), None), "ensemble_spec_abs")
            if last_wins:  # uvr_min_spec / uvr_max_spec: the sequential np.where(|new| <= |cur|, new, cur) (>= for max)
                cur = z[0].copy()
                for m in range(1, M):
                    better = (np.abs(z[m]) >= np.abs(cur)) if take_max else (np.abs(z[m]) <= np.abs(cur))
                    cur = np.where(better, z[m], cur)
                want = cur
            else:  # min_fft / max_fft: np.argmin / np.argmax, the first extremum
                idx = a.argmax(0) if take_max else a.argmin(0)
                want = np.take_along_axis(z, idx[None], 0)[0]
            ref = np.stack([want[0].real, want[0].imag, want[1].real, want[1].imag]).astype(np.float32)
            assert np.array_equal(out.cpu().numpy(), ref), (take_max, last_wins)
            assert tuple(out[0:2, 0].tolist()) == tuple(axes[M - 1 if last_wins else 0])


# ================================================================================================================ DConv statistics
@pytest.mark.timeout(180)
@pytest.mark.parametrize("B,C,Fr,L_,hid,dil,u_in", [(2, 48, 3, 700, 6, 1, False), (1, 384, 1, 300, 48, 2, True)])
def test_fused_dconv_large_conv_bias(L, B, C, Fr, L_, hid, dil, u_in):
    """test_fused_dconv_layer_vs_torch with a first-convolution bias of 30: u's mean is about 30 times its standard deviation, so the GroupNorm
    statistics of the fused layer (fp32 per-position sums merged in double, then E[u^2] - mean^2) must not cancel."""
    g = gen(B * 7 + C + Fr + L_ + hid)
    x = torch.randn(B, C, Fr, L_, generator=g)
    w0 = torch.randn(hid, C, 3, generator=g) / (3 * C) ** 0.5
    b0 = 30.0 + torch.randn(hid, generator=g) * 0.1
    g1, be1 = torch.rand(hid, generator=g) + 0.5, torch.randn(hid, generator=g) * 0.1
    w3 = torch.randn(2 * C, hid, generator=g) / hid**0.5
    b3 = torch.randn(2 * C, generator=g) * 0.1
    g4, be4 = torch.rand(2 * C, generator=g) + 0.5, torch.randn(2 * C, generator=g) * 0.1
    ls = torch.rand(C, generator=g) * 0.5
    xs = x.double().permute(0, 2, 1, 3).reshape(B * Fr, C, L_)
    u = F.conv1d(xs, w0.double(), b0.double(), padding=dil, dilation=dil)
    assert u.mean().item() > 20 * u.std(dim=(1, 2)).max().item()
    h = F.gelu(F.group_norm(u, 1, g1.double(), be1.double(), eps=1e-5))
    z = F.group_norm(F.conv1d(h, w3.double()[:, :, None], b3.double()), 1, g4.double(), be4.double(), eps=1e-5)
    ref = (xs + ls.double()[None, :, None] * F.glu(z, dim=1)).reshape(B, Fr, C, L_).permute(0, 2, 1, 3)
    d = [cu(t) for t in (x, w0, b0, g1, be1, w3, b3, g4, be4, ls)]
    y = torch.full_like(d[0], float("nan"))
    uin = cu(u.float().reshape(B, Fr, hid, L_).permute(0, 2, 1, 3)) if u_in else None
    work = torch.empty(L.lib.b200sep_dconv_work_floats(B, C, Fr, L_, hid), device="cuda")
    run(L, L.lib.b200sep_dconv_f32(p(d[0]), p(y), *[p(t) for t in d[1:]], B, C, Fr, L_, hid, dil, p(uin), p(work), None), "dconv_f32")
    assert torch.isfinite(y).all()
    assert (y.cpu().double() - ref).abs().max().item() <= 2e-5 * max(1.0, ref.abs().max().item())
