"""GPU parity of the HTDemucs path: the fp32 operator kernels against ATen on the CPU, HTDemucsNet.forward / apply_model /
demix_demucs against golden vectors produced by the UNMODIFIED reference (oracle/make_golden_demucs.py), and one full-size
segment (343980 samples, 42 M parameters) against the oracle.  Audio tolerance: 1e-4 max-abs (BASELINE gate)."""
import math
import os
from fractions import Fraction

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import demucs_oracle as D
import mdx_oracle as M

pytestmark = pytest.mark.gpu

SMALL = dict(channels=8, bottom_channels=32, t_layers=3, t_heads=4, segment=Fraction(1, 2))


def dev(x):
    return torch.as_tensor(np.ascontiguousarray(x)).cuda()


@pytest.fixture(scope="module")
def dm(lib_built):
    assert torch.cuda.is_available()
    from audio_separator.separator.b200 import demucs

    return demucs


@pytest.fixture(scope="module")
def ops(lib_built):
    assert torch.cuda.is_available()
    from audio_separator.separator.b200 import ops

    return ops


@pytest.fixture(scope="module")
def small(dm, golden_dir):
    z = np.load(os.path.join(golden_dir, "demucs_small.npz"))
    ocfg = D.HTConfig(**SMALL)
    w = D.make_weights(ocfg, seed=int(z["weights_seed"]))
    cfg = dm.HTDemucsConfig(**SMALL)
    net = dm.HTDemucsNet(cfg, w)
    mix = M.synth_music(3 * ocfg.seg_len, seed=int(z["mix_seed"]))
    return z, ocfg, w, net, mix


# ------------------------------------------------------------------------------------------------ operators
@pytest.mark.parametrize(
    "geom",
    [
        dict(cin=5, cout=7, k=(1, 1), s=(1, 1), p=(0, 0), dw=1, hw=(3, 200)),
        dict(cin=9, cout=50, k=(3, 3), s=(1, 1), p=(1, 1), dw=1, hw=(11, 133)),
        dict(cin=8, cout=3, k=(1, 3), s=(1, 1), p=(0, 1), dw=1, hw=(1, 517)),
        dict(cin=8, cout=3, k=(1, 3), s=(1, 1), p=(0, 2), dw=2, hw=(4, 130)),
        dict(cin=4, cout=48, k=(8, 1), s=(4, 1), p=(2, 0), dw=1, hw=(64, 37)),
        dict(cin=2, cout=10, k=(1, 8), s=(1, 4), p=(0, 2), dw=1, hw=(1, 1026)),
    ],
)
def test_conv2d_f32(ops, geom):
    g = torch.Generator().manual_seed(1)
    x = torch.randn((2, geom["cin"]) + geom["hw"], generator=g)
    w = torch.randn((geom["cout"], geom["cin"]) + geom["k"], generator=g) * 0.2
    b = torch.randn(geom["cout"], generator=g)
    ref = F.gelu(F.conv2d(x.double(), w.double(), b.double(), stride=geom["s"], padding=geom["p"], dilation=(1, geom["dw"])))
    wb = dev(ops.block_conv_weight(w.numpy()))
    got = ops.conv2d(x.cuda(), wb, b.cuda(), geom["cout"], geom["k"], geom["s"], geom["p"], geom["dw"], act=ops.ACT_GELU).cpu()
    assert got.shape == ref.shape
    assert (got.double() - ref).abs().max() <= 2e-5 * max(1.0, ref.abs().max())


def test_conv2d_f32_ragged_time_pad_and_add(ops):
    """The time encoder pads its input to a multiple of the stride (hdemucs.py:126-129): implicit zero columns."""
    g = torch.Generator().manual_seed(2)
    x = torch.randn((1, 3, 1, 1023), generator=g)
    w = torch.randn((6, 3, 1, 8), generator=g) * 0.2
    b = torch.randn(6, generator=g)
    ref = F.conv2d(F.pad(x, (0, 1)), w, b, stride=(1, 4), padding=(0, 2))
    add = torch.randn(ref.shape, generator=g)
    got = ops.conv2d(x.cuda(), dev(ops.block_conv_weight(w.numpy())), b.cuda(), 6, (1, 8), (1, 4), (0, 2), out_hw=(1, 256), add=add.cuda(), add_before_act=True, act=ops.ACT_RELU).cpu()
    assert (got - F.relu(ref + add)).abs().max() <= 2e-5


@pytest.mark.parametrize("axis", [1, 2])
def test_conv_transpose_f32(ops, axis):
    g = torch.Generator().manual_seed(3)
    cin, cout = 12, 5
    if axis == 1:
        x = torch.randn((2, cin, 9, 70), generator=g)
        w = torch.randn((cin, cout, 8, 1), generator=g) * 0.2
        b = torch.randn(cout, generator=g)
        ref = F.gelu(F.conv_transpose2d(x.double(), w.double(), b.double(), stride=(4, 1))[..., 2:-2, :])
        got = ops.conv_transpose(x.cuda(), dev(ops.block_convtr_weight(w.numpy().reshape(cin, cout, 8), 4)), b.cuda(), cout, 1, 4, 2, 36, ops.ACT_GELU).cpu()
    else:
        x = torch.randn((2, cin, 1, 301), generator=g)
        w = torch.randn((cin, cout, 8), generator=g) * 0.2
        b = torch.randn(cout, generator=g)
        length = 1201  # the skip length of the time decoder: odd, shorter than 4 * 301
        ref = F.conv_transpose1d(x[:, :, 0].double(), w.double(), b.double(), stride=4)[..., 2 : 2 + length][:, :, None]
        got = ops.conv_transpose(x.cuda(), dev(ops.block_convtr_weight(w.numpy(), 4)), b.cuda(), cout, 2, 4, 2, length).cpu()
    assert got.shape == ref.shape
    assert (got.double() - ref).abs().max() <= 2e-5 * max(1.0, ref.abs().max())


@pytest.mark.parametrize("axis", [1, 2])
def test_conv_transpose_f32_tensor_core_route(ops, axis):
    """Same operator at shapes the wgmma kernel takes (real output channels a multiple of 16, >= 512 coarse pixels): the scatter epilogue of tc_f32.cu."""
    g = torch.Generator().manual_seed(5)
    cin, cout = 96, 48
    if axis == 1:
        x = torch.randn((2, cin, 8, 90), generator=g)
        w = torch.randn((cin, cout, 8, 1), generator=g) / cin**0.5
        b = torch.randn(cout, generator=g)
        ref = F.gelu(F.conv_transpose2d(x.double(), w.double(), b.double(), stride=(4, 1))[..., 2:-2, :])
        got = ops.conv_transpose(x.cuda(), dev(ops.block_convtr_weight(w.numpy().reshape(cin, cout, 8), 4)), b.cuda(), cout, 1, 4, 2, 32, ops.ACT_GELU).cpu()
    else:
        x = torch.randn((2, cin, 1, 700), generator=g)
        w = torch.randn((cin, cout, 8), generator=g) / cin**0.5
        b = torch.randn(cout, generator=g)
        length = 2797
        ref = F.conv_transpose1d(x[:, :, 0].double(), w.double(), b.double(), stride=4)[..., 2 : 2 + length][:, :, None]
        got = ops.conv_transpose(x.cuda(), dev(ops.block_convtr_weight(w.numpy(), 4)), b.cuda(), cout, 2, 4, 2, length).cpu()
    assert got.shape == ref.shape and torch.isfinite(got).all()
    assert (got.double() - ref).abs().max() <= 5e-5 * max(1.0, ref.abs().max())


def test_groupnorm_glu_layernorm_softmax_permute(ops):
    g = torch.Generator().manual_seed(4)
    x = torch.randn((2, 6, 5, 77), generator=g) * 3 + 1
    ga, be = torch.rand(6, generator=g) + 0.5, torch.randn(6, generator=g)
    # DConv applied per frequency row: samples are (b, fr), statistics over (C, T)
    ref = F.gelu(F.group_norm(x.permute(0, 2, 1, 3).reshape(10, 6, 77), 1, ga, be)).view(2, 5, 6, 77).permute(0, 2, 1, 3)
    got = ops.groupnorm1(x.cuda().clone(), ga.cuda(), be.cuda(), ops.ACT_GELU).cpu()
    assert (got - ref).abs().max() <= 1e-5
    tok = torch.randn((3, 50, 6), generator=g) * 2 - 1
    ref = F.group_norm(tok.transpose(1, 2), 1, ga, be).transpose(1, 2)
    got = ops.groupnorm1(tok.cuda().clone(), ga.cuda(), be.cuda(), channel_last=True).cpu()
    assert (got - ref).abs().max() <= 1e-5
    a = torch.randn((2, 12, 5, 33), generator=g)
    res, sc = torch.randn((2, 6, 5, 33), generator=g), torch.rand(6, generator=g)
    assert (ops.glu(a.cuda()).cpu() - F.glu(a, 1)).abs().max() <= 1e-6
    assert (ops.glu(a.cuda(), res.cuda(), sc.cuda()).cpu() - (res + sc[None, :, None, None] * F.glu(a, 1))).abs().max() <= 1e-6
    t = torch.randn((7, 9, 40), generator=g) * 4
    g2, b2 = torch.rand(40, generator=g), torch.randn(40, generator=g)
    assert (ops.layernorm(t.cuda(), g2.cuda(), b2.cuda()).cpu() - F.layer_norm(t, (40,), g2, b2)).abs().max() <= 1e-5
    from audio_separator.separator.b200._lib import check, lib

    s = (torch.randn((33, 300), generator=g) * 5).cuda()
    ref = torch.softmax(s.cpu(), -1)
    check(lib.b200sep_softmax_rows_f32(s.data_ptr(), 33, 300, 300, 0))
    torch.cuda.synchronize()
    assert (s.cpu() - ref).abs().max() <= 1e-6
    p = torch.randn((2, 3, 4, 5), generator=g).cuda()
    out = torch.empty((2, 5, 4, 3), device="cuda")
    check(lib.b200sep_permute4_f32(p.data_ptr(), out.data_ptr(), 2, 3, 4, 5, 0, 3, 2, 1, 0))
    torch.cuda.synchronize()
    assert torch.equal(out.cpu(), p.cpu().permute(0, 3, 2, 1).contiguous())


def test_gemm_f32_and_attention_pattern(ops):
    g = torch.Generator().manual_seed(5)
    x = torch.randn((130, 72), generator=g)
    w = torch.randn((200, 72), generator=g) * 0.1
    b = torch.randn(200, generator=g)
    res, rs = torch.randn((130, 200), generator=g), torch.rand(200, generator=g)
    ref = res + rs * F.gelu(F.linear(x.double(), w.double(), b.double()))
    got = ops.linear(x.cuda(), w.cuda(), b.cuda(), act=ops.ACT_GELU, res=res.cuda(), res_scale=rs.cuda()).cpu()
    assert (got.double() - ref).abs().max() <= 2e-5
    # odd K / unaligned leading dimensions take the scalar load path
    x2, w2 = torch.randn((17, 45), generator=g), torch.randn((9, 45), generator=g)
    assert (ops.linear(x2.cuda(), w2.cuda(), None).cpu() - x2 @ w2.t()).abs().max() <= 2e-5


@pytest.mark.timeout(180)
@pytest.mark.parametrize("B,C,Fr,L,hid,dil,u_in", [(2, 48, 5, 336, 6, 1, False), (1, 96, 3, 130, 12, 2, False), (2, 48, 1, 5000, 6, 2, False), (1, 192, 2, 336, 24, 1, False),
                                                  (1, 384, 2, 200, 48, 2, True), (1, 32, 1, 2500, 4, 1, False), (1, 64, 2, 77, 8, 2, False)])
def test_fused_dconv_layer_vs_torch(dm, B, C, Fr, L, hid, dil, u_in):
    """b200sep_dconv_f32 (csrc/dconv_fused.cu) against the operator-by-operator definition of one DConv residual layer (demucs.py:124-168), fp64 on the CPU."""
    from audio_separator.separator.b200._lib import check, lib

    g = torch.Generator().manual_seed(B * 7 + C + Fr + L + hid)
    x = torch.randn(B, C, Fr, L, generator=g)
    w0 = torch.randn(hid, C, 3, generator=g) / (3 * C) ** 0.5
    b0 = torch.randn(hid, generator=g) * 0.1
    g1, be1 = torch.rand(hid, generator=g) + 0.5, torch.randn(hid, generator=g) * 0.1
    w3 = torch.randn(2 * C, hid, generator=g) / hid**0.5
    b3 = torch.randn(2 * C, generator=g) * 0.1
    g4, be4 = torch.rand(2 * C, generator=g) + 0.5, torch.randn(2 * C, generator=g) * 0.1
    ls = torch.rand(C, generator=g) * 0.5
    xs = x.double().permute(0, 2, 1, 3).reshape(B * Fr, C, L)  # one sample per (b, fr) row
    u = F.conv1d(xs, w0.double(), b0.double(), padding=dil, dilation=dil)
    h = F.gelu(F.group_norm(u, 1, g1.double(), be1.double(), eps=1e-5))
    z = F.group_norm(F.conv1d(h, w3.double()[:, :, None], b3.double()), 1, g4.double(), be4.double(), eps=1e-5)
    ref = (xs + ls.double()[None, :, None] * F.glu(z, dim=1)).reshape(B, Fr, C, L).permute(0, 2, 1, 3)
    d = [t.cuda().contiguous() for t in (x, w0, b0, g1, be1, w3, b3, g4, be4, ls)]
    y = torch.full_like(d[0], float("nan"))
    uin = u.float().reshape(B, Fr, hid, L).permute(0, 2, 1, 3).contiguous().cuda() if u_in else None
    work = torch.empty(lib.b200sep_dconv_work_floats(B, C, Fr, L, hid), device="cuda")
    check(lib.b200sep_dconv_f32(d[0].data_ptr(), y.data_ptr(), *[t.data_ptr() for t in d[1:]], B, C, Fr, L, hid, dil, uin.data_ptr() if u_in else None, work.data_ptr(), None), "dconv_f32")
    torch.cuda.synchronize()
    assert torch.isfinite(y).all()
    assert (y.cpu().double() - ref).abs().max().item() <= 2e-5 * max(1.0, ref.abs().max().item())
    # in place (y aliases x), as HTDemucsNet uses it
    check(lib.b200sep_dconv_f32(d[0].data_ptr(), d[0].data_ptr(), *[t.data_ptr() for t in d[1:]], B, C, Fr, L, hid, dil, uin.data_ptr() if u_in else None, work.data_ptr(), None), "dconv_f32")
    assert torch.equal(d[0], y)


def test_meanstd_and_stats_ops(ops):
    from audio_separator.separator.b200._lib import check, lib

    g = torch.Generator().manual_seed(6)
    x = (torch.randn(100_003, generator=g) * 3 + 0.7).cuda()
    st = torch.empty(2, device="cuda")
    check(lib.b200sep_meanstd_f32(x.data_ptr(), x.numel(), st.data_ptr(), 0))
    m, s = st.cpu().tolist()
    assert abs(m - x.double().mean().item()) <= 1e-6 and abs(s - x.double().std().item()) <= 1e-5
    y = ops.ew(x, st, torch.empty_like(x), op=2)
    assert (y.cpu() - (x.cpu() - m) / (1e-5 + s)).abs().max() <= 1e-6
    z = ops.ew(y, st, torch.empty_like(x), op=3)
    assert (z.cpu() - x.cpu()).abs().max() <= 1e-4


def test_spec_ispec_vs_torch(dm, small):
    """HTDemucs._spec / _ispec (htdemucs.py:383-413) through stft_forward_ex / stft_inverse_ex against torch.stft / istft."""
    from audio_separator.separator.b200._lib import LAYOUT_CFT, check, lib

    z, ocfg, w, net, mix = small
    T_len, hl, nfft = 22050, 1024, 4096
    x = torch.from_numpy(mix[None, :, :T_len])
    le = math.ceil(T_len / hl)
    pad = hl // 2 * 3
    xp = F.pad(x, (pad, pad + le * hl - T_len), mode="reflect")
    zz = torch.stft(xp.reshape(-1, xp.shape[-1]), nfft, hl, window=torch.hann_window(nfft), normalized=True, center=True, return_complex=True, pad_mode="reflect")
    zz = zz.view(1, 2, zz.shape[-2], zz.shape[-1])[..., :-1, :][..., 2 : 2 + le]
    ref = torch.view_as_real(zz).permute(0, 1, 4, 2, 3).reshape(1, 4, nfft // 2, le)
    spec = torch.empty((1, 4, nfft // 2, le), device="cuda")
    xd = x.cuda().contiguous()
    check(lib.b200sep_stft_forward_ex(net.stft.handle, xd.data_ptr(), 2 * T_len, T_len, 0, 1, T_len, le, pad, 1.0 / math.sqrt(nfft), nfft // 2, 0, LAYOUT_CFT, 0, spec.data_ptr(), 0))
    torch.cuda.synchronize()
    assert (spec.cpu() - ref).abs().max() <= 2e-5 * max(1.0, ref.abs().max())
    # inverse of an arbitrary (non-consistent) spectrogram
    g = torch.Generator().manual_seed(7)
    sp = torch.randn((3, 4, nfft // 2, le), generator=g)
    zc = torch.view_as_complex(sp.view(3, 2, 2, nfft // 2, le).permute(0, 1, 3, 4, 2).contiguous())
    zc = F.pad(F.pad(zc, (0, 0, 0, 1)), (2, 2))
    lei = hl * le + 2 * pad
    xi = torch.istft(zc.reshape(-1, zc.shape[-2], zc.shape[-1]), nfft, hl, window=torch.hann_window(nfft), normalized=True, length=lei, center=True)
    xi = xi.view(3, 2, lei)[..., pad : pad + T_len]
    wave = torch.empty((3, 2, T_len), device="cuda")
    work = torch.empty(lib.b200sep_stft_inverse_work_floats(net.stft.handle, 3, le, nfft // 2, LAYOUT_CFT), device="cuda")
    spd = sp.cuda()
    check(lib.b200sep_stft_inverse_ex(net.stft.handle, spd.data_ptr(), 3, le, nfft // 2, LAYOUT_CFT, T_len, pad, 2, math.sqrt(nfft), wave.data_ptr(), work.data_ptr(), 0))
    torch.cuda.synchronize()
    assert (wave.cpu() - xi).abs().max() <= 2e-5 * max(1.0, xi.abs().max())


def test_triangle_overlap_add_vs_oracle(dm):
    from audio_separator.separator.b200._lib import check, lib

    ocfg = D.HTConfig(**SMALL)
    seg, S = ocfg.seg_len, 4
    rng = np.random.default_rng(8)
    N = int(2.6 * seg) + 17
    x = rng.standard_normal((1, 2, N)).astype(np.float32)
    # a "model" whose output is a fixed per-sample transform of the padded chunk lets the oracle's apply_split define the truth
    gains = np.array([1.0, -0.5, 0.25, 2.0], np.float32)

    def fn(c):
        return c[:, None] * gains[None, :, None, None]

    ref = D.apply_split(fn, ocfg, x, 0, N, 0.25)[0].reshape(S * 2, N)
    stride = int(0.75 * seg)
    offs = list(range(0, N, stride))
    segs = np.zeros((len(offs), S * 2, seg), np.float32)
    for i, off in enumerate(offs):
        clen = min(N - off, seg)
        segs[i, :, :clen] = D.center_trim(fn(D.padded(x, off, clen, seg)), clen)[0].reshape(S * 2, clen)
    out = torch.empty((S * 2, N), device="cuda")
    sd = dev(segs)
    check(lib.b200sep_triangle_overlap_add(sd.data_ptr(), len(offs), S * 2, seg, stride, N, 0, N, 1.0, None, 0, out.data_ptr(), 0))
    torch.cuda.synchronize()
    assert np.abs(out.cpu().numpy() - ref).max() <= 1e-5
    # windowed, scaled, accumulated read-out (shift trick / bag weights)
    cs = torch.rand(S * 2).cuda()
    out2 = torch.ones((S * 2, 1000), device="cuda")
    check(lib.b200sep_triangle_overlap_add(sd.data_ptr(), len(offs), S * 2, seg, stride, N, 333, 1000, 0.5, cs.data_ptr(), 1, out2.data_ptr(), 0))
    torch.cuda.synchronize()
    assert np.abs(out2.cpu().numpy() - (1.0 + 0.5 * cs.cpu().numpy()[:, None] * ref[:, 333:1333])).max() <= 1e-5


# ------------------------------------------------------------------------------------------------ the network and its callers
def test_forward_vs_reference_golden(small):
    z, ocfg, w, net, mix = small
    L = ocfg.seg_len
    y = net.forward(dev(mix[None, :, :L])).cpu().numpy()
    assert y.shape == z["forward_ref"].shape == (1, 4, 2, L)
    assert np.abs(y - z["forward_ref"]).max() <= 1e-4, np.abs(y - z["forward_ref"]).max()
    ys = net.forward(dev(mix[None, :, : L - 1234])).cpu().numpy()  # shorter than the training segment: zero-padded, cut back
    assert ys.shape == z["forward_short_ref"].shape
    assert np.abs(ys - z["forward_short_ref"]).max() <= 1e-4


def test_forward_batch_matches_single(small):
    z, ocfg, w, net, mix = small
    L = ocfg.seg_len
    batch = np.stack([mix[:, i * 5000 : i * 5000 + L] for i in range(3)])
    yb = net.forward(dev(batch)).cpu().numpy()
    for i in range(3):
        yi = net.forward(dev(batch[i : i + 1])).cpu().numpy()
        assert np.abs(yb[i] - yi[0]).max() <= 2e-5  # batch size moves some layers between the tensor-core and the SIMT kernels


def test_apply_model_and_demix_vs_reference_golden(dm, small):
    z, ocfg, w, net, mix = small
    N = int(z["n_apply"])
    m2 = mix[:, :N]
    offs = [int(v) for v in z["shift_offsets"]]
    eng = dm.DemucsEngine([net], batch_size=3)
    ref = torch.from_numpy(m2).mean(0)
    mn = ((torch.from_numpy(m2) - ref.mean()) / ref.std()).numpy()
    got = eng.apply_model(dev(mn), offs).cpu().numpy().reshape(1, 4, 2, N)
    assert np.abs(got - z["apply_ref"]).max() <= 1e-4, np.abs(got - z["apply_ref"]).max()
    src = eng.demix(m2, [offs])
    assert src.shape == z["demix_ref"].shape == (4, 2, N)
    assert np.abs(src - z["demix_ref"]).max() <= 1e-4
    # shifts = 0 and a two-model bag with one-hot-ish weights against the oracle
    w2 = D.make_weights(ocfg, seed=77)
    net2 = dm.HTDemucsNet(dm.HTDemucsConfig(**SMALL), w2)
    bag = [[1.0, 0.0, 1.0, 0.5], [0.0, 1.0, 1.0, 0.5]]
    fns = [lambda c: D.forward(w, ocfg, c), lambda c: D.forward(w2, ocfg, c)]
    short = m2[:, : ocfg.seg_len + 4321]
    ref_bag = D.demix_demucs(fns, bag, ocfg, short, [[], [777]], 0.25)
    got_bag = dm.DemucsEngine([net, net2], bag_weights=bag, batch_size=2).demix(short, [[], [777]])
    assert np.abs(got_bag - ref_bag).max() <= 1e-4


def test_full_size_segment_vs_oracle(dm):
    """The released geometry: 48 channels, 512-d 5-layer cross-transformer, 343980-sample segment (SURVEY section 8 a10)."""
    ocfg = D.HTConfig()
    w = D.make_weights(ocfg, seed=11)
    net = dm.HTDemucsNet(dm.HTDemucsConfig(), w)
    mix = M.synth_music(ocfg.seg_len, seed=12)[None]
    mix = (mix / np.abs(mix).max() * 0.9).astype(np.float32)
    ref = D.forward(w, ocfg, mix)
    got = net.forward(dev(mix)).cpu().numpy()
    assert got.shape == ref.shape == (1, 4, 2, ocfg.seg_len)
    err = np.abs(got - ref).max()
    assert err <= 1e-4 * max(1.0, np.abs(ref).max()), (err, np.abs(ref).max())


def _write_package(path, ocfg, w, half=False):
    """A `.th` package as demucs/states.py serialises it, with the class pickled by reference to a module that is NOT importable
    when the package is read back (the product must not need the reference's classes)."""
    import sys
    import types

    mod = types.ModuleType("demucs_fake_pkg.htdemucs")
    parent = types.ModuleType("demucs_fake_pkg")
    HT = type("HTDemucs", (), {"__module__": "demucs_fake_pkg.htdemucs"})
    mod.HTDemucs = HT
    sys.modules["demucs_fake_pkg"], sys.modules["demucs_fake_pkg.htdemucs"] = parent, mod
    try:
        state = {k: (torch.from_numpy(v).half() if half else torch.from_numpy(v)) for k, v in w.items()}
        torch.save({"klass": HT, "args": (), "kwargs": ocfg.kwargs(), "state": state}, path)
    finally:
        del sys.modules["demucs_fake_pkg"], sys.modules["demucs_fake_pkg.htdemucs"]


def test_demucs_separator_plugin_end_to_end(dm, tmp_path):
    """Separator(...).load_model(bag.yaml); separate(wav) -> four WAVs named as the reference names them; PCM within 3 LSB of the oracle."""
    import random
    import wave

    from audio_separator.separator import Separator

    ocfg = D.HTConfig(**SMALL)
    w_a, w_b = D.make_weights(ocfg, seed=21), D.make_weights(ocfg, seed=22)
    _write_package(str(tmp_path / "aaaa1111.th"), ocfg, w_a)
    _write_package(str(tmp_path / "bbbb2222-0123abcd.th"), ocfg, w_b)
    (tmp_path / "tiny_ft.yaml").write_text("models: ['aaaa1111', 'bbbb2222']\nweights: [[1, 0, 1, 1], [0, 1, 1, 0]]\n")
    mix = M.synth_music(30000, seed=3)
    pcm = (mix.T * 32767).astype("<i2")
    with wave.open(str(tmp_path / "song.wav"), "wb") as wf:
        wf.setnchannels(2); wf.setsampwidth(2); wf.setframerate(44100); wf.writeframes(pcm.tobytes())
    sep = Separator(model_file_dir=str(tmp_path), output_dir=str(tmp_path / "out"), demucs_params={"shifts": 1, "batch_size": 2})
    sep.load_model("tiny_ft.yaml")
    random.seed(1234)
    files = sep.separate(str(tmp_path / "song.wav"))
    assert files == ["song_(Bass)_tiny_ft.wav", "song_(Drums)_tiny_ft.wav", "song_(Other)_tiny_ft.wav", "song_(Vocals)_tiny_ft.wav"]
    random.seed(1234)
    offs = [[random.randint(0, 22050)], [random.randint(0, 22050)]]
    loaded = pcm.astype(np.float32).T / 32768.0
    fns = [lambda c: D.forward(w_a, ocfg, c), lambda c: D.forward(w_b, ocfg, c)]
    ref = D.demix_demucs(fns, [[1, 0, 1, 1], [0, 1, 1, 0]], ocfg, loaded, offs, 0.25)
    for k, fname in enumerate(files):
        with wave.open(str(tmp_path / "out" / fname)) as wf:
            assert wf.getnframes() == 30000 and wf.getnchannels() == 2
            got = np.frombuffer(wf.readframes(30000), dtype="<i2").astype(np.int32)
        want = M.to_pcm16(ref[k].T.copy(), 0.9, 0.0).astype(np.int32)  # final_process receives (N, 2)
        assert np.abs(got - want).max() <= 3  # <= 1e-4 * 32767 LSB


def test_dconv_mode_1_without_bottom_channels_vs_reference_golden(dm, small):
    """The constructor defaults dconv_mode=1 / bottom_channels=0 (DConv in the encoders only, transformer at the encoder width)."""
    z, ocfg, w, net, mix = small
    kw = dict(SMALL, bottom_channels=0, t_layers=2)
    ocfg1 = D.HTConfig(**dict(kw, dconv_mode=1))
    w1 = D.make_weights(ocfg1, seed=6)
    net1 = dm.HTDemucsNet(dm.HTDemucsConfig(**kw), w1)
    y = net1.forward(dev(mix[None, :, : ocfg1.seg_len])).cpu().numpy()
    assert np.abs(y - z["forward_dm1_ref"]).max() <= 1e-4
