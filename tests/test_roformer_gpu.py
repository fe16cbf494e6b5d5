"""GPU parity of the BS-Roformer path (the Roformer branch of the MDXC plugin): operator kernels against ATen, BSRoformerNet.forward and
RoformerEngine against golden vectors produced by the UNMODIFIED reference (oracle/make_golden_roformer.py; rotary-embedding-torch restated),
one full-size chunk (dim 512, depth 12, 62 bands, 801 frames) against the oracle.  Audio tolerance 1e-4 max-abs."""
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import mdx_oracle as M
import roformer_oracle as R

pytestmark = pytest.mark.gpu

SMALL = dict(dim=32, depth=2, time_transformer_depth=1, freq_transformer_depth=2, freqs_per_bands=(2, 2, 4, 4, 8, 12, 16, 17), dim_head=8, heads=4, stft_n_fft=128,
             stft_hop_length=32, stft_win_length=128)


def dev(x):
    return torch.as_tensor(np.ascontiguousarray(x)).cuda()


@pytest.fixture(scope="module")
def rf(lib_built):
    assert torch.cuda.is_available()
    from audio_separator.separator.b200 import roformer

    return roformer


@pytest.fixture(scope="module")
def gold(golden_dir):
    return np.load(os.path.join(golden_dir, "roformer_small.npz"))


def _net(rf, seed=3, **over):
    kw = dict(SMALL, **over)
    ocfg = R.BSRoformerConfig(**dict(kw, dim_t=65, overlap=8))
    w = R.make_weights(ocfg, seed=seed)
    return rf.BSRoformerNet(rf.BSRoformerConfig(**kw), w), ocfg, w


def test_roformer_operator_kernels(rf):
    from audio_separator.separator.b200._lib import check, lib

    g = torch.Generator().manual_seed(1)
    # RMSNorm on a column slice
    x = torch.randn((37, 50), generator=g)
    gam = torch.rand(12, generator=g) + 0.5
    xd, gd = x.cuda(), gam.cuda()
    y = torch.empty((37, 12), device="cuda")
    check(lib.b200sep_rmsnorm_f32(xd.data_ptr() + 20 * 4, gd.data_ptr(), y.data_ptr(), 37, 12, 50, 12, 0))
    ref = F.normalize(x[:, 20:32], dim=-1) * 12**0.5 * gam
    assert (y.cpu() - ref).abs().max() <= 1e-5
    # rotary + head split
    B, n, H, dh = 3, 13, 4, 8
    qkv = torch.randn((B, n, 3 * H * dh), generator=g)
    fr = torch.from_numpy(R.rotary_freqs(dh))
    qd, fd = qkv.cuda(), fr.cuda()
    q, k, v = (torch.empty((B, H, n, dh), device="cuda") for _ in range(3))
    check(lib.b200sep_rope_split_heads_f32(qd.data_ptr(), fd.data_ptr(), q.data_ptr(), k.data_ptr(), v.data_ptr(), B, n, H, dh, 0))
    qr, kr, vr = qkv.view(B, n, 3, H, dh).permute(2, 0, 3, 1, 4)
    assert (q.cpu() - R.apply_rotary(qr, fr)).abs().max() <= 1e-5 and (k.cpu() - R.apply_rotary(kr, fr)).abs().max() <= 1e-5
    assert torch.equal(v.cpu(), vr.contiguous())
    # P @ V with V given (K, N) row-major and P on a padded row stride
    P, V = torch.rand((6, 70, 72), generator=g), torch.randn((6, 70, 64), generator=g)
    Pd, Vd = P.cuda(), V.cuda()
    O = torch.empty((6, 70, 64), device="cuda")
    check(lib.b200sep_gemm_kn_f32(Pd.data_ptr(), Vd.data_ptr(), O.data_ptr(), 70, 64, 70, 72, 64, 64, 6, 70 * 72, 70 * 64, 70 * 64, 1.0, 0))
    ref = torch.einsum("bik,bkd->bid", P[:, :, :70].double(), V.double())
    assert (O.cpu().double() - ref).abs().max() <= 3e-5 * ref.abs().max()
    # gates + head merge
    o, gates = torch.randn((B, H, n, dh), generator=g), torch.randn((B * n, H), generator=g)
    od, gd2 = o.cuda(), gates.cuda()
    m = torch.empty((B * n, H * dh), device="cuda")
    check(lib.b200sep_gate_merge_heads_f32(od.data_ptr(), gd2.data_ptr(), m.data_ptr(), B, n, H, dh, 0))
    ref = (o * gates.view(B, n, H).permute(0, 2, 1)[..., None].sigmoid()).permute(0, 2, 1, 3).reshape(B * n, H * dh)
    assert (m.cpu() - ref).abs().max() <= 1e-6
    # GLU over the last dimension into a column slice
    a = torch.randn((21, 14), generator=g)
    ad = a.cuda()
    out = torch.zeros((21, 30), device="cuda")
    check(lib.b200sep_glu_rows_f32(ad.data_ptr(), out.data_ptr() + 5 * 4, 21, 7, 14, 30, 0))
    assert (out.cpu()[:, 5:12] - F.glu(a, -1)).abs().max() <= 1e-6 and not out.cpu()[:, :5].any() and not out.cpu()[:, 12:].any()
    # complex mask product + plane re-ordering
    b, S, T, Fq = 2, 2, 9, 5
    st, mk = torch.randn((b, T, Fq, 2, 2), generator=g), torch.randn((b, S, T, Fq, 2, 2), generator=g)
    sd_, md = st.cuda(), mk.cuda()
    planes = torch.empty((b * S, 4, Fq, T), device="cuda")
    check(lib.b200sep_roformer_mask_apply(sd_.data_ptr(), md.data_ptr(), planes.data_ptr(), b, S, T, Fq, 0))
    prod = torch.view_as_complex(st)[:, None] * torch.view_as_complex(mk)  # (b, S, T, F, s)
    ref = torch.view_as_real(prod.permute(0, 1, 4, 3, 2)).permute(0, 1, 2, 5, 3, 4).reshape(b * S, 4, Fq, T)
    assert (planes.cpu() - ref).abs().max() <= 1e-6
    # Hamming overlap-add with counter at explicit starts (tail chunk overlapping the previous one)
    C, N = 50, 133
    starts = [0, 40, 80, N - C]
    ch = torch.randn((4, 3, C), generator=g)
    win = torch.from_numpy(np.hamming(C).astype(np.float32))
    cd, wd, sdv = ch.cuda(), win.cuda(), torch.tensor(starts, dtype=torch.int64).cuda()
    out = torch.empty((3, N), device="cuda")
    check(lib.b200sep_overlap_add_starts(cd.data_ptr(), sdv.data_ptr(), wd.data_ptr(), 4, 3, C, N, out.data_ptr(), 0))
    res, cnt = torch.zeros((3, N)), torch.zeros(N)
    for i, s in enumerate(starts):
        res[:, s : s + C] += ch[i] * win
        cnt[s : s + C] += win
    assert (out.cpu() - res / cnt.clamp(min=1e-10)).abs().max() <= 1e-5
    # softmax on rows with a padded stride (register path, and the streaming path for very long rows)
    for n, ld in ((801, 804), (62, 64), (200, 200), (1500, 1504), (3000, 3000)):
        sc = torch.randn((19, ld), generator=g) * 6
        sdv2 = sc.cuda()
        check(lib.b200sep_softmax_rows_f32(sdv2.data_ptr(), 19, n, ld, 0))
        got = sdv2.cpu()
        assert (got[:, :n] - torch.softmax(sc[:, :n], -1)).abs().max() <= 1e-6 and torch.equal(got[:, n:], sc[:, n:])
    # tiny-N GEMM (the attention gates): warp-per-row kernel
    from audio_separator.separator.b200.ops import linear

    xg, wg, bg = torch.randn((2500, 96), generator=g), torch.randn((8, 96), generator=g) * 0.1, torch.randn(8, generator=g)
    assert (linear(xg.cuda(), wg.cuda(), bg.cuda()).cpu() - F.linear(xg, wg, bg)).abs().max() <= 2e-5
    torch.cuda.synchronize()


def test_forward_vs_reference_golden(rf, gold):
    net, ocfg, w = _net(rf)
    mix = M.synth_music(int(gold["n_samples"]), seed=int(gold["mix_seed"]))
    y = net.forward(dev(mix[None, :, : ocfg.chunk_size])).cpu().numpy()
    assert y.shape == gold["forward_ref"].shape
    assert np.abs(y - gold["forward_ref"]).max() <= 1e-4, np.abs(y - gold["forward_ref"]).max()
    yb = net.forward(dev(np.stack([mix[:, :1500], mix[:, 700:2200]]))).cpu().numpy()  # batch 2; 1500 is not a multiple of the hop: L' = hop * (L // hop)
    assert yb.shape == gold["forward_short_ref"].shape and np.abs(yb - gold["forward_short_ref"]).max() <= 1e-4
    net2, ocfg2, _ = _net(rf, seed=4, num_stems=2, mask_estimator_depth=3, depth=1)
    y2 = net2.forward(dev(mix[None, :, : ocfg2.chunk_size])).cpu().numpy()
    assert y2.shape == gold["forward_2stem_ref"].shape and np.abs(y2 - gold["forward_2stem_ref"]).max() <= 1e-4


def test_demix_vs_reference_golden(rf, gold):
    net, ocfg, w = _net(rf)
    mix = M.synth_music(int(gold["n_samples"]), seed=int(gold["mix_seed"]))
    eng = rf.RoformerEngine(net, 65, 8, 44100, n_instruments=2, batch_size=2)
    out = eng.demix_device(dev(mix)).cpu().numpy()
    assert out.shape == (1, 2, mix.shape[1]) and np.abs(out[0] - gold["demix_ref"]).max() <= 1e-4
    eng_o = rf.RoformerEngine(net, 65, 0.03, 44100, n_instruments=2, batch_size=3)  # step 1323 < chunk 2048: weighted overlap
    assert eng_o.step == 1323
    out_o = eng_o.demix_device(dev(mix)).cpu().numpy()
    assert np.abs(out_o[0] - gold["demix_overlap_ref"]).max() <= 1e-4
    net2, _, _ = _net(rf, seed=4, num_stems=2, mask_estimator_depth=3, depth=1)
    out2 = rf.RoformerEngine(net2, 65, 8, 44100, n_instruments=2, batch_size=1).demix_device(dev(mix)).cpu().numpy()
    assert out2.shape == gold["demix_2stem_ref"].shape and np.abs(out2 - gold["demix_2stem_ref"]).max() <= 1e-4
    with pytest.raises(NotImplementedError):
        eng.demix_device(dev(mix[:, :1000]))


def test_full_size_chunk_vs_oracle(rf):
    """The reference's default model geometry: dim 512, depth 12, 8 heads x 64, 62 bands, n_fft 2048 / hop 441, 801 frames (8 s)."""
    kw = dict(stft_hop_length=441)
    ocfg = R.BSRoformerConfig(**kw)
    w = R.make_weights(ocfg, seed=8)
    net = rf.BSRoformerNet(rf.BSRoformerConfig(**kw), w)
    mix = M.synth_music(ocfg.chunk_size, seed=9)[None]
    mix = (mix / np.abs(mix).max() * 0.9).astype(np.float32)
    ref = R.forward(w, ocfg, mix)
    got = net.forward(dev(mix)).cpu().numpy()
    assert got.shape == ref.shape == (1, 2, ocfg.chunk_size)
    err = np.abs(got - ref).max()
    assert err <= 1e-4 * max(1.0, np.abs(ref).max()), (err, np.abs(ref).max())


def test_mdxc_plugin_roformer_end_to_end(rf, tmp_path):
    import wave as wavmod

    import yaml

    from audio_separator.separator import Separator

    ocfg = R.BSRoformerConfig(**dict(SMALL, dim_t=65, overlap=8))
    w = R.make_weights(ocfg, seed=12)
    np.savez(tmp_path / "tiny_bs_roformer.npz", **w)
    model = dict(SMALL, freqs_per_bands=list(SMALL["freqs_per_bands"]), stereo=True, num_stems=1, mask_estimator_depth=2)
    (tmp_path / "tiny_bs_roformer.yaml").write_text(yaml.safe_dump({"audio": {"sample_rate": 44100, "hop_length": 32, "n_fft": 128, "dim_f": 65}, "model": model,
                                                                    "training": {"instruments": ["Vocals", "Instrumental"], "target_instrument": "Vocals"}, "inference": {"dim_t": 65}}))
    mix = M.synth_music(30000, seed=13)
    pcm = (mix.T * 32767).astype("<i2")
    with wavmod.open(str(tmp_path / "song.wav"), "wb") as wf:
        wf.setnchannels(2); wf.setsampwidth(2); wf.setframerate(44100); wf.writeframes(pcm.tobytes())
    sep = Separator(model_file_dir=str(tmp_path), output_dir=str(tmp_path / "out"), mdxc_params={"batch_size": 4, "segment_size": 65})  # < 10 s: dim_t = segment_size (:137-143)
    sep.load_model("tiny_bs_roformer.npz")
    files = sep.separate(str(tmp_path / "song.wav"))
    assert files == ["song_(Instrumental)_tiny_bs_roformer.wav", "song_(Vocals)_tiny_bs_roformer.wav"]  # secondary (residual) first, then the target
    loaded = M.normalize(pcm.astype(np.float32).T / 32768.0, 0.9, 0.0)
    prim = R.demix(loaded, ocfg, lambda c: R.forward(w, ocfg, c), n_instruments=2)[0]
    for fname, ref in zip(files, (loaded - prim, prim)):
        with wavmod.open(str(tmp_path / "out" / fname)) as wf:
            assert wf.getnframes() == 30000 and wf.getnchannels() == 2
            got = np.frombuffer(wf.readframes(30000), dtype="<i2").astype(np.int32)
        want = M.to_pcm16(ref.T.copy(), 0.9, 0.0).astype(np.int32)
        assert np.abs(got - want).max() <= 3


# ------------------------------------------------------------------------------------------------ Mel-Band Roformer
MSMALL = dict(dim=32, depth=2, time_transformer_depth=1, freq_transformer_depth=1, num_bands=12, dim_head=8, heads=4, mask_estimator_depth=2, stft_n_fft=128, stft_hop_length=32,
              stft_win_length=128)


def test_melband_gather_and_average_kernels(rf):
    from audio_separator.separator.b200._lib import check, lib

    g = torch.Generator().manual_seed(2)
    cfg = rf.MelBandRoformerConfig(**MSMALL)
    mask_b, idx, nfpb, nbpf = rf.mel_band_layout(cfg)
    FS, G = 65 * 2, len(idx)
    src = torch.randn((7, FS, 2), generator=g)
    sd, idd = src.cuda(), torch.from_numpy(idx.astype(np.int32)).cuda()
    dst = torch.empty((7, G, 2), device="cuda")
    check(lib.b200sep_gather_pairs_f32(sd.data_ptr(), idd.data_ptr(), dst.data_ptr(), 7, FS, G, 0))
    assert torch.equal(dst.cpu(), src[:, torch.from_numpy(idx)])
    mg = torch.randn((7, G, 2), generator=g)
    order = np.argsort(idx, kind="stable")
    off = np.concatenate([[0], np.cumsum(np.bincount(idx, minlength=FS))]).astype(np.int32)
    mgd, od, pd = mg.cuda(), torch.from_numpy(off).cuda(), torch.from_numpy(order.astype(np.int32)).cuda()
    out = torch.empty((7, FS, 2), device="cuda")
    check(lib.b200sep_mask_average_f32(mgd.data_ptr(), od.data_ptr(), pd.data_ptr(), out.data_ptr(), 7, G, FS, 0))
    summed = torch.zeros((7, FS, 2)).index_add_(1, torch.from_numpy(idx), mg)
    ref = summed / torch.from_numpy(np.repeat(nbpf, 2)).float()[None, :, None]
    assert (out.cpu() - ref).abs().max() <= 1e-6
    torch.cuda.synchronize()


def test_melband_forward_and_demix_vs_reference_golden(rf, gold):
    ocfg = R.MelBandRoformerConfig(**dict(MSMALL, dim_t=65))
    w = R.make_mel_weights(ocfg, seed=6)
    net = rf.BSRoformerNet(rf.MelBandRoformerConfig(**MSMALL), w)
    mix = M.synth_music(int(gold["n_samples"]), seed=int(gold["mix_seed"]))
    y = net.forward(dev(mix[None, :, : ocfg.chunk_size])).cpu().numpy()
    assert y.shape == gold["mel_forward_ref"].shape and np.abs(y - gold["mel_forward_ref"]).max() <= 1e-4
    kw2 = dict(MSMALL, num_stems=2, mask_estimator_depth=1, depth=1, freq_transformer_depth=2)
    ocfg2 = R.MelBandRoformerConfig(**dict(kw2, dim_t=65))
    net2 = rf.BSRoformerNet(rf.MelBandRoformerConfig(**kw2), R.make_mel_weights(ocfg2, seed=7))
    y2 = net2.forward(dev(mix[None, :, : ocfg2.chunk_size])).cpu().numpy()
    assert y2.shape == gold["mel_forward_2stem_ref"].shape and np.abs(y2 - gold["mel_forward_2stem_ref"]).max() <= 1e-4
    out = rf.RoformerEngine(net, 65, 8, 44100, n_instruments=2, batch_size=2).demix_device(dev(mix)).cpu().numpy()
    assert np.abs(out[0] - gold["mel_demix_ref"]).max() <= 1e-4


def test_melband_full_size_chunk_vs_oracle(rf):
    """A released Mel-Band geometry: dim 384, depth 6, 60 mel bands over 1025 bins (3958 gathered bin-channel pairs), hop 441, 801 frames."""
    ocfg = R.MelBandRoformerConfig()
    w = R.make_mel_weights(ocfg, seed=14)
    net = rf.BSRoformerNet(rf.MelBandRoformerConfig(stft_hop_length=441, mask_estimator_depth=2), w)
    mix = M.synth_music(ocfg.chunk_size, seed=15)[None]
    mix = (mix / np.abs(mix).max() * 0.9).astype(np.float32)
    ref = R.forward_mel(w, ocfg, mix)
    got = net.forward(dev(mix)).cpu().numpy()
    assert got.shape == ref.shape == (1, 2, ocfg.chunk_size)
    err = np.abs(got - ref).max()
    assert err <= 1e-4 * max(1.0, np.abs(ref).max()), (err, np.abs(ref).max())
