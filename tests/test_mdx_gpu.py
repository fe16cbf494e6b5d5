"""GPU parity tests: the CUDA path, called through the C ABI (ctypes), against the oracle on the same seeded
inputs and against the committed golden vectors produced by the unmodified reference.

Tolerances (BASELINE.json north_star: <= 1e-4 max-abs per PCM sample, sample count / stem order exact):
  * audio-domain outputs: 1e-4 max-abs hard gate; the fp32 SIMT path is additionally held to 2e-5
  * spectrogram / network outputs: relative to the tensor's max (1e-5 fp32 path, 1e-4 split-bf16 path)
"""
import os

import numpy as np
import pytest
import torch

import mdx_oracle as O

pytestmark = pytest.mark.gpu

SMALL = dict(n_fft=1536, hop_length=256, dim_f=768, dim_t=32, segment_size=32, g=8)
MID = dict(n_fft=1024, hop_length=256, dim_f=512, dim_t=32, segment_size=32, g=16, num_blocks=7)  # channel counts the wgmma conv accepts


@pytest.fixture(scope="module")
def eng(lib_built):
    assert torch.cuda.is_available(), "-m gpu tests need a CUDA device"
    from audio_separator.separator.b200 import engine

    return engine


def maxabs(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    assert a.shape == b.shape, (a.shape, b.shape)
    fa, fb = np.isfinite(a), np.isfinite(b)
    assert (fa == fb).all()
    return np.abs(a[fa] - b[fa]).max() if fa.any() else 0.0


def dev(x):
    return torch.as_tensor(np.ascontiguousarray(x)).cuda()


def make_net(eng, cfg, w, max_batch=2, precision=0, dim_t=None):
    from audio_separator.separator.b200 import mdx_weights

    hp = mdx_weights.infer_hparams_from_state(w)
    return eng.MdxNet(mdx_weights.flatten_state(w, **hp), dim_t=dim_t or cfg.dim_t, max_batch=max_batch, precision=precision, **hp)


# ---------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n_fft,hop,dim_f,frames", [(1536, 256, 768, 32), (6144, 1024, 3072, 16), (4096, 1024, 2048, 12), (8192, 1024, 4096, 9), (640, 80, 321, 20), (960, 480, 481, 7), (512, 160, 257, 11)])
def test_stft_forward_inverse_vs_oracle(eng, n_fft, hop, dim_f, frames):
    """Every FFT size on the reference's four paths (6144 MDX, 4096 Demucs, 8192 MDX23C, VR band sizes), both layouts."""
    T = hop * (frames - 1)
    if T <= n_fft // 2:
        frames = n_fft // 2 // hop + 3
        T = hop * (frames - 1)
    x = O.synth_music(3 * T, seed=5)[:, : 3 * T].reshape(2, 3, T).transpose(1, 0, 2).copy()  # (3,2,T)
    plan = eng.StftPlan(n_fft, hop)
    ref = O.stft_forward(x, n_fft, hop, dim_f)
    for layout in (eng.LAYOUT_CFT, eng.LAYOUT_CTF):
        got = plan.forward(dev(x), dim_f, 0, layout).cpu().numpy()
        if layout == eng.LAYOUT_CTF:
            got = got.transpose(0, 1, 3, 2)
        assert maxabs(got, ref) <= 2e-6 * n_fft  # un-normalised DFT: error scales with sum(window) ~ n_fft/2
        spec = ref if layout == eng.LAYOUT_CFT else np.ascontiguousarray(ref.transpose(0, 1, 3, 2))
        inv = plan.inverse(dev(spec), layout).cpu().numpy()
        assert inv.shape == (3, 2, T)
        assert maxabs(inv, O.stft_inverse(ref, n_fft, hop)) <= 5e-6
    z = plan.forward(dev(x), dim_f, 3, eng.LAYOUT_CFT).cpu().numpy()  # fused `spek[:, :, :3, :] *= 0`
    assert not z[:, :, :3].any() and maxabs(z[:, :, 3:], ref[:, :, 3:]) <= 2e-6 * n_fft


def test_stft_vs_reference_golden(eng, golden_dir):
    z = np.load(os.path.join(golden_dir, "mdx_small.npz"))
    cfg = O.MDXConfig(**SMALL)
    mix = O.synth_music(int(z["n_samples"]), seed=int(z["mix_seed"]))
    plan = eng.StftPlan(cfg.n_fft, cfg.hop_length)
    spec = plan.forward(dev(mix[None, :, : cfg.chunk_size]), cfg.dim_f).cpu().numpy()
    assert spec.shape == z["spec_ref"].shape and maxabs(spec, z["spec_ref"]) <= 1e-3
    wav = plan.inverse(dev(z["spec_ref"])).cpu().numpy()
    assert wav.shape == z["istft_ref"].shape and maxabs(wav, z["istft_ref"]) <= 5e-6


def test_stft_class_mirror(eng):
    """Same call pattern as the reference's tests/unit/test_stft.py:43-138: mono (1,16000) input -> (..., dim_f, N//hop+1)."""
    import logging

    from audio_separator.separator.uvr_lib_v5.stft import STFT

    st = STFT(logging.getLogger("t"), 2048, 512, 1025, "cuda")
    x1 = torch.rand(1, 16000, device="cuda")
    s1 = st(x1)
    assert tuple(s1.shape[-2:]) == (1025, 16000 // 512 + 1) and s1.shape[0] == 2
    ref = O.stft_forward(x1.cpu().numpy()[None], 2048, 512, 1025)[0]
    assert maxabs(s1.cpu().numpy(), ref) <= 2e-6 * 2048
    x = torch.randn(3, 2, 7680, device="cuda")
    s = st(x)
    assert tuple(s.shape) == (3, 4, 1025, 16)
    y = st.inverse(s)
    assert tuple(y.shape) == (3, 2, 7680)
    assert (y - x).abs().max().item() < 1e-4  # COLA round trip with the full one-sided spectrum
    with pytest.raises(RuntimeError):
        st(x.cpu())


# ---------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("precision", [0, 1])
def test_network_small_vs_oracle_and_golden(eng, golden_dir, precision):
    z = np.load(os.path.join(golden_dir, "mdx_small.npz"))
    cfg = O.MDXConfig(**SMALL)
    w = O.make_convtdfnet_weights(cfg, seed=int(z["weights_seed"]), out_gain=float(z["out_gain"]))
    net = make_net(eng, cfg, w, max_batch=2, precision=precision)
    rel = 1e-5 if precision == 0 else 1e-4
    spec = z["spec_ref"]
    got = net.forward(dev(spec)).cpu().numpy()
    assert maxabs(got, z["net_ref"]) <= rel * np.abs(z["net_ref"]).max()
    # batch of 3 distinct inputs through max_batch=2 (ragged last batch), CTF layout
    rng = np.random.default_rng(1)
    x3 = (rng.standard_normal((3, 4, cfg.dim_f, cfg.dim_t)) * 3).astype(np.float32)
    ref3 = O.convtdfnet_forward(w, cfg, x3)
    got3 = net.forward(dev(x3.transpose(0, 1, 3, 2)), eng.LAYOUT_CTF).cpu().numpy().transpose(0, 1, 3, 2)
    assert maxabs(got3, ref3) <= rel * np.abs(ref3).max()


@pytest.mark.parametrize("precision", [0, 1])
def test_network_mid_vs_oracle(eng, precision):
    """A 7-block net with 16..64 channels: every TFC conv and most TDF linears take the tensor-core path at precision 1."""
    cfg = O.MDXConfig(**MID)
    w = O.make_convtdfnet_weights(cfg, seed=21)
    net = make_net(eng, cfg, w, max_batch=3, precision=precision)
    rng = np.random.default_rng(2)
    x = (rng.standard_normal((3, 4, cfg.dim_f, cfg.dim_t)) * 3).astype(np.float32)
    ref = O.convtdfnet_forward(w, cfg, x, dtype="float64")
    got = net.forward(dev(x)).cpu().numpy()
    assert maxabs(got, ref) <= (1e-5 if precision == 0 else 1e-4) * np.abs(ref).max()
    got1 = net.forward(dev(x[:1])).cpu().numpy()  # batch smaller than max_batch uses a prefix of the arena
    assert maxabs(got1, ref[:1]) <= (1e-5 if precision == 0 else 1e-4) * np.abs(ref).max()


@pytest.mark.parametrize("precision", [0, 1])
def test_network_full_size_chunk_vs_golden(eng, golden_dir, precision):
    """UVR-MDX-NET-Inst_HQ_3 topology (g=48, 3072x256), one chunk, against the subsampled reference output."""
    z = np.load(os.path.join(golden_dir, "mdx_full_chunk.npz"))
    cfg = O.MDXConfig()
    w = O.make_convtdfnet_weights(cfg, seed=int(z["weights_seed"]), out_gain=float(z["out_gain"]))
    mix = O.normalize(O.synth_music(cfg.chunk_size, seed=int(z["mix_seed"])), 0.9, 0.0)
    net = make_net(eng, cfg, w, max_batch=1, precision=precision)
    e = eng.MdxEngine(net, cfg.n_fft, cfg.hop_length, cfg.dim_f, cfg.segment_size, cfg.overlap, cfg.compensate)
    spec = e.plan.forward(dev(mix[None]), cfg.dim_f, 3, eng.LAYOUT_CFT)
    assert maxabs(spec.cpu().numpy()[0, :, ::16, ::4], z["spec_ref_sub"]) <= 5e-3
    out = net.forward(spec).cpu().numpy()
    # network-output domain: fp32 path 1e-5 of max; split-bf16 path measured 1.0e-4 of max (1.2e-5 of rms) after ~65
    # sequential layers -> gate 3e-4; the binding gate is the audio-domain one below (1e-4 abs, measured 1.1e-5)
    rel = 1e-5 if precision == 0 else 3e-4
    assert maxabs(out[0, :, ::16, ::4], z["net_ref_sub"]) <= rel * np.abs(z["net_ref_sub"]).max()
    assert abs(np.abs(out.astype(np.float64)).sum() / float(z["net_abs_sum"]) - 1) < 1e-4
    wav = e.run_model(dev(mix[None])).cpu().numpy()
    assert wav.shape == (1, 2, cfg.chunk_size)
    assert maxabs(wav[0, :, ::16], z["wav_ref_sub"]) <= (2e-5 if precision == 0 else 1e-4)


# ---------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("precision", [0, 1])
def test_demix_and_separate_vs_golden(eng, golden_dir, precision):
    z = np.load(os.path.join(golden_dir, "mdx_small.npz"))
    cfg = O.MDXConfig(**SMALL)
    w = O.make_convtdfnet_weights(cfg, seed=int(z["weights_seed"]), out_gain=float(z["out_gain"]))
    mix = O.synth_music(int(z["n_samples"]), seed=int(z["mix_seed"]))
    net = make_net(eng, cfg, w, max_batch=2, precision=precision)
    e = eng.MdxEngine(net, cfg.n_fft, cfg.hop_length, cfg.dim_f, cfg.segment_size, cfg.overlap, cfg.compensate)
    tol = 2e-5 if precision == 0 else 1e-4
    mixn = O.normalize(mix, 0.9, 0.0)
    dem = e.demix_device(dev(mixn)).cpu().numpy()
    assert dem.shape == z["demix_ref"].shape == (2, mix.shape[1])  # sample count exact
    assert maxabs(dem, z["demix_ref"]) <= tol
    mm = e.demix_device(dev(mixn), is_match_mix=True).cpu().numpy()
    assert maxabs(mm, z["matchmix_ref"]) <= 2e-5
    prim, sec = e.separate_device(dev(mix))
    prim, sec = prim.cpu().numpy(), sec.cpu().numpy()
    assert prim.shape == sec.shape == (mix.shape[1], 2)  # (N,2), primary/secondary order as mdx_separator.py:163,182
    assert maxabs(prim, z["primary_ref"]) <= tol and maxabs(sec, z["secondary_ref"]) <= tol
    # PCM16 after write_audio's normalise+truncate: off by at most a few LSB of 1/32767 given the float tolerance
    for stem, ref in ((prim, z["primary_ref"]), (sec, z["secondary_ref"])):
        pcm = e.to_pcm16(dev(stem)).cpu().numpy()
        ref_pcm = O.to_pcm16(ref, 0.9, 0.0)
        assert pcm.shape == ref_pcm.shape and pcm.dtype == np.int16
        assert np.abs(pcm.astype(np.int32) - ref_pcm.astype(np.int32)).max() <= int(np.ceil(tol * 32767 * 4)) + 1
        assert np.array_equal(pcm, O.to_pcm16(stem, 0.9, 0.0))  # the device conversion itself is bit-exact
    for amplification_threshold in (0.0, 0.5):  # an all-zero stem is near-silent, also where amplifying would divide by its zero peak
        assert e.to_pcm16(dev(np.zeros_like(prim)), 0.9, amplification_threshold) is None
    # denoise branch (mdx_separator.py:435-440)
    ed = eng.MdxEngine(net, cfg.n_fft, cfg.hop_length, cfg.dim_f, cfg.segment_size, cfg.overlap, cfg.compensate, enable_denoise=True)
    den = ed.run_model(dev(mix[None, :, : cfg.chunk_size])).cpu().numpy()
    assert maxabs(den, z["denoise_ref"]) <= tol


@pytest.mark.parametrize("n", [1, 777, 6399, 6400, 6401, 12805])
def test_demix_edge_grids_vs_golden(eng, golden_dir, n):
    """Ragged / degenerate lengths through the reference's chunk grid with the identity*0.5 'network' replaced by
    is_match_mix (spectrum passes straight through; the golden was made with 0.5*spec so scale by 0.5)."""
    cfg = O.MDXConfig(**SMALL)
    edge = np.load(os.path.join(golden_dir, "mdx_edge.npz"))
    m = O.synth_music(max(n, 64), seed=99)[:, :n]
    e = eng.MdxEngine(None, cfg.n_fft, cfg.hop_length, cfg.dim_f, cfg.segment_size, cfg.overlap, cfg.compensate)
    L, step, n_chunks, _ = e.grid(n)
    assert (L, step, n_chunks) == (O.chunk_starts(n, cfg)[0], O.chunk_starts(n, cfg)[1], len(O.chunk_starts(n, cfg)[2]))
    # run the normal-overlap grid but with the pass-through spectrum: drive the C ABI pieces directly
    import ctypes as C

    from audio_separator.separator.b200._lib import check, lib

    T = cfg.chunk_size
    mixture = torch.zeros((2, L), device="cuda")
    mixture[:, cfg.trim : cfg.trim + n] = dev(m)
    chunks = torch.empty((n_chunks, 2, T), device="cuda")
    work = torch.empty(lib.b200sep_mdx_run_model_work_floats(e.plan.handle, n_chunks, T, cfg.dim_f), device="cuda")
    check(lib.b200sep_mdx_run_model(e.plan.handle, None, mixture.data_ptr(), step, L, L, n_chunks, T, cfg.dim_f, 0, chunks.data_ptr(), work.data_ptr(), None))
    out = torch.empty((2, n), device="cuda")
    check(lib.b200sep_demix_overlap_add(chunks.data_ptr(), n_chunks, T, step, L, cfg.trim, n, 1, 0.5, None, 0.0, 0, out.data_ptr(), None, None))
    torch.cuda.synchronize()
    assert maxabs(out.cpu().numpy(), edge[f"n{n}"]) <= 2e-5


def test_full_size_grid_against_oracle(eng):
    """BASELINE-size chunk grid (n_fft 6144, chunk 261120): one minute of audio through STFT -> iSTFT -> Hann
    overlap-add with the pass-through spectrum (the reference's always-run is_match_mix pass, mdx_separator.py:175),
    compared sample-for-sample with the oracle; plus linearity and the 5-minute grid sizes."""
    cfg = O.MDXConfig()
    e = eng.MdxEngine(None, cfg.n_fft, cfg.hop_length, cfg.dim_f, cfg.segment_size, cfg.overlap, cfg.compensate)
    assert e.grid(13_230_000)[2] == 68 and e.grid(13_230_000, True)[2] == 52
    N = 44100 * 60 + 123
    x = O.normalize(O.synth_music(N, seed=77), 0.9, 0.0)
    for match in (True,):
        ref = O.demix(x, cfg, None, is_match_mix=match)
        got = e.demix_device(dev(x), is_match_mix=match).cpu().numpy()
        assert got.shape == ref.shape == (2, N)
        assert maxabs(got, ref) <= 2e-5
    # normal overlap (0.25) grid with the pass-through spectrum, driven through the C ABI
    from audio_separator.separator.b200._lib import check, lib

    L, step, n_chunks, _ = e.grid(N)
    T = cfg.chunk_size
    mixture = torch.zeros((2, L), device="cuda")
    mixture[:, cfg.trim : cfg.trim + N] = dev(x)
    chunks = torch.empty((n_chunks, 2, T), device="cuda")
    work = torch.empty(lib.b200sep_mdx_run_model_work_floats(e.plan.handle, n_chunks, T, cfg.dim_f), device="cuda")
    check(lib.b200sep_mdx_run_model(e.plan.handle, None, mixture.data_ptr(), step, L, L, n_chunks, T, cfg.dim_f, 0, chunks.data_ptr(), work.data_ptr(), None))
    out = torch.empty((2, N), device="cuda")
    check(lib.b200sep_demix_overlap_add(chunks.data_ptr(), n_chunks, T, step, L, cfg.trim, N, 1, 1.0, None, 0.0, 0, out.data_ptr(), None, None))
    ref = O.demix(x, cfg, lambda s: s)
    assert maxabs(out.cpu().numpy(), ref) <= 2e-5
    got_half = e.demix_device(dev(0.5 * x), is_match_mix=True).cpu().numpy()
    assert np.abs(got_half - 0.5 * got).max() < 1e-6  # linearity


@pytest.mark.timeout(900)
def test_baseline_config1_full_size_net_three_chunks_vs_oracle(eng, golden_dir):
    """BASELINE configs[0]: 10 s of 44.1 kHz stereo through the WHOLE path at the Inst_HQ_3 sizes -- 3 overlapping chunks, the full-size ConvTDFNet
    (16.7 M parameters), STFT / iSTFT 6144, Hann overlap-add, peak normalisation, secondary = mix - compensate * primary -- MdxEngine.separate_device
    against oracle.separate_arrays (the reference's algorithm on the CPU), both arithmetic paths of the library.  Gate: 1e-4 max-abs per sample."""
    from audio_separator.separator.b200 import mdx_weights

    cfg = O.MDXConfig()
    N = 441_000
    assert eng.MdxEngine(None, cfg.n_fft, cfg.hop_length, cfg.dim_f, cfg.segment_size, cfg.overlap).grid(N)[2] == 3
    z = np.load(os.path.join(golden_dir, "mdx_full_chunk.npz"))  # the weights of the full-size golden: output gain chosen for a 0.5 peak on this programme material
    w = O.make_convtdfnet_weights(cfg, seed=int(z["weights_seed"]), out_gain=float(z["out_gain"]))
    mix = O.synth_music(N, seed=1234)
    torch.set_num_threads(min(32, os.cpu_count() or 8))
    ref_p, ref_s = O.separate_arrays(mix, cfg, lambda s: O.convtdfnet_forward(w, cfg, s))
    assert ref_p.shape == (N, 2) and float(np.abs(ref_p).max()) > 0.05  # a real signal level: 1e-4 absolute is then a meaningful gate
    hp = mdx_weights.infer_hparams_from_state(w)
    flat = mdx_weights.flatten_state(w, **hp)
    for precision, batch in ((1, 2), (0, 1)):
        net = eng.MdxNet(flat, dim_t=cfg.dim_t, max_batch=batch, precision=precision, **hp)
        e = eng.MdxEngine(net, cfg.n_fft, cfg.hop_length, cfg.dim_f, cfg.segment_size, cfg.overlap, cfg.compensate, batch_size=batch)
        p, s = e.separate_device(dev(mix))
        ep, es = maxabs(p.cpu().numpy(), ref_p), maxabs(s.cpu().numpy(), ref_s)
        print(f"config 1, precision {precision}: max|gpu - oracle| primary {ep:.2e} secondary {es:.2e}")
        assert ep <= 1e-4 and es <= 1e-4, (precision, ep, es)
        del e, net


def test_device_output_pipeline_matches_host_writer(eng, tmp_path):
    """CommonSeparator.pcm_bytes on a CUDA stem (absmax / normalize / to_pcm_bytes kernels, bytes downloaded) == the numpy path on the same stem, every bit depth and both writers."""
    import logging

    from audio_separator.separator.common_separator import CommonSeparator, DeviceStem

    x = (O.synth_music(50_001, seed=4) * 1.3).T.copy()  # peak above the 0.9 threshold: the normalisation is active
    for bits in (16, 24, 32):
        for use_sf in (False, True):
            cs = CommonSeparator(dict(logger=logging.getLogger("t"), model_name="m", model_path="/x/m.onnx", model_data={"primary_stem": "Vocals"}, output_dir=str(tmp_path),
                                      output_format="WAV", normalization_threshold=0.9, amplification_threshold=0.0, sample_rate=44100, use_soundfile=use_sf))
            cs.input_bit_depth = bits
            host = cs.pcm_bytes(x)
            devb = cs.pcm_bytes(dev(x))
            assert host[0] == devb[0] == bits and len(devb[1]) == x.size * bits // 8
            a, b = np.frombuffer(host[1], np.uint8).astype(np.int32), np.frombuffer(devb[1], np.uint8).astype(np.int32)
            if use_sf and bits > 16:  # x * scale is rounded once on the device and once in numpy: identical inputs, identical fp32 products
                assert np.array_equal(a, b)
            else:
                assert np.array_equal(a, b), (bits, use_sf)
    assert cs.pcm_bytes(dev(np.zeros((100, 2), np.float32))) is None  # near-silent stems are skipped like the reference does
    st = DeviceStem(dev(x))
    assert np.array_equal(np.asarray(st), x) and st.shape == x.shape


def test_mdx_separator_plugin_end_to_end(eng, tmp_path):
    """Separator(...).load_model(); separate(wav) -> two WAVs, secondary first, names as the reference builds them."""
    import wave

    from audio_separator.separator import Separator

    cfg = O.MDXConfig(**SMALL)
    w = O.make_convtdfnet_weights(cfg, seed=7, out_gain=0.05)
    np.savez(tmp_path / "tiny-mdx.npz", **w)
    (tmp_path / "tiny-mdx.json").write_text('{"compensate": 1.022, "mdx_dim_f_set": 768, "mdx_dim_t_set": 5, "mdx_n_fft_scale_set": 1536, "primary_stem": "Instrumental"}')
    mix = O.synth_music(30000, seed=3)
    pcm = (mix.T * 32767).astype("<i2")
    with wave.open(str(tmp_path / "song.wav"), "wb") as wf:
        wf.setnchannels(2); wf.setsampwidth(2); wf.setframerate(44100); wf.writeframes(pcm.tobytes())
    sep = Separator(model_file_dir=str(tmp_path), output_dir=str(tmp_path / "out"), mdx_params={"hop_length": 256, "segment_size": 32, "overlap": 0.25, "batch_size": 2, "enable_denoise": False, "b200_precision": 0})
    sep.load_model("tiny-mdx.npz")
    files = sep.separate(str(tmp_path / "song.wav"))
    assert files == ["song_(Vocals)_tiny-mdx.wav", "song_(Instrumental)_tiny-mdx.wav"]
    loaded = pcm.astype(np.float32).T / 32768.0
    prim, sec = O.separate_arrays(loaded, cfg, lambda s: O.convtdfnet_forward(w, cfg, s))
    for fname, ref in zip(files, (sec, prim)):
        with wave.open(str(tmp_path / "out" / fname)) as wf:
            assert wf.getnframes() == 30000 and wf.getnchannels() == 2
            got = np.frombuffer(wf.readframes(30000), dtype="<i2").astype(np.int32)
        want = O.to_pcm16(ref, 0.9, 0.0).astype(np.int32)
        assert np.abs(got - want).max() <= 3  # <= 1e-4 * 32767 LSB
