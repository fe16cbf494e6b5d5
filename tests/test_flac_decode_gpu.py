"""GPU FLAC decoder (csrc/flac_decode.cu, b200/flac.py decode, CommonSeparator.prepare_mix on FLAC input): real encoders' frames, GPU encoder
round trips, every writer stream, false sync patterns, damaged streams, prepare_mix parity with the WAV reader, and the plugins on FLAC input."""
import json
import logging
import os
import wave

import numpy as np
import pytest
import torch

import flac_oracle as F
import flac_stream_oracle as S
import flac_writer as W
import mdx_oracle as O

pytestmark = pytest.mark.gpu

SR = 44100


@pytest.fixture(scope="module")
def flac(lib_built):
    assert torch.cuda.is_available()
    from audio_separator.separator.b200 import flac

    return flac


def gpu_ints(flac, data):
    """Decode on the GPU -> (N, C') int64, checking that every float is exactly int * 2^-(bps-1)."""
    mix, info = flac.decode(data)
    x = mix.cpu().numpy().astype(np.float64) * float(1 << (info["bps"] - 1))
    ints = np.rint(x).astype(np.int64)
    assert np.array_equal(ints.astype(np.float64), x), "a decoded float is not an integer times 2^-(bps-1)"
    return ints.T, info


def stream_of(streaminfo, frames):
    return b"fLaC" + bytes([0x80]) + len(streaminfo).to_bytes(3, "big") + streaminfo + frames


def test_golden_frames_of_real_encoders(flac, golden_dir):
    for name in ("flac_frames.npz", "flac_decode.npz"):
        g = dict(np.load(os.path.join(golden_dir, name)))
        tags = sorted({k[: -len("_frames")] for k in g if k.endswith("_frames")})
        assert tags
        for tag in tags:
            data = stream_of(g[f"{tag}_streaminfo"].tobytes(), g[f"{tag}_frames"].tobytes())
            got, info = gpu_ints(flac, data)
            want = g[f"{tag}_samples"].astype(np.int64)
            assert np.array_equal(got, want[:, :2]), tag
            d = S.decode(data, first_anywhere=True)
            assert np.array_equal(got, d.samples[:, :2]), tag
            assert info["frames"] == len(d.frames) and info["first_number"] == d.streaminfo.get("first_number", 0), tag


def test_encoder_roundtrip_matrix(flac):
    from test_flac_gpu import LENGTHS, SIGNALS, WRITERS, separator, signal, wav_samples

    import tempfile

    with tempfile.TemporaryDirectory() as tmp:
        for kind in SIGNALS:
            for n in LENGTHS:
                for bits, use_sf in WRITERS:
                    cs = separator(tmp, bits, use_sf)
                    bps = flac.stream_bps(bits, use_sf)
                    if bps is None:
                        continue
                    x = torch.as_tensor(signal(kind, n, seed=n)).cuda()
                    data = flac.encode(cs._normalized_on_device(x), bits, not use_sf, bps, SR)
                    got, info = gpu_ints(flac, data)
                    _, want = wav_samples(cs, signal(kind, n, seed=n))
                    assert np.array_equal(got << (bits - bps), want), (kind, n, bits, use_sf)
                    again, _ = gpu_ints(flac, data)
                    assert np.array_equal(again, got)


@pytest.mark.parametrize("bits", (16, 24))
def test_five_minute_roundtrip(flac, tmp_path, bits):
    from test_flac_gpu import separator, wav_samples

    n = 5 * 60 * SR
    rng = np.random.default_rng(bits)
    x = np.cumsum(rng.standard_normal((n, 2)), axis=0)
    x = (0.8 * x / np.abs(x).max()).astype(np.float32)
    cs = separator(tmp_path, bits, False)
    data = flac.encode(cs._normalized_on_device(torch.as_tensor(x).cuda()), bits, True, bits, SR)
    got, info = gpu_ints(flac, data)
    _, want = wav_samples(cs, x)
    assert info["n_samples"] == n and np.array_equal(got, want)
    mix1, _ = flac.decode(data)
    mix2, _ = flac.decode(data)
    assert torch.equal(mix1, mix2)


@pytest.fixture(scope="module")
def writer_cases():
    return W.cases()


def test_writer_streams(flac, writer_cases):
    seen = set()
    for name, (data, want, tools) in writer_cases.items():
        got, info = gpu_ints(flac, data)
        assert np.array_equal(got, want[:, :2]), name
        seen |= tools
    assert W.REQUIRED_TOOLS <= seen, sorted(W.REQUIRED_TOOLS - seen)


def _verbatim_frame_with(payload: bytes, bs=1024):
    """Samples of a stereo 16-bit VERBATIM frame whose channel-0 bytes begin with `payload` (VERBATIM 16-bit samples are byte aligned)."""
    rng = np.random.default_rng(len(payload))
    x = rng.integers(-3000, 3000, (bs, 2))
    pad = payload + bytes(len(payload) & 1)
    vals = np.frombuffer(pad, ">i2").astype(np.int64)
    x[: len(vals), 0] = vals
    return x


def _fake_header(number, bs_code=12):
    h = bytes([0xFF, 0xF8, (bs_code << 4) | 9, (1 << 4) | (4 << 1)]) + W.utf8_number(number)
    return h + bytes([W.crc8(h)])


def test_false_sync_patterns(flac, writer_cases):
    frames = []
    for k in range(4):
        fakes = _fake_header(k + 1) + b"\x12\x34" + _fake_header(k) + _fake_header(k + 2, bs_code=10) + _fake_header(k + 1)
        frames.append(W.Frame(_verbatim_frame_with(fakes), subs=[W.Sub("verbatim")]))
    # a fake header with the next frame's number in the last bytes of the last subframe, right before the CRC-16 where a real frame could start
    x = frames[1].samples.copy()
    fake = _fake_header(2)
    tail = np.frombuffer(fake + bytes(len(fake) & 1), ">i2").astype(np.int64)
    x[-len(tail):, 1] = tail
    frames[1] = W.Frame(x, subs=[W.Sub("verbatim")])
    data, want = W.stream(frames, SR, 16)
    assert data.count(_fake_header(2)) >= 3
    assert np.array_equal(F.decode(data).samples, want)
    got, info = gpu_ints(flac, data)
    assert info["frames"] == 4 and np.array_equal(got, want)


def _gpu_stream(flac, n=3 * 4096 + 100, seed=3):
    x = torch.as_tensor(np.ascontiguousarray(O.synth_music(n, seed=seed).T * 0.5, dtype=np.float32)).cuda()
    data = flac.encode(x, 16, True, 16, SR)
    return data, F.decode(data)


def test_damaged_streams(flac, writer_cases):
    good, dg = _gpu_stream(flac)
    want_good = dg.samples
    (s1, l1, _) = dg.frames[1]
    cases = {}
    b = bytearray(good); b[s1 + 2] ^= 0x01; cases["header bit"] = bytes(b)
    b = bytearray(good); b[s1 + l1 // 2] ^= 0x08; cases["residual bit"] = bytes(b)
    b = bytearray(good); b[s1 + l1 - 1] ^= 0x40; cases["CRC-16 bit"] = bytes(b)
    cases["truncated last frame"] = good[:-10]
    # a reserved subframe type and a residual that runs past its frame, both with valid CRCs
    data, _ = W.stream([W.Frame(W.signal(4096, 16, 2, 1))], SR, 16)
    begin = flac.parse(data)[1]
    frame = bytearray(data[begin:])
    frame[6] = 2 << 1  # subframe type 2 is reserved
    cases["reserved subframe type"] = data[:begin] + bytes(frame[:-2]) + W.crc16(frame[:-2]).to_bytes(2, "big")
    frame = bytearray(data[begin:-200])
    cases["residual overruns its frame"] = data[:begin] + bytes(frame) + W.crc16(frame).to_bytes(2, "big")
    for name, bad in cases.items():
        with pytest.raises(ValueError, match=r"FLAC frame \d+ at byte \d+"):
            flac.decode(bad)
        got, _ = gpu_ints(flac, good)  # nothing latched
        assert np.array_equal(got, want_good), name
    for cut in (3, 20, 41):
        with pytest.raises(ValueError, match="truncated FLAC metadata|no fLaC"):
            flac.decode(good[:cut])
    assert np.array_equal(gpu_ints(flac, good)[0], want_good)


def _separator(tmp, fmt="WAV"):
    from audio_separator.separator.common_separator import CommonSeparator

    return CommonSeparator(dict(logger=logging.getLogger("flac-in"), model_name="m", model_path="/x/m.onnx", model_data={"primary_stem": "Vocals"},
                                output_dir=str(tmp), output_format=fmt, normalization_threshold=0.9, amplification_threshold=0.0, sample_rate=SR,
                                torch_device=torch.device("cuda", 0)))


def _write_wav(path, ints, width, rate=SR):
    q = np.ascontiguousarray(ints, dtype=np.int64)
    raw = q.astype("<i4").view(np.uint8).reshape(-1, 4)[:, :width]
    with wave.open(str(path), "wb") as wf:
        wf.setnchannels(q.shape[1]); wf.setsampwidth(width); wf.setframerate(rate); wf.writeframes(raw.tobytes())


@pytest.mark.parametrize("bps", (8, 12, 16, 20, 24))
def test_prepare_mix_equals_wav(flac, tmp_path, bps):
    from audio_separator.separator.common_separator import DeviceStem

    x = W.signal(10000, bps, 2, bps)
    data, _ = W.stream([W.Frame(y) for y in np.array_split(x, 3)], SR, bps)
    (tmp_path / "a.flac").write_bytes(data)
    width = 2 if bps <= 16 else 3
    _write_wav(tmp_path / "a.wav", x << (8 * width - bps), width)
    cf, cw = _separator(tmp_path), _separator(tmp_path)
    mf, mw = cf.prepare_mix(str(tmp_path / "a.flac")), cw.prepare_mix(str(tmp_path / "a.wav"))
    assert isinstance(mf, DeviceStem) and mf.tensor.is_cuda and mf.shape == mw.shape
    assert np.array_equal(mf.tensor.cpu().numpy(), mw)
    assert cf.input_bit_depth == cw.input_bit_depth == 8 * width


def test_prepare_mix_channels_rate_and_silence(flac, tmp_path):
    cs = _separator(tmp_path)
    mono = W.signal(5000, 16, 1, 1)
    (tmp_path / "m.flac").write_bytes(W.stream([W.Frame(mono)], SR, 16)[0])
    _write_wav(tmp_path / "m.wav", mono, 2)
    m = cs.prepare_mix(str(tmp_path / "m.flac")).tensor.cpu().numpy()
    assert m.shape == (2, 5000) and np.array_equal(m[0], m[1]) and np.array_equal(m, cs.prepare_mix(str(tmp_path / "m.wav")))
    x6 = W.signal(5000, 16, 6, 2)
    (tmp_path / "s.flac").write_bytes(W.stream([W.Frame(x6)], SR, 16)[0])
    _write_wav(tmp_path / "s.wav", x6, 2)
    assert np.array_equal(cs.prepare_mix(str(tmp_path / "s.flac")).tensor.cpu().numpy(), cs.prepare_mix(str(tmp_path / "s.wav")))
    (tmp_path / "r.flac").write_bytes(W.stream([W.Frame(W.signal(4800, 16, 2, 3))], 48000, 16)[0])
    with pytest.raises(RuntimeError, match="cannot decode"):
        cs.prepare_mix(str(tmp_path / "r.flac"))
    (tmp_path / "z.flac").write_bytes(W.stream([W.Frame(np.zeros((4096, 2), np.int64), subs=[W.Sub("constant")])], SR, 16)[0])
    with pytest.raises(ValueError, match="empty or not valid"):
        cs.prepare_mix(str(tmp_path / "z.flac"))
    # content, not the extension, selects the decoder: a FLAC stream behind an ID3v2 tag, named .wav
    data, want = W.stream([W.Frame(W.signal(3000, 16, 2, 4))], SR, 16, id3v2_tag=W.id3v2(25))
    (tmp_path / "tagged.wav").write_bytes(data)
    got = cs.prepare_mix(str(tmp_path / "tagged.wav")).tensor.cpu().numpy()
    assert np.array_equal(got, (want.T / 32768.0).astype(np.float32))


def _song_pair(tmp, n=30000, seed=3):
    ints = (O.synth_music(n, seed=seed).T * 32767).astype(np.int64)
    _write_wav(tmp / "song.wav", ints, 2)
    (tmp / "songf.flac").write_bytes(W.stream([W.Frame(y) for y in np.array_split(ints, 8)], SR, 16)[0])
    os.makedirs(tmp / "flacdir", exist_ok=True)
    return ints


def _separate_both(tmp, model, out, **params):
    from audio_separator.separator import Separator

    res = {}
    for fmt in ("WAV", "FLAC"):
        sep = Separator(model_file_dir=str(tmp), output_dir=str(tmp / f"{out}_{fmt}"), output_format=fmt, **params)
        sep.load_model(model)
        for src in ("song.wav", "songf.flac"):
            import random

            random.seed(1234)
            files = sep.separate(str(tmp / src))
            res[fmt, src] = [open(tmp / f"{out}_{fmt}" / f, "rb").read() for f in files]
    return res


def _assert_same(res):
    for fmt in ("WAV", "FLAC"):
        a, b = res[fmt, "song.wav"], res[fmt, "songf.flac"]
        assert len(a) >= 2 and a == b, fmt


def test_mdx_plugin_flac_input_stays_on_device(flac, tmp_path, monkeypatch):
    from audio_separator.separator.common_separator import DeviceStem

    cfg = O.MDXConfig(n_fft=1536, hop_length=256, dim_f=768, dim_t=32, segment_size=32, g=8)
    np.savez(tmp_path / "tiny-mdx.npz", **O.make_convtdfnet_weights(cfg, seed=7, out_gain=0.05))
    (tmp_path / "tiny-mdx.json").write_text('{"compensate": 1.022, "mdx_dim_f_set": 768, "mdx_dim_t_set": 5, "mdx_n_fft_scale_set": 1536, "primary_stem": "Instrumental"}')
    _song_pair(tmp_path)

    def no_download(self, dtype=None, copy=None):
        raise AssertionError("the mix was downloaded to the host")

    monkeypatch.setattr(DeviceStem, "__array__", no_download)
    params = {"hop_length": 256, "segment_size": 32, "overlap": 0.25, "batch_size": 2, "enable_denoise": False, "b200_precision": 0}
    _assert_same(_separate_both(tmp_path, "tiny-mdx.npz", "mdx", mdx_params=params))


def test_mdxc_demucs_vr_plugins_flac_input(flac, tmp_path):
    import demucs_oracle as D
    import vr_oracle as V
    from test_autocast_separator_gpu import _mdx23c_files, _roformer_files
    from test_demucs_gpu import SMALL, _write_package

    _song_pair(tmp_path)
    _roformer_files(tmp_path)
    _assert_same(_separate_both(tmp_path, "tiny_bs_roformer.npz", "rof", mdxc_params={"batch_size": 4, "segment_size": 65}))
    _mdx23c_files(tmp_path)
    _assert_same(_separate_both(tmp_path, "tiny-mdx23c.npz", "mdx23c", mdxc_params={"overlap": 4, "batch_size": 2, "segment_size": 16}))
    ocfg = D.HTConfig(**SMALL)
    _write_package(str(tmp_path / "aaaa1111.th"), ocfg, D.make_weights(ocfg, seed=21))
    _write_package(str(tmp_path / "bbbb2222.th"), ocfg, D.make_weights(ocfg, seed=22))
    (tmp_path / "tiny_ft.yaml").write_text("models: ['aaaa1111', 'bbbb2222']\nweights: [[1, 0, 1, 1], [0, 1, 1, 0]]\n")
    _assert_same(_separate_both(tmp_path, "tiny_ft.yaml", "demucs", demucs_params={"shifts": 1, "batch_size": 2}))
    np.savez(tmp_path / "tiny-vr51.npz", **V.make_weights_51(256, 8, 16, seed=5))
    (tmp_path / "tiny-vr51.json").write_text('{"vr_model_param": "tiny_1band_51", "primary_stem": "Vocals", "nout": 8, "nout_lstm": 16}')
    p = V.single_band_param(n_fft=256, hl=64, bins=128, pre_filter_start=120, pre_filter_stop=127)
    (tmp_path / "tiny_1band_51.json").write_text(json.dumps({k: v for k, v in p.items() if not isinstance(v, bool)}))
    _assert_same(_separate_both(tmp_path, "tiny-vr51.npz", "vr", vr_params={"window_size": 160, "batch_size": 4, "aggression": 5}))


def test_separate_directory_with_flac_and_wav(flac, tmp_path):
    from audio_separator.separator import Separator

    cfg = O.MDXConfig(n_fft=1536, hop_length=256, dim_f=768, dim_t=32, segment_size=32, g=8)
    np.savez(tmp_path / "tiny-mdx.npz", **O.make_convtdfnet_weights(cfg, seed=7, out_gain=0.05))
    (tmp_path / "tiny-mdx.json").write_text('{"compensate": 1.022, "mdx_dim_f_set": 768, "mdx_dim_t_set": 5, "mdx_n_fft_scale_set": 1536, "primary_stem": "Instrumental"}')
    _song_pair(tmp_path)
    d = tmp_path / "in"
    d.mkdir()
    os.replace(tmp_path / "song.wav", d / "a.wav")
    os.replace(tmp_path / "songf.flac", d / "b.flac")
    params = {"hop_length": 256, "segment_size": 32, "overlap": 0.25, "batch_size": 2, "enable_denoise": False, "b200_precision": 0}
    sep = Separator(model_file_dir=str(tmp_path), output_dir=str(tmp_path / "out"), output_format="WAV", mdx_params=params)
    sep.load_model("tiny-mdx.npz")
    files = sorted(os.path.basename(f) for f in sep.separate(str(d)))
    assert files == ["a_(Instrumental)_tiny-mdx.wav", "a_(Vocals)_tiny-mdx.wav", "b_(Instrumental)_tiny-mdx.wav", "b_(Vocals)_tiny-mdx.wav"], files
    for stem in ("Instrumental", "Vocals"):
        assert (tmp_path / "out" / f"a_({stem})_tiny-mdx.wav").read_bytes() == (tmp_path / "out" / f"b_({stem})_tiny-mdx.wav").read_bytes()
