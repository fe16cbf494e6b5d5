"""GPU PCM decoder (csrc/pcm_decode.cu, b200/pcm_reader.py decode, CommonSeparator.prepare_mix on float / 8-bit WAV, RF64 and AIFF input): the
kernel bit for bit against the numpy restatement for every format, channel count and tile boundary, prepare_mix parity with the integer WAV
reader, and the plugins and Separator.separate(directory) on these inputs."""
import json
import os
import wave

import numpy as np
import pytest
import torch

import mdx_oracle as O
import pcm_writer as W
from test_flac_decode_gpu import _separator, _write_wav

pytestmark = pytest.mark.gpu

SR = 44100
FIVE_MINUTES = 5 * 60 * SR


@pytest.fixture(scope="module")
def pcm(lib_built):
    assert torch.cuda.is_available()
    from audio_separator.separator.b200 import pcm_reader

    return pcm_reader


def tile_frames(frame_bytes):
    """Frames per CTA of pcm_decode_kernel (csrc/pcm_decode.cu)."""
    return min(1024, max(1, 32768 // frame_bytes))


def random_payload(n, frame_bytes, fmt, seed):
    """Random bytes (every integer value, and for floats every class: normals, subnormals, infinities, NaNs with payloads), plus specials."""
    rng = np.random.default_rng(seed)
    raw = rng.integers(0, 256, size=n * frame_bytes, dtype=np.uint8)
    b = W.SAMPLE_BYTES[fmt]
    if fmt in W.FLOATS and n >= 8:
        specials = [np.inf, -np.inf, np.nan, -0.0, 1e-40, 3.4e38, 1.0, -1.0]
        for i, v in enumerate(specials):
            raw[i * frame_bytes:i * frame_bytes + b] = np.frombuffer(W.payload(np.array([[v]]), fmt), np.uint8)
    return raw.tobytes()


def gpu_decode(pcm, data, n, frame_bytes, channels, fmt, out_channels):
    from audio_separator.separator.b200._lib import check, lib

    host = np.zeros(max(16, (len(data) + 15) // 16 * 16), np.uint8)
    host[:len(data)] = np.frombuffer(data, np.uint8)
    buf = torch.from_numpy(host).cuda()
    out = torch.full((out_channels, n), float("nan"), dtype=torch.float32, device="cuda")
    check(lib.b200sep_pcm_decode_f32(buf.data_ptr(), n, frame_bytes, channels, fmt, out_channels, out.data_ptr(), n,
                                     torch.cuda.current_stream().cuda_stream), "pcm_decode_f32")
    torch.cuda.synchronize()
    return out.cpu().numpy()


def assert_bits_equal(got, want):
    assert got.shape == want.shape
    bad = np.flatnonzero(got.view(np.uint32) != want.view(np.uint32))
    assert bad.size == 0, f"{bad.size} samples differ, first at {bad[0]}: {got.flat[bad[0]]!r} vs {want.flat[bad[0]]!r}"


@pytest.mark.parametrize("fmt", range(12), ids=W.NAMES)
def test_kernel_every_format_channels_and_tile_boundary(pcm, fmt):
    b = W.SAMPLE_BYTES[fmt]
    for channels in (1, 2, 3, 6):
        for frame_bytes in (channels * b, channels * b + 3):  # tight, and a padded block align
            t = tile_frames(frame_bytes)
            for n in (0, 1, t - 1, t, t + 1, 3 * t + 5):
                data = random_payload(n, frame_bytes, fmt, seed=1000 * fmt + 10 * channels + n % 7)
                oc = min(channels, 2)
                got = gpu_decode(pcm, data, n, frame_bytes, channels, fmt, oc)
                assert_bits_equal(got, W.restate(data, n, frame_bytes, channels, fmt, oc))
            # every channel of the frame, not only the two a mix keeps
            data = random_payload(t + 3, frame_bytes, fmt, seed=fmt)
            assert_bits_equal(gpu_decode(pcm, data, t + 3, frame_bytes, channels, fmt, channels), W.restate(data, t + 3, frame_bytes, channels, fmt, channels))


@pytest.mark.parametrize("fmt", range(12), ids=W.NAMES)
def test_kernel_five_minutes(pcm, fmt):
    fb = 2 * W.SAMPLE_BYTES[fmt]
    data = random_payload(FIVE_MINUTES, fb, fmt, seed=fmt)
    assert_bits_equal(gpu_decode(pcm, data, FIVE_MINUTES, fb, 2, fmt, 2), W.restate(data, FIVE_MINUTES, fb, 2, fmt, 2))


def test_kernel_rejects_bad_arguments(pcm):
    from audio_separator.separator.b200._lib import lib

    buf = torch.zeros(64, dtype=torch.uint8, device="cuda")
    out = torch.empty(64, dtype=torch.float32, device="cuda")
    st = torch.cuda.current_stream().cuda_stream
    assert lib.b200sep_pcm_decode_f32(buf.data_ptr(), 4, 4, 2, 12, 2, out.data_ptr(), 4, st) != 0  # unknown format
    assert lib.b200sep_pcm_decode_f32(buf.data_ptr(), 4, 3, 2, W.S16LE, 2, out.data_ptr(), 4, st) != 0  # frame too small for 2 x 16 bits
    assert lib.b200sep_pcm_decode_f32(buf.data_ptr(), 4, 4, 2, W.S16LE, 3, out.data_ptr(), 4, st) != 0  # more output rows than channels
    assert lib.b200sep_pcm_decode_f32(buf.data_ptr(), 4, 4, 2, W.S16LE, 0, out.data_ptr(), 4, st) != 0
    assert lib.b200sep_pcm_decode_f32(buf.data_ptr() + 1, 4, 4, 2, W.S16LE, 2, out.data_ptr(), 4, st) != 0  # misaligned payload
    assert lib.b200sep_pcm_decode_f32(buf.data_ptr(), 4, 4, 2, W.S16LE, 2, out.data_ptr(), 4, st) == 0


def test_decode_writer_streams(pcm):
    """Every writer stream through pcm_reader.decode equals the restatement of its payload."""
    for name, blob, want in W.cases():
        mix, info = pcm.decode(blob)
        ref = W.restate(blob[info["begin"]:], info["n_frames"], info["block_align"], info["channels"], info["format"], min(info["channels"], 2))
        assert info["bytes_uploaded"] == want["nbytes"] - want["nbytes"] % want["block_align"], name
        assert_bits_equal(mix.cpu().numpy(), ref)


# ---- prepare_mix -----------------------------------------------------------------------------------------------------------------------

def _write(path, blob):
    path.write_bytes(blob)
    return str(path)


@pytest.mark.parametrize("bits", (8, 16, 24))
def test_prepare_mix_aiff_equals_wav(pcm, tmp_path, bits):
    from audio_separator.separator.common_separator import DeviceStem

    x = W.ints(10000, 2, bits, seed=bits)
    fmt = {8: W.S8, 16: W.S16BE, 24: W.S24BE}[bits]
    width = max(2, bits // 8)
    _write_wav(tmp_path / "a.wav", x << (8 * width - bits), width)  # an 8-bit sample is the 16-bit sample << 8: the same float
    ca, cw = _separator(tmp_path), _separator(tmp_path)
    ma = ca.prepare_mix(_write(tmp_path / "a.aiff", W.aiff(W.payload(x, fmt), 2, SR, bits)))
    mw = cw.prepare_mix(str(tmp_path / "a.wav"))
    assert isinstance(ma, DeviceStem) and ma.tensor.is_cuda and isinstance(mw, np.ndarray)
    assert np.array_equal(ma.tensor.cpu().numpy(), mw)
    assert ca.input_bit_depth == cw.input_bit_depth == 8 * width
    assert ca.input_subtype == {8: "PCM_S8", 16: "PCM_16", 24: "PCM_24"}[bits]


def test_prepare_mix_float_rf64_rate_and_silence(pcm, tmp_path):
    from audio_separator.separator.common_separator import DeviceStem

    cs = _separator(tmp_path)
    k = W.ints(8000, 2, 16, seed=4)
    _write_wav(tmp_path / "k.wav", k, 2)
    m16 = cs.prepare_mix(str(tmp_path / "k.wav"))
    for fmt, tag, bits in ((W.F32LE, 3, 32), (W.F64LE, 3, 64)):
        m = cs.prepare_mix(_write(tmp_path / f"f{bits}.wav", W.wav(W.payload(k / 32768.0, fmt), tag, 2, SR, bits // 4, bits)))
        assert isinstance(m, DeviceStem) and np.array_equal(m.tensor.cpu().numpy(), m16)
    riff = W.wav(W.payload(k, W.S24LE), 1, 2, SR, 6, 24)
    rf64 = W.wav(W.payload(k, W.S24LE), 1, 2, SR, 6, 24, rf64=True)
    a = cs.prepare_mix(_write(tmp_path / "r.wav", riff))
    b = cs.prepare_mix(_write(tmp_path / "r64.wav", rf64))
    assert isinstance(b, DeviceStem) and np.array_equal(np.asarray(a), b.tensor.cpu().numpy())
    # 8-bit WAV (unsigned) and mono
    u = W.ints(3000, 1, 8, seed=6)
    m8 = cs.prepare_mix(_write(tmp_path / "u8.wav", W.wav(W.payload(u + 128, W.U8), 1, 1, SR, 1, 8)))
    assert m8.shape == (2, 3000) and np.array_equal(m8.tensor.cpu().numpy(), np.repeat((u.T / 128.0).astype(np.float32), 2, 0))
    assert (cs.input_bit_depth, cs.input_subtype) == (16, "PCM_U8")
    # the rate rule of the WAV and FLAC readers holds: no resampling here
    _write(tmp_path / "r48.wav", W.wav(W.payload(k / 32768.0, W.F32LE), 3, 2, 48000, 8, 32))
    with pytest.raises(RuntimeError, match="cannot decode"):
        cs.prepare_mix(str(tmp_path / "r48.wav"))
    _write(tmp_path / "z.wav", W.wav(W.payload(np.zeros((4096, 2)), W.F32LE), 3, 2, SR, 8, 32))
    with pytest.raises(ValueError, match="empty or not valid"):
        cs.prepare_mix(str(tmp_path / "z.wav"))


def test_input_bit_depth_every_format(pcm, tmp_path):
    cs = _separator(tmp_path)
    x = W.ints(500, 2, 8, seed=1)
    files = {
        (16, "PCM_U8"): W.wav(W.payload(x + 128, W.U8), 1, 2, SR, 2, 8),
        (16, "PCM_S8"): W.aiff(W.payload(x, W.S8), 2, SR, 8),
        (16, "PCM_16"): W.aiff(W.payload(x, W.S16LE), 2, SR, 16, compression=b"sowt"),
        (24, "PCM_24"): W.aiff(W.payload(x, W.S24BE), 2, SR, 20),
        (32, "PCM_32"): W.wav(W.payload(x, W.S32LE), 1, 2, SR, 8, 32, extensible=True, valid_bits=24, rf64=True),
        (32, "FLOAT"): W.aiff(W.payload(x / 128.0, W.F32BE), 2, SR, 32, compression=b"fl32"),
        (32, "DOUBLE"): W.wav(W.payload(x / 128.0, W.F64LE), 3, 2, SR, 16, 64),
    }
    for (depth, sub), blob in files.items():
        cs.prepare_mix(_write(tmp_path / f"{sub}.aif", blob))
        assert (cs.input_bit_depth, cs.input_subtype) == (depth, sub)


# ---- plugins and directories ---------------------------------------------------------------------------------------------------------

def _song_set(tmp, n=30000, seed=3):
    """song.wav (16-bit, the host reader), songa.aiff (the same integers, 16-bit AIFF) and songf.wav (32-bit float k / 32768)."""
    k = (O.synth_music(n, seed=seed).T * 32767).astype(np.int64)
    _write_wav(tmp / "song.wav", k, 2)
    (tmp / "songa.aiff").write_bytes(W.aiff(W.payload(k, W.S16BE), 2, SR, 16))
    (tmp / "songf.wav").write_bytes(W.wav(W.payload(k / 32768.0, W.F32LE), 3, 2, SR, 8, 32))


def _separate_all(tmp, model, out, **params):
    import random

    from audio_separator.separator import Separator

    res = {}
    for fmt in ("WAV", "FLAC"):
        sep = Separator(model_file_dir=str(tmp), output_dir=str(tmp / f"{out}_{fmt}"), output_format=fmt, **params)
        sep.load_model(model)
        for src in ("song.wav", "songa.aiff", "songf.wav"):
            random.seed(1234)
            files = sep.separate(str(tmp / src))
            res[fmt, src] = [str(tmp / f"{out}_{fmt}" / f) for f in files]
    return res


def _wav_ints(path):
    with wave.open(path, "rb") as wf:
        width, raw = wf.getsampwidth(), wf.readframes(wf.getnframes())
    return width, np.frombuffer(raw, {2: "<i2", 4: "<i4"}[width]).astype(np.int64)


def _assert_stems(res):
    from audio_separator.separator.b200 import flac

    a, b, f = res["WAV", "song.wav"], res["WAV", "songa.aiff"], res["WAV", "songf.wav"]
    assert len(a) >= 2 and len(a) == len(b) == len(f)
    for pa, pb, pf in zip(a, b, f):
        assert open(pa, "rb").read() == open(pb, "rb").read()
        (wa, qa), (wf, qf) = _wav_ints(pa), _wav_ints(pf)
        assert (wa, wf) == (2, 4) and np.array_equal(qf >> 16, qa)  # the pydub writer's 32-bit samples are int16 << 16
    a, b, f = res["FLAC", "song.wav"], res["FLAC", "songa.aiff"], res["FLAC", "songf.wav"]
    for pa, pb, pf in zip(a, b, f):
        da, db, df = (open(p, "rb").read() for p in (pa, pb, pf))
        assert da == db
        (ma, ia), (mf, inf) = flac.decode(da), flac.decode(df)
        assert (ia["bps"], inf["bps"]) == (16, 24) and torch.equal(ma, mf)  # int16 << 8 at 24 bits: the same floats


def test_mdx_plugin_pcm_input_stays_on_device(pcm, tmp_path, monkeypatch):
    from audio_separator.separator.common_separator import DeviceStem

    cfg = O.MDXConfig(n_fft=1536, hop_length=256, dim_f=768, dim_t=32, segment_size=32, g=8)
    np.savez(tmp_path / "tiny-mdx.npz", **O.make_convtdfnet_weights(cfg, seed=7, out_gain=0.05))
    (tmp_path / "tiny-mdx.json").write_text('{"compensate": 1.022, "mdx_dim_f_set": 768, "mdx_dim_t_set": 5, "mdx_n_fft_scale_set": 1536, "primary_stem": "Instrumental"}')
    _song_set(tmp_path)

    def no_download(self, dtype=None, copy=None):
        raise AssertionError("the mix was downloaded to the host")

    params = {"hop_length": 256, "segment_size": 32, "overlap": 0.25, "batch_size": 2, "enable_denoise": False, "b200_precision": 0}
    monkeypatch.setattr(DeviceStem, "__array__", no_download)
    _assert_stems(_separate_all(tmp_path, "tiny-mdx.npz", "mdx", mdx_params=params))


def test_mdxc_demucs_vr_plugins_pcm_input(pcm, tmp_path):
    import demucs_oracle as D
    import vr_oracle as V
    from test_autocast_separator_gpu import _mdx23c_files, _roformer_files
    from test_demucs_gpu import SMALL, _write_package

    _song_set(tmp_path)
    _roformer_files(tmp_path)
    _assert_stems(_separate_all(tmp_path, "tiny_bs_roformer.npz", "rof", mdxc_params={"batch_size": 4, "segment_size": 65}))
    _mdx23c_files(tmp_path)
    _assert_stems(_separate_all(tmp_path, "tiny-mdx23c.npz", "mdx23c", mdxc_params={"overlap": 4, "batch_size": 2, "segment_size": 16}))
    ocfg = D.HTConfig(**SMALL)
    _write_package(str(tmp_path / "aaaa1111.th"), ocfg, D.make_weights(ocfg, seed=21))
    _write_package(str(tmp_path / "bbbb2222.th"), ocfg, D.make_weights(ocfg, seed=22))
    (tmp_path / "tiny_ft.yaml").write_text("models: ['aaaa1111', 'bbbb2222']\nweights: [[1, 0, 1, 1], [0, 1, 1, 0]]\n")
    _assert_stems(_separate_all(tmp_path, "tiny_ft.yaml", "demucs", demucs_params={"shifts": 1, "batch_size": 2}))
    np.savez(tmp_path / "tiny-vr51.npz", **V.make_weights_51(256, 8, 16, seed=5))
    (tmp_path / "tiny-vr51.json").write_text('{"vr_model_param": "tiny_1band_51", "primary_stem": "Vocals", "nout": 8, "nout_lstm": 16}')
    p = V.single_band_param(n_fft=256, hl=64, bins=128, pre_filter_start=120, pre_filter_stop=127)
    (tmp_path / "tiny_1band_51.json").write_text(json.dumps({k: v for k, v in p.items() if not isinstance(v, bool)}))
    _assert_stems(_separate_all(tmp_path, "tiny-vr51.npz", "vr", vr_params={"window_size": 160, "batch_size": 4, "aggression": 5}))


def test_separate_directory_with_aiff_and_wav(pcm, tmp_path):
    from audio_separator.separator import Separator

    cfg = O.MDXConfig(n_fft=1536, hop_length=256, dim_f=768, dim_t=32, segment_size=32, g=8)
    np.savez(tmp_path / "tiny-mdx.npz", **O.make_convtdfnet_weights(cfg, seed=7, out_gain=0.05))
    (tmp_path / "tiny-mdx.json").write_text('{"compensate": 1.022, "mdx_dim_f_set": 768, "mdx_dim_t_set": 5, "mdx_n_fft_scale_set": 1536, "primary_stem": "Instrumental"}')
    _song_set(tmp_path)
    d = tmp_path / "in"
    d.mkdir()
    os.replace(tmp_path / "song.wav", d / "a.wav")
    os.replace(tmp_path / "songa.aiff", d / "b.aiff")
    params = {"hop_length": 256, "segment_size": 32, "overlap": 0.25, "batch_size": 2, "enable_denoise": False, "b200_precision": 0}
    sep = Separator(model_file_dir=str(tmp_path), output_dir=str(tmp_path / "out"), output_format="WAV", mdx_params=params)
    sep.load_model("tiny-mdx.npz")
    files = sorted(os.path.basename(f) for f in sep.separate(str(d)))
    assert files == ["a_(Instrumental)_tiny-mdx.wav", "a_(Vocals)_tiny-mdx.wav", "b_(Instrumental)_tiny-mdx.wav", "b_(Vocals)_tiny-mdx.wav"], files
    for stem in ("Instrumental", "Vocals"):
        assert (tmp_path / "out" / f"a_({stem})_tiny-mdx.wav").read_bytes() == (tmp_path / "out" / f"b_({stem})_tiny-mdx.wav").read_bytes()
