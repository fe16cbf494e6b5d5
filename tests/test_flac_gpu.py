"""GPU FLAC writer (csrc/flac.cu, b200/flac.py, CommonSeparator.write_flac) checked with the RFC 9639 oracle decoder (oracle/flac_oracle.py):
lossless round trips to the WAV writer's samples across signals, lengths and writer rules, coverage of the coding tools, compression against
libFLAC / ffmpeg on the golden frames, and the plugins and the ensemble writing FLAC."""
import json
import logging
import os
import wave

import numpy as np
import pytest
import torch

import flac_oracle as F
import mdx_oracle as O

pytestmark = pytest.mark.gpu

SR = 44100
LENGTHS = (1, 15, 16, 4095, 4096, 4097, 3 * 4096 + 1)
WRITERS = ((16, False), (16, True), (24, False), (24, True), (32, False))  # (input bits, use_soundfile); 32 + soundfile writes no file


def signal(kind, n, seed=0):
    rng = np.random.default_rng(seed)
    t = np.arange(n)
    if kind == "click":
        x = np.zeros((n, 2))
        x[n // 2] = 0.5
    elif kind == "dc":
        x = np.full((n, 2), 0.3)
    elif kind == "noise":
        x = rng.uniform(-1, 1, (n, 2))
    elif kind == "square":
        x = np.where((t // 50) % 2 == 0, 1.0, -1.0)[:, None].repeat(2, 1)
    elif kind == "sine":
        x = 0.5 * np.stack([np.sin(2 * np.pi * 440 * t / SR), np.sin(2 * np.pi * 440 * t / SR + 1.0)], 1)
    elif kind in ("music", "same", "opposite", "near_right"):
        x = O.synth_music(n, seed=seed + 1).T.astype(np.float64)
        if kind == "same":
            x[:, 1] = x[:, 0]
        elif kind == "opposite":
            x[:, 1] = -x[:, 0]
        elif kind == "near_right":  # the left channel is the right one plus a little noise: right + side is the cheapest pair
            x[:, 0] = x[:, 1] + 0.003 * rng.standard_normal(n)
    elif kind == "half_noise":  # every 4096-sample frame: silence, then full-scale noise (escape partitions); a shorter stem: its first half silent
        x = rng.uniform(-1, 1, (n, 2)) * ((t % 4096) >= min(2048, n // 2))[:, None]
    else:
        raise ValueError(kind)
    return np.ascontiguousarray(x, dtype=np.float32)


SIGNALS = ("click", "dc", "noise", "square", "sine", "music", "same", "opposite", "half_noise", "near_right")


def separator(tmp_path, bits, use_sf):
    from audio_separator.separator.common_separator import CommonSeparator

    cs = CommonSeparator(dict(logger=logging.getLogger("flac-test"), model_name="m", model_path="/x/m.onnx", model_data={"primary_stem": "Vocals"},
                              output_dir=str(tmp_path), output_format="FLAC", normalization_threshold=0.9, amplification_threshold=0.0,
                              sample_rate=SR, use_soundfile=use_sf))
    cs.input_bit_depth = bits
    return cs


def wav_samples(cs, x):
    """The WAV writer's samples for this stem (pcm_bytes of the device path) as int64, (N, 2)."""
    bits, data = cs.pcm_bytes(torch.as_tensor(x).cuda())
    a = np.frombuffer(data, np.uint8).reshape(-1, bits // 8)
    v = np.zeros(a.shape[0], np.int64)
    for b in range(bits // 8):
        v |= a[:, b].astype(np.int64) << (8 * b)
    v = np.where(v >= 1 << (bits - 1), v - (1 << bits), v)
    return bits, v.reshape(-1, 2)


def roundtrip(tmp_path, x, bits, use_sf, name="s.flac"):
    """write_flac twice; checks the stream against the oracle and the WAV path.  Returns the oracle's Decoded."""
    cs = separator(tmp_path, bits, use_sf)
    path = tmp_path / name
    cs.write_flac(name, torch.as_tensor(x).cuda())
    data = path.read_bytes()
    os.remove(path)
    cs.write_flac(name, torch.as_tensor(x).cuda())
    assert path.read_bytes() == data, "two encodes of the same stem differ"
    os.remove(path)
    d = F.decode(data)  # every CRC-8 / CRC-16 is checked
    info = d.streaminfo
    bps = 16 if bits == 16 else 24
    lengths = [f[1] for f in d.frames]
    assert (info["total_samples"], info["bps"], info["channels"], info["sample_rate"]) == (x.shape[0], bps, 2, SR)
    assert (info["min_block"], info["max_block"], info["min_frame"], info["max_frame"]) == (4096, 4096, min(lengths), max(lengths))
    assert info["md5"] == bytes(16) and sum(lengths) + 42 == len(data)
    wbits, want = wav_samples(cs, x)
    assert wbits == bits
    assert np.array_equal(d.samples << (bits - bps), want)
    return d


@pytest.fixture(scope="module")
def matrix(lib_built, tmp_path_factory):
    """Every signal at every length through every writer, plus 10-s streams of music (every writer) and noise; returns the union of what the
    oracle saw."""
    tmp = tmp_path_factory.mktemp("flac")
    seen = set()
    for kind in SIGNALS:
        for n in LENGTHS:
            for bits, use_sf in WRITERS:
                x = signal(kind, n, seed=n)
                try:
                    seen |= roundtrip(tmp, x, bits, use_sf).seen
                except Exception as e:
                    raise AssertionError(f"{kind} n={n} bits={bits} soundfile={use_sf}: {e!r}") from e
    for bits, use_sf in WRITERS:
        seen |= roundtrip(tmp, signal("music", 10 * SR, seed=3), bits, use_sf).seen
    seen |= roundtrip(tmp, signal("noise", 10 * SR, seed=4), 16, False).seen
    return seen


def test_lossless_roundtrip_matrix(matrix):
    assert matrix


def test_coverage_of_coding_tools(matrix):
    want = {"CONSTANT", "VERBATIM", "FIXED", "LPC", "wasted", "escape", "independent", "left/side", "right/side", "mid/side"}
    assert want <= matrix, sorted(want - matrix)


def test_32bit_soundfile_writes_no_file(lib_built, tmp_path, caplog):
    cs = separator(tmp_path, 32, True)
    with caplog.at_level(logging.ERROR, logger="flac-test"):
        cs.write_flac("s.flac", torch.as_tensor(signal("music", 5000)).cuda())
    assert not (tmp_path / "s.flac").exists()
    assert any("32-bit FLAC" in r.getMessage() for r in caplog.records)


def test_near_silent_stem_writes_no_file(lib_built, tmp_path):
    cs = separator(tmp_path, 16, False)
    cs.write_flac("s.flac", torch.zeros((5000, 2), device="cuda"))
    cs.write_flac("h.flac", np.full((5000, 2), 1e-8, np.float32))
    assert not os.listdir(tmp_path)


def test_host_stem_is_uploaded(lib_built, tmp_path):
    x = signal("music", 9000, seed=5)
    a, b = separator(tmp_path / "a", 24, False), separator(tmp_path / "b", 24, False)
    a.write_flac("s.flac", x)
    b.write_flac("s.flac", torch.as_tensor(x).cuda())
    assert (tmp_path / "a" / "s.flac").read_bytes() == (tmp_path / "b" / "s.flac").read_bytes()


def test_compression_against_libflac_and_ffmpeg(lib_built, golden_dir):
    """The GPU stream's frame bytes for the golden frames' samples against the real encoder's bytes for the same samples (target: within 3 %)."""
    from audio_separator.separator.b200 import flac

    g = dict(np.load(os.path.join(golden_dir, "flac_frames.npz")))
    report = {}
    for tag in ("libflac16", "ffmpeg16", "ffmpeg24"):
        s = g[f"{tag}_samples"].astype(np.int64)
        bps = F.parse_streaminfo(g[f"{tag}_streaminfo"].tobytes())["bps"]
        q = s >> (bps - 16)  # the 24-bit file holds int16 << 8: the pydub writer's samples
        x = torch.as_tensor(((q + 0.5 * np.sign(q)) / 32767.0).astype(np.float32)).cuda()  # truncates back to q exactly
        data = flac.encode(x, bps, True, bps, SR)
        d = F.decode(data)
        assert np.array_equal(d.samples, s)
        ours = len(data) - 42
        report[tag] = (ours, int(g[f"{tag}_encoder_bytes"]), ours / int(g[f"{tag}_encoder_bytes"]))
    print("FLAC compression, GPU bytes / encoder bytes:", json.dumps(report))
    for tag, (_, _, ratio) in report.items():
        assert ratio <= 1.03, f"{tag}: GPU stream is {100 * (ratio - 1):.1f} % larger than the reference encoder's"


def _read_wav(path):
    with wave.open(str(path)) as wf:
        w, raw = wf.getsampwidth(), wf.readframes(wf.getnframes())
    a = np.frombuffer(raw, np.uint8).reshape(-1, w)
    v = np.zeros(a.shape[0], np.int64)
    for b in range(w):
        v |= a[:, b].astype(np.int64) << (8 * b)
    return np.where(v >= 1 << (8 * w - 1), v - (1 << (8 * w)), v).reshape(-1, 2)


def _write_wav(path, mix, width):
    q = np.ascontiguousarray((mix.T * 32767).astype(np.int64) << (8 * width - 16))
    raw = q.astype("<i4").view(np.uint8).reshape(-1, 4)[:, :width]
    with wave.open(str(path), "wb") as wf:
        wf.setnchannels(2); wf.setsampwidth(width); wf.setframerate(SR); wf.writeframes(raw.tobytes())


@pytest.mark.parametrize("width", (2, 3))
def test_mdx_plugin_writes_flac(lib_built, tmp_path, width):
    from audio_separator.separator import Separator

    cfg = O.MDXConfig(n_fft=1536, hop_length=256, dim_f=768, dim_t=32, segment_size=32, g=8)
    np.savez(tmp_path / "tiny-mdx.npz", **O.make_convtdfnet_weights(cfg, seed=7, out_gain=0.05))
    (tmp_path / "tiny-mdx.json").write_text('{"compensate": 1.022, "mdx_dim_f_set": 768, "mdx_dim_t_set": 5, "mdx_n_fft_scale_set": 1536, "primary_stem": "Instrumental"}')
    _write_wav(tmp_path / "song.wav", O.synth_music(30000, seed=3), width)
    params = {"hop_length": 256, "segment_size": 32, "overlap": 0.25, "batch_size": 2, "enable_denoise": False, "b200_precision": 0}
    got = {}
    for fmt in ("WAV", "FLAC"):
        sep = Separator(model_file_dir=str(tmp_path), output_dir=str(tmp_path / fmt), output_format=fmt, mdx_params=params)
        sep.load_model("tiny-mdx.npz")
        got[fmt] = sep.separate(str(tmp_path / "song.wav"))
    assert got["FLAC"] == ["song_(Vocals)_tiny-mdx.flac", "song_(Instrumental)_tiny-mdx.flac"]
    for wf, ff in zip(got["WAV"], got["FLAC"]):
        d = F.decode((tmp_path / "FLAC" / ff).read_bytes())
        assert d.streaminfo["bps"] == 8 * width
        assert np.array_equal(d.samples, _read_wav(tmp_path / "WAV" / wf))


def test_ensemble_writes_flac(lib_built, tmp_path):
    from audio_separator.separator import Separator

    cfg = O.MDXConfig(n_fft=1536, hop_length=256, dim_f=768, dim_t=32, segment_size=32, g=8)
    md = {"compensate": cfg.compensate, "mdx_dim_f_set": cfg.dim_f, "mdx_dim_t_set": 5, "mdx_n_fft_scale_set": cfg.n_fft, "primary_stem": "Vocals"}
    for name, seed in (("UVR-MDX-NET-tinyA", 7), ("UVR-MDX-NET-tinyB", 8)):
        np.savez(tmp_path / f"{name}.npz", **O.make_convtdfnet_weights(cfg, seed=seed, out_gain=0.05))
        (tmp_path / f"{name}.json").write_text(json.dumps(md))
    _write_wav(tmp_path / "song.wav", O.synth_music(30000, seed=3), 2)
    params = {"segment_size": cfg.segment_size, "hop_length": cfg.hop_length, "overlap": cfg.overlap, "batch_size": 2}
    got = {}
    for fmt in ("WAV", "FLAC"):
        sep = Separator(model_file_dir=str(tmp_path), output_dir=str(tmp_path / fmt), output_format=fmt, mdx_params=params, ensemble_algorithm="avg_wave")
        sep.load_model(["UVR-MDX-NET-tinyA.npz", "UVR-MDX-NET-tinyB.npz"])
        got[fmt] = sorted(os.path.basename(f) for f in sep.separate(str(tmp_path / "song.wav")))
    assert got["FLAC"] == ["song_(Instrumental)_custom_ensemble_tinyA_tinyB.flac", "song_(Vocals)_custom_ensemble_tinyA_tinyB.flac"]
    for wf, ff in zip(got["WAV"], got["FLAC"]):
        d = F.decode((tmp_path / "FLAC" / ff).read_bytes())
        assert np.array_equal(d.samples, _read_wav(tmp_path / "WAV" / wf))
