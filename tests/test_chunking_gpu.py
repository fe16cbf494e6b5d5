"""Separator(chunk_duration=...) on the H100: every plugin's joined stems equal the concatenation of its normal runs on WAV files holding each
chunk's samples (cut by the restated splitter, oracle/chunking_oracle.py), at 16 and 24 bits, as WAV and FLAC, from WAV and FLAC input."""
import json
import logging
import os
import random
import re
import socket
import tempfile
import wave

import numpy as np
import pytest
import torch

import chunking_oracle as C
import flac_writer as FW
import mdx_oracle as O
import pcm_writer as W
from test_flac_decode_gpu import _write_wav

pytestmark = pytest.mark.gpu

SR = 44100
N = 30011  # 681 ms: four chunks of 200 ms, the last one ragged
CHUNK = 0.2
MDX_PARAMS = {"hop_length": 256, "segment_size": 32, "overlap": 0.25, "batch_size": 2, "enable_denoise": False, "b200_precision": 0}


def _mdx_files(tmp, name="tiny-mdx", seed=7):
    cfg = O.MDXConfig(n_fft=1536, hop_length=256, dim_f=768, dim_t=32, segment_size=32, g=8)
    np.savez(tmp / f"{name}.npz", **O.make_convtdfnet_weights(cfg, seed=seed, out_gain=0.05))
    (tmp / f"{name}.json").write_text('{"compensate": 1.022, "mdx_dim_f_set": 768, "mdx_dim_t_set": 5, "mdx_n_fft_scale_set": 1536, "primary_stem": "Instrumental"}')
    return f"{name}.npz", dict(mdx_params=MDX_PARAMS)


def _roformer(tmp):
    from test_autocast_separator_gpu import _roformer_files

    _roformer_files(tmp)
    return "tiny_bs_roformer.npz", dict(mdxc_params={"batch_size": 4, "segment_size": 65})


def _mdx23c(tmp):
    from test_autocast_separator_gpu import _mdx23c_files

    _mdx23c_files(tmp)
    return "tiny-mdx23c.npz", dict(mdxc_params={"overlap": 4, "batch_size": 2, "segment_size": 16})


def _demucs(tmp):
    import demucs_oracle as D
    from test_demucs_gpu import SMALL, _write_package

    ocfg = D.HTConfig(**SMALL)
    _write_package(str(tmp / "aaaa1111.th"), ocfg, D.make_weights(ocfg, seed=21))
    _write_package(str(tmp / "bbbb2222.th"), ocfg, D.make_weights(ocfg, seed=22))
    (tmp / "tiny_ft.yaml").write_text("models: ['aaaa1111', 'bbbb2222']\nweights: [[1, 0, 1, 1], [0, 1, 1, 0]]\n")
    return "tiny_ft.yaml", dict(demucs_params={"shifts": 2, "batch_size": 2})


def _vr(tmp):
    import vr_oracle as V

    np.savez(tmp / "tiny-vr51.npz", **V.make_weights_51(256, 8, 16, seed=5))
    (tmp / "tiny-vr51.json").write_text('{"vr_model_param": "tiny_1band_51", "primary_stem": "Vocals", "nout": 8, "nout_lstm": 16}')
    p = V.single_band_param(n_fft=256, hl=64, bins=128, pre_filter_start=120, pre_filter_stop=127)
    (tmp / "tiny_1band_51.json").write_text(json.dumps({k: v for k, v in p.items() if not isinstance(v, bool)}))
    return "tiny-vr51.npz", dict(vr_params={"window_size": 160, "batch_size": 4, "aggression": 5})


MODELS = {"mdx": _mdx_files, "roformer": _roformer, "mdx23c": _mdx23c, "demucs": _demucs, "vr": _vr}


def _ints(n=N, seed=3, bits=16):
    return (O.synth_music(n, seed=seed).T * ((1 << (bits - 1)) - 1)).astype(np.int64)  # (n, 2)


def _run(tmp, model, params, src, out, seed=1234, **kw):
    from audio_separator.separator import Separator

    sep = Separator(model_file_dir=str(tmp), output_dir=str(tmp / out), **params, **kw)
    sep.load_model(model)
    random.seed(seed)
    files = sep.separate(str(src)) if isinstance(src, (str, os.PathLike)) else [f for s in src for f in sep.separate(str(s))]
    return [f if os.path.isabs(f) else str(tmp / out / f) for f in files]


def _read_wav(path):
    with wave.open(path, "rb") as wf:
        width, raw = wf.getsampwidth(), wf.readframes(wf.getnframes())
        assert wf.getnchannels() == 2 and wf.getframerate() == SR
    return width, np.frombuffer(raw, {2: "<i2", 3: "u1", 4: "<i4"}[width])


def _as_int(width, data):
    if width == 3:
        b = data.reshape(-1, 3).astype(np.int32)
        return ((b[:, 0] | (b[:, 1] << 8) | (b[:, 2] << 16)) << 8) >> 8
    return data.astype(np.int64)


def _per_chunk_expected(tmp, model, params, ints, width, out, seed=1234, **kw):
    """The reference's pipeline on chunk files: the restated splitter writes chunk_NNNN.wav, the plugin separates them one after the other, and the
    stems are grouped by the name inside `_(...)`, sorted and concatenated.  -> {joined file name: (width, int samples)}."""
    d = tmp / f"{out}_chunks"
    d.mkdir()
    paths = []
    for i, (_, _, a, b) in enumerate(C.boundaries(len(ints), SR, CHUNK)):
        piece = np.concatenate([ints[a:min(b, len(ints))], np.zeros((max(0, b - len(ints)), 2), np.int64)])
        _write_wav(d / f"chunk_{i:04d}.wav", piece, width)
        paths.append(d / f"chunk_{i:04d}.wav")
    files = [f for f in _run(tmp, model, params, paths, f"{out}_chunkout", seed=seed, **kw) if os.path.exists(f)]
    groups = {}
    for f in files:
        key = re.search(r"_\(([^)]+)\)", os.path.basename(f)).group(1)
        w, data = _read_wav(f)
        groups.setdefault(key, []).append(_as_int(w, data))
    return {key: np.concatenate(groups[key]) for key in sorted(groups)}


def _check_joined(files, expected, base, width):
    assert [os.path.basename(f) for f in files] == [f"{base}_({k}).wav" for k in expected]
    for f, (key, want) in zip(files, expected.items()):
        w, data = _read_wav(f)
        if width == 3:  # a 24-bit input joins into a 32-bit WAV holding the 24-bit samples << 8
            assert w == 4 and np.array_equal(data.astype(np.int64) >> 8, want), key
        else:
            assert w == width and np.array_equal(data.astype(np.int64), want), key


@pytest.mark.parametrize("arch", list(MODELS))
def test_plugin_chunked_equals_per_chunk_runs(lib_built, tmp_path, arch, monkeypatch):
    from audio_separator.separator.b200 import flac

    model, params = MODELS[arch](tmp_path)
    temp = tmp_path / "tmp"
    temp.mkdir()
    monkeypatch.setattr(tempfile, "tempdir", str(temp))
    for width in (2, 3):
        ints = _ints(bits=8 * width)
        _write_wav(tmp_path / f"song{width}.wav", ints, width)
        expected = _per_chunk_expected(tmp_path, model, params, ints, width, f"ref{width}")
        assert len(expected) >= 2
        files = _run(tmp_path, model, params, tmp_path / f"song{width}.wav", f"chunked{width}", chunk_duration=CHUNK)
        _check_joined(files, expected, f"song{width}", width)
        assert sorted(os.listdir(tmp_path / f"chunked{width}")) == sorted(os.path.basename(f) for f in files)
        # FLAC output decodes to the WAV run's samples
        ffiles = _run(tmp_path, model, params, tmp_path / f"song{width}.wav", f"chunkedf{width}", chunk_duration=CHUNK, output_format="FLAC")
        assert [os.path.basename(f) for f in ffiles] == [os.path.basename(f)[:-4] + ".flac" for f in files]
        for fw, ff in zip(files, ffiles):
            w, data = _read_wav(fw)
            mix, info = flac.decode(open(ff, "rb").read())
            assert info["bps"] == 8 * width
            want = torch.from_numpy((data.astype(np.float64) / 2.0 ** (8 * w - 1)).astype(np.float32).reshape(-1, 2).T.copy())
            assert torch.equal(mix.cpu(), want)
    assert os.listdir(temp) == []  # no chunk files, no temporary directory left behind


def test_flac_input_equals_wav_input(lib_built, tmp_path):
    model, params = _mdx_files(tmp_path)
    ints = _ints()
    _write_wav(tmp_path / "song.wav", ints, 2)
    data, _ = FW.stream([FW.Frame(y) for y in np.array_split(ints, 12)], SR, 16)
    (tmp_path / "song.flac").write_bytes(data)
    a = _run(tmp_path, model, params, tmp_path / "song.wav", "w", chunk_duration=CHUNK)
    b = _run(tmp_path, model, params, tmp_path / "song.flac", "f", chunk_duration=CHUNK)
    assert [os.path.basename(p) for p in a] == [os.path.basename(p) for p in b] and len(a) == 2
    for pa, pb in zip(a, b):
        assert open(pa, "rb").read() == open(pb, "rb").read()


@pytest.mark.parametrize("arch,chunk", [(a, 0.681) for a in MODELS] + [("mdx", 1.0)])  # 681 ms: longer than the 680.5-ms file
def test_chunk_not_shorter_than_file_is_the_normal_run(lib_built, tmp_path, monkeypatch, arch, chunk):
    from audio_separator.separator.common_separator import CommonSeparator

    model, params = MODELS[arch](tmp_path)
    _write_wav(tmp_path / "song.wav", _ints(), 2)
    plain = _run(tmp_path, model, params, tmp_path / "song.wav", "plain")
    decodes = []
    read = CommonSeparator._read_audio
    monkeypatch.setattr(CommonSeparator, "_read_audio", lambda self, path: decodes.append(path) or read(self, path))
    ch = _run(tmp_path, model, params, tmp_path / "song.wav", "ch", chunk_duration=chunk)
    assert decodes == [str(tmp_path / "song.wav")]  # the decode that decides against chunking is the one the separation uses
    assert [os.path.basename(p) for p in plain] == [os.path.basename(p) for p in ch] and len(plain) >= 2
    for pa, pb in zip(plain, ch):
        assert open(pa, "rb").read() == open(pb, "rb").read()


def test_near_silent_chunk_is_left_out(lib_built, tmp_path, caplog):
    """A float WAV whose second chunk is ~1e-9: both of its stems are near-silent, so the joined stems skip that chunk."""
    model, params = _mdx_files(tmp_path)
    x = O.synth_music(N, seed=5).T.astype(np.float32)
    bounds = C.boundaries(N, SR, CHUNK)
    a, b = bounds[1][2], bounds[1][3]
    x[a:b] *= np.float32(1e-9)
    (tmp_path / "song.wav").write_bytes(W.wav(W.payload(x, W.F32LE), 3, 2, SR, 8, 32))
    d = tmp_path / "chunks"
    d.mkdir()
    for i, (_, _, s, e) in enumerate(bounds):
        piece = np.concatenate([x[s:min(e, N)], np.zeros((max(0, e - N), 2), np.float32)])
        (d / f"chunk_{i:04d}.wav").write_bytes(W.wav(W.payload(piece, W.F32LE), 3, 2, SR, 8, 32))
    ref = [f for f in _run(tmp_path, model, params, [d / f"chunk_{i:04d}.wav" for i in range(len(bounds))], "ref") if os.path.exists(f)]
    assert len(ref) == 2 * (len(bounds) - 1) and not any("chunk_0001" in os.path.basename(f) for f in ref)
    with caplog.at_level(logging.WARNING):
        files = _run(tmp_path, model, params, tmp_path / "song.wav", "ch", chunk_duration=CHUNK)
    assert any("Chunk 2/" in r.getMessage() and "near-silent" in r.getMessage() for r in caplog.records)
    assert len(files) == 2
    for f in files:
        key = re.search(r"_\(([^)]+)\)", os.path.basename(f)).group(1)
        want = np.concatenate([_read_wav(r)[1] for r in ref if f"_({key})_" in os.path.basename(r)])
        w, data = _read_wav(f)
        assert w == 4 and np.array_equal(data, want)
        assert len(data) == 2 * sum(e - s for i, (_, _, s, e) in enumerate(bounds) if i != 1)


def test_single_stem_and_custom_names(lib_built, tmp_path):
    model, params = _mdx_files(tmp_path)
    _write_wav(tmp_path / "song.wav", _ints(), 2)
    full = _run(tmp_path, model, params, tmp_path / "song.wav", "full", chunk_duration=CHUNK)
    single = _run(tmp_path, model, params, tmp_path / "song.wav", "single", chunk_duration=CHUNK, output_single_stem="vocals")
    assert [os.path.basename(f) for f in single] == ["song_(Vocals).wav"]
    assert open(single[0], "rb").read() == open(full[1], "rb").read()
    from audio_separator.separator import Separator

    sep = Separator(model_file_dir=str(tmp_path), output_dir=str(tmp_path / "named"), mdx_params=MDX_PARAMS, chunk_duration=CHUNK)
    sep.load_model(model)
    named = sep.separate(str(tmp_path / "song.wav"), {"Vocals": "lead", "Instrumental": "backing"})
    assert [os.path.basename(f) for f in named] == ["backing.wav", "lead.wav"]
    assert [open(f, "rb").read() for f in named] == [open(f, "rb").read() for f in full]


def test_ensemble_with_chunking(lib_built, tmp_path):
    """Two-model ensemble with chunking equals the ensemble of the two chunked single-model runs: each model's joined stems are kept apart."""
    from audio_separator.separator import Separator
    from audio_separator.separator.ensembler import Ensembler
    from test_flac_decode_gpu import _separator

    a, params = _mdx_files(tmp_path, "tiny-mdx-a", seed=7)
    b, _ = _mdx_files(tmp_path, "tiny-mdx-b", seed=8)
    _write_wav(tmp_path / "song.wav", _ints(), 2)
    ra = _run(tmp_path, a, params, tmp_path / "song.wav", "a", chunk_duration=CHUNK)
    rb = _run(tmp_path, b, params, tmp_path / "song.wav", "b", chunk_duration=CHUNK)
    assert [open(f, "rb").read() for f in ra] != [open(f, "rb").read() for f in rb]
    sep = Separator(model_file_dir=str(tmp_path), output_dir=str(tmp_path / "ens"), mdx_params=MDX_PARAMS, chunk_duration=CHUNK)
    sep.load_model([a, b])
    ens = sep.separate(str(tmp_path / "song.wav"))
    assert sorted(os.path.basename(f) for f in ens) == ["song_(Instrumental)_custom_ensemble_tiny-mdx-a_tiny-mdx-b.wav", "song_(Vocals)_custom_ensemble_tiny-mdx-a_tiny-mdx-b.wav"]
    writer = _separator(tmp_path / "want")
    for fa, fb in zip(ra, rb):
        key = re.search(r"_\(([^)]+)\)", os.path.basename(fa)).group(1)
        waves = [writer.prepare_mix(fa), writer.prepare_mix(fb)]
        writer.write_audio(f"{key}.wav", np.ascontiguousarray(np.asarray(Ensembler(logging.getLogger("t"), "avg_wave").ensemble(waves)).T))
        got = [f for f in ens if f"_({key})_" in os.path.basename(f)][0]
        assert open(got, "rb").read() == open(tmp_path / "want" / f"{key}.wav", "rb").read(), key


def test_sharded_world1_mdx(lib_built, tmp_path):
    import torch.distributed as dist

    model, params = _mdx_files(tmp_path)
    _write_wav(tmp_path / "song.wav", _ints(), 2)
    plain = _run(tmp_path, model, params, tmp_path / "song.wav", "plain", chunk_duration=CHUNK)
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        port = s.getsockname()[1]
    dev = torch.cuda.current_device()
    dist.init_process_group("nccl", init_method=f"tcp://127.0.0.1:{port}", rank=0, world_size=1, device_id=torch.device("cuda", dev))
    try:
        sharded = _run(tmp_path, model, dict(mdx_params=dict(MDX_PARAMS, b200_sharded=True)), tmp_path / "song.wav", "sharded", chunk_duration=CHUNK)
    finally:
        dist.destroy_process_group()
    assert [os.path.basename(p) for p in plain] == [os.path.basename(p) for p in sharded] and len(plain) == 2
    for pa, pb in zip(plain, sharded):
        assert open(pa, "rb").read() == open(pb, "rb").read()
