"""Separator(use_autocast=True) end to end, on the seeded small models of the other plugin tests: the switch reaches the nets of the Roformer branch of
MDXC, Demucs and VR (fp16 tensor-core mode: stems written, close to the default mode's but not equal to them); MDX-Net and MDX23C write files
byte-identical to use_autocast=False (ONNX Runtime in the reference, which autocast does not touch / pair-format kernels without an fp16 mode); and
the time-sharded MDXC plugin at world size 1 writes the same files as the plain one with use_autocast=True."""
import json
import os
import socket
import wave

import numpy as np
import pytest
import torch
import yaml

import demucs_oracle as D
import mdx_oracle as M
import mdxc_oracle as X
import roformer_oracle as R
import vr_oracle as V

pytestmark = pytest.mark.gpu

RSMALL = dict(dim=32, depth=2, time_transformer_depth=1, freq_transformer_depth=2, freqs_per_bands=(2, 2, 4, 4, 8, 12, 16, 17), dim_head=8, heads=4, stft_n_fft=128,
              stft_hop_length=32, stft_win_length=128)


@pytest.fixture(scope="module")
def lib(lib_built):
    assert torch.cuda.is_available()
    from audio_separator.separator.b200 import _lib

    return _lib


def _song(path, n=30000, seed=13):
    pcm = (M.synth_music(n, seed=seed).T * 32767).astype("<i2")
    with wave.open(str(path), "wb") as wf:
        wf.setnchannels(2); wf.setsampwidth(2); wf.setframerate(44100); wf.writeframes(pcm.tobytes())


def _run(tmp, model, autocast, out, **params):
    from audio_separator.separator import Separator

    sep = Separator(model_file_dir=str(tmp), output_dir=str(tmp / out), use_autocast=autocast, **params)
    sep.load_model(model)
    files = sep.separate(str(tmp / "song.wav"))
    return sep.model_instance, files, [open(tmp / out / f, "rb").read() for f in files]


def _pcm(b):
    import io

    with wave.open(io.BytesIO(b)) as wf:
        return np.frombuffer(wf.readframes(wf.getnframes()), dtype="<i2").astype(np.float64)


def _assert_fp16_stems(files16, bytes16, files32, bytes32):
    assert files16 == files32 and len(files16) >= 2
    assert bytes16 != bytes32  # the fp16 mode is in effect ...
    for a, b in zip(bytes16, bytes32):
        x, y = _pcm(a), _pcm(b)
        assert x.shape == y.shape
        snr = 10 * np.log10(np.sum(y**2) / max(np.sum((x - y) ** 2), 1e-9))
        assert snr >= 40.0, snr  # ... and changes the stems by fp16 rounding, not more


def _roformer_files(tmp):
    ocfg = R.BSRoformerConfig(**dict(RSMALL, dim_t=65, overlap=8))
    np.savez(tmp / "tiny_bs_roformer.npz", **R.make_weights(ocfg, seed=12))
    model = dict(RSMALL, freqs_per_bands=list(RSMALL["freqs_per_bands"]), stereo=True, num_stems=1, mask_estimator_depth=2)
    (tmp / "tiny_bs_roformer.yaml").write_text(yaml.safe_dump({"audio": {"sample_rate": 44100, "hop_length": 32, "n_fft": 128, "dim_f": 65}, "model": model,
                                                               "training": {"instruments": ["Vocals", "Instrumental"], "target_instrument": "Vocals"},
                                                               "inference": {"dim_t": 65}}))


def test_mdxc_roformer_writes_fp16_stems(lib, tmp_path):
    _roformer_files(tmp_path)
    _song(tmp_path / "song.wav")
    params = dict(mdxc_params={"batch_size": 4, "segment_size": 65})
    inst16, f16, b16 = _run(tmp_path, "tiny_bs_roformer.npz", True, "o16", **params)
    inst32, f32, b32 = _run(tmp_path, "tiny_bs_roformer.npz", False, "o32", **params)
    assert inst16.net.math == lib.MATH_FP16 and inst32.net.math == lib.MATH_BF16X3
    _assert_fp16_stems(f16, b16, f32, b32)


def test_demucs_writes_fp16_stems(lib, tmp_path):
    from test_demucs_gpu import SMALL, _write_package

    ocfg = D.HTConfig(**SMALL)
    _write_package(str(tmp_path / "aaaa1111.th"), ocfg, D.make_weights(ocfg, seed=21))
    _write_package(str(tmp_path / "bbbb2222.th"), ocfg, D.make_weights(ocfg, seed=22))
    (tmp_path / "tiny_ft.yaml").write_text("models: ['aaaa1111', 'bbbb2222']\nweights: [[1, 0, 1, 1], [0, 1, 1, 0]]\n")
    _song(tmp_path / "song.wav", seed=3)
    import random

    params = dict(demucs_params={"shifts": 1, "batch_size": 2})
    random.seed(1234)
    inst16, f16, b16 = _run(tmp_path, "tiny_ft.yaml", True, "o16", **params)
    random.seed(1234)
    inst32, f32, b32 = _run(tmp_path, "tiny_ft.yaml", False, "o32", **params)
    assert [n.math for n in inst16.engine.nets] == [lib.MATH_FP16] * 2 and [n.math for n in inst32.engine.nets] == [lib.MATH_BF16X3] * 2
    _assert_fp16_stems(f16, b16, f32, b32)


def test_vr51_writes_fp16_stems(lib, tmp_path):
    np.savez(tmp_path / "tiny-vr51.npz", **V.make_weights_51(256, 8, 16, seed=5))
    (tmp_path / "tiny-vr51.json").write_text('{"vr_model_param": "tiny_1band_51", "primary_stem": "Vocals", "nout": 8, "nout_lstm": 16}')
    p = V.single_band_param(n_fft=256, hl=64, bins=128, pre_filter_start=120, pre_filter_stop=127)
    (tmp_path / "tiny_1band_51.json").write_text(json.dumps({k: v for k, v in p.items() if not isinstance(v, bool)}))
    _song(tmp_path / "song.wav", seed=8)
    params = dict(vr_params={"window_size": 160, "batch_size": 4, "aggression": 5})
    inst16, f16, b16 = _run(tmp_path, "tiny-vr51.npz", True, "o16", **params)
    inst32, f32, b32 = _run(tmp_path, "tiny-vr51.npz", False, "o32", **params)
    assert inst16.net.math == lib.MATH_FP16 and inst32.net.math == lib.MATH_BF16X3
    _assert_fp16_stems(f16, b16, f32, b32)


def _mdx23c_files(tmp):
    xcfg = X.MDXCConfig(n_fft=1024, hop_length=256, dim_f=512, dim_t=16, num_scales=2, num_channels_model=16, growth=16, bottleneck_factor=4, overlap=4)
    np.savez(tmp / "tiny-mdx23c.npz", **X.make_weights(xcfg, seed=4, out_gain=0.3))
    (tmp / "tiny-mdx23c.json").write_text(json.dumps({
        "audio": {"n_fft": xcfg.n_fft, "hop_length": xcfg.hop_length, "dim_f": xcfg.dim_f, "num_channels": 2, "chunk_size": xcfg.chunk_size, "sample_rate": 44100},
        "model": {"norm": "InstanceNorm", "act": "gelu", "num_subbands": 4, "num_scales": xcfg.num_scales, "scale": [2, 2], "num_blocks_per_scale": 2,
                  "num_channels": xcfg.num_channels_model, "growth": xcfg.growth, "bottleneck_factor": xcfg.bottleneck_factor},
        "training": {"instruments": ["Vocals", "Instrumental"], "target_instrument": None}, "inference": {"dim_t": xcfg.dim_t}}))


def test_mdx_and_mdx23c_files_are_byte_identical(lib, tmp_path):
    cfg = M.MDXConfig(n_fft=1536, hop_length=256, dim_f=768, dim_t=32, segment_size=32, g=8)
    np.savez(tmp_path / "tiny-mdx.npz", **M.make_convtdfnet_weights(cfg, seed=7, out_gain=0.05))
    (tmp_path / "tiny-mdx.json").write_text('{"compensate": 1.022, "mdx_dim_f_set": 768, "mdx_dim_t_set": 5, "mdx_n_fft_scale_set": 1536, "primary_stem": "Instrumental"}')
    _mdx23c_files(tmp_path)
    _song(tmp_path / "song.wav", seed=3)
    cases = (("tiny-mdx.npz", dict(mdx_params={"hop_length": 256, "segment_size": 32, "overlap": 0.25, "batch_size": 2, "enable_denoise": False})),
             ("tiny-mdx23c.npz", dict(mdxc_params={"overlap": 4, "batch_size": 2, "segment_size": 16})))
    for model, params in cases:
        _, f16, b16 = _run(tmp_path, model, True, f"o16_{model}", **params)
        _, f32, b32 = _run(tmp_path, model, False, f"o32_{model}", **params)
        assert f16 == f32 and len(f16) == 2
        assert b16 == b32, model


def test_sharded_mdxc_world1_with_autocast(lib, tmp_path):
    """The time-sharded MDXC plugin (mdxc_params b200_sharded) builds the same fp16 net: world size 1 writes the same bytes as the plain plugin."""
    import torch.distributed as dist

    _roformer_files(tmp_path)
    _song(tmp_path / "song.wav")
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        port = s.getsockname()[1]
    dev = torch.cuda.current_device()
    dist.init_process_group("nccl", init_method=f"tcp://127.0.0.1:{port}", rank=0, world_size=1, device_id=torch.device("cuda", dev))
    try:
        params = {"batch_size": 4, "segment_size": 65}
        inst_s, fs, bs = _run(tmp_path, "tiny_bs_roformer.npz", True, "sharded", mdxc_params=dict(params, b200_sharded=True))
        inst_p, fp, bp = _run(tmp_path, "tiny_bs_roformer.npz", True, "plain", mdxc_params=params)
    finally:
        dist.destroy_process_group()
    assert inst_s.net.math == inst_p.net.math == lib.MATH_FP16
    assert fs == fp and len(fs) == 2 and bs == bp
