"""GPU: the band-limited resampler (b200sep_resample_sinc_f32) against its float64 restatement (oracle/resample_oracle.py), and the two features
built on it -- MDXC `pitch_shift` and VR models at 32 / 48 kHz -- against the goldens of oracle/make_golden_resample.py, through the plugins'
demix / engine and through Separator(...).separate() writing WAV, on one GPU and time-sharded over two.  A run that needs no resampling at another
ratio (pitch_shift=0, a 44.1 kHz VR model) must never launch the new kernel."""
import json
import math
import os
import socket
import tempfile
import wave

import numpy as np
import pytest
import torch

import mdx_oracle as M
import mdxc_oracle as X
import resample_oracle as RO
import roformer_oracle as R
import vr_oracle as V
from make_golden_resample import MDXC_SMALL, PITCHES, RF_SMALL, VR_PARAMS, pcm_wave, rf_cfg, vr_loading_mix, vr_param

pytestmark = pytest.mark.gpu

DESIGNS = ("soxr_hq", "sinc_medium", "sinc_fastest", "kaiser_fast")
RATES = [(48000, 44100), (44100, 48000), (32000, 44100), (44100, 32000), (32000, 6000)] + [(44100, 44100 * 2 ** (k / 12)) for k in (-12, -7, -1, 1, 5, 12)] \
    + [(16, 1), (1, 16)]


@pytest.fixture(scope="module")
def rs(lib_built):
    from audio_separator.separator.b200 import resample

    return resample


def _signal(c, n, seed):
    return (np.random.default_rng(seed).uniform(-1.0, 1.0, (c, n)) * 0.7).astype(np.float32)


def _check(rs, x, orig_sr, target_sr, res_type, idx=None):
    got = rs.resample(torch.from_numpy(x).cuda(), orig_sr, target_sr, res_type).cpu().numpy()
    ratio = float(target_sr) / orig_sr
    assert got.shape == (x.shape[0], int(np.ceil(x.shape[1] * ratio)))
    want = RO.sinc_resample(x, ratio, *RO.table(res_type), idx=idx)
    g = got if idx is None else got[:, idx]
    err = float(np.abs(g - want).max())
    assert err <= 1e-5, (orig_sr, target_sr, res_type, x.shape, err)


@pytest.mark.parametrize("res_type", DESIGNS)
@pytest.mark.parametrize("orig_sr,target_sr", RATES)
def test_kernel_vs_oracle_ratios(rs, res_type, orig_sr, target_sr):
    c = 1 + (RATES.index((orig_sr, target_sr)) + DESIGNS.index(res_type)) % 2
    _check(rs, _signal(c, 10007, 3), orig_sr, target_sr, res_type)


@pytest.mark.parametrize("res_type", DESIGNS)
@pytest.mark.parametrize("c", [1, 2])
def test_kernel_vs_oracle_short_inputs(rs, res_type, c):
    nz = RO.FILTERS[res_type][0]
    for n in (1, 7, nz // 2 + 1):  # the last is shorter than one filter half-width at every ratio
        for orig_sr, target_sr in ((44100, 32000), (32000, 44100), (16, 1), (1, 16), (44100, 44100 * 2 ** (5 / 12))):
            _check(rs, _signal(c, n, n), orig_sr, target_sr, res_type)


@pytest.mark.parametrize("orig_sr,target_sr,res_type", [(44100, 32000, "soxr_hq"), (32000, 44100, "soxr_hq"), (44100, 44100 * 2 ** (-3 / 12), "sinc_fastest")])
def test_kernel_vs_oracle_five_minutes(rs, orig_sr, target_sr, res_type):
    """a 5-minute stereo track: positions far from 0 (a float32 running position would be off by whole samples here), checked at the start, the
    middle and the end"""
    n = 44100 * 300 if orig_sr == 44100 else 32000 * 300
    x = _signal(2, n, 9)
    n_out = int(np.ceil(n * (float(target_sr) / orig_sr)))
    idx = np.concatenate([np.arange(0, 3000), np.arange(n_out // 2 - 1500, n_out // 2 + 1500), np.arange(n_out - 3000, n_out)])
    _check(rs, x, orig_sr, target_sr, res_type, idx=idx)


def test_ratio_outside_range_raises(rs):
    from audio_separator.separator.b200._lib import B200SepError

    x = torch.zeros((2, 1000), device="cuda")
    for a, b in ((17, 1), (1, 17)):
        with pytest.raises(B200SepError, match=r"ratio .* outside \[1/16, 16\]"):
            rs.resample(x, a, b, "soxr_hq")
    with pytest.raises(NotImplementedError, match="soxr_vhq"):
        rs.resample(x, 44100, 32000, "soxr_vhq")
    assert rs.resample(x, 44100, 44100, "sinc_fastest") is x


# ------------------------------------------------------------------------------------------------ plugins: model files
def _write_wav(path, x):
    pcm = np.round(x.T * 32768).astype("<i2")
    with wave.open(path, "wb") as wf:
        wf.setnchannels(2); wf.setsampwidth(2); wf.setframerate(44100); wf.writeframes(pcm.tobytes())


def _read_wav(path):
    with wave.open(path) as wf:
        n = wf.getnframes()
        return np.frombuffer(wf.readframes(n), dtype="<i2").astype(np.int32).reshape(n, 2)


def _model_files(tmp, z_pitch):
    import yaml

    cfg = X.MDXCConfig(**MDXC_SMALL)
    np.savez(os.path.join(tmp, "tiny-mdx23c.npz"), **X.make_weights(cfg, seed=int(z_pitch["tfc_weights_seed"]), out_gain=float(z_pitch["tfc_out_gain"])))
    with open(os.path.join(tmp, "tiny-mdx23c.json"), "w") as f:
        json.dump({"audio": {"n_fft": cfg.n_fft, "hop_length": cfg.hop_length, "dim_f": cfg.dim_f, "num_channels": 2, "chunk_size": cfg.chunk_size, "sample_rate": 44100},
                   "model": {"norm": "InstanceNorm", "act": "gelu", "num_subbands": 4, "num_scales": cfg.num_scales, "scale": [2, 2], "num_blocks_per_scale": 2,
                             "num_channels": cfg.num_channels_model, "growth": cfg.growth, "bottleneck_factor": cfg.bottleneck_factor},
                   "training": {"instruments": ["Vocals", "Instrumental"], "target_instrument": None}, "inference": {"dim_t": cfg.dim_t}}, f)
    rcfg = rf_cfg(overlap=int(z_pitch["rf_overlap"]))
    np.savez(os.path.join(tmp, "tiny_bs_roformer.npz"), **R.make_weights(rcfg, seed=int(z_pitch["rf_weights_seed"])))
    model = {k: v for k, v in RF_SMALL.items() if k not in ("dim_t", "overlap")}
    model.update(freqs_per_bands=list(RF_SMALL["freqs_per_bands"]), stereo=True, num_stems=1, mask_estimator_depth=2)
    with open(os.path.join(tmp, "tiny_bs_roformer.yaml"), "w") as f:
        yaml.safe_dump({"audio": {"sample_rate": 44100, "hop_length": rcfg.stft_hop_length, "n_fft": rcfg.stft_n_fft, "dim_f": 65}, "model": model,
                        "training": {"instruments": ["Vocals", "Instrumental"], "target_instrument": "Vocals"}, "inference": {"dim_t": rcfg.dim_t}}, f)
    for i, name in enumerate(VR_PARAMS):
        np.savez(os.path.join(tmp, f"tiny-vr-{name}.npz"), **V.make_weights(31191, seed=11 + i))
        with open(os.path.join(tmp, f"tiny-vr-{name}.json"), "w") as f:
            json.dump({"vr_model_param": name, "primary_stem": "Instrumental", "b200_nn_architecture": 31191}, f)
    _write_wav(os.path.join(tmp, "song.wav"), pcm_wave(int(z_pitch["n_samples"]), int(z_pitch["mix_seed"])))


MDXC_RUNS = {"tfc": ("tiny-mdx23c.npz", {"overlap": MDXC_SMALL["overlap"], "batch_size": 2, "segment_size": MDXC_SMALL["dim_t"]}),
             "rf": ("tiny_bs_roformer.npz", {"overlap": 2, "batch_size": 4, "segment_size": RF_SMALL["dim_t"]})}
VR_RUN = {"window_size": 272, "batch_size": 2, "aggression": 5}


@pytest.fixture(scope="module")
def gold(lib_built, golden_dir):
    return np.load(os.path.join(golden_dir, "pitch_small.npz")), np.load(os.path.join(golden_dir, "vr_rates_small.npz"))


@pytest.fixture(scope="module")
def model_dir(gold, tmp_path_factory):
    tmp = str(tmp_path_factory.mktemp("resample-models"))
    _model_files(tmp, gold[0])
    return tmp


@pytest.mark.parametrize("family", ["tfc", "rf"])
@pytest.mark.parametrize("s", PITCHES)
def test_mdxc_pitch_shift_vs_reference_golden(gold, model_dir, tmp_path, family, s):
    from audio_separator.separator import Separator

    z = gold[0]
    want = z[f"{family}_pitch{s:+d}"]  # rows: Vocals, Instrumental (the residual for the single-target Roformer)
    model_file, params = MDXC_RUNS[family]
    sep = Separator(model_file_dir=model_dir, output_dir=str(tmp_path), mdxc_params=dict(params, pitch_shift=s))
    sep.load_model(model_file)
    mix = M.normalize(pcm_wave(int(z["n_samples"]), int(z["mix_seed"])), 0.9, 0.0)
    src = sep.model_instance.demix(mix)  # segment_size is the model's dim_t: the < 10 s switch of separate() changes no engine here
    got = np.stack([src["Vocals"], src["Instrumental"]])
    assert got.shape == want.shape == (2, 2, mix.shape[1])
    err = float(np.abs(got - want).max())
    # pitched down, the mix is empty above 0.8 of the old Nyquist frequency, and the tiny random BS-Roformer's RMSNorm over those near-silent bands
    # turns a 1e-6 change of its input into ~5e-3 of output (measured on the oracle itself): 1e-3 there, 1e-4 everywhere else
    assert err <= (1e-3 if (family, s) == ("rf", -3) else 1e-4), err
    files = Separator(model_file_dir=model_dir, output_dir=str(tmp_path / "out"), mdxc_params=dict(params, pitch_shift=s))
    files.load_model(model_file)
    written = files.separate(os.path.join(model_dir, "song.wav"))
    stem = os.path.splitext(model_file)[0]
    assert written == [f"song_(Instrumental)_{stem}.wav", f"song_(Vocals)_{stem}.wav"]
    for fname, ref in zip(written, (want[1], want[0])):
        pcm = _read_wav(str(tmp_path / "out" / fname))
        assert pcm.shape == (mix.shape[1], 2)
        assert np.abs(pcm - M.to_pcm16(ref.T.copy(), 0.9, 0.0).astype(np.int32).reshape(-1, 2)).max() <= (40 if (family, s) == ("rf", -3) else 4)


@pytest.mark.parametrize("name", VR_PARAMS)
def test_vr_model_rates_vs_reference_golden(gold, model_dir, tmp_path, name):
    from audio_separator.separator import Separator

    z = gold[1]
    wave_ = pcm_wave(int(z["n_samples"]), int(z["wave_seed"]))
    p = vr_param(name)
    sep = Separator(model_file_dir=model_dir, output_dir=str(tmp_path), vr_params=VR_RUN)
    sep.load_model(f"tiny-vr-{name}.npz")
    eng = sep.model_instance.engine
    top = p["band"][len(p["band"])]
    X_got = eng.loading_mix(torch.from_numpy(RO.resample(wave_, 44100, top["sr"], top["res_type"])).cuda()).cpu().numpy()
    X_want = vr_loading_mix(wave_, p)
    assert np.abs((X_got[0::2] + 1j * X_got[1::2]) - X_want).max() <= 1e-4 * np.abs(X_want).max()
    prim, sec = eng.separate(wave_, sr=44100)
    for got, key in ((prim, "primary"), (sec, "secondary")):
        want = z[f"{name}_{key}"]
        assert got.shape == want.shape and want.shape[1] == math.ceil(top["hl"] * (int(z[f"{name}_frames"]) - 1) * 44100 / p["sr"])
        err = float(np.abs(got - want).max())
        assert err <= 1e-4, (key, err)
    _write_wav(str(tmp_path / "vr_song.wav"), wave_)
    written = sep.separate(str(tmp_path / "vr_song.wav"))
    assert written == [f"vr_song_(Instrumental)_tiny-vr-{name}.wav", f"vr_song_(Vocals)_tiny-vr-{name}.wav"]
    for fname, key in zip(written, ("primary", "secondary")):
        pcm = _read_wav(str(tmp_path / fname))
        want = z[f"{name}_{key}"]
        assert pcm.shape == (want.shape[1], 2)
        assert np.abs(pcm - M.to_pcm16(want.T.copy(), 0.9, 0.0).astype(np.int32).reshape(-1, 2)).max() <= 3


def test_no_sinc_launch_without_a_rate_change(gold, model_dir, tmp_path, monkeypatch):
    """pitch_shift=0 and a 44.1 kHz VR model (its top band's res_type is sinc_best, at the file's rate) never call the new kernel"""
    from audio_separator.separator import Separator
    from audio_separator.separator.b200 import _lib

    calls = []
    monkeypatch.setattr(_lib.lib, "b200sep_resample_sinc_f32", lambda *a: calls.append(a) or 0)
    model_file, params = MDXC_RUNS["tfc"]
    sep = Separator(model_file_dir=model_dir, output_dir=str(tmp_path / "mdxc"), mdxc_params=dict(params, pitch_shift=0))
    sep.load_model(model_file)
    assert len(sep.separate(os.path.join(model_dir, "song.wav"))) == 2
    with open(os.path.join(model_dir, "tiny-vr-44k.json"), "w") as f:
        json.dump({"vr_model_param": "1band_sr44100_hl512", "primary_stem": "Instrumental", "b200_nn_architecture": 31191}, f)
    np.savez(os.path.join(model_dir, "tiny-vr-44k.npz"), **V.make_weights(31191, seed=5))
    sep = Separator(model_file_dir=model_dir, output_dir=str(tmp_path / "vr"), vr_params=VR_RUN)
    sep.load_model("tiny-vr-44k.npz")
    assert sep.model_instance.model_params["band"][1]["res_type"] == "sinc_best"
    assert len(sep.separate(os.path.join(model_dir, "song.wav"))) == 2
    assert calls == []


# ------------------------------------------------------------------------------------------------ time-sharded (b200_sharded)
SHARDED_RUNS = [("tiny-mdx23c.npz", "mdxc_params", dict(MDXC_RUNS["tfc"][1], pitch_shift=-3)),
                ("tiny_bs_roformer.npz", "mdxc_params", dict(MDXC_RUNS["rf"][1], pitch_shift=2)),
                ("tiny-vr-2band_32000.npz", "vr_params", VR_RUN)]


def _worker(rank, world, port, tmp, q):
    import torch.distributed as dist

    from audio_separator.separator import Separator

    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", rank))
    res = []
    for model_file, key, params in SHARDED_RUNS:
        out_dir = os.path.join(tmp, f"sharded_{model_file}")
        sep = Separator(model_file_dir=tmp, output_dir=out_dir, **{key: dict(params, b200_sharded=True)})
        sep.load_model(model_file)
        files = sep.separate(os.path.join(tmp, "song.wav"))
        if rank == 0:
            res.append((model_file, files))  # the bytes stay on disk: a large item in the queue would block the child's exit and so the join
        else:
            res_ok = files == [] and (not os.path.isdir(out_dir) or not any(os.scandir(out_dir)))
            assert res_ok, files
    dist.barrier()
    if rank == 0:
        q.put(res)
    dist.destroy_process_group()


def _free_port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


@pytest.mark.timeout(600)
@pytest.mark.parametrize("world", [1, 2])
def test_sharded_pitch_shift_and_vr_rates_equal_one_gpu(gold, world):
    import torch.multiprocessing as mp

    from audio_separator.separator import Separator

    if torch.cuda.device_count() < world:
        pytest.skip(f"needs {world} GPUs")
    with tempfile.TemporaryDirectory(prefix="b200sep-resample-sharded-") as tmp:
        _model_files(tmp, gold[0])
        plain = []
        for model_file, key, params in SHARDED_RUNS:
            out_dir = os.path.join(tmp, f"plain_{model_file}")
            sep = Separator(model_file_dir=tmp, output_dir=out_dir, **{key: params})
            sep.load_model(model_file)
            files = sep.separate(os.path.join(tmp, "song.wav"))
            plain.append((model_file, files, [open(os.path.join(out_dir, f), "rb").read() for f in files]))
        ctx = mp.get_context("spawn")
        q = ctx.Queue()
        port = _free_port()
        procs = [ctx.Process(target=_worker, args=(r, world, port, tmp, q)) for r in range(world)]
        for p in procs:
            p.start()
        for p in procs:
            p.join(900)
        codes = [p.exitcode for p in procs]
        for p in procs:  # a rank that died leaves its peers waiting in NCCL: do not let them hold the GPUs
            if p.is_alive():
                p.kill()
        assert codes == [0] * world, codes
        sharded = q.get(timeout=10)
        assert sharded == [(m, f) for m, f, _ in plain]
        for m, f, b_pl in plain:
            assert len(f) == 2 and [open(os.path.join(tmp, f"sharded_{m}", x), "rb").read() for x in f] == b_pl, m
