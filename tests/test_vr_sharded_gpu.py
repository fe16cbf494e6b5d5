"""GPU: VREngine(dist=...) -- the patches of one VR track split over the ranks -- and the `b200_sharded` switch of the VR and Demucs plugins.

World size 1 (always runs on a one-GPU box, spawned nccl group): the sharded engine must reproduce the plain engine bit for bit for a small
CascadedASPPNet (one band and 4band_v2) and a small VR 5.1 net, with test-time augmentation, post-processing and the high-end mirror each on and off;
the sharded VR and Demucs plugins must write the same WAV bytes as the plain ones.  World size 2 (skipped unless two GPUs are visible): the same
equalities against a single-GPU run inside rank 0, and rank 1 returns [] and writes nothing.  The planner gives every patch the forward (batch
size and slot) it has on one GPU; separately, at the released geometries, a patch's prediction must not depend on the batch it ran in at all."""
import json
import os
import random
import socket
import tempfile
import wave

import numpy as np
import pytest
import torch

import demucs_oracle as D
import mdx_oracle as M
import vr_oracle as V

pytestmark = pytest.mark.gpu

COMBOS = [(tta, pp, he) for tta in (False, True) for pp in (None, 0.05) for he in (False, True)]


def _nets():
    from audio_separator.separator.b200 import vr

    p1 = V.single_band_param(n_fft=256, hl=64, bins=128)
    p51 = V.single_band_param(n_fft=256, hl=64, bins=128, pre_filter_start=120, pre_filter_stop=127)
    p51["band"][1]["convert_channels"] = "mid_side_c"
    return vr, [  # (name, net, model parameters, window_size, batch_size, samples)
        ("aspp 1band", vr.VRNet(31191, 256, V.make_weights(31191, seed=31191 % 97)), p1, 272, 3, 40000),
        ("aspp 4band_v2", vr.VRNet(33966, 1344, V.make_weights(33966, seed=5)), V.four_band_v2_param(), 272, 2, 90000),
        ("vr51 1band", vr.VRNet51(256, 8, 16, V.make_weights_51(256, 8, 16, seed=3)), p51, 160, 3, 40000),
    ]


def _check_engines(rank, world, results):
    """On every rank of an initialised nccl group; rank 0 appends (name, equal)."""
    import torch.distributed as dist

    vr, nets = _nets()
    for name, net, param, window, batch, n in nets:
        wave_ = M.synth_music(n, seed=n % 97)
        sharded = vr.VREngine(net, param, window, aggression=5, primary_stem="Instrumental", batch_size=batch, dist=dist)
        plain = vr.VREngine(net, param, window, aggression=5, primary_stem="Instrumental", batch_size=batch) if rank == 0 else None
        for tta, pp, he in COMBOS:
            got = sharded.separate(wave_, enable_tta=tta, post_process_threshold=pp, high_end_process=he)
            tag = f"{name} tta={tta} post_process={pp} high_end={he}"
            if rank != 0:
                assert got is None, tag
                continue
            ref = plain.separate(wave_, enable_tta=tta, post_process_threshold=pp, high_end_process=he)
            results.append((tag, all(np.array_equal(a, b) for a, b in zip(got, ref)) and got[0].shape == ref[0].shape))
        if rank == 0:  # the mask itself, and `inference` on the rank that holds it
            spec = plain.loading_mix(torch.from_numpy(wave_).cuda())
            for tta in (False, True):
                m = sharded.masks(spec, tta)
                results.append((f"{name} masks tta={tta}", torch.equal(m, plain.masks(spec, tta))))
        else:
            spec = sharded.loading_mix(torch.from_numpy(wave_).cuda())
            for tta in (False, True):
                assert sharded.masks(spec, tta) is None
        dist.barrier()


def _song(path, n=30000, seed=13):
    pcm = (M.synth_music(n, seed=seed).T * 32767).astype("<i2")
    with wave.open(str(path), "wb") as wf:
        wf.setnchannels(2); wf.setsampwidth(2); wf.setframerate(44100); wf.writeframes(pcm.tobytes())


def _model_files(tmp):
    from test_demucs_gpu import SMALL, _write_package

    np.savez(os.path.join(tmp, "tiny-vr.npz"), **V.make_weights(31191, seed=3))
    with open(os.path.join(tmp, "tiny-vr.json"), "w") as f:
        f.write('{"vr_model_param": "tiny_1band", "primary_stem": "Instrumental", "b200_nn_architecture": 31191}')
    p = V.single_band_param(n_fft=256, hl=64, bins=128)
    with open(os.path.join(tmp, "tiny_1band.json"), "w") as f:
        json.dump({k: v for k, v in p.items() if not isinstance(v, bool)}, f)
    np.savez(os.path.join(tmp, "tiny-vr51.npz"), **V.make_weights_51(256, 8, 16, seed=5))
    with open(os.path.join(tmp, "tiny-vr51.json"), "w") as f:
        f.write('{"vr_model_param": "tiny_1band_51", "primary_stem": "Vocals", "nout": 8, "nout_lstm": 16}')
    p = V.single_band_param(n_fft=256, hl=64, bins=128, pre_filter_start=120, pre_filter_stop=127)
    with open(os.path.join(tmp, "tiny_1band_51.json"), "w") as f:
        json.dump({k: v for k, v in p.items() if not isinstance(v, bool)}, f)
    ocfg = D.HTConfig(**SMALL)
    _write_package(os.path.join(tmp, "aaaa1111.th"), ocfg, D.make_weights(ocfg, seed=21))
    _write_package(os.path.join(tmp, "bbbb2222.th"), ocfg, D.make_weights(ocfg, seed=22))
    with open(os.path.join(tmp, "tiny_ft.yaml"), "w") as f:
        f.write("models: ['aaaa1111', 'bbbb2222']\nweights: [[1, 0, 1, 1], [0, 1, 1, 0]]\n")
    _song(os.path.join(tmp, "song.wav"))


PLUGIN_RUNS = [("tiny-vr.npz", "vr_params", {"window_size": 272, "batch_size": 4, "aggression": 5, "enable_tta": True}),
               ("tiny-vr51.npz", "vr_params", {"window_size": 160, "batch_size": 3, "aggression": 5, "enable_post_process": True, "high_end_process": True}),
               ("tiny_ft.yaml", "demucs_params", {"shifts": 2, "batch_size": 2})]


def _check_plugins(rank, results):
    """The plugins with b200_sharded write the bytes the plain plugins write (plain runs on rank 0 only); the other ranks write nothing."""
    from audio_separator.separator import Separator

    with tempfile.TemporaryDirectory(prefix="b200sep-vr-sharded-") as tmp:
        _model_files(tmp)
        for model_file, key, params in PLUGIN_RUNS:
            written = []
            for sharded in ((False, True) if rank == 0 else (True,)):
                out_dir = os.path.join(tmp, f"out_{model_file}_{sharded}")
                random.seed(1234 + rank)  # the Demucs shift draws: the sharded plugin uses rank 0's on every rank
                sep = Separator(model_file_dir=tmp, output_dir=out_dir, **{key: dict(params, b200_sharded=sharded)})
                sep.load_model(model_file)
                files = sep.separate(os.path.join(tmp, "song.wav"))
                if rank != 0:
                    assert files == [], files
                    assert not os.path.isdir(out_dir) or not any(os.scandir(out_dir)), os.listdir(out_dir)
                    continue
                written.append((files, [open(os.path.join(out_dir, f), "rb").read() for f in files]))
            if rank == 0:
                (f0, b0), (f1, b1) = written
                results.append((f"plugin {model_file}", f0 == f1 and len(f0) >= 2 and b0 == b1))


def _worker(rank, world, port, q):
    import torch.distributed as dist

    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", rank))
    res = []
    _check_engines(rank, world, res)
    _check_plugins(rank, res)
    dist.barrier()
    if rank == 0:
        q.put(res)
    dist.destroy_process_group()


def _free_port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def _run(world):
    import torch.multiprocessing as mp

    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_worker, args=(r, world, port, q)) for r in range(world)]
    for p in procs:
        p.start()
    for p in procs:
        p.join(900)
    codes = [p.exitcode for p in procs]
    for p in procs:  # a rank that died leaves its peers waiting in NCCL: do not let them hold the GPUs
        if p.is_alive():
            p.kill()
    assert codes == [0] * world, codes
    return q.get(timeout=10)


def _assert_all_equal(res):
    assert len(res) == 3 * len(COMBOS) + 3 * 2 + len(PLUGIN_RUNS)
    bad = [name for name, same in res if not same]
    assert not bad, bad


@pytest.mark.timeout(1200)
def test_vr_sharded_world1_equals_plain_engine_and_plugins(lib_built):
    _assert_all_equal(_run(1))


@pytest.mark.timeout(1200)
@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs two GPUs")
def test_vr_sharded_world2_equals_single_gpu(lib_built):
    _assert_all_equal(_run(2))


@pytest.mark.parametrize("model_file,key", [("tiny-vr.npz", "vr_params"), ("tiny_ft.yaml", "demucs_params")])
def test_sharded_plugins_need_torch_distributed(lib_built, tmp_path, model_file, key):
    import torch.distributed as dist
    from audio_separator.separator import Separator

    assert not dist.is_initialized()
    _model_files(str(tmp_path))
    sep = Separator(model_file_dir=str(tmp_path), output_dir=str(tmp_path / "out"), **{key: {"b200_sharded": True}})
    with pytest.raises(RuntimeError, match="torch.distributed"):
        sep.load_model(model_file)


@pytest.mark.timeout(900)
@pytest.mark.parametrize("geometry", ["9_HP2 (CascadedASPPNet 537238, 4band_v2)", "VR 5.1 (nout 48, nout_lstm 128)"])
def test_patch_prediction_does_not_depend_on_its_batch(lib_built, geometry):
    """Four 512-frame patches at a released geometry, predicted as one forward of 4, as 2 + 2, as 3 + 1 and one by one: every patch's mask must be
    bit-identical, so a rank that runs a patch in another forward than one GPU would gets the same result."""
    from audio_separator.separator.b200 import vr

    if geometry.startswith("9_HP2"):
        net = vr.VRNet(537238, 1344, V.make_weights(537238, seed=9))
    else:
        net = vr.VRNet51(1344, 48, 128, V.make_weights_51(1344, 48, 128, seed=12))
    x = torch.from_numpy(np.abs(np.random.default_rng(11).standard_normal((4, 2, 673, 512))).astype(np.float32)).cuda()
    x /= x.max()
    whole = net.predict_mask(x)
    for split in ((2, 2), (3, 1), (1, 3), (1, 1, 1, 1)):
        parts, i = [], 0
        for b in split:
            parts.append(net.predict_mask(x[i : i + b].contiguous()))
            i += b
        got = torch.cat(parts)
        assert torch.equal(got, whole), (split, float((got - whole).abs().max()))
