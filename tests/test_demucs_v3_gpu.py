"""GPU parity of the time-domain Demucs v3 path: the two resampling kernels against an fp64 restatement, DemucsNet's layers and forward against the
oracle and the golden vectors of the UNMODIFIED reference (oracle/make_golden_demucs_v3.py), a bag mixing Demucs and HDemucs members through
apply_model, the released 48-channel geometry, the fp16 mode, the Separator plugin on a bag file, and the time-sharded run.
Audio tolerance: 1e-4 max-abs relative to the signal peak."""
import os
import random
import socket
import sys
import types

import numpy as np
import pytest
import torch

import demucs_v3_oracle as V
import hdemucs_oracle as H
import mdx_oracle as M

pytestmark = pytest.mark.gpu

SMALL = dict(channels=8, depth=4, norm_starts=2, dconv_lstm=2, dconv_attn=2, dconv_mode=3, segment=0.1)
SMALL_B = dict(channels=8, depth=3, dconv_mode=1, context=0, segment=0.15)
HD_SMALL = dict(channels=8, nfft=256, depth=4, norm_starts=2, dconv_lstm=2, dconv_attn=2, segment=0.5)


def dev(x):
    return torch.as_tensor(np.ascontiguousarray(x)).cuda()


@pytest.fixture(scope="module")
def dv(lib_built):
    assert torch.cuda.is_available()
    from audio_separator.separator.b200 import demucs_v3

    return demucs_v3


def _bag(dv, z):
    from audio_separator.separator.b200 import hdemucs as hd

    seeds = [int(s) for s in z["weights_seed"]]
    w, w_b, hw = V.make_weights(V.V3Config(**SMALL), seeds[0]), V.make_weights(V.V3Config(**SMALL_B), seeds[1]), H.make_weights(H.HDConfig(**HD_SMALL), seeds[2])
    nets = [dv.DemucsNet(dv.DemucsConfig(**SMALL), w), dv.DemucsNet(dv.DemucsConfig(**SMALL_B), w_b), hd.HDemucsNet(hd.HDemucsConfig(**HD_SMALL), hw)]
    return (w, w_b, hw), nets


@pytest.fixture(scope="module")
def small(dv, golden_dir):
    z = np.load(os.path.join(golden_dir, "demucs_v3_small.npz"))
    weights, nets = _bag(dv, z)
    mix = M.synth_music(3 * int(z["n_apply"]), seed=int(z["mix_seed"]))
    return z, weights, nets, mix


# ------------------------------------------------------------------------------------------------ the two kernels
@pytest.mark.parametrize("B,length,extra", [(1, 2, 0), (2, 17, 6), (3, 40, 0), (1, 1000, 1), (2, 4095, 321), (1, 44101, 2048), (4, 123457, 0)])
def test_resample_kernels_vs_fp64(dv, B, length, extra):
    """Both kernels on ragged lengths, lengths shorter than the filters (replicate edges dominate) and batches, against the oracle's ends of the forward
    evaluated in float64 with the same float32 taps."""
    from audio_separator.separator.b200._lib import check, lib
    from audio_separator.separator.b200.engine import _ptr, _stream

    g = torch.Generator().manual_seed(length)
    x = torch.randn((B, 2, length), generator=g) * 0.3 + 0.05
    valid = length + extra
    up, uw = dv.julius_taps(1, 2)
    down, dw = dv.julius_taps(2, 1)
    up_d, down_d = dev(up.astype(np.float32)), dev(down.astype(np.float32))
    xd = x.cuda()
    y = torch.empty((B, 2, 2 * valid), device="cuda")
    stats = torch.empty((B, 2), device="cuda")
    work = torch.empty((lib.b200sep_meanstd_work_floats(B),), device="cuda")
    check(lib.b200sep_demucs_upsample2_f32(_ptr(xd), B, length, valid, _ptr(up_d), uw, _ptr(stats), _ptr(y), _ptr(work), _stream()), "demucs_upsample2_f32")
    ref, mean, std = V.resample_in(x.double(), valid)
    torch.cuda.synchronize()
    assert (stats.cpu().double()[:, 0] - mean.view(B)).abs().max() <= 1e-6 and (stats.cpu().double()[:, 1] / std.view(B) - 1).abs().max() <= 1e-6
    assert (y.cpu().double() - ref).abs().max() <= 2e-5 * max(1.0, float(ref.abs().max()))
    C = 6
    x2 = torch.randn((B, C, 2 * valid), generator=g)
    st = torch.stack([torch.randn(B, generator=g) * 0.1, torch.rand(B, generator=g) + 0.2], 1)
    x2d, std_d = x2.cuda(), st.cuda()
    out = torch.empty((B, C, length), device="cuda")
    check(lib.b200sep_demucs_downsample2_f32(_ptr(x2d), B, C, valid, length, _ptr(down_d), dw, _ptr(std_d), _ptr(out), _stream()), "demucs_downsample2_f32")
    ref2 = V.resample_out(x2.double(), st[:, 0].double().view(B, 1, 1), st[:, 1].double().view(B, 1, 1), length)
    torch.cuda.synchronize()
    assert (out.cpu().double() - ref2).abs().max() <= 2e-5 * max(1.0, float(ref2.abs().max()))


# ------------------------------------------------------------------------------------------------ the network
def _check(got, ref, tol=1e-4):
    assert got.shape == ref.shape, (got.shape, ref.shape)
    err = float(np.abs(got - ref).max())
    assert err <= tol * max(1.0, float(np.abs(ref).max())), (err, float(np.abs(ref).max()))


def test_forward_vs_reference_golden(small):
    z, _, nets, mix = small
    n, nl = int(z["fwd_len"]), int(z["long_len"])
    _check(nets[0].forward(dev(mix[None, :, :n])).cpu().numpy(), z["forward_b2_ref"][:1])  # one chunk = entry 0 of the batch-2 golden
    _check(nets[0].forward(dev(mix[None, :, :nl])).cpu().numpy(), z["forward_long_ref"])
    _check(nets[0].forward(dev(np.stack([mix[:, :n], mix[:, n : 2 * n]]))).cpu().numpy(), z["forward_b2_ref"])


def test_encoder_decoder_taps_vs_oracle(small):
    """Every encoder and decoder output against the oracle's intermediate tensors (localises a failure of the forward tests)."""
    z, (w, _, _), nets, mix = small
    net = nets[0]
    seg = mix[None, :, : int(z["long_len"])]
    taps = {}
    V.forward(w, V.V3Config(**SMALL), seg, taps=taps)
    got = {}
    orig_enc, orig_dec = net._enc_layer, net._dec_layer

    def enc(x, prefix, L, inject=None):
        y = orig_enc(x, prefix, L, inject)
        got["enc" + prefix.split(".")[1]] = y.clone()
        return y

    def dec(x, skip, length, prefix, L):
        zz, y = orig_dec(x, skip, length, prefix, L)
        got["dec" + prefix.split(".")[1]] = zz.clone()
        return zz, y

    net._enc_layer, net._dec_layer = enc, dec
    try:
        net.forward(dev(seg))
    finally:
        del net._enc_layer, net._dec_layer
    torch.cuda.synchronize()
    assert set(got) == set(taps)
    report = [(k, float(np.abs(t.cpu().numpy().reshape(taps[k].shape) - taps[k]).max()), float(np.abs(taps[k]).max())) for k, t in got.items()]
    assert not [r for r in report if r[1] > 1e-4 * max(1.0, r[2])], report


@pytest.mark.parametrize("split", [True, False])
def test_mixed_bag_apply_model_vs_reference_golden(small, split):
    """apply_model on a BagOfModels of two Demucs and one HDemucs with per-source weights and their own segments: split + shifts, and split=False."""
    from audio_separator.separator.b200.demucs import DemucsEngine

    z, _, nets, mix = small
    name = "split" if split else "nosplit"
    N = int(z["n_apply"])
    m2 = torch.from_numpy(mix[:, :N])
    mn = dev(((m2 - m2.mean(0).mean()) / m2.mean(0).std()).numpy())
    bw = np.asarray(z["bag_weights"], np.float64)
    eng = DemucsEngine(nets, bag_weights=bw.tolist(), batch_size=3, split=split)
    out = torch.empty((8, N), device="cuda")
    for mi, offs in enumerate(z[f"bag_{name}_offsets"].tolist()):
        cs = dev(np.repeat(bw[mi] / bw.sum(0), 2).astype(np.float32))
        eng.apply_model(mn, offs, mi, out, cs, accumulate=mi > 0)
    _check(out.cpu().numpy().reshape(1, 4, 2, N), z[f"bag_{name}_ref"])


def test_released_geometry_5s_vs_oracle(dv):
    """48 channels, depth 6 (DConv hidden 12 ... 384, BLSTM / LocalState and GroupNorm from index 4 on) on 5 seconds against the oracle."""
    ocfg = V.V3Config(channels=48)
    w = V.make_weights(ocfg, seed=31)
    mix = M.synth_music(220500, seed=78)[None]
    ref = V.forward(w, ocfg, mix)
    _check(dv.DemucsNet(dv.DemucsConfig(channels=48), w).forward(dev(mix)).cpu().numpy(), ref)


def test_fp16_mode(small, dv):
    from audio_separator.separator.b200 import _lib

    z, (w, _, _), nets, mix = small
    seg = dev(mix[None, :, : int(z["long_len"])])
    y16 = dv.DemucsNet(dv.DemucsConfig(**SMALL), w, math=_lib.MATH_FP16).forward(seg).cpu().numpy()
    y32 = nets[0].forward(seg).cpu().numpy()
    assert np.isfinite(y16).all() and np.abs(y16 - y32).max() > 1e-5
    snr = 10 * np.log10(np.sum(y32.astype(np.float64) ** 2) / np.sum((y16 - y32).astype(np.float64) ** 2))
    print(f"small Demucs v3: fp16 vs bf16x3 {snr:.1f} dB")
    assert snr >= 50.0, snr  # the gate of the HDemucs fp16 test


# ------------------------------------------------------------------------------------------------ the plugin
def _package(path, module, name, kwargs, weights):
    parts = module.split(".")
    mods = {".".join(parts[: i + 1]): types.ModuleType(".".join(parts[: i + 1])) for i in range(len(parts))}
    K = type(name, (), {"__module__": module})
    setattr(mods[module], name, K)
    saved = {m: sys.modules.get(m) for m in mods}
    sys.modules.update(mods)
    try:
        torch.save({"klass": K, "args": (), "kwargs": kwargs, "state": {k: torch.from_numpy(v) for k, v in weights.items()}}, path)
    finally:
        for m, v in saved.items():
            if v is None:
                del sys.modules[m]
            else:
                sys.modules[m] = v


def test_separator_mixed_bag_end_to_end(small, tmp_path):
    """Separator().load_model(bag.yaml) on a bag of two Demucs v3 and one HDemucs package; separate(wav) -> four stems within 3 LSB of the oracle pipeline."""
    import wave

    from audio_separator.separator import Separator

    z, (w, w_b, hw), _, _ = small
    _package(str(tmp_path / "aaaa0001.th"), "demucs.demucs", "Demucs", V.V3Config(**SMALL).kwargs(), w)
    _package(str(tmp_path / "aaaa0002-0123abcd.th"), "demucs.demucs", "Demucs", V.V3Config(**SMALL_B).kwargs(), w_b)
    _package(str(tmp_path / "aaaa0003.th"), "demucs.hdemucs", "HDemucs", H.HDConfig(**HD_SMALL).kwargs(), hw)
    bw = z["bag_weights"].tolist()
    (tmp_path / "mixed.yaml").write_text(f"models: ['aaaa0001', 'aaaa0002', 'aaaa0003']\nweights: {bw}\n")
    n = 30000
    pcm = (M.synth_music(n, seed=44).T * 32767).astype("<i2")
    with wave.open(str(tmp_path / "song.wav"), "wb") as wf:
        wf.setnchannels(2); wf.setsampwidth(2); wf.setframerate(44100); wf.writeframes(pcm.tobytes())
    sep = Separator(model_file_dir=str(tmp_path), output_dir=str(tmp_path / "out"), demucs_params={"shifts": 1, "batch_size": 2})
    sep.load_model("mixed.yaml")
    random.seed(77)
    files = sep.separate(str(tmp_path / "song.wav"))
    assert files == ["song_(Bass)_mixed.wav", "song_(Drums)_mixed.wav", "song_(Other)_mixed.wav", "song_(Vocals)_mixed.wav"]
    random.seed(77)
    offs = [[random.randint(0, 22050)] for _ in range(3)]
    m = torch.from_numpy(pcm.astype(np.float32).T / 32768.0)
    ref_ = m.mean(0)
    mn = ((m - ref_.mean()) / ref_.std()).numpy()[None]
    members = [(lambda c: V.forward(w, V.V3Config(**SMALL), c), V.V3Config(**SMALL)), (lambda c: V.forward(w_b, V.V3Config(**SMALL_B), c), V.V3Config(**SMALL_B)),
               (lambda c: H.forward(hw, H.HDConfig(**HD_SMALL), c), H.HDConfig(**HD_SMALL))]
    est = V.apply_bag(members, bw, mn, offs)[0]
    src = (torch.from_numpy(est) * ref_.std() + ref_.mean()).numpy()
    src[[0, 1]] = src[[1, 0]]
    for k, fname in enumerate(files):
        with wave.open(str(tmp_path / "out" / fname)) as wf:
            got = np.frombuffer(wf.readframes(n), dtype="<i2").astype(np.int32)
        want = M.to_pcm16(src[k].T.copy(), 0.9, 0.0).astype(np.int32)
        assert np.abs(got - want).max() <= 3


# ------------------------------------------------------------------------------------------------ time-sharded
def _worker(rank, world, port, q):
    import torch.distributed as dist

    from audio_separator.separator.b200 import demucs_v3
    from audio_separator.separator.b200.demucs import DemucsEngine

    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", rank))
    z = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "demucs_v3_small.npz"))
    _, nets = _bag(demucs_v3, z)
    n = 7 * nets[0].cfg.seg_len + 1234
    mix = torch.from_numpy(M.synth_music(n, seed=9)).cuda()
    offs, bag = [[1000, 15000], [22050, 7], [3, 11111]], z["bag_weights"].tolist()
    eng = DemucsEngine(nets, bag_weights=bag, batch_size=3, dist=dist)
    got = eng.gather(eng.demix_device(mix, offs), n)
    if rank == 0:
        ref = DemucsEngine(nets, bag_weights=bag, batch_size=3).demix_device(mix, offs)
        q.put(float((got - ref).abs().max()))
    dist.barrier()
    dist.destroy_process_group()


def _run(world):
    import torch.multiprocessing as mp

    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        port = s.getsockname()[1]
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=_worker, args=(r, world, port, q)) for r in range(world)]
    for p in procs:
        p.start()
    for p in procs:
        p.join(600)
    codes = [p.exitcode for p in procs]
    for p in procs:  # a rank that died leaves its peers waiting in NCCL: do not let them hold the GPUs
        if p.is_alive():
            p.kill()
    assert codes == [0] * world, codes
    return q.get(timeout=10)


@pytest.mark.timeout(900)
@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs two GPUs")
def test_sharded_world2_equals_world1(lib_built):
    """A mixed bag time-sharded over two GPUs gives the single-GPU result (the gate of test_sharded_gpu.py's Demucs case)."""
    assert _run(2) <= 1e-5
