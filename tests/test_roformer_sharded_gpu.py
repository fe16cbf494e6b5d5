"""GPU: the time-sharded Roformer path -- b200sep_overlap_add_starts_range, RoformerEngine(dist=...) and the MDXC plugin's `b200_sharded` switch.

World size 1 (always runs on a one-GPU box): the sharded code path must reproduce the plain engine bit for bit and the reference goldens within
1e-4, and the sharded plugin must write the same WAV bytes as the plain one.  World size 2 (skipped unless two GPUs are visible): two NCCL
processes, halo exchange + gather, compared with a single-GPU run inside rank 0."""
import os
import socket

import numpy as np
import pytest
import torch

import mdx_oracle as M
import roformer_oracle as R

pytestmark = pytest.mark.gpu

SMALL = dict(dim=32, depth=2, time_transformer_depth=1, freq_transformer_depth=2, freqs_per_bands=(2, 2, 4, 4, 8, 12, 16, 17), dim_head=8, heads=4, stft_n_fft=128,
             stft_hop_length=32, stft_win_length=128)
MSMALL = dict(dim=32, depth=2, time_transformer_depth=1, freq_transformer_depth=1, num_bands=12, dim_head=8, heads=4, mask_estimator_depth=2, stft_n_fft=128, stft_hop_length=32,
              stft_win_length=128)
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "roformer_small.npz")


def dev(x):
    return torch.as_tensor(np.ascontiguousarray(x)).cuda()


# ------------------------------------------------------------------------------------------------ ranged kernel
def test_overlap_add_starts_range_partitions_equal_full(lib_built):
    from audio_separator.separator.b200._lib import check, lib

    g = torch.Generator().manual_seed(4)
    C, N, step, ch = 50, 1000, 17, 3
    starts = [i if i + C <= N else N - C for i in range(0, N, step)]
    assert starts.count(N - C) > 1  # repeated tail starts
    n = len(starts)
    chunks = torch.randn((n, ch, C), generator=g).cuda()
    win = torch.from_numpy(np.hamming(C).astype(np.float32)).cuda()
    sd = torch.tensor(starts, dtype=torch.int64).cuda()
    full = torch.empty((ch, N), device="cuda")
    check(lib.b200sep_overlap_add_starts(chunks.data_ptr(), sd.data_ptr(), win.data_ptr(), n, ch, C, N, full.data_ptr(), 0), "overlap_add_starts")
    for cuts in ([0, N], [0, 500, N], [0, 1, 333, 334, 990, N], [0, 120, 120, 640, N], [0, 17, 51, 52, 400, 401, 951, N]):
        parts = []
        for q0, q1 in zip(cuts, cuts[1:]):
            cover = [i for i, s in enumerate(starts) if s < q1 and s + C > q0] or [0]
            lo, hi = cover[0], cover[-1] + 1  # only the chunks that overlap [q0, q1)
            base = max(0, q0 - 3)
            ld = q1 - base + 5
            out = torch.full((ch, ld), float("nan"), device="cuda")
            check(lib.b200sep_overlap_add_starts_range(chunks[lo:hi].data_ptr(), sd[lo:hi].data_ptr(), hi - lo, win.data_ptr(), ch, C, N, q0, q1, out.data_ptr(), ld, base, 0),
                  "overlap_add_starts_range")
            o = out.cpu()
            assert o[:, : q0 - base].isnan().all() and o[:, q1 - base :].isnan().all()  # nothing outside the range is written
            parts.append(o[:, q0 - base : q1 - base])
        assert torch.equal(torch.cat(parts, 1), full.cpu()), cuts
    out = torch.empty((ch, N), device="cuda")
    p = (chunks.data_ptr(), sd.data_ptr(), n, win.data_ptr(), ch, C, N)
    for bad in ((10, 5, out.data_ptr(), N, 0), (-1, 5, out.data_ptr(), N, 0), (0, N + 1, out.data_ptr(), N + 1, 0), (100, 200, out.data_ptr(), N, 101),
                (100, 200, out.data_ptr(), 50, 100), (0, N, None, N, 0)):
        q0, q1, optr, ld, base = bad
        rc = lib.b200sep_overlap_add_starts_range(*p, q0, q1, optr, ld, base, 0)
        assert rc != 0 and b"overlap_add_starts" in lib.b200sep_last_error(), bad
    assert lib.b200sep_overlap_add_starts_range(chunks.data_ptr(), sd.data_ptr(), 0, win.data_ptr(), ch, C, N, 0, N, out.data_ptr(), N, 0, 0) != 0
    torch.cuda.synchronize()


# ------------------------------------------------------------------------------------------------ engines, world size 1 and 2
def _nets():
    from audio_separator.separator.b200 import roformer as rf

    bs1 = rf.BSRoformerNet(rf.BSRoformerConfig(**SMALL), R.make_weights(R.BSRoformerConfig(**dict(SMALL, dim_t=65, overlap=8)), seed=3))
    kw2 = dict(SMALL, num_stems=2, mask_estimator_depth=3, depth=1)
    bs2 = rf.BSRoformerNet(rf.BSRoformerConfig(**kw2), R.make_weights(R.BSRoformerConfig(**dict(kw2, dim_t=65, overlap=8)), seed=4))
    mel = rf.BSRoformerNet(rf.MelBandRoformerConfig(**MSMALL), R.make_mel_weights(R.MelBandRoformerConfig(**dict(MSMALL, dim_t=65)), seed=6))
    return rf, {"bs": bs1, "bs2": bs2, "mel": mel}


GOLDEN_KEYS = {("bs", 8): "demix_ref", ("bs", 0.03): "demix_overlap_ref", ("bs2", 8): "demix_2stem_ref", ("mel", 8): "mel_demix_ref"}


def _check_engines(rank, world, results):
    """Runs on every rank of an initialised nccl group; rank 0 appends (name, bit_identical, max_abs_diff, batch)."""
    import torch.distributed as dist

    rf, nets = _nets()
    gold = np.load(GOLDEN)
    mixes = {"gold": M.synth_music(int(gold["n_samples"]), seed=int(gold["mix_seed"])), "long": M.synth_music(11 * 1024 + 77, seed=21)}
    for name, net in nets.items():
        for overlap in (8, 0.03):  # step == chunk (2048), step 1323 < chunk
            for batch in (1, 3) if world > 1 else (2,):
                sharded = rf.RoformerEngine(net, 65, overlap, 44100, n_instruments=2, batch_size=batch, dist=dist)
                plain = rf.RoformerEngine(net, 65, overlap, 44100, n_instruments=2, batch_size=1 if world > 1 else batch)
                for mname, mix in mixes.items():
                    N = mix.shape[1]
                    part = sharded.demix_device(dev(mix))
                    assert part.shape[-1] == sharded.out_range(N)[1] - sharded.out_range(N)[0]
                    got = sharded.gather(part, N)
                    if rank != 0:
                        assert got is None
                        continue
                    ref = plain.demix_device(dev(mix))
                    tag = f"{name} overlap={overlap} {mname}"
                    results.append((tag, bool(torch.equal(got, ref)), float((got - ref).abs().max()), batch))
                    key = GOLDEN_KEYS.get((name, overlap))
                    if key and mname == "gold":
                        g = gold[key]
                        out = got.cpu().numpy()
                        out = out[0] if g.ndim == 2 else out
                        results.append((tag + " vs golden", None, float(np.abs(out - g).max()), batch))
    dist.barrier()


def _check_plugin(results):
    """World size 1: the plugin with b200_sharded writes the same bytes as without, for a Roformer and an MDX23C model."""
    import tempfile

    # the plugin takes any model whose path contains "roformer" for a Roformer: keep the MDX23C model out of a directory named after this test
    with tempfile.TemporaryDirectory(prefix="b200sep-plugin-") as tmp:
        _check_plugin_in(tmp, results)


def _check_plugin_in(tmp, results):
    import json
    import wave

    import yaml

    import mdxc_oracle as X
    from audio_separator.separator import Separator

    ocfg = R.BSRoformerConfig(**dict(SMALL, dim_t=65, overlap=8))
    np.savez(os.path.join(tmp, "tiny_bs_roformer.npz"), **R.make_weights(ocfg, seed=12))
    model = dict(SMALL, freqs_per_bands=list(SMALL["freqs_per_bands"]), stereo=True, num_stems=1, mask_estimator_depth=2)
    with open(os.path.join(tmp, "tiny_bs_roformer.yaml"), "w") as f:
        f.write(yaml.safe_dump({"audio": {"sample_rate": 44100, "hop_length": 32, "n_fft": 128, "dim_f": 65}, "model": model,
                                "training": {"instruments": ["Vocals", "Instrumental"], "target_instrument": "Vocals"}, "inference": {"dim_t": 65}}))
    xcfg = X.MDXCConfig(n_fft=1024, hop_length=256, dim_f=512, dim_t=16, num_scales=2, num_channels_model=16, growth=16, bottleneck_factor=4, overlap=4)
    np.savez(os.path.join(tmp, "tiny-mdx23c.npz"), **X.make_weights(xcfg, seed=4, out_gain=0.3))
    with open(os.path.join(tmp, "tiny-mdx23c.json"), "w") as f:
        json.dump({"audio": {"n_fft": xcfg.n_fft, "hop_length": xcfg.hop_length, "dim_f": xcfg.dim_f, "num_channels": 2, "chunk_size": xcfg.chunk_size, "sample_rate": 44100},
                   "model": {"norm": "InstanceNorm", "act": "gelu", "num_subbands": 4, "num_scales": xcfg.num_scales, "scale": [2, 2], "num_blocks_per_scale": 2,
                             "num_channels": xcfg.num_channels_model, "growth": xcfg.growth, "bottleneck_factor": xcfg.bottleneck_factor},
                   "training": {"instruments": ["Vocals", "Instrumental"], "target_instrument": None}, "inference": {"dim_t": xcfg.dim_t}}, f)
    mix = M.synth_music(30000, seed=13)
    with wave.open(os.path.join(tmp, "song.wav"), "wb") as wf:
        wf.setnchannels(2); wf.setsampwidth(2); wf.setframerate(44100); wf.writeframes((mix.T * 32767).astype("<i2").tobytes())
    for model_file, params in (("tiny_bs_roformer.npz", {"batch_size": 4, "segment_size": 65}), ("tiny-mdx23c.npz", {"overlap": 4, "batch_size": 2, "segment_size": 16})):
        written = []
        for sharded in (False, True):
            out_dir = os.path.join(tmp, f"out_{model_file}_{sharded}")
            sep = Separator(model_file_dir=tmp, output_dir=out_dir, mdxc_params=dict(params, b200_sharded=sharded))
            sep.load_model(model_file)
            files = sep.separate(os.path.join(tmp, "song.wav"))
            written.append((files, [open(os.path.join(out_dir, f), "rb").read() for f in files]))
        (f0, b0), (f1, b1) = written
        results.append((f"plugin {model_file}", f0 == f1 and len(f0) == 2 and b0 == b1, 0.0, 0))


def _worker(rank, world, port, q):
    import torch.distributed as dist

    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", rank))
    res = []
    _check_engines(rank, world, res)
    if world == 1:
        _check_plugin(res)
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
        p.join(600)
    codes = [p.exitcode for p in procs]
    for p in procs:  # a rank that died leaves its peers waiting in NCCL: do not let them hold the GPUs
        if p.is_alive():
            p.kill()
    assert codes == [0] * world, codes
    return q.get(timeout=10)


@pytest.mark.timeout(900)
def test_roformer_sharded_world1_equals_plain_engine_and_goldens(lib_built):
    res = _run(1)
    assert len(res) == 3 * 2 * 2 + 4 + 2
    for name, same, diff, _ in res:
        if same is None:
            assert diff <= 1e-4, (name, diff)  # against the reference goldens
        else:
            assert same and diff == 0.0, (name, diff)


@pytest.mark.timeout(900)
@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs two GPUs")
def test_roformer_sharded_world2_equals_single_gpu(lib_built):
    for name, same, diff, batch in _run(2):
        if same is None:
            assert diff <= 1e-4, (name, diff)
        elif batch == 1:  # every forward has the same shape on both sides: the same arithmetic
            assert same, (name, diff)
        else:
            # the ranks batch their chunks differently from the single-GPU run, and b200sep_gemm_f32 picks the SIMT or the tensor-core kernel by
            # M*N*batch (tc_gemm_usable), and the small-N kernel from M = 1024 rows on: at these toy sizes a different batch can move a
            # mask-estimator GEMM across either threshold
            assert diff <= 1e-5, (name, diff)


def test_sharded_plugin_needs_torch_distributed(lib_built, tmp_path):
    import yaml

    import torch.distributed as dist
    from audio_separator.separator import Separator

    assert not dist.is_initialized()
    ocfg = R.BSRoformerConfig(**dict(SMALL, dim_t=65, overlap=8))
    np.savez(tmp_path / "tiny_bs_roformer.npz", **R.make_weights(ocfg, seed=12))
    model = dict(SMALL, freqs_per_bands=list(SMALL["freqs_per_bands"]), stereo=True, num_stems=1, mask_estimator_depth=2)
    (tmp_path / "tiny_bs_roformer.yaml").write_text(yaml.safe_dump({"audio": {"sample_rate": 44100, "hop_length": 32, "n_fft": 128, "dim_f": 65}, "model": model,
                                                                    "training": {"instruments": ["Vocals", "Instrumental"], "target_instrument": "Vocals"}, "inference": {"dim_t": 65}}))
    sep = Separator(model_file_dir=str(tmp_path), output_dir=str(tmp_path / "out"), mdxc_params={"b200_sharded": True})
    with pytest.raises(RuntimeError, match="torch.distributed"):
        sep.load_model("tiny_bs_roformer.npz")


@pytest.mark.timeout(900)
def test_released_geometry_batch_size_does_not_change_the_result(lib_built):
    """dim 512, depth 12, 8 x 64 heads, 62 bands, n_fft 2048, hop 441, dim_t 801, overlap 2 s: 10 chunks (the last four at the clamped tail
    start) as forwards of 1, of 2, or of 3 + 3 + 2 + 2 chunks."""
    from audio_separator.separator.b200 import roformer as rf

    kw = dict(stft_hop_length=441)
    net = rf.BSRoformerNet(rf.BSRoformerConfig(**kw), R.make_weights(R.BSRoformerConfig(**kw), seed=8))
    C = 441 * 800
    mix = dev(M.synth_music(C + 5 * 88200 + 1234, seed=9))
    one, two, three = (rf.RoformerEngine(net, 801, 2, 44100, batch_size=b).demix_device(mix) for b in (1, 2, 3))
    assert torch.equal(two, three), float((two - three).abs().max())
    # A forward of one chunk is not bit-identical to a batched one: the mask estimator's last Linear of a 2-bin band has N = 16 outputs and
    # M = batch * 801 rows, and b200sep_gemm_f32 runs such a GEMM on the warp-per-row small-N kernel only from M = 1024 on (the tiled SIMT kernel
    # below), so batch 1 sums in a different order.  1.7e-7 was measured on an H100.
    assert float((one - three).abs().max()) <= 1e-6
