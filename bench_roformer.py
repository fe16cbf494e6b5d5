"""bench_roformer.py -- real-time factor of the BS-Roformer demix on N H100s, one track time-sharded over the GPUs.

  python -m torch.distributed.run --nproc-per-node N bench_roformer.py [--steps K] [--warmup W] [--batch-size B] [--seconds S]
  python bench_roformer.py ...                       (one GPU, no process group)

Workload: the released BS-Roformer geometry (dim 512, depth 12, 8 x 64 heads, 62 bands, n_fft 2048, hop 441, dim_t 801 -> 352 800-sample
chunks) with seeded synthetic weights (oracle/roformer_oracle.make_weights; there are no model files offline) on a seeded S-second stereo
track (default 5 min), at two overlap settings of the MDXC plugin:
  overlap 8 -- the plugin default: step = chunk, only the clamped tail chunk overlaps its neighbour;
  overlap 2 -- step 88 200, about four chunks cover each sample, so every rank past the first receives a halo of its left neighbour's chunks.
One step = RoformerEngine.demix_device + gather to rank 0 with the mix resident in HBM; CUDA events on the launch stream, `warmup` untimed steps
first, max over ranks.  parity: rank 0 compares the gathered stems of the last timed step with a single-GPU RoformerEngine on the same mix.
Prints one JSON line (rank 0).  Writes nothing to disk.
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(ROOT, "python-audio-separator_b200"))
sys.path.insert(0, os.path.join(ROOT, "oracle"))

SR = 44100


def gpu_info(index):
    q = "name,power.limit,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader,nounits", "-i", str(index)], capture_output=True, text=True, timeout=20).stdout
        name, power, clock = (v.strip() for v in out.strip().split(","))
        return {"gpu": name, "power_limit_w": float(power), "clocks_max_sm_mhz": float(clock)}
    except Exception as e:  # the numbers are reported as missing rather than guessed
        import torch

        return {"gpu": torch.cuda.get_device_name(index), "power_limit_w": None, "clocks_max_sm_mhz": None, "nvidia_smi_error": str(e)}


def music(n, seed):
    """Seeded programme material: a 30-s pattern of the oracle generator, tiled."""
    import numpy as np

    import mdx_oracle as O

    base = O.synth_music(min(n, 30 * SR), seed=seed)
    return np.tile(base, (1, -(-n // base.shape[1])))[:, :n].copy()


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--steps", type=int, default=1)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--batch-size", type=int, default=1)
    ap.add_argument("--seconds", type=float, default=300.0)
    ap.add_argument("--overlaps", default="8,2", help="comma-separated mdxc_params['overlap'] values (seconds)")
    args = ap.parse_args()

    import torch

    assert torch.cuda.is_available(), "bench_roformer.py needs a CUDA device"
    local = int(os.environ.get("LOCAL_RANK", "0"))
    torch.cuda.set_device(local)
    dist = None
    if "RANK" in os.environ:  # launched by torch.distributed.run: the sharded path, also at world size 1
        import torch.distributed as dist

        dist.init_process_group("nccl", device_id=torch.device("cuda", local))
    rank = dist.get_rank() if dist else 0
    world = dist.get_world_size() if dist else 1

    import roformer_oracle as R
    from audio_separator.separator.b200 import roformer as rf

    kw = dict(stft_hop_length=441)
    net = rf.BSRoformerNet(rf.BSRoformerConfig(**kw), R.make_weights(R.BSRoformerConfig(**kw), seed=8))
    N = int(args.seconds * SR)
    mix = torch.from_numpy(music(N, seed=21) * 0.5).cuda()

    def sync():
        if dist:
            dist.barrier()
        torch.cuda.synchronize()

    results = []
    for overlap in (float(v) for v in args.overlaps.split(",")):
        eng = rf.RoformerEngine(net, 801, overlap, SR, batch_size=args.batch_size, dist=dist)
        step_fn = lambda: eng.gather(eng.demix_device(mix), N)  # noqa: E731
        for _ in range(args.warmup):
            step_fn()
        sync()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(args.steps):
            out = step_fn()
        e1.record()
        sync()
        ms = torch.tensor([e0.elapsed_time(e1) / args.steps], dtype=torch.float64, device="cuda")
        if dist:
            dist.all_reduce(ms, op=dist.ReduceOp.MAX)
        ms = float(ms)
        res = {"overlap": overlap, "step": eng.step, "chunks": len(eng.chunk_starts(N)), "ms_per_step": round(ms, 3), "rtf": round(args.seconds / (ms / 1000.0), 3)}
        if rank == 0:
            ref = rf.RoformerEngine(net, 801, overlap, SR, batch_size=args.batch_size).demix_device(mix)
            res["parity"] = {"bit_identical": bool(torch.equal(out, ref)), "max_abs_diff": float((out - ref).abs().max())}
            del ref
        del eng, out
        sync()
        results.append(res)
    if rank == 0:
        line = {"workload": "bs_roformer", "metric": "real-time factor (audio-sec/device-sec) @44.1kHz stereo", "world": world, **gpu_info(local),
                "track_seconds": args.seconds, "batch_size": args.batch_size, "steps": args.steps, "warmup": args.warmup, "data": "synthetic (seeded)",
                "results": results}
        print(json.dumps(line), flush=True)
    if dist:
        dist.destroy_process_group()


if __name__ == "__main__":
    main()
