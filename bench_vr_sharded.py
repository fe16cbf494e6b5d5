"""bench_vr_sharded.py -- seconds per track of the VR separation on N H100s, the patches of one track split over the GPUs.

  python -m torch.distributed.run --nproc-per-node N bench_vr_sharded.py [--steps K] [--warmup W] [--batch-size B] [--seconds S]
  python bench_vr_sharded.py ...                       (one GPU, no process group)

Workload: the 9_HP2-UVR geometry (CascadedASPPNet 537238, 4band_v2 parameters, 1344 bins, window 512, aggression 10) with seeded synthetic
weights (oracle/vr_oracle.make_weights; there are no model files offline) on a seeded S-second stereo track (default 3 min, 65 patches at
window 512), batch_size 4 -- the VREngine path of VRSeparator.separate without the file I/O.
One step = upload of the track, then three phases, each timed with CUDA events on the launch stream:
  front   -- loading_mix (band resampling, STFTs, combine): every rank, on the whole track;
  patches -- VREngine.masks: magnitude, normalisation, this rank's patches, gather of the mask to rank 0;
  tail    -- rank 0 only: the mask products (apply_mask), both stems' band synthesis (iSTFT, band sum, up-sampling) and the download.
`warmup` untimed steps first; seconds per track is the max over the ranks.  The front end and the tail do not shrink with N, so
serial = (front + tail) / step bounds the speedup at N GPUs by 1 / (serial + (1 - serial) / N) (Amdahl); `amdahl_limit` gives it for N = 8 from
this run's split.  parity: rank 0 compares the stems of the last timed step with a single-GPU VREngine on the same track.
Prints one JSON line (rank 0).  Writes nothing to disk.
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(ROOT, "python-audio-separator_b200"))
sys.path.insert(0, os.path.join(ROOT, "oracle"))

from bench_roformer import SR, gpu_info, music  # noqa: E402


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--batch-size", type=int, default=4)
    ap.add_argument("--seconds", type=float, default=180.0)
    args = ap.parse_args()

    import numpy as np
    import torch

    assert torch.cuda.is_available(), "bench_vr_sharded.py needs a CUDA device"
    local = int(os.environ.get("LOCAL_RANK", "0"))
    torch.cuda.set_device(local)
    dist = None
    if "RANK" in os.environ:  # launched by torch.distributed.run: the sharded path, also at world size 1
        import torch.distributed as dist

        dist.init_process_group("nccl", device_id=torch.device("cuda", local))
    rank = dist.get_rank() if dist else 0
    world = dist.get_world_size() if dist else 1

    import vr_oracle as V
    from audio_separator.separator.b200 import vr

    arch = 537238
    net = vr.VRNet(arch, 1344, V.make_weights(arch, seed=9))
    param = V.four_band_v2_param()
    eng = vr.VREngine(net, param, window_size=512, aggression=10, batch_size=args.batch_size, dist=dist)
    N = int(args.seconds * SR)
    wave = (music(N, seed=21) * 0.5).astype(np.float32)

    def sync():
        if dist:
            dist.barrier()
        torch.cuda.synchronize()

    n_frames = [0]

    def step(ev):
        wd = torch.from_numpy(wave).to(eng.device)
        ev[0].record()
        spec = eng.loading_mix(wd)
        n_frames[0] = spec.shape[2]  # make_padding at roi 256: frames // 256 + 1 patches
        ev[1].record()
        mask = eng.masks(spec)
        ev[2].record()
        out = None
        if mask is not None:
            y, v = eng.apply_mask(spec, mask)
            out = eng.spec_to_wav(y).cpu().numpy(), eng.spec_to_wav(v).cpu().numpy()
        ev[3].record()
        return out

    for _ in range(args.warmup):
        step([torch.cuda.Event(enable_timing=True) for _ in range(4)])
    sync()
    phases = np.zeros(4)
    for _ in range(args.steps):
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(4)]
        out = step(ev)
        torch.cuda.synchronize()
        phases += [ev[0].elapsed_time(ev[1]), ev[1].elapsed_time(ev[2]), ev[2].elapsed_time(ev[3]), ev[0].elapsed_time(ev[3])]
        if dist:
            dist.barrier()
    phases /= args.steps
    total = torch.tensor([phases[3]], dtype=torch.float64, device="cuda")
    if dist:
        dist.all_reduce(total, op=dist.ReduceOp.MAX)
    if rank == 0:
        front, patches, tail = (float(v) / 1000.0 for v in phases[:3])
        sec = float(total) / 1000.0
        serial = (front + tail) / sec
        ref = vr.VREngine(net, param, window_size=512, aggression=10, batch_size=args.batch_size).separate(wave)
        line = {"workload": "vr_9_HP2_one_track_sharded", "metric": "seconds per track (device) and real-time factor @44.1kHz stereo", "world": world, **gpu_info(local),
                "track_seconds": args.seconds, "batch_size": args.batch_size, "patches": n_frames[0] // 256 + 1,
                "steps": args.steps, "warmup": args.warmup, "data": "synthetic (seeded)",
                "seconds_per_track": round(sec, 4), "rtf": round(args.seconds / sec, 2),
                "split_rank0_s": {"front": round(front, 4), "patches": round(patches, 4), "tail": round(tail, 4)},
                "serial_share": round(serial, 4), "amdahl_limit": {"n": 8, "speedup": round(1.0 / (serial + (1.0 - serial) / 8), 2)},
                "parity": {"bit_identical": all(np.array_equal(a, b) for a, b in zip(out, ref)), "max_abs_diff": max(float(np.abs(a - b).max()) for a, b in zip(out, ref))}}
        print(json.dumps(line), flush=True)
    if dist:
        dist.barrier()
        dist.destroy_process_group()


if __name__ == "__main__":
    main()
