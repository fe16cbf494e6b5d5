"""bench_autocast.py -- real-time factor of the fp16 tensor-core mode (Separator(use_autocast=True)) against the default mode, on one H100.

  python bench_autocast.py [--runs R] [--seconds S] [--workloads bs_roformer,htdemucs_ft]

Workloads (seeded synthetic weights from the oracles -- there are no model files offline -- on a seeded S-second stereo track, default 5 min):
  bs_roformer  the released BS-Roformer geometry (dim 512, depth 12, 8 x 64 heads, 62 bands, n_fft 2048, hop 441, 801 frames), MDXC plugin defaults
               (overlap 8, batch 1): RoformerEngine.demix_device;
  htdemucs_ft  bag of 4 HTDemucs (htdemucs_ft geometry, one-hot bag weights), shifts 2, overlap 0.25, batch 4: DemucsEngine.demix_device.
Each workload builds one net set per math mode (0 = bf16x3, 1 = fp16), warms both up, then times R runs of each, alternated 0, 1, 0, 1, ...
with CUDA events around one full demix (mix resident in HBM).  Prints one JSON line per workload: median real-time factor and spread
(max/min - 1) per mode, the speed-up of the medians, the GPU name, power limit and max SM clock read in the same run, and the max-abs
difference and SNR of the fp16 stems against the default-mode stems.  Writes nothing to disk.
"""
import argparse
import json
import os
import random
import subprocess
import sys

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(ROOT, "python-audio-separator_b200"))
sys.path.insert(0, os.path.join(ROOT, "oracle"))

SR = 44100


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader,nounits", "-i", "0"], capture_output=True, text=True,
                             timeout=20).stdout
        name, power, clock = (v.strip() for v in out.strip().split(","))
        return {"gpu": name, "power_limit_w": float(power), "clocks_max_sm_mhz": float(clock)}
    except Exception as e:  # reported as missing rather than guessed
        import torch

        return {"gpu": torch.cuda.get_device_name(0), "power_limit_w": None, "clocks_max_sm_mhz": None, "nvidia_smi_error": str(e)}


def music(n, seed):
    import numpy as np

    import mdx_oracle as O

    base = O.synth_music(min(n, 30 * SR), seed=seed)
    return np.tile(base, (1, -(-n // base.shape[1])))[:, :n].copy()


def roformer_runner(math):
    import roformer_oracle as R
    from audio_separator.separator.b200 import roformer as rf

    kw = dict(stft_hop_length=441)
    net = rf.BSRoformerNet(rf.BSRoformerConfig(**kw), R.make_weights(R.BSRoformerConfig(**kw), seed=8), math=math)
    eng = rf.RoformerEngine(net, 801, 8.0, SR, batch_size=1)
    return lambda mix: eng.demix_device(mix)


def htdemucs_runner(math):
    import torch

    import demucs_oracle as D
    from audio_separator.separator.b200 import demucs as dm

    ocfg = D.HTConfig()
    nets = [dm.HTDemucsNet(dm.HTDemucsConfig(), D.make_weights(ocfg, seed=11 + i), device=torch.device("cuda", 0), math=math) for i in range(4)]
    bag = [[1.0 if s == m else 0.0 for s in range(4)] for m in range(4)]
    eng = dm.DemucsEngine(nets, bag_weights=bag, overlap=0.25, batch_size=4)
    rng = random.Random(0)
    offsets = [[rng.randint(0, SR // 2) for _ in range(2)] for _ in nets]
    return lambda mix: eng.demix_device(mix, offsets)


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--seconds", type=float, default=300.0)
    ap.add_argument("--workloads", default="bs_roformer,htdemucs_ft")
    args = ap.parse_args()

    import numpy as np
    import torch

    assert torch.cuda.is_available(), "bench_autocast.py needs a CUDA device"
    torch.cuda.set_device(0)
    info = gpu_info()
    N = int(args.seconds * SR)
    mix = torch.from_numpy(music(N, seed=21) * 0.5).cuda()
    makers = {"bs_roformer": roformer_runner, "htdemucs_ft": htdemucs_runner}
    for name in args.workloads.split(","):
        run = {m: makers[name](m) for m in (0, 1)}
        out = {}
        for m in (0, 1):  # warm-up: module loads, graph captures, packed weights
            out[m] = run[m](mix)
        torch.cuda.synchronize()
        ms = {0: [], 1: []}
        for _ in range(args.runs):
            for m in (0, 1):
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                out[m] = run[m](mix)
                e1.record()
                torch.cuda.synchronize()
                ms[m].append(e0.elapsed_time(e1))
        a, b = out[0].double(), out[1].double()
        snr = 10 * np.log10(float((a**2).sum()) / max(float(((b - a) ** 2).sum()), 1e-30))
        rtf = {m: [args.seconds / (t / 1000.0) for t in ms[m]] for m in (0, 1)}
        med = {m: float(np.median(rtf[m])) for m in (0, 1)}
        line = {"workload": name, "metric": "real-time factor (audio-sec/device-sec) @44.1kHz stereo", **info, "track_seconds": args.seconds, "runs": args.runs,
                "data": "synthetic (seeded)", "rtf_bf16x3": round(med[0], 3), "rtf_fp16": round(med[1], 3), "speedup": round(med[1] / med[0], 4),
                "spread_bf16x3": round(max(rtf[0]) / min(rtf[0]) - 1, 4), "spread_fp16": round(max(rtf[1]) / min(rtf[1]) - 1, 4),
                "rtf_runs_bf16x3": [round(v, 3) for v in rtf[0]], "rtf_runs_fp16": [round(v, 3) for v in rtf[1]],
                "fp16_vs_bf16x3": {"max_abs_diff": float((b - a).abs().max()), "snr_db": round(snr, 2)}}
        print(json.dumps(line), flush=True)
        del run, out, a, b
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
