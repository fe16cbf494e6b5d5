"""Time the band-limited resampler (b200sep_resample_sinc_f32) on a seeded 5-minute stereo track.

    python bench_resample.py [--steps K] [--warmup W] [--seconds S]

Prints one JSON line.  Per case (44.1 -> 32 kHz and 32 -> 44.1 kHz with soxr_hq, the VR model-rate conversions; the -3 / +3 semitone pitch
ratios with sinc_fastest, the MDXC pitch_shift path): kernel_ms (CUDA events around K launches after W warm-ups, mean per launch), the taps the
filter reaches per output, GFLOP/s at 4 FLOP per tap (the table interpolation's subtract and FMA, the multiply-accumulate), and GB/s of the
samples read and written once.  Both rates come from shapes, not from counters.  The card's name, power limit and max SM clock are read in the
same call.  Needs a CUDA device; writes nothing.
"""
import argparse
import json
import math
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(ROOT, "python-audio-separator_b200"))


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True,
                       timeout=30).stdout.strip()
    name, power, clock = [s.strip() for s in q.split(",")]
    return dict(name=name, power_limit=power, max_sm_clock=clock)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--seconds", type=float, default=300.0)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_resample.py needs a CUDA device")
    from audio_separator.separator.b200 import resample

    cases = [("44100->32000 soxr_hq", 44100, 32000, "soxr_hq"), ("32000->44100 soxr_hq", 32000, 44100, "soxr_hq"),
             ("pitch -3 semitones sinc_fastest", 44100, 44100 * 2 ** (-3 / 12), "sinc_fastest"),
             ("pitch +3 semitones sinc_fastest", 44100, 44100 * 2 ** (3 / 12), "sinc_fastest")]
    report = dict(card=card(), seconds=a.seconds, steps=a.steps, warmup=a.warmup, cases={})
    rng = np.random.default_rng(0)
    for name, orig, target, res_type in cases:
        n_in = int(a.seconds * orig)
        x = torch.from_numpy(rng.uniform(-0.7, 0.7, (2, n_in)).astype(np.float32)).cuda()
        for _ in range(a.warmup):
            y = resample.resample(x, orig, target, res_type)
        torch.cuda.synchronize()
        t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        t0.record()
        for _ in range(a.steps):
            y = resample.resample(x, orig, target, res_type)
        t1.record()
        torch.cuda.synchronize()
        ms = t0.elapsed_time(t1) / a.steps
        ratio = float(target) / orig
        n_zeros = resample.filter_design(res_type)[0]
        taps = 2 * n_zeros / min(1.0, ratio)  # input samples the filter reaches per output
        outputs = y.numel()
        report["cases"][name] = dict(kernel_ms=round(ms, 4), outputs=outputs, taps_per_output=round(taps, 1),
                                     gflops=round(4 * taps * outputs / (ms * 1e-3) / 1e9, 1),
                                     gbytes_per_s=round((x.numel() + outputs) * 4 / (ms * 1e-3) / 1e9, 1))
        assert math.isfinite(float(y.abs().max()))
    print(json.dumps(report))


if __name__ == "__main__":
    main()
