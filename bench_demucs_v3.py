"""Benchmark of the time-domain Demucs v3 path: the mdx_extra bag geometry end to end, the two resampling kernels, and parity against the oracle.

  python bench_demucs_v3.py [--minutes 5] [--reps 20]

Prints one JSON line:
  * the card's name and power limit, read in the same run;
  * real-time factor (track seconds per wall second) of a bag shaped like mdx_extra -- two time-domain Demucs (48 channels, depth 6) and two
    HDemucs (48 channels, depth 6, nfft 4096), four sources, seeded synthetic weights -- through DemucsEngine at the plugin defaults (shifts 2,
    overlap 0.25, each member's own 40-s segment, 4 segments per forward) on a synthetic stereo track;
  * CUDA-event time per launch of b200sep_demucs_upsample2_f32 / b200sep_demucs_downsample2_f32 at one full 40-s segment batch, the bytes each
    must move, and that over the time as a share of the 3.35 TB/s HBM3 data-sheet bandwidth (the bound of both: a few FLOP per byte);
  * the largest deviation of one Demucs member's forward from the oracle on a 10-s slice, relative to the output peak.
Nothing is written to the tree."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.abspath(__file__))
for p in (os.path.join(ROOT, "python-audio-separator_b200"), os.path.join(ROOT, "oracle")):
    sys.path.insert(0, p)

HBM_BYTES_PER_S = 3.35e12


def card():
    name = torch.cuda.get_device_name()
    try:
        q = subprocess.run(["nvidia-smi", "-i", str(torch.cuda.current_device()), "--query-gpu=power.limit", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30)
        power = q.stdout.strip() or "unknown"
    except (OSError, subprocess.SubprocessError):
        power = "unknown"
    return name, power


def event_ms(fn, reps):
    fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / reps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--minutes", type=float, default=5.0)
    ap.add_argument("--reps", type=int, default=20)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_demucs_v3.py measures on a CUDA device; none is visible")
    import demucs_v3_oracle as V
    import hdemucs_oracle as H
    import mdx_oracle as M
    from audio_separator.separator.b200 import demucs_v3 as dv
    from audio_separator.separator.b200 import hdemucs as hd
    from audio_separator.separator.b200._lib import check, lib
    from audio_separator.separator.b200.demucs import DemucsEngine
    from audio_separator.separator.b200.engine import _ptr, _stream

    name, power = card()
    out = {"bench": "demucs_v3", "card": name, "power_limit": power}

    # ---- the two kernels at one batch of 4 full 40-s segments
    cfg = dv.DemucsConfig(channels=48)
    B, L = 4, cfg.seg_len
    valid = cfg.valid_length(L)
    up, uw = dv.julius_taps(1, 2)
    down, dw = dv.julius_taps(2, 1)
    up_d = torch.from_numpy(up.astype(np.float32)).cuda()
    down_d = torch.from_numpy(down.astype(np.float32)).cuda()
    x = torch.randn((B, 2, L), device="cuda")
    y = torch.empty((B, 2, 2 * valid), device="cuda")
    stats = torch.empty((B, 2), device="cuda")
    work = torch.empty((lib.b200sep_meanstd_work_floats(B),), device="cuda")
    C = 8
    x2 = torch.randn((B, C, 2 * valid), device="cuda")
    o2 = torch.empty((B, C, L), device="cuda")
    t_up = event_ms(lambda: check(lib.b200sep_demucs_upsample2_f32(_ptr(x), B, L, valid, _ptr(up_d), uw, _ptr(stats), _ptr(y), _ptr(work), _stream()), "up"), args.reps)
    t_dn = event_ms(lambda: check(lib.b200sep_demucs_downsample2_f32(_ptr(x2), B, C, valid, L, _ptr(down_d), dw, _ptr(stats), _ptr(o2), _stream()), "down"), args.reps)
    up_bytes = 4 * (2 * B * 2 * L + B * 2 * 2 * valid)  # the input read twice (statistics, filter), the x2 output written once
    dn_bytes = 4 * (B * C * 2 * valid + B * C * L)
    for key, t, nb in (("upsample2", t_up, up_bytes), ("downsample2", t_dn, dn_bytes)):
        out[key] = {"shape": f"B={B} L={L} valid={valid}" + (f" channels={C}" if key == "downsample2" else ""), "ms": round(t, 4), "bytes": nb,
                    "GB_per_s": round(nb / t / 1e6, 1), "share_of_3.35TB_per_s": round(nb / t / 1e6 / (HBM_BYTES_PER_S / 1e9), 3)}

    # ---- parity of one Demucs member against the oracle on 10 s
    w = V.make_weights(V.V3Config(channels=48), seed=7)
    net = dv.DemucsNet(cfg, w)
    clip = M.synth_music(441000, seed=5)[None]
    got = net.forward(torch.from_numpy(clip).cuda()).cpu().numpy()
    ref = V.forward(w, V.V3Config(channels=48), clip)
    out["parity_10s_max_abs_over_peak"] = float(np.abs(got - ref).max() / np.abs(ref).max())
    del net

    # ---- the mdx_extra geometry end to end
    nets = [dv.DemucsNet(dv.DemucsConfig(channels=48), V.make_weights(V.V3Config(channels=48), seed=s)) for s in (11, 12)]
    nets += [hd.HDemucsNet(hd.HDemucsConfig(), H.make_weights(H.HDConfig(), seed=s)) for s in (13, 14)]
    n = int(args.minutes * 60 * 44100)
    mix = torch.from_numpy(M.synth_music(n, seed=3)).cuda()
    rng = np.random.default_rng(0)
    offs = [[int(v) for v in rng.integers(0, 22050, 2)] for _ in nets]
    eng = DemucsEngine(nets, bag_weights=[[1.0] * 4] * 4, overlap=0.25, batch_size=4)
    eng.demix_device(mix[:, : 44100 * 50].contiguous(), offs)  # warm-up: module loads, weight images, workspace sizes of every segment width
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    src = eng.demix_device(mix, offs)
    torch.cuda.synchronize()
    dt = time.perf_counter() - t0
    assert torch.isfinite(src).all()
    out["mdx_extra_geometry"] = {"track_s": round(n / 44100, 1), "wall_s": round(dt, 3), "rtf": round(n / 44100 / dt, 2), "shifts": 2, "overlap": 0.25,
                                 "segment_s": 40, "batch": 4}
    print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()
