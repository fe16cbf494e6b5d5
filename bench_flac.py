"""bench_flac.py -- time of the GPU FLAC writer on one H100.

  python bench_flac.py [--steps K] [--warmup W] [--seconds S]

Workload: a seeded S-second (default 5 min) stereo stem already on the device (bench_roformer.music: the oracle's programme generator), written
  * at 16 bits and at 24 bits through the pydub rule (int16 << 8, the default writer), i.e. CommonSeparator with input_bit_depth 16 / 24.
Two timings per bit depth:
  encode_ms      -- CUDA events around b200/flac.encode's device work (analysis, offsets and pack kernels) on the normalised stem, after W warm-up
                    encodes; the median of K;
  write_flac_ms  -- host clock around CommonSeparator.write_audio(".flac") end to end: normalisation, encode, the copy of the stream to the host and
                    the file write, alternated in the same loop with write_audio(".wav") (write_wav_ms: normalisation, PCM packing, download and the
                    stdlib WAV write); medians of K.
bytes / ratio_to_wav: the FLAC file against the WAV file of the same stem.  The card's name and power limit are read in the same call.
Writes only to a temporary directory.  Prints one JSON line.
"""
import argparse
import json
import logging
import os
import statistics
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(ROOT, "python-audio-separator_b200"))
sys.path.insert(0, os.path.join(ROOT, "oracle"))

from bench_roformer import SR, gpu_info, music  # noqa: E402


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--seconds", type=float, default=300.0)
    args = ap.parse_args()

    import numpy as np
    import torch

    from audio_separator.separator.b200 import flac
    from audio_separator.separator.common_separator import CommonSeparator

    if not torch.cuda.is_available():
        sys.exit("bench_flac.py needs a CUDA device")
    torch.cuda.set_device(0)
    n = int(args.seconds * SR)
    stem = torch.as_tensor(np.ascontiguousarray(music(n, seed=11).T)).cuda()
    out = {"workload": f"{args.seconds:g}-s stereo stem at {SR} Hz on the device", "samples": n, "steps": args.steps, "warmup": args.warmup}
    out.update(gpu_info(0))
    with tempfile.TemporaryDirectory(prefix="bench-flac-") as tmp:
        for bits in (16, 24):
            cs = CommonSeparator(dict(logger=logging.getLogger("bench_flac"), model_name="m", model_path="/x/m.onnx", model_data={"primary_stem": "Vocals"},
                                      output_dir=tmp, output_format="FLAC", normalization_threshold=0.9, amplification_threshold=0.0, sample_rate=SR,
                                      use_soundfile=False))
            cs.input_bit_depth = bits
            norm = cs._normalized_on_device(stem)
            bps = flac.stream_bps(bits, False)
            for _ in range(args.warmup):
                flac.encode(norm, bits, True, bps, SR)
            times = []
            for _ in range(args.steps):
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                n_bytes = int(lib_encode_only(flac, norm, bits, bps, e0, e1))
                times.append(e0.elapsed_time(e1))
            flac_ms, wav_ms = [], []
            for _ in range(args.warmup):
                cs.write_audio("b.flac", stem)
                cs.write_audio("b.wav", stem)
            for _ in range(args.steps):
                for name, acc in (("b.flac", flac_ms), ("b.wav", wav_ms)):
                    torch.cuda.synchronize()
                    t0 = time.perf_counter()
                    cs.write_audio(name, stem)
                    acc.append(1e3 * (time.perf_counter() - t0))
            fb, wb = os.path.getsize(os.path.join(tmp, "b.flac")), os.path.getsize(os.path.join(tmp, "b.wav"))
            assert fb == n_bytes + 42
            out[f"bits{bits}"] = {"stream_bps": bps, "encode_ms": round(statistics.median(times), 3), "encode_ms_min": round(min(times), 3),
                                  "write_flac_ms": round(statistics.median(flac_ms), 2), "write_wav_ms": round(statistics.median(wav_ms), 2),
                                  "flac_bytes": fb, "wav_bytes": wb, "ratio_to_wav": round(fb / wb, 4)}
    print(json.dumps(out), flush=True)


def lib_encode_only(flac, norm, bits, bps, e0, e1):
    """The device part of flac.encode between two CUDA events; returns the stream's frame bytes."""
    import torch

    from audio_separator.separator.b200._lib import check, lib

    n = int(norm.shape[0])
    st = torch.cuda.current_stream()
    work = torch.empty(lib.b200sep_flac_work_bytes(n), dtype=torch.uint8, device="cuda")
    buf = torch.empty(lib.b200sep_flac_max_bytes(n, bps), dtype=torch.uint8, device="cuda")
    result = torch.empty(4, dtype=torch.int64, device="cuda")
    e0.record(st)
    check(lib.b200sep_flac_encode(norm.data_ptr(), n, bits, 1, bps, SR, work.data_ptr(), buf.data_ptr(), result.data_ptr(), st.cuda_stream), "flac_encode")
    e1.record(st)
    e1.synchronize()
    total, _, _, bad = result.tolist()
    assert bad == 0
    return total


if __name__ == "__main__":
    main()
