"""Time the GPU PCM input path on a seeded 5-minute stereo track stored as 32-bit float WAV, 24-bit AIFF and 24-bit RF64, against the same track as
16-bit WAV through the host reader.

    python bench_pcm_input.py [--steps K] [--warmup W] [--launches L] [--seconds S]

Prints one JSON line: per file, prepare_mix_ms (host clock around CommonSeparator.prepare_mix, ending in a device sync; for the 16-bit WAV the
host mix is uploaded as the MDX plugin does; median of K steps after W warm-ups), kernel_ms (CUDA events around L back-to-back launches of
b200sep_pcm_decode_f32 on the payload in HBM, per launch) with the HBM bytes it moves per second, the bytes uploaded, and the card's name, power
limit and max SM clock read in the same run.  Files go to a temporary directory.
"""
import argparse
import json
import logging
import os
import sys
import tempfile
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(ROOT, "python-audio-separator_b200"))
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.dont_write_bytecode = True
SR = 44100


def main():
    from bench_flac_decode import card

    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--launches", type=int, default=100)
    ap.add_argument("--seconds", type=float, default=300.0)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "bench_pcm_input.py needs a CUDA device"
    import pcm_writer as W
    from audio_separator.separator.b200 import pcm_reader
    from audio_separator.separator.b200._lib import check, lib
    from audio_separator.separator.common_separator import CommonSeparator, DeviceStem

    n = int(a.seconds * SR)
    rng = np.random.default_rng(0)
    x = np.cumsum(rng.standard_normal((n, 2)), axis=0)
    x = 0.8 * x / np.abs(x).max()
    i16, i24 = np.round(x * 32767).astype(np.int64), np.round(x * 8388607).astype(np.int64)
    files = {
        "wav_float32": W.wav(W.payload(x.astype(np.float32), W.F32LE), 3, 2, SR, 8, 32),
        "aiff_24": W.aiff(W.payload(i24, W.S24BE), 2, SR, 24),
        "rf64_24": W.wav(W.payload(i24, W.S24LE), 1, 2, SR, 6, 24, rf64=True),
        "wav_16_host": W.wav(W.payload(i16, W.S16LE), 1, 2, SR, 4, 16),
    }
    report = dict(card=card(), seconds=a.seconds, steps=a.steps, warmup=a.warmup, launches=a.launches)
    cs = CommonSeparator(dict(logger=logging.getLogger("bench"), sample_rate=SR, torch_device=torch.device("cuda", 0)))
    stream = torch.cuda.current_stream().cuda_stream
    with tempfile.TemporaryDirectory() as tmp:
        for name, blob in files.items():
            path = os.path.join(tmp, name + (".aiff" if "aiff" in name else ".wav"))
            with open(path, "wb") as f:
                f.write(blob)
            t = []
            for step in range(a.warmup + a.steps):
                t0 = time.perf_counter()
                m = cs.prepare_mix(path)
                m = m.tensor if isinstance(m, DeviceStem) else torch.from_numpy(np.ascontiguousarray(m)).cuda()
                torch.cuda.synchronize()
                if step >= a.warmup:
                    t.append(1e3 * (time.perf_counter() - t0))
            row = dict(prepare_mix_ms=float(np.median(t)), file_bytes=len(blob), on_device=name != "wav_16_host")
            if name != "wav_16_host":
                info = pcm_reader.parse(blob)
                nb = info["n_frames"] * info["block_align"]
                host = np.zeros((nb + 15) // 16 * 16, np.uint8)
                host[:nb] = np.frombuffer(blob, np.uint8, nb, info["begin"])
                buf = torch.from_numpy(host).cuda()
                out = torch.empty((2, info["n_frames"]), dtype=torch.float32, device="cuda")
                args = (buf.data_ptr(), info["n_frames"], info["block_align"], 2, info["format"], 2, out.data_ptr(), info["n_frames"], stream)
                for _ in range(a.warmup):
                    check(lib.b200sep_pcm_decode_f32(*args), "pcm_decode_f32")
                ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
                ev[0].record()
                for _ in range(a.launches):
                    check(lib.b200sep_pcm_decode_f32(*args), "pcm_decode_f32")
                ev[1].record()
                torch.cuda.synchronize()
                ms = ev[0].elapsed_time(ev[1]) / a.launches
                moved = nb + out.numel() * 4
                row.update(kernel_ms=ms, kernel_hbm_gb_s=moved / ms / 1e6, bytes_uploaded=nb)
            report[name] = row
        report["aiff_24_equals_rf64_24"] = bool(torch.equal(cs.prepare_mix(os.path.join(tmp, "aiff_24.aiff")).tensor,
                                                            cs.prepare_mix(os.path.join(tmp, "rf64_24.wav")).tensor))
    print(json.dumps(report))


if __name__ == "__main__":
    main()
