"""Time the GPU FLAC decoder on a seeded 5-minute stereo track encoded by the GPU encoder at 16 and at 24 bits.

    python bench_flac_decode.py [--steps K] [--warmup W] [--seconds S]

Prints one JSON line: per bit depth, decode_ms (CUDA events around b200sep_flac_locate + b200sep_flac_decode, from the compressed bytes in HBM to
the float mix; median of K steps after W warm-ups) with its split into the two calls, prepare_mix_flac_ms against prepare_mix_wav_ms (host clock
around CommonSeparator.prepare_mix of the same samples as .flac and as .wav, ending in a device sync), the bytes uploaded, and the card's name,
power limit and max SM clock.  Nothing is written outside a temporary directory.
"""
import argparse
import json
import logging
import os
import subprocess
import sys
import tempfile
import time
import wave

import numpy as np
import torch

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(ROOT, "python-audio-separator_b200"))
SR = 44100


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"], capture_output=True,
                           text=True, timeout=30).stdout.strip()
        name, power, clock = [s.strip() for s in q.split(",")]
        return dict(name=name, power_limit=power, max_sm_clock=clock)
    except Exception as e:  # noqa: BLE001
        return dict(name=torch.cuda.get_device_name(0), error=str(e))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--seconds", type=float, default=300.0)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "bench_flac_decode.py needs a CUDA device"
    from audio_separator.separator.b200 import flac
    from audio_separator.separator.b200._lib import check, lib
    from audio_separator.separator.common_separator import CommonSeparator

    n = int(a.seconds * SR)
    rng = np.random.default_rng(0)
    x = np.cumsum(rng.standard_normal((n, 2)), axis=0)
    x = np.ascontiguousarray(0.8 * x / np.abs(x).max(), dtype=np.float32)
    xd = torch.as_tensor(x).cuda()
    stream = torch.cuda.current_stream().cuda_stream
    report = dict(card=card(), seconds=a.seconds, steps=a.steps, warmup=a.warmup)
    with tempfile.TemporaryDirectory() as tmp:
        for bits in (16, 24):
            data = flac.encode(xd, bits, True, bits, SR)
            info, begin, end = flac.parse(data)
            nb = end - begin
            host = torch.empty((nb + 15) // 16 * 16, dtype=torch.uint8, pin_memory=True)
            host.numpy()[:nb] = np.frombuffer(data, np.uint8, nb, begin)
            buf = host.cuda()
            work = torch.empty(lib.b200sep_flac_decode_work_bytes(nb), dtype=torch.uint8, device="cuda")
            result = torch.empty(8, dtype=torch.int64, device="cuda")
            ev = [torch.cuda.Event(enable_timing=True) for _ in range(3)]
            locate_ms, decode_ms, total_ms = [], [], []
            out = None
            for step in range(a.warmup + a.steps):
                ev[0].record()
                check(lib.b200sep_flac_locate(buf.data_ptr(), nb, SR, bits, 2, 0, work.data_ptr(), result.data_ptr(), stream), "flac_locate")
                ev[1].record()
                r = result.tolist()  # the one host read between the calls
                assert r[2] == 0, r
                if out is None:
                    out = torch.empty((2, r[1]), dtype=torch.float32, device="cuda")
                check(lib.b200sep_flac_decode(buf.data_ptr(), nb, work.data_ptr(), r[0], r[5], out.data_ptr(), r[1], result.data_ptr(), stream), "flac_decode")
                ev[2].record()
                torch.cuda.synchronize()
                if step >= a.warmup:
                    locate_ms.append(ev[0].elapsed_time(ev[1]))
                    decode_ms.append(ev[1].elapsed_time(ev[2]))
                    total_ms.append(ev[0].elapsed_time(ev[2]))
            ints = (out.cpu().numpy().T.astype(np.float64) * (1 << (bits - 1))).astype(np.int64)
            width = bits // 8
            fpath, wpath = os.path.join(tmp, f"t{bits}.flac"), os.path.join(tmp, f"t{bits}.wav")
            with open(fpath, "wb") as f:
                f.write(data)
            raw = np.ascontiguousarray(ints, dtype="<i4").view(np.uint8).reshape(-1, 4)[:, :width]
            with wave.open(wpath, "wb") as wf:
                wf.setnchannels(2); wf.setsampwidth(width); wf.setframerate(SR); wf.writeframes(raw.tobytes())
            cs = CommonSeparator(dict(logger=logging.getLogger("bench"), sample_rate=SR, torch_device=torch.device("cuda", 0)))
            times = {}
            for kind, path in (("flac", fpath), ("wav", wpath)):
                t = []
                for step in range(a.warmup + a.steps):
                    t0 = time.perf_counter()
                    m = cs.prepare_mix(path)
                    if kind == "wav":
                        m = torch.from_numpy(np.ascontiguousarray(m)).cuda()  # what the MDX plugin uploads
                    else:
                        m = m.tensor
                    torch.cuda.synchronize()
                    if step >= a.warmup:
                        t.append(1e3 * (time.perf_counter() - t0))
                times[kind] = float(np.median(t))
                last = m
            fm = cs.prepare_mix(fpath).tensor
            same = bool(torch.equal(fm, last))
            report[f"bits{bits}"] = dict(decode_ms=float(np.median(total_ms)), locate_ms=float(np.median(locate_ms)), decode_call_ms=float(np.median(decode_ms)),
                                         prepare_mix_flac_ms=times["flac"], prepare_mix_wav_ms=times["wav"], flac_equals_wav=same, bytes_uploaded=nb,
                                         wav_bytes=n * 2 * width, frames=r[0], samples=r[1])
    print(json.dumps(report))


if __name__ == "__main__":
    main()
