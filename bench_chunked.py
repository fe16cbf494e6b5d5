"""Benchmark of `Separator(chunk_duration=...)` against the same separation without chunking, end to end through the Separator facade.

  python bench_chunked.py [--minutes 60] [--chunk 600] [--models mdx,htdemucs_ft] [--repeats 2]

A seeded synthetic stereo track (44.1 kHz, 16-bit WAV, `--minutes` long) is separated by synthetic-weight models of the UVR-MDX-NET-Inst_HQ_3
geometry (MDX defaults: segment_size 256, overlap 0.25) and the htdemucs_ft geometry (bag of 4 HTDemucs, shifts 2, overlap 0.25), once with
`chunk_duration=--chunk` and once without, `--repeats` times, alternating which of the two goes first.  Before the timed runs each model
separates a 1-minute track once with 20-s chunks and once without, so module loads, first launches and allocator growth are not timed.  Prints one JSON line with the card's name and power limit (read in the same run) and, per run:
  * wall seconds (host clock around `separate`, which ends in file writes) and the real-time factor (track seconds per wall second);
  * peak device memory (torch.cuda.max_memory_allocated, reset before the run), or the out-of-memory error when the run does not fit;
  * the wall time split into decode (prepare_mix of the file), separation (the plugin's separate / separate_mix, less decode and stem output),
    stem output (CommonSeparator.write_stems: normalisation, packing and, without chunking, the file writes) and join + write (the rest:
    the chunked path's slicing, byte downloads, joining and file writes).
Every phase timer synchronises the device.  Model and audio files go to a temporary directory that is removed afterwards."""
import argparse
import gc
import json
import logging
import os
import shutil
import subprocess
import sys
import tempfile
import time
import wave

import numpy as np
import torch

ROOT = os.path.dirname(os.path.abspath(__file__))
for p in (os.path.join(ROOT, "python-audio-separator_b200"), os.path.join(ROOT, "oracle"), os.path.join(ROOT, "tests")):
    sys.path.insert(0, p)
SR = 44100


def card():
    name = torch.cuda.get_device_name()
    try:
        q = subprocess.run(["nvidia-smi", "-i", str(torch.cuda.current_device()), "--query-gpu=power.limit", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30)
        power = q.stdout.strip() or "unknown"
    except (OSError, subprocess.SubprocessError):
        power = "unknown"
    return name, power


def write_track(path, minutes):
    import mdx_oracle as O

    n = int(minutes * 60 * SR)
    base = (O.synth_music(30 * SR, seed=5).T * 32767 * 0.5).astype("<i2")  # a 30-s pattern tiled
    with wave.open(path, "wb") as wf:
        wf.setnchannels(2), wf.setsampwidth(2), wf.setframerate(SR)
        for start in range(0, n, base.shape[0]):
            wf.writeframes(base[: min(base.shape[0], n - start)].tobytes())
    return n


def write_models(d):
    import demucs_oracle as D
    import mdx_oracle as O
    from test_demucs_gpu import _write_package

    cfg = O.MDXConfig()
    np.savez(os.path.join(d, "Inst_HQ_3_geometry.npz"), **O.make_convtdfnet_weights(cfg, seed=11, out_gain=66.97557067871094))
    with open(os.path.join(d, "Inst_HQ_3_geometry.json"), "w") as f:
        json.dump({"compensate": cfg.compensate, "mdx_dim_f_set": cfg.dim_f, "mdx_dim_t_set": 8, "mdx_n_fft_scale_set": cfg.n_fft, "primary_stem": "Instrumental"}, f)
    ocfg = D.HTConfig()
    sigs = []
    for i in range(4):
        sig = f"ft{i:06d}"
        _write_package(os.path.join(d, f"{sig}.th"), ocfg, D.make_weights(ocfg, seed=11 + i))
        sigs.append(sig)
    with open(os.path.join(d, "htdemucs_ft_geometry.yaml"), "w") as f:
        f.write(f"models: {sigs!r}\nweights: [[1, 0, 0, 0], [0, 1, 0, 0], [0, 0, 1, 0], [0, 0, 0, 1]]\n")
    return {"mdx": ("Inst_HQ_3_geometry.npz", {}), "htdemucs_ft": ("htdemucs_ft_geometry.yaml", {"demucs_params": {"shifts": 2, "overlap": 0.25}})}


class PhaseTimer:
    """Accumulates synchronised wall time of the wrapped CommonSeparator methods."""

    def __init__(self):
        from audio_separator.separator.common_separator import CommonSeparator

        self.cls, self.t = CommonSeparator, {}
        self.orig = {k: getattr(CommonSeparator, k) for k in ("prepare_mix", "write_stems", "separate_mix")}

        def timed(key, fn, when=lambda obj, *a: True):
            def wrapper(obj, *a, **k):
                if not when(obj, *a):
                    return fn(obj, *a, **k)
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                try:
                    return fn(obj, *a, **k)
                finally:
                    torch.cuda.synchronize()
                    self.t[key] = self.t.get(key, 0.0) + time.perf_counter() - t0
            return wrapper

        CommonSeparator.prepare_mix = timed("decode", self.orig["prepare_mix"], lambda obj, mix, *a: isinstance(mix, str) and obj._mix_slice is None)
        CommonSeparator.write_stems = timed("stem_output", self.orig["write_stems"])
        CommonSeparator.separate_mix = timed("chunk_separate", self.orig["separate_mix"])

    def restore(self):
        for k, v in self.orig.items():
            setattr(self.cls, k, v)


def run(d, track, model, params, chunk, n):
    from audio_separator.separator import Separator

    out = tempfile.mkdtemp(dir=d, prefix="out_")
    sep = Separator(log_level=logging.WARNING, model_file_dir=d, output_dir=out, chunk_duration=chunk, **params)
    sep.load_model(model)
    timer = PhaseTimer()
    gc.collect()  # the previous run's model and buffers must not count towards this run's peak
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    res = {"chunk_duration": chunk}
    t0 = time.perf_counter()
    try:
        files = sep._separate_file(track)
        torch.cuda.synchronize()
        wall = time.perf_counter() - t0
        res.update(wall_s=round(wall, 3), rtf=round(n / SR / wall, 2), peak_mem_gib=round(torch.cuda.max_memory_allocated() / 2 ** 30, 3),
                   files=len(files), output_bytes=sum(os.path.getsize(os.path.join(out, f)) for f in os.listdir(out)))
        t = timer.t
        decode, stems = t.get("decode", 0.0), t.get("stem_output", 0.0)
        if chunk is None:
            sep_s, join = wall - decode - stems, 0.0
        else:
            sep_s = t.get("chunk_separate", 0.0) - stems
            join = wall - decode - sep_s - stems
        res["split_s"] = {"decode": round(decode, 3), "separation": round(sep_s, 3), "stem_output": round(stems, 3), "join_and_write": round(join, 3)}
    except torch.cuda.OutOfMemoryError as e:
        res.update(error="out of device memory", detail=str(e).splitlines()[0], peak_mem_gib=round(torch.cuda.max_memory_allocated() / 2 ** 30, 3))
    finally:
        timer.restore()
        sep.model_instance = None
        del sep
        gc.collect()
        shutil.rmtree(out, ignore_errors=True)
        torch.cuda.empty_cache()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--minutes", type=float, default=60.0)
    ap.add_argument("--chunk", type=float, default=600.0)
    ap.add_argument("--models", default="mdx,htdemucs_ft")
    ap.add_argument("--repeats", type=int, default=2)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_chunked.py measures on a CUDA device; none is visible")
    name, power = card()
    d = tempfile.mkdtemp(prefix="b200sep_bench_chunked_")
    try:
        track, warm = os.path.join(d, "track.wav"), os.path.join(d, "warm.wav")
        n = write_track(track, args.minutes)
        n_warm = write_track(warm, 1.0)
        models = write_models(d)
        results = {}
        for key in args.models.split(","):
            model, params = models[key]
            run(d, warm, model, params, 20.0, n_warm)
            run(d, warm, model, params, None, n_warm)
            runs = {"chunked": [], "unchunked": []}
            for r in range(args.repeats):
                order = [("chunked", args.chunk), ("unchunked", None)]
                for label, chunk in (order if r % 2 == 0 else order[::-1]):
                    runs[label].append(run(d, track, model, params, chunk, n))
                    print(key, label, json.dumps(runs[label][-1]), file=sys.stderr, flush=True)  # progress: a 60-minute run takes minutes
            results[key] = runs
        print(json.dumps({"card": name, "power_limit": power, "track_minutes": args.minutes, "results": results}))
    finally:
        shutil.rmtree(d, ignore_errors=True)


if __name__ == "__main__":
    main()
