"""Pin oracle/flac_oracle.py against real encoders and write tests/golden/flac_frames.npz.

Decodes three whole FLAC files of the reference's test inputs -- the libFLAC 1.4.2 `mardy20s.flac` (16-bit, block 4096) and the ffmpeg (pydub)
outputs `ref_clocks_piano_bass_htdemucs_ft.flac` (16-bit) and `ref_levee_drums_vocals.flac` (24-bit, block 4608) -- and asserts that
  * the MD5 of the decoded samples equals each file's STREAMINFO MD5;
  * the 24-bit pydub file's samples are all multiples of 256 (ffmpeg stored int16 << 8: the writer rule of b200/flac.py).
The fixture keeps, per file, the STREAMINFO, the raw bytes of the first frames (under 0.5 s of audio), their decoded samples and the byte count of
those frames: the real encoder's size for those samples, which the GPU encoder's output is compared with.

    python oracle/make_golden_flac.py            (needs the reference tree; B200SEP_REFERENCE_ROOT overrides its location)
"""
import os
import sys
import time

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import flac_oracle as F  # noqa: E402
from ref_shim import REF_ROOT  # noqa: E402

GOLD = os.path.join(os.path.dirname(HERE), "tests", "golden", "flac_frames.npz")
FILES = {
    "libflac16": "tests/inputs/mardy20s.flac",
    "ffmpeg16": "tests/inputs/reference/ref_clocks_piano_bass_htdemucs_ft.flac",
    "ffmpeg24": "tests/inputs/reference/ref_levee_drums_vocals.flac",
}
MAX_SECONDS = 0.5


def present() -> bool:
    return all(os.path.exists(os.path.join(REF_ROOT, p)) for p in FILES.values())


def build(out_path=GOLD, verbose=True):
    out = {}
    for tag, rel in FILES.items():
        data = open(os.path.join(REF_ROOT, rel), "rb").read()
        t0 = time.perf_counter()
        d = F.decode(data)
        info = d.streaminfo
        assert d.samples.shape == (info["total_samples"], info["channels"]), (tag, d.samples.shape)
        assert F.pcm_md5(d.samples, info["bps"]) == info["md5"], f"{tag}: decoded samples do not match the STREAMINFO MD5"
        if tag == "ffmpeg24":
            assert info["bps"] == 24 and np.all(d.samples % 256 == 0), "24-bit pydub output should hold int16 << 8"
        keep, n = 0, 0
        while keep < len(d.frames) and n + d.frames[keep][2] <= MAX_SECONDS * info["sample_rate"]:
            n += d.frames[keep][2]
            keep += 1
        first, last = d.frames[0], d.frames[keep - 1]
        si_pos = data.index(b"fLaC") + 8  # the first metadata block is STREAMINFO
        out[f"{tag}_streaminfo"] = np.frombuffer(data[si_pos:si_pos + 34], np.uint8)
        out[f"{tag}_frames"] = np.frombuffer(data[first[0]:last[0] + last[1]], np.uint8)
        out[f"{tag}_samples"] = d.samples[:n].astype(np.int32)
        out[f"{tag}_encoder_bytes"] = np.int64(last[0] + last[1] - first[0])
        if verbose:
            print(f"{tag}: {info['total_samples']} samples x {info['channels']} at {info['bps']} bits, block {info['max_block']}, MD5 ok, "
                  f"seen {sorted(d.seen)}; kept {keep} frames = {n} samples in {int(out[f'{tag}_encoder_bytes'])} bytes "
                  f"({time.perf_counter() - t0:.1f} s)", flush=True)
    np.savez_compressed(out_path, **out)
    return out


if __name__ == "__main__":
    if not present():
        sys.exit(f"reference inputs not found under {REF_ROOT}")
    build()
    print("wrote", GOLD)
