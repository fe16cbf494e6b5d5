"""Write tests/golden/flac_decode.npz: excerpts of real FLAC files for the GPU decoder, decoded by oracle/flac_stream_oracle.py.

Each excerpt keeps the file's STREAMINFO, the raw bytes of whole frames (under 0.5 s of audio) and the oracle's samples for them:
  * clocks      the first frames of tests/inputs/clocks_piano.flac (ffmpeg, block 4608, right/side and mid/side);
  * levee       the first frames of tests/inputs/levee_drums.flac (24-bit, RICE2);
  * mardy_mid   frames from the middle of tests/inputs/mardy20s.flac (libFLAC 1.4.2, block 4096): the first frame number is not zero;
    these three are pinned by the MD5 of their whole file: the oracle decodes the whole file and its samples must match the STREAMINFO MD5;
  * fallen      the first frames of tests/inputs/fallen24bit20s.flac (24-bit, 96 kHz), an excerpt cut from a longer stream: its first frame is
    number 703 and its STREAMINFO (total samples, MD5) belongs to the original stream, so this excerpt is pinned by its frame CRCs only.

    python oracle/make_golden_flac_decode.py     (needs the reference tree; B200SEP_REFERENCE_ROOT overrides its location)
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import flac_oracle as F  # noqa: E402
import flac_stream_oracle as S  # noqa: E402
from ref_shim import REF_ROOT  # noqa: E402

GOLD = os.path.join(os.path.dirname(HERE), "tests", "golden", "flac_decode.npz")
# tag -> (file, first frame kept, pinned by the whole file's MD5)
FILES = {
    "clocks": ("tests/inputs/clocks_piano.flac", 0, True),
    "levee": ("tests/inputs/levee_drums.flac", 0, True),
    "mardy_mid": ("tests/inputs/mardy20s.flac", 100, True),
    "fallen": ("tests/inputs/fallen24bit20s.flac", 0, False),
}
MAX_SECONDS = 0.5


def present() -> bool:
    return all(os.path.exists(os.path.join(REF_ROOT, f)) for f, _, _ in FILES.values())


def build(out_path=GOLD, verbose=True):
    out = {}
    for tag, (rel, first, whole) in FILES.items():
        data = open(os.path.join(REF_ROOT, rel), "rb").read()
        d = S.decode(data, first_anywhere=not whole, max_frames=None if whole else 64)  # every CRC-8 / CRC-16 is checked
        info = d.streaminfo
        if whole:
            assert d.samples.shape == (info["total_samples"], info["channels"]), (tag, d.samples.shape)
            assert F.pcm_md5(d.samples, info["bps"]) == info["md5"], f"{tag}: decoded samples do not match the STREAMINFO MD5"
        keep, n = first, 0
        while keep < len(d.frames) and n + d.frames[keep][2] <= MAX_SECONDS * info["sample_rate"]:
            n += d.frames[keep][2]
            keep += 1
        s0 = sum(f[2] for f in d.frames[:first])
        a, b = d.frames[first], d.frames[keep - 1]
        si_pos = data.index(b"fLaC") + 8  # the first metadata block is STREAMINFO
        out[f"{tag}_streaminfo"] = np.frombuffer(data[si_pos:si_pos + 34], np.uint8)
        out[f"{tag}_frames"] = np.frombuffer(data[a[0]:b[0] + b[1]], np.uint8)
        out[f"{tag}_samples"] = d.samples[s0:s0 + n].astype(np.int32)
        if verbose:
            print(f"{tag}: {info['channels']} x {info['bps']} bits at {info['sample_rate']} Hz, frames {first}-{keep - 1} = {n} samples, "
                  f"{'MD5 ok' if whole else 'CRCs only'}, first number {info.get('first_number', 0)}, seen {sorted(d.seen)}", flush=True)
    np.savez_compressed(out_path, **out)
    return out


if __name__ == "__main__":
    if not present():
        sys.exit(f"reference inputs not found under {REF_ROOT}")
    build()
    print("wrote", GOLD)
