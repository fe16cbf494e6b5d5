"""FLAC stream decoder for the GPU decoder's tests: oracle/flac_oracle.py extended to every frame layout a FLAC reader meets.

TEST INFRASTRUCTURE -- never imported by the product path.  flac_oracle.py checks the GPU encoder, whose streams always use fixed blocking and
number their frames from 0.  A reader also meets variable-blocking streams (the header codes a sample number of up to 36 bits) and excerpts cut
from a longer stream, whose first frame or sample number is not zero.  This module parses those frame headers and reuses flac_oracle's bit
reader, subframe decoder (CONSTANT / VERBATIM / FIXED / LPC, wasted bits, RICE / RICE2, escapes) and CRCs.  A stream flac_oracle accepts decodes
here to the same samples.
"""
import numpy as np

import flac_oracle as F
from flac_oracle import BitReader, CRCError, Decoded, FlacError, crc8, crc16


def _frame(buf: bytes, pos: int, info: dict, expect_number, seen: set):
    """One frame at byte `pos`; expect_number None accepts any number (the first frame of an excerpt).  Returns (samples, end, number)."""
    r = BitReader(buf, pos)
    if r.u(15) != 0x7FFC:
        raise FlacError(f"no frame sync at byte {pos}")
    variable = r.u(1)
    if info.setdefault("variable", variable) != variable:
        raise FlacError("blocking strategy changes within the stream")
    bs_code, sr_code, ca, ss_code = r.u(4), r.u(4), r.u(4), r.u(3)
    if r.u(1):
        raise FlacError("reserved header bit set")
    first = r.u(8)  # frame number (fixed blocking) or sample number (variable blocking), UTF-8 style
    n_more = 0
    while n_more < 7 and (first << n_more) & 0x80:
        n_more += 1
    if n_more == 1 or n_more > (7 if variable else 6):
        raise FlacError("invalid coded frame number")
    number = first & (0x7F >> n_more) if n_more else first
    for _ in range(max(0, n_more - 1)):
        c = r.u(8)
        if c >> 6 != 2:
            raise FlacError("invalid coded frame number")
        number = (number << 6) | (c & 0x3F)
    if bs_code == 0:
        raise FlacError("reserved block size code")
    if bs_code == 1:
        bs = 192
    elif bs_code == 6:
        bs = r.u(8) + 1
    elif bs_code == 7:
        bs = r.u(16) + 1
    elif bs_code <= 5:
        bs = 576 << (bs_code - 2)
    else:
        bs = 256 << (bs_code - 8)
    if sr_code == 12:
        rate = r.u(8) * 1000
    elif sr_code == 13:
        rate = r.u(16)
    elif sr_code == 14:
        rate = r.u(16) * 10
    elif sr_code == 15:
        raise FlacError("invalid sample rate code")
    else:
        rate = F.RATE_CODES.get(sr_code, info["sample_rate"])
    if ss_code == 3:
        raise FlacError("reserved sample size code")
    bps = F.BPS_CODES.get(ss_code, info["bps"]) if ss_code else info["bps"]
    hdr_end = r.p >> 3
    if r.u(8) != crc8(buf[pos:hdr_end]):
        raise CRCError(f"frame at byte {pos}: header CRC-8 mismatch")
    if expect_number is not None and number != expect_number:
        raise FlacError(f"{'sample' if variable else 'frame'} number {number}, expected {expect_number}")
    if rate != info["sample_rate"] or bps != info["bps"]:
        raise FlacError("frame header disagrees with STREAMINFO")
    nch = info["channels"]
    if ca < 8:
        if ca + 1 != nch:
            raise FlacError("channel count disagrees with STREAMINFO")
        chans = [F._subframe(r, bs, bps, seen) for _ in range(nch)]
        seen.add("independent")
    elif ca <= 10:
        if nch != 2:
            raise FlacError("stereo decorrelation in a non-stereo stream")
        a = F._subframe(r, bs, bps + (ca == 9), seen)
        b = F._subframe(r, bs, bps + (ca != 9), seen)
        if ca == 8:
            chans = [a, a - b]
        elif ca == 9:
            chans = [a + b, b]
        else:
            mid = (a << 1) | (b & 1)
            chans = [(mid + b) >> 1, (mid - b) >> 1]
        seen.add(F.ASSIGNMENTS[ca])
    else:
        raise FlacError(f"reserved channel assignment {ca}")
    r.align()
    body_end = r.p >> 3
    if r.u(16) != crc16(buf[pos:body_end]):
        raise CRCError(f"frame at byte {pos}: CRC-16 mismatch")
    seen.add("variable" if variable else "fixed")
    return np.stack(chans, 1), r.p >> 3, number


def decode(data: bytes, max_frames=None, first_anywhere=False) -> Decoded:
    """Decode a FLAC stream (from `fLaC` to its last frame), fixed or variable blocking.  The frames are numbered from 0, or from any number when
    first_anywhere (an excerpt of a longer stream), and then on consecutively (fixed blocking) or by the running sample count (variable
    blocking); streaminfo["first_number"] is the first frame's number.  Raises CRCError on a CRC mismatch, FlacError on anything malformed."""
    if data[:4] != b"fLaC":
        raise FlacError("no fLaC marker")
    p, info = 4, None
    while True:
        if p + 4 > len(data):
            raise FlacError("truncated metadata")
        h = data[p]
        length = int.from_bytes(data[p + 1:p + 4], "big")
        if h & 0x7F == 0:
            info = F.parse_streaminfo(data[p + 4:p + 4 + length])
        p += 4 + length
        if h & 0x80:
            break
    if info is None:
        raise FlacError("no STREAMINFO")
    out = Decoded(info, np.zeros((0, info["channels"]), np.int64))
    blocks, expect, done = [], None if first_anywhere else 0, 0
    while p < len(data) and (max_frames is None or len(blocks) < max_frames):
        x, end, number = _frame(data, p, info, expect, out.seen)
        if not blocks:
            info["first_number"] = number
        done += x.shape[0]
        expect = info["first_number"] + (done if info["variable"] else len(blocks) + 1)
        out.frames.append((p, end - p, x.shape[0]))
        blocks.append(x)
        p = end
    if blocks:
        out.samples = np.concatenate(blocks)
    return out


def decode_frames(streaminfo_body: bytes, frames: bytes, first_anywhere=False) -> Decoded:
    """Decode raw frame bytes given the STREAMINFO they belong to (the golden fixtures store only some frames of a file)."""
    return decode(b"fLaC" + bytes([0x80]) + len(streaminfo_body).to_bytes(3, "big") + streaminfo_body + frames, first_anywhere=first_anywhere)
