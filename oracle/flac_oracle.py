"""FLAC decoder written from RFC 9639: the checker of the GPU FLAC encoder (csrc/flac.cu, b200/flac.py).

TEST INFRASTRUCTURE -- never imported by the product path.  Pure Python + numpy, meant for correctness, not speed (a 10-s stereo stream decodes in
a few seconds).  It handles the STREAMINFO block, frame headers with CRC-8, CONSTANT / VERBATIM / FIXED / LPC subframes, wasted bits, RICE and
RICE2 residuals with escape partitions, the four stereo channel assignments and the frame CRC-16, and reports which of these it met.
"""
import hashlib
from dataclasses import dataclass, field

import numpy as np


class FlacError(ValueError):
    pass


class CRCError(FlacError):
    pass


def _crc_table(poly, width):
    top, mask = 1 << (width - 1), (1 << width) - 1
    tab = []
    for i in range(256):
        c = i << (width - 8)
        for _ in range(8):
            c = ((c << 1) ^ poly) if c & top else (c << 1)
        tab.append(c & mask)
    return tab


_CRC8 = _crc_table(0x07, 8)
_CRC16 = _crc_table(0x8005, 16)


def crc8(data: bytes) -> int:
    c = 0
    for b in data:
        c = _CRC8[c ^ b]
    return c


def crc16(data: bytes) -> int:
    c = 0
    for b in data:
        c = ((c << 8) & 0xFFFF) ^ _CRC16[(c >> 8) ^ b]
    return c


class BitReader:
    def __init__(self, buf: bytes, byte_pos: int = 0):
        self.buf, self.p, self.end = buf, byte_pos * 8, len(buf) * 8

    def u(self, n: int) -> int:
        if n == 0:
            return 0
        p = self.p
        if p + n > self.end:
            raise FlacError("read past the end of the stream")
        b = p >> 3
        w = int.from_bytes(self.buf[b:b + 8].ljust(8, b"\0"), "big")
        self.p = p + n
        return (w >> (64 - (p & 7) - n)) & ((1 << n) - 1)

    def s(self, n: int) -> int:
        v = self.u(n)
        return v - (1 << n) if n and v >> (n - 1) else v

    def unary(self) -> int:
        zeros = 0
        while True:
            p = self.p
            if p >= self.end:
                raise FlacError("unterminated unary code")
            b = p >> 3
            avail = 64 - (p & 7)
            w = int.from_bytes(self.buf[b:b + 8].ljust(8, b"\0"), "big") & ((1 << avail) - 1)
            if w:
                z = avail - w.bit_length()
                self.p = p + z + 1
                if self.p > self.end:
                    raise FlacError("unterminated unary code")
                return zeros + z
            zeros += avail
            self.p = p + avail

    def align(self):
        self.p = (self.p + 7) & ~7


FIXED_COEFS = ([], [1], [2, -1], [3, -3, 1], [4, -6, 4, -1])
ASSIGNMENTS = {8: "left/side", 9: "right/side", 10: "mid/side"}
BPS_CODES = {1: 8, 2: 12, 4: 16, 5: 20, 6: 24, 7: 32}
RATE_CODES = {1: 88200, 2: 176400, 3: 192000, 4: 8000, 5: 16000, 6: 22050, 7: 24000, 8: 32000, 9: 44100, 10: 48000, 11: 96000}


def parse_streaminfo(body: bytes) -> dict:
    if len(body) != 34:
        raise FlacError(f"STREAMINFO is 34 bytes, got {len(body)}")
    x = int.from_bytes(body[10:18], "big")
    return dict(min_block=int.from_bytes(body[0:2], "big"), max_block=int.from_bytes(body[2:4], "big"), min_frame=int.from_bytes(body[4:7], "big"),
                max_frame=int.from_bytes(body[7:10], "big"), sample_rate=x >> 44, channels=((x >> 41) & 7) + 1, bps=((x >> 36) & 31) + 1,
                total_samples=x & ((1 << 36) - 1), md5=body[18:34])


@dataclass
class Decoded:
    streaminfo: dict
    samples: np.ndarray  # (N, channels) int64
    frames: list = field(default_factory=list)  # (byte offset, byte length, block size) per frame
    seen: set = field(default_factory=set)  # subframe types, "wasted", "escape", "RICE", "RICE2", channel assignments


def _residual(r: BitReader, bs: int, order: int, seen: set) -> list:
    method = r.u(2)
    if method > 1:
        raise FlacError(f"reserved residual coding method {method}")
    seen.add("RICE2" if method else "RICE")
    pbits = 5 if method else 4
    esc = (1 << pbits) - 1
    po = r.u(4)
    if bs % (1 << po) or (bs >> po) < order:
        raise FlacError(f"partition order {po} does not fit block size {bs} / predictor order {order}")
    out = []
    for p in range(1 << po):
        n = (bs >> po) - (order if p == 0 else 0)
        k = r.u(pbits)
        if k == esc:
            seen.add("escape")
            w = r.u(5)
            out.extend(r.s(w) if w else 0 for _ in range(n))
        else:
            for _ in range(n):
                v = (r.unary() << k) | r.u(k)
                out.append((v >> 1) ^ -(v & 1))
    return out


def _predict(warm: list, res: list, coefs: list, shift: int) -> list:
    x = list(warm)
    order = len(coefs)
    for e in res:
        acc = 0
        for j in range(order):
            acc += coefs[j] * x[-1 - j]
        x.append(e + (acc >> shift))
    return x


def _subframe(r: BitReader, bs: int, bps: int, seen: set) -> np.ndarray:
    if r.u(1):
        raise FlacError("subframe padding bit set")
    t = r.u(6)
    wasted = 0
    if r.u(1):
        wasted = r.unary() + 1
        seen.add("wasted")
    bps -= wasted
    if bps < 1:
        raise FlacError("more wasted bits than sample bits")
    if t == 0:
        seen.add("CONSTANT")
        x = [r.s(bps)] * bs
    elif t == 1:
        seen.add("VERBATIM")
        x = [r.s(bps) for _ in range(bs)]
    elif 8 <= t <= 12:
        seen.add("FIXED")
        order = t - 8
        if order > bs:
            raise FlacError("predictor order above block size")
        warm = [r.s(bps) for _ in range(order)]
        x = _predict(warm, _residual(r, bs, order, seen), FIXED_COEFS[order], 0)
    elif t >= 32:
        seen.add("LPC")
        order = t - 31
        if order > bs:
            raise FlacError("predictor order above block size")
        warm = [r.s(bps) for _ in range(order)]
        prec = r.u(4) + 1
        if prec == 16:
            raise FlacError("invalid LPC precision")
        shift = r.s(5)
        if shift < 0:
            raise FlacError("negative LPC shift")
        coefs = [r.s(prec) for _ in range(order)]
        x = _predict(warm, _residual(r, bs, order, seen), coefs, shift)
    else:
        raise FlacError(f"reserved subframe type {t}")
    return np.asarray(x, dtype=np.int64) << wasted


def _frame(buf: bytes, pos: int, info: dict, expect_number: int, seen: set):
    r = BitReader(buf, pos)
    if r.u(15) != 0x7FFC:
        raise FlacError(f"no frame sync at byte {pos}")
    if r.u(1):
        raise FlacError("variable block size streams are not produced by this encoder")
    bs_code, sr_code, ca, ss_code = r.u(4), r.u(4), r.u(4), r.u(3)
    if r.u(1):
        raise FlacError("reserved header bit set")
    first = r.u(8)  # frame number, UTF-8 style
    n_more = 0
    while n_more < 6 and (first << n_more) & 0x80:
        n_more += 1
    if n_more == 1 or n_more > 6:
        raise FlacError("invalid coded frame number")
    number = first & (0x7F >> n_more) if n_more else first
    for _ in range(max(0, n_more - 1)):
        c = r.u(8)
        if c >> 6 != 2:
            raise FlacError("invalid coded frame number")
        number = (number << 6) | (c & 0x3F)
    if bs_code == 0:
        raise FlacError("reserved block size code")
    bs = {1: 192, 6: None, 7: None}.get(bs_code)
    if bs_code == 6:
        bs = r.u(8) + 1
    elif bs_code == 7:
        bs = r.u(16) + 1
    elif 2 <= bs_code <= 5:
        bs = 576 << (bs_code - 2)
    elif bs_code >= 8:
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
        rate = RATE_CODES.get(sr_code, info["sample_rate"])
    bps = BPS_CODES.get(ss_code, info["bps"]) if ss_code else info["bps"]
    if ss_code == 3:
        raise FlacError("reserved sample size code")
    hdr_end = r.p >> 3
    if r.u(8) != crc8(buf[pos:hdr_end]):
        raise CRCError(f"frame {expect_number}: header CRC-8 mismatch")
    if number != expect_number:
        raise FlacError(f"frame number {number}, expected {expect_number}")
    if rate != info["sample_rate"] or bps != info["bps"]:
        raise FlacError("frame header disagrees with STREAMINFO")
    nch = info["channels"]
    if ca < 8:
        if ca + 1 != nch:
            raise FlacError("channel count disagrees with STREAMINFO")
        chans = [_subframe(r, bs, bps, seen) for _ in range(nch)]
        seen.add("independent")
    elif ca <= 10:
        if nch != 2:
            raise FlacError("stereo decorrelation in a non-stereo stream")
        a = _subframe(r, bs, bps + (ca == 9), seen)
        b = _subframe(r, bs, bps + (ca != 9), seen)
        if ca == 8:
            chans = [a, a - b]
        elif ca == 9:
            chans = [a + b, b]
        else:
            mid = (a << 1) | (b & 1)
            chans = [(mid + b) >> 1, (mid - b) >> 1]
        seen.add(ASSIGNMENTS[ca])
    else:
        raise FlacError(f"reserved channel assignment {ca}")
    r.align()
    body_end = r.p >> 3
    if r.u(16) != crc16(buf[pos:body_end]):
        raise CRCError(f"frame {expect_number}: CRC-16 mismatch")
    return np.stack(chans, 1), r.p >> 3


def decode(data: bytes, max_frames=None) -> Decoded:
    """Decode a whole FLAC stream (or its first max_frames frames).  Raises CRCError on a CRC mismatch, FlacError on anything malformed."""
    if data[:4] != b"fLaC":
        raise FlacError("no fLaC marker")
    p, info = 4, None
    while True:
        if p + 4 > len(data):
            raise FlacError("truncated metadata")
        h = data[p]
        length = int.from_bytes(data[p + 1:p + 4], "big")
        if h & 0x7F == 0:
            info = parse_streaminfo(data[p + 4:p + 4 + length])
        p += 4 + length
        if h & 0x80:
            break
    if info is None:
        raise FlacError("no STREAMINFO")
    out = Decoded(info, np.zeros((0, info["channels"]), np.int64))
    blocks = []
    while p < len(data) and (max_frames is None or len(blocks) < max_frames):
        x, end = _frame(data, p, info, len(blocks), out.seen)
        out.frames.append((p, end - p, x.shape[0]))
        blocks.append(x)
        p = end
    if blocks:
        out.samples = np.concatenate(blocks)
    return out


def decode_frames(streaminfo_body: bytes, frames: bytes) -> Decoded:
    """Decode raw frame bytes given the STREAMINFO they belong to (the golden fixtures store only the first frames of a file)."""
    return decode(b"fLaC" + bytes([0x80]) + len(streaminfo_body).to_bytes(3, "big") + streaminfo_body + frames)


def pcm_md5(samples: np.ndarray, bps: int) -> bytes:
    """MD5 of the interleaved little-endian PCM at ceil(bps / 8) bytes per sample: what STREAMINFO's MD5 covers."""
    width = (bps + 7) // 8
    raw = samples.astype("<i8").view(np.uint8).reshape(-1, 8)[:, :width]
    return hashlib.md5(raw.tobytes()).digest()
