"""Plain-Python writer of uncompressed PCM containers for the tests of b200/pcm_reader.py and csrc/pcm_decode.cu, and the numpy restatement of
the decoder's conversion table (libsndfile's sf_read_float with normalisation on).

Containers: RIFF/WAVE (PCM, IEEE float, WAVE_FORMAT_EXTENSIBLE with either sub-format), RF64 with ds64, streamed data sizes (0 and 0xFFFFFFFF),
extra, odd-length and unknown chunks; FORM/AIFF and AIFC (NONE, twos, sowt, fl32 / FL32, fl64 / FL64, raw ) with padded pstrings, SSND
offsets and block sizes, COMM before or after SSND, and sample rates written as exact 80-bit extended values.
"""
import struct
from fractions import Fraction

import numpy as np

U8, S8, S16LE, S16BE, S24LE, S24BE, S32LE, S32BE, F32LE, F32BE, F64LE, F64BE = range(12)
SAMPLE_BYTES = (1, 1, 2, 2, 3, 3, 4, 4, 4, 4, 8, 8)
NAMES = ("U8", "S8", "S16LE", "S16BE", "S24LE", "S24BE", "S32LE", "S32BE", "F32LE", "F32BE", "F64LE", "F64BE")
BIG_ENDIAN = {S16BE, S24BE, S32BE, F32BE, F64BE}
FLOATS = {F32LE, F32BE, F64LE, F64BE}
_GUID_TAIL = bytes.fromhex("000000001000800000aa00389b71")


# ---- samples -> payload bytes ---------------------------------------------------------------------------------------------------------

def payload(x, fmt, frame_bytes=None, pad=0xA5):
    """(N, C) samples -> interleaved payload bytes.  Integer formats take the stored integers (U8: 0..255), float formats floats.  Frames wider
    than C samples (a padded block align) are filled with `pad`."""
    x = np.asarray(x)
    n, c = x.shape
    b = SAMPLE_BYTES[fmt]
    if fmt in FLOATS:
        raw = np.ascontiguousarray(x, dtype=(">" if fmt in BIG_ENDIAN else "<") + ("f4" if b == 4 else "f8")).view(np.uint8).reshape(n, c * b)
    else:
        u = x.astype(np.int64) & ((1 << (8 * b)) - 1)
        shifts = 8 * (np.arange(b)[::-1] if fmt in BIG_ENDIAN else np.arange(b))
        raw = ((u[:, :, None] >> shifts) & 0xFF).astype(np.uint8).reshape(n, c * b)
    fb = c * b if frame_bytes is None else frame_bytes
    out = np.full((n, fb), pad, np.uint8)
    out[:, :c * b] = raw
    return out.tobytes()


def restate(data: bytes, n: int, frame_bytes: int, channels: int, fmt: int, out_channels: int) -> np.ndarray:
    """numpy restatement of b200sep_pcm_decode_f32: the first n frames of `data` -> (out_channels, n) float32.
      U8: (u - 128) / 2^7;  S8..S32: v / 2^(8*bytes-1) in float64, rounded once to float32;  F32: the bits;  F64: numpy's float64 -> float32 cast."""
    b = SAMPLE_BYTES[fmt]
    raw = np.frombuffer(data, np.uint8, n * frame_bytes).reshape(n, frame_bytes)[:, :channels * b].reshape(n, channels, b)[:, :out_channels]
    raw = np.ascontiguousarray(raw.transpose(1, 0, 2))
    if fmt in (F32LE, F32BE):
        return raw.view(">u4" if fmt == F32BE else "<u4")[..., 0].astype("<u4").view(np.float32)
    if fmt in (F64LE, F64BE):
        with np.errstate(over="ignore", invalid="ignore"):  # NaN and out-of-range doubles are part of the table
            return raw.view(">f8" if fmt == F64BE else "<f8")[..., 0].astype(np.float32)
    cols = raw.astype(np.int64)
    order = range(b) if fmt in BIG_ENDIAN else range(b - 1, -1, -1)
    u = np.zeros(cols.shape[:2], np.int64)
    for k in order:
        u = (u << 8) | cols[..., k]
    if fmt == U8:
        v = u - 128
        scale = 128.0
    else:
        v = np.where(u >= 1 << (8 * b - 1), u - (1 << (8 * b)), u)
        scale = float(1 << (8 * b - 1))
    return (v.astype(np.float64) / scale).astype(np.float32)


# ---- RIFF / RF64 ----------------------------------------------------------------------------------------------------------------------

def chunk(cid: bytes, body: bytes, size=None, pad=True, endian="<") -> bytes:
    """One chunk: id, size (the body length unless given), body, and the pad byte after an odd body."""
    n = len(body) if size is None else size
    return cid + struct.pack(endian + "I", n) + body + (b"\0" if pad and len(body) & 1 else b"")


def fmt_chunk(tag, channels, rate, block_align, bits, extensible_tag=None, valid_bits=None) -> bytes:
    body = struct.pack("<HHIIHH", 0xFFFE if extensible_tag is not None else tag, channels, rate, rate * block_align, block_align, bits)
    if extensible_tag is not None:
        body += struct.pack("<HHI", 22, valid_bits or bits, 3) + struct.pack("<H", extensible_tag) + _GUID_TAIL
    elif tag != 1:
        body += struct.pack("<H", 0)
    return chunk(b"fmt ", body)


def wav(data: bytes, tag, channels, rate, block_align, bits, extensible=False, valid_bits=None, before=(), after=(), data_size=None,
        rf64=False) -> bytes:
    """A RIFF/WAVE (or RF64) file holding `data`.  `before` / `after`: extra chunks (bytes) around the data chunk; `data_size` overrides the
    data chunk's size field (0 or 0xFFFFFFFF: streamed; a larger value: a file cut short).  RF64 puts the sizes in ds64 and 0xFFFFFFFF in the
    RIFF and data size fields."""
    f = fmt_chunk(tag, channels, rate, block_align, bits, tag if extensible else None, valid_bits)
    if rf64:
        n_frames = len(data) // block_align
        body = f + b"".join(before) + chunk(b"data", data, size=0xFFFFFFFF) + b"".join(after)
        riff = 4 + 36 + len(body)
        ds64 = chunk(b"ds64", struct.pack("<QQQI", riff, len(data) if data_size is None else data_size, n_frames, 0))
        return b"RF64" + struct.pack("<I", 0xFFFFFFFF) + b"WAVE" + ds64 + body
    body = b"".join(before) + f + chunk(b"data", data, size=data_size) + b"".join(after)
    return b"RIFF" + struct.pack("<I", min(4 + len(body), 0xFFFFFFFF)) + b"WAVE" + body


# ---- AIFF / AIFC ----------------------------------------------------------------------------------------------------------------------

def extended(rate) -> bytes:
    """An exact 80-bit IEEE 754 extended value (sign 0, 15-bit exponent, 64-bit mantissa with its explicit integer bit) of a positive int or
    Fraction whose binary expansion fits 64 bits."""
    v = Fraction(rate)
    e = v.numerator.bit_length() - v.denominator.bit_length()
    while v >= Fraction(2) ** (e + 1):
        e += 1
    while v < Fraction(2) ** e:
        e -= 1
    m = v * Fraction(2) ** (63 - e)
    assert m.denominator == 1 and 1 << 63 <= m.numerator < 1 << 64, "value needs more than 64 mantissa bits"
    return struct.pack(">HQ", e + 16383, m.numerator)


def pstring(s: bytes) -> bytes:
    """Pascal string padded to even total length."""
    out = bytes([len(s)]) + s
    return out + (b"\0" if len(out) & 1 else b"")


def aiff(data: bytes, channels, rate, bits, n_frames=None, compression=None, name=b"not compressed", offset=0, block_size=0, before=(),
         ssnd_first=False, ssnd_size=None) -> bytes:
    """A FORM/AIFF file (compression None) or FORM/AIFC (a 4-byte compression type) holding `data` in SSND after `offset` filler bytes.
    `rate` is an int / Fraction (exactly encoded) or the 10 COMM bytes themselves; n_frames defaults to the frames in `data`."""
    nb = {b"fl32": 4, b"FL32": 4, b"fl64": 8, b"FL64": 8, b"raw ": 1}.get(compression, (bits + 7) // 8)
    if n_frames is None:
        n_frames = len(data) // (channels * nb)
    rate_bytes = rate if isinstance(rate, bytes) else extended(rate)
    comm = struct.pack(">HIH", channels, n_frames, bits) + rate_bytes
    if compression is not None:
        comm += compression + pstring(name)
    ssnd_body = struct.pack(">II", offset, block_size) + b"\x5a" * offset + data
    ssnd = chunk(b"SSND", ssnd_body, size=ssnd_size, endian=">")
    comm_c = chunk(b"COMM", comm, endian=">")
    chunks = b"".join(before) + (ssnd + comm_c if ssnd_first else comm_c + ssnd)
    kind = b"AIFC" if compression is not None else b"AIFF"
    if compression is not None:
        chunks = chunk(b"FVER", struct.pack(">I", 0xA2805140), endian=">") + chunks
    return b"FORM" + struct.pack(">I", 4 + len(chunks)) + kind + chunks


# ---- test signals ---------------------------------------------------------------------------------------------------------------------

def ints(n, channels, bits, seed=0):
    """(n, channels) signed integers spanning the full `bits`-bit range, extremes included."""
    rng = np.random.default_rng(seed)
    x = rng.integers(-(1 << (bits - 1)), 1 << (bits - 1), size=(n, channels), dtype=np.int64)
    if n >= 2:
        x[0, 0], x[1, 0] = -(1 << (bits - 1)), (1 << (bits - 1)) - 1
    return x


def cases():
    """Every writer stream with what parse() must report: list of (name, file bytes, expected fields)."""
    out = []

    def add(name, blob, **want):
        out.append((name, blob, want))

    sig = ints(300, 2, 16, seed=1)
    for bits, fmt in ((8, U8), (16, S16LE), (24, S24LE), (32, S32LE)):
        b = SAMPLE_BYTES[fmt]
        x = ints(257, 2, bits, seed=bits)
        if fmt == U8:
            x = x + 128
        d = payload(x, fmt)
        add(f"wav_pcm{bits}", wav(d, 1, 2, 44100, 2 * b, bits), format=fmt, channels=2, sample_rate=44100, block_align=2 * b, n_frames=257, nbytes=len(d))
    for bits, fmt in ((32, F32LE), (64, F64LE)):
        d = payload(np.linspace(-1, 1, 3 * 101).reshape(101, 3), fmt)
        add(f"wav_float{bits}", wav(d, 3, 3, 48000, 3 * bits // 8, bits), format=fmt, channels=3, sample_rate=48000, block_align=3 * bits // 8,
            n_frames=101, nbytes=len(d))
    d = payload(ints(99, 6, 24, seed=5) << 8, S32LE)
    add("wav_ext_pcm24in32", wav(d, 1, 6, 44100, 24, 32, extensible=True, valid_bits=24), format=S32LE, channels=6, sample_rate=44100,
        block_align=24, n_frames=99, nbytes=len(d))
    d = payload(np.linspace(-2, 2, 64).reshape(64, 1), F32LE)
    add("wav_ext_float", wav(d, 3, 1, 44100, 4, 32, extensible=True), format=F32LE, channels=1, sample_rate=44100, block_align=4, n_frames=64, nbytes=len(d))
    d = payload(sig, S16LE, frame_bytes=6)
    add("wav_padded_block_align", wav(d, 1, 2, 44100, 6, 16), format=S16LE, channels=2, sample_rate=44100, block_align=6, n_frames=300, nbytes=len(d))
    d = payload(sig, S16LE)
    extra = (chunk(b"LIST", b"INFOISFT\x05\x00\x00\x00abcd\x00"), chunk(b"JUNK", bytes(7)), chunk(b"bext", bytes(3)), chunk(b"zzzz", b"odd"))
    add("wav_odd_and_unknown_chunks", wav(d, 1, 2, 44100, 4, 16, before=extra[:2], after=extra[2:]), format=S16LE, channels=2, sample_rate=44100,
        block_align=4, n_frames=300, nbytes=len(d))
    add("wav_fact_peak", wav(payload(sig, F32LE), 3, 2, 44100, 8, 32, before=(chunk(b"fact", struct.pack("<I", 300)), chunk(b"PEAK", bytes(24)))),
        format=F32LE, channels=2, sample_rate=44100, block_align=8, n_frames=300, nbytes=2400)
    for size in (0, 0xFFFFFFFF):
        add(f"wav_streamed_{size:x}", wav(d, 1, 2, 44100, 4, 16, data_size=size), format=S16LE, channels=2, sample_rate=44100, block_align=4,
            n_frames=300, nbytes=len(d))
    d3 = payload(ints(300, 3, 24, seed=3), S24LE)
    add("wav_odd_data_pcm24_mono_pad", wav(payload(ints(301, 1, 24, seed=4), S24LE), 1, 1, 44100, 3, 24, after=(chunk(b"LIST", b"x"),)),
        format=S24LE, channels=1, sample_rate=44100, block_align=3, n_frames=301, nbytes=903)
    add("rf64_pcm24", wav(d3, 1, 3, 44100, 9, 24, rf64=True), format=S24LE, channels=3, sample_rate=44100, block_align=9, n_frames=300, nbytes=len(d3))
    add("rf64_float_unknown_chunks", wav(payload(sig, F32LE), 3, 2, 44100, 8, 32, rf64=True, before=(chunk(b"JUNK", bytes(5)),)), format=F32LE,
        channels=2, sample_rate=44100, block_align=8, n_frames=300, nbytes=2400)
    # AIFF: 8 / 12 / 16 / 20 / 24 / 32 bits, by container bytes
    for bits, fmt in ((8, S8), (12, S16BE), (16, S16BE), (20, S24BE), (24, S24BE), (32, S32BE)):
        b = SAMPLE_BYTES[fmt]
        x = ints(211, 2, bits, seed=bits) << (8 * b - bits)
        dd = payload(x, fmt)
        add(f"aiff_{bits}", aiff(dd, 2, 44100, bits), format=fmt, channels=2, sample_rate=44100, block_align=2 * b, n_frames=211, nbytes=len(dd))
    # AIFC compression types
    for comp, bits, fmt, ch in ((b"NONE", 16, S16BE, 1), (b"twos", 24, S24BE, 3), (b"sowt", 16, S16LE, 2), (b"sowt", 24, S24LE, 6),
                                (b"sowt", 32, S32LE, 2), (b"sowt", 8, S8, 2), (b"fl32", 32, F32BE, 2), (b"FL32", 32, F32BE, 1),
                                (b"fl64", 64, F64BE, 2), (b"FL64", 64, F64BE, 3), (b"raw ", 8, U8, 2)):
        b = SAMPLE_BYTES[fmt]
        x = np.linspace(-1.5, 1.5, 97 * ch).reshape(97, ch) if fmt in FLOATS else ints(97, ch, 8 * b, seed=ch) + (128 if fmt == U8 else 0)
        dd = payload(x, fmt)
        add(f"aifc_{comp.decode().strip()}_{bits}_{ch}ch", aiff(dd, ch, 44100, bits, compression=comp, name=b"odd"), format=fmt, channels=ch,
            sample_rate=44100, block_align=ch * b, n_frames=97, nbytes=len(dd))
    dd = payload(ints(50, 2, 16, seed=8), S16BE)
    add("aifc_ssnd_offset_block_first", aiff(dd, 2, 44100, 16, compression=b"NONE", name=b"", offset=13, block_size=4096, ssnd_first=True),
        format=S16BE, channels=2, sample_rate=44100, block_align=4, n_frames=50, nbytes=len(dd), offset=13)
    add("aiff_unknown_chunks", aiff(dd, 2, 44100, 16, before=(chunk(b"NAME", b"abc", endian=">"), chunk(b"ANNO", b"x" * 6, endian=">"))),
        format=S16BE, channels=2, sample_rate=44100, block_align=4, n_frames=50, nbytes=len(dd))
    # sample rates: small, large and fractional (the truncated integer is the rate, as libsndfile reads it)
    for rate, want in ((1, 1), (3, 3), (8000, 8000), (192000, 192000), ((1 << 31) - 1, (1 << 31) - 1), (Fraction(88200 * (1 << 40) + 1, 1 << 41), 44100),
                       (Fraction((1 << 64) - 1, 1 << 48), 65535)):
        add(f"aiff_rate_{want}", aiff(dd, 2, rate, 16), format=S16BE, channels=2, sample_rate=want, block_align=4, n_frames=50, nbytes=len(dd))
    return out
