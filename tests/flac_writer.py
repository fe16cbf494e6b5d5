"""A plain-Python FLAC (RFC 9639) writer for tests, in the manner of onnx_writer.py.

TEST INFRASTRUCTURE -- not product code.  It encodes given integer samples with explicitly chosen tools, so that the decoder meets what the GPU
encoder never emits: variable blocking, every block-size / sample-rate / sample-size header code, 1-8 channels, FIXED 0-4, LPC 1-32 at any
precision, RICE2, high partition orders, escape partitions, wasted bits, every metadata block type, and ID3 tags around the stream.  The
expected samples of a stream are the writer's input; the stream oracle (oracle/flac_stream_oracle.py) decodes every stream independently.
"""
from dataclasses import dataclass, field

import numpy as np

FIXED_COEFS = ([], [1], [2, -1], [3, -3, 1], [4, -6, 4, -1])
RATE_CODES = {88200: 1, 176400: 2, 192000: 3, 8000: 4, 16000: 5, 22050: 6, 24000: 7, 32000: 8, 44100: 9, 48000: 10, 96000: 11}
BPS_CODES = {8: 1, 12: 2, 16: 4, 20: 5, 24: 6}


def _table(poly, width):
    top, mask, tab = 1 << (width - 1), (1 << width) - 1, []
    for i in range(256):
        c = i << (width - 8)
        for _ in range(8):
            c = ((c << 1) ^ poly) if c & top else (c << 1)
        tab.append(c & mask)
    return tab


_T8, _T16 = _table(0x07, 8), _table(0x8005, 16)


def crc8(data):
    c = 0
    for b in data:
        c = _T8[c ^ b]
    return c


def crc16(data):
    c = 0
    for b in data:
        c = ((c << 8) & 0xFFFF) ^ _T16[(c >> 8) ^ b]
    return c


class BitWriter:
    def __init__(self):
        self.chunks, self.acc, self.n = bytearray(), 0, 0

    def u(self, v, n):
        assert 0 <= v < (1 << n) or n == 0 and v == 0, (v, n)
        self.acc, self.n = (self.acc << n) | v, self.n + n
        while self.n >= 8:
            self.n -= 8
            self.chunks.append((self.acc >> self.n) & 0xFF)
        self.acc &= (1 << self.n) - 1

    def s(self, v, n):
        assert -(1 << (n - 1)) <= v < (1 << (n - 1)) if n else v == 0, (v, n)
        self.u(v & ((1 << n) - 1), n)

    def unary(self, q):
        while q >= 32:
            self.u(0, 32)
            q -= 32
        self.u(1, q + 1)

    def align(self):
        if self.n:
            self.u(0, 8 - self.n)

    def bytes(self):
        assert self.n == 0
        return bytes(self.chunks)


def utf8_number(v):
    if v < 0x80:
        return bytes([v])
    n = 2
    while v >= 1 << (5 * n + 1):
        n += 1
    assert n <= 7
    out = [((0xFF00 >> n) & 0xFF) | (v >> (6 * (n - 1)))]
    out += [0x80 | ((v >> (6 * j)) & 0x3F) for j in range(n - 2, -1, -1)]
    return bytes(out)


@dataclass
class Sub:
    """How one subframe is coded.  params: per-partition Rice parameter, "esc" (escape partition at the smallest width) or ("esc", width);
    None picks the cheapest parameter per partition."""
    kind: str = "fixed"  # constant | verbatim | fixed | lpc
    order: int = 2
    coefs: tuple = ()
    precision: int = 15
    shift: int = 0
    method: int = 0  # 0 RICE, 1 RICE2
    po: int = 0
    params: object = None
    wasted: int = 0


def _rice_cost(res, k):
    zz = np.where(res >= 0, 2 * res, -2 * res - 1)
    return int(np.sum((zz >> k) + 1 + k))


def _residual(w, res, bs, order, sub, tools):
    w.u(sub.method, 2)
    tools.add("RICE2" if sub.method else "RICE")
    w.u(sub.po, 4)
    tools.add(f"po{sub.po}")
    pbits, kmax = (5, 30) if sub.method else (4, 14)
    psz = bs >> sub.po
    assert bs % (1 << sub.po) == 0 and psz >= order
    start = 0
    for p in range(1 << sub.po):
        part = res[start:start + psz - (order if p == 0 else 0)]
        start += len(part)
        want = sub.params[p] if isinstance(sub.params, (list, tuple)) else sub.params
        if want is None:
            want = min(range(kmax + 1), key=lambda k: _rice_cost(part, k))
        if want == "esc" or isinstance(want, tuple):
            width = max([0] + [int(v).bit_length() + 1 for v in part if v])
            if isinstance(want, tuple):
                width = max(width, want[1])
            tools.add("escape0" if width == 0 else "escape")
            w.u((1 << pbits) - 1, pbits)
            w.u(width, 5)
            for v in part:
                w.s(int(v), width)
        else:
            assert 0 <= want <= kmax
            w.u(want, pbits)
            for v in part:
                zz = 2 * int(v) if v >= 0 else -2 * int(v) - 1
                w.unary(zz >> want)
                w.u(zz & ((1 << want) - 1), want)


def _subframe(w, x, bps, sub, tools):
    x = [int(v) for v in x]
    bs = len(x)
    types = {"constant": 0, "verbatim": 1}
    if sub.kind == "fixed":
        t = 8 + sub.order
    elif sub.kind == "lpc":
        t = 31 + sub.order
    else:
        t = types[sub.kind]
    w.u(0, 1)
    w.u(t, 6)
    if sub.wasted:
        assert all(v % (1 << sub.wasted) == 0 for v in x)
        x = [v >> sub.wasted for v in x]
        w.u(1, 1)
        w.unary(sub.wasted - 1)
        tools.add("wasted")
    else:
        w.u(0, 1)
    b = bps - sub.wasted
    if sub.kind == "constant":
        assert len(set(x)) == 1
        w.s(x[0], b)
        tools.add("CONSTANT")
        return
    if sub.kind == "verbatim":
        for v in x:
            w.s(v, b)
        tools.add("VERBATIM")
        return
    order = sub.order
    for v in x[:order]:
        w.s(v, b)
    if sub.kind == "fixed":
        coefs, shift = FIXED_COEFS[order], 0
        tools.add(f"FIXED{order}")
    else:
        coefs, shift = list(sub.coefs), sub.shift
        assert len(coefs) == order and 1 <= sub.precision <= 15 and 0 <= shift <= 15
        w.u(sub.precision - 1, 4)
        w.s(shift, 5)
        for c in coefs:
            w.s(c, sub.precision)
        tools.add(f"LPC{order}")
        tools.add(f"prec{sub.precision}")
    res = np.array([x[i] - (sum(c * x[i - 1 - j] for j, c in enumerate(coefs)) >> shift) for i in range(order, bs)], dtype=np.int64)
    assert res.size == 0 or (res.min() >= -(1 << 31) and res.max() < (1 << 31)), "residual does not fit 32 bits"
    _residual(w, res, bs, order, sub, tools)


@dataclass
class Frame:
    samples: np.ndarray  # (bs, channels) int
    assign: int = 1  # 1 independent, 8 left/side, 9 right/side, 10 mid/side
    subs: list = field(default_factory=lambda: [Sub()])  # one per coded channel (the last one repeats)
    bs_code: object = None  # None: natural code
    rate_code: object = None  # None: the table code or 0
    bps_code: object = None  # None: the table code or 0


def _bs_code(bs, want):
    natural = {192: 1, 576: 2, 1152: 3, 2304: 4, 4608: 5, **{256 << k: 8 + k for k in range(8)}}
    if want is None:
        want = natural.get(bs, 6 if bs <= 256 else 7)
    if want in (6, 7):
        return want, (bs - 1).to_bytes(1 if want == 6 else 2, "big")
    assert natural.get(bs) == want, (bs, want)
    return want, b""


def _rate_code(rate, want):
    if want is None:
        want = RATE_CODES.get(rate, 0)
    if want == 12:
        assert rate % 1000 == 0
        return 12, bytes([rate // 1000])
    if want == 13:
        return 13, rate.to_bytes(2, "big")
    if want == 14:
        assert rate % 10 == 0
        return 14, (rate // 10).to_bytes(2, "big")
    assert want == 0 or RATE_CODES[rate] == want
    return want, b""


def frame_bytes(fr: Frame, number, rate, bps, variable, tools):
    x = np.asarray(fr.samples, dtype=np.int64)
    bs, nch = x.shape
    bsc, bse = _bs_code(bs, fr.bs_code)
    src, sre = _rate_code(rate, fr.rate_code)
    ssc = BPS_CODES.get(bps, 0) if fr.bps_code is None else fr.bps_code
    tools.update({f"bs{bsc}", f"sr{src}", f"ss{ssc}", f"ch{nch}", f"bps{bps}"})
    head = bytes([0xFF, 0xF8 | variable, (bsc << 4) | src, (fr.assign if fr.assign >= 8 else nch - 1) << 4 | ssc << 1])
    head += utf8_number(number) + bse + sre
    head += bytes([crc8(head)])
    if fr.assign == 8:
        chans, widths = [x[:, 0], x[:, 0] - x[:, 1]], [bps, bps + 1]
    elif fr.assign == 9:
        chans, widths = [x[:, 0] - x[:, 1], x[:, 1]], [bps + 1, bps]
    elif fr.assign == 10:
        chans, widths = [(x[:, 0] + x[:, 1]) >> 1, x[:, 0] - x[:, 1]], [bps, bps + 1]
    else:
        chans, widths = [x[:, c] for c in range(nch)], [bps] * nch
    tools.add({1: "independent", 8: "left/side", 9: "right/side", 10: "mid/side"}[fr.assign])
    w = BitWriter()
    for c, (ch, width) in enumerate(zip(chans, widths)):
        _subframe(w, ch, width, fr.subs[min(c, len(fr.subs) - 1)], tools)
    w.align()
    body = head + w.bytes()
    return body + crc16(body).to_bytes(2, "big")


def streaminfo(rate, bps, channels, total, min_block=0, max_block=0, md5=bytes(16)):
    packed = (rate << 44) | ((channels - 1) << 41) | ((bps - 1) << 36) | total
    return min_block.to_bytes(2, "big") + max_block.to_bytes(2, "big") + bytes(6) + packed.to_bytes(8, "big") + md5


def metadata_block(kind, body, last):
    return bytes([(0x80 if last else 0) | kind]) + len(body).to_bytes(3, "big") + body


# a plausible body for every metadata block type after STREAMINFO
EXTRA_BLOCKS = {
    1: bytes(37),  # PADDING
    2: b"test" + b"application data",  # APPLICATION
    3: (0).to_bytes(8, "big") + (0).to_bytes(8, "big") + (4096).to_bytes(2, "big"),  # SEEKTABLE, one point
    4: (6).to_bytes(4, "little") + b"writer" + (1).to_bytes(4, "little") + (9).to_bytes(4, "little") + b"TITLE=abc",  # VORBIS_COMMENT
    5: bytes(128 + 8 + 1 + 258 + 1),  # CUESHEET with no tracks
    6: (3).to_bytes(4, "big") + (9).to_bytes(4, "big") + b"image/png" + (0).to_bytes(4, "big") + bytes(16) + (0).to_bytes(4, "big"),  # PICTURE
}


def id3v2(size=30, footer=False):
    ss = bytes([(size >> 21) & 0x7F, (size >> 14) & 0x7F, (size >> 7) & 0x7F, size & 0x7F])
    tag = b"ID3" + bytes([4, 0, 0x10 if footer else 0]) + ss + bytes(size)
    return tag + (b"3DI" + bytes([4, 0, 0x10]) + ss if footer else b"")


def stream(frames, rate, bps, variable=False, first_number=0, blocks=(), id3v2_tag=b"", id3v1=False, total=None, tools=None):
    """Whole file: [ID3v2] fLaC STREAMINFO [blocks] frames [ID3v1].  Returns (bytes, (N, channels) int64 samples)."""
    tools = set() if tools is None else tools
    nch = frames[0].samples.shape[1]
    n = sum(f.samples.shape[0] for f in frames)
    sizes = [f.samples.shape[0] for f in frames]
    meta = [(0, streaminfo(rate, bps, nch, n if total is None else total, min(sizes), max(sizes)))] + [(k, EXTRA_BLOCKS[k]) for k in blocks]
    out = id3v2_tag + b"fLaC" + b"".join(metadata_block(k, b, i == len(meta) - 1) for i, (k, b) in enumerate(meta))
    tools.update(f"meta{k}" for k, _ in meta)
    if id3v2_tag:
        tools.add("id3v2")
    number = first_number
    for f in frames:
        out += frame_bytes(f, number, rate, bps, int(variable), tools)
        number += f.samples.shape[0] if variable else 1
    if variable:
        tools.add("variable")
    if id3v1:
        out += b"TAG" + bytes(125)
        tools.add("id3v1")
    return out, np.concatenate([np.asarray(f.samples, np.int64) for f in frames])


# ---- the catalogue of test streams ------------------------------------------------------------------------------------------------------

def signal(n, bps, channels, seed):
    """A smooth random walk at half of full scale: small prediction residuals, every channel different."""
    rng = np.random.default_rng(seed)
    x = np.cumsum(rng.standard_normal((n, channels)), axis=0)
    x = x - x.mean(axis=0)
    x = x / max(1e-9, np.abs(x).max()) * ((1 << (bps - 1)) - 1) * 0.5
    return np.rint(x).astype(np.int64)


def _lpc_coefs(order, precision, rng):
    lim = (1 << (precision - 1)) - 1
    return tuple(int(c) for c in rng.integers(-lim, lim + 1, order) // order)


# every tool and header code the catalogue must exercise (the coverage check of the decoder tests)
REQUIRED_TOOLS = (
    {"variable", "independent", "left/side", "right/side", "mid/side", "CONSTANT", "VERBATIM", "wasted", "escape", "escape0", "RICE", "RICE2",
     "id3v2", "id3v1"}
    | {f"FIXED{o}" for o in range(5)} | {f"LPC{o}" for o in range(1, 33)} | {f"prec{p}" for p in range(1, 16)}
    | {f"bs{c}" for c in range(1, 16)} | {f"sr{c}" for c in range(15)} | {f"ss{c}" for c in (0, 1, 2, 4, 5, 6)}
    | {f"bps{b}" for b in range(4, 25)} | {f"ch{c}" for c in range(1, 9)} | {f"meta{k}" for k in range(7)} | {f"po{p}" for p in range(16)}
)


def cases():
    """name -> (FLAC bytes, (N, channels) int64 expected samples, tools used)."""
    out = {}

    def add(name, frames, rate=44100, bps=16, **kw):
        tools = set()
        data, want = stream(frames, rate, bps, tools=tools, **kw)
        out[name] = (data, want, tools)

    rng = np.random.default_rng(1)
    x = signal(5 * 4096, 16, 2, 1)
    add("fixed_orders", [Frame(x[i * 4096:(i + 1) * 4096], subs=[Sub("fixed", order=i, po=i)]) for i in range(5)])
    frames = []
    for o in range(1, 33):
        p = 1 + (o - 1) % 15
        frames.append(Frame(signal(1152, 16, 2, o), subs=[Sub("lpc", order=o, precision=p, shift=p - 1, coefs=_lpc_coefs(o, p, rng), method=o & 1)]))
    add("lpc_orders_16bit", frames)
    frames = [Frame(signal(4608, 24, 2, 40 + o), subs=[Sub("lpc", order=o, precision=15, shift=14, coefs=_lpc_coefs(o, 15, rng), po=3, method=1)])
              for o in (8, 12, 32)]
    add("lpc_24bit_wide_accumulator", frames, bps=24)
    x = signal(4 * 4096, 16, 2, 2)
    add("stereo_modes", [Frame(x[i * 4096:(i + 1) * 4096], assign=a, subs=[Sub("fixed", order=2, method=1, po=5 + i)])
                         for i, a in enumerate((1, 8, 9, 10))])
    x = signal(4096, 16, 2, 3)
    x[:2048] = 1000
    add("escapes", [Frame(x, subs=[Sub("fixed", order=1, po=4, params=["esc"] * 8 + [("esc", 20)] * 4 + [None] * 4, method=1)])])
    x = signal(2 * 4096, 16, 2, 4) & ~7
    c = np.full((4096, 2), -96, np.int64)
    add("wasted_constant_verbatim", [Frame(x[:4096], subs=[Sub("fixed", order=3, wasted=3)]), Frame(x[4096:], subs=[Sub("verbatim", wasted=2)]),
                                     Frame(c, subs=[Sub("constant", wasted=5)]), Frame(c, subs=[Sub("constant")])])
    sizes = (192, 576, 1152, 2304, 4608) + tuple(256 << k for k in range(8)) + (1, 17, 256, 300, 65535)
    codes = (1, 2, 3, 4, 5) + tuple(range(8, 16)) + (6, 6, 6, 7, 7)
    x = signal(sum(sizes), 16, 1, 5)
    frames, at = [], 0
    for bs, code in zip(sizes, codes):
        frames.append(Frame(x[at:at + bs], bs_code=code, subs=[Sub("fixed", order=min(2, bs), po=0)]))
        at += bs
    add("block_size_codes_variable", frames, variable=True, first_number=123456)
    add("variable_seven_byte_number", [Frame(signal(4096, 16, 2, 6))], variable=True, first_number=1 << 35)
    add("fixed_first_frame_703", [Frame(y) for y in np.split(signal(3 * 4608, 16, 2, 7), 3)], first_number=703)
    add("fixed_six_byte_number", [Frame(signal(576, 16, 2, 8))], first_number=(1 << 31) - 1)
    for rate, code in RATE_CODES.items():
        add(f"rate_code_{code}", [Frame(signal(192, 16, 2, code), rate_code=code)], rate=rate)
    add("rate_code_0", [Frame(signal(192, 16, 2, 20), rate_code=0)], rate=44100)
    add("rate_code_12", [Frame(signal(192, 16, 2, 21), rate_code=12)], rate=37000)
    add("rate_code_13", [Frame(signal(192, 16, 2, 22), rate_code=13)], rate=44100)
    add("rate_code_14", [Frame(signal(192, 16, 2, 23), rate_code=14)], rate=88210)
    for bps in range(4, 25):
        add(f"bps_{bps}", [Frame(signal(1000, bps, 2, 100 + bps), subs=[Sub("fixed", order=2, method=1, po=3)])], bps=bps)
    add("bps_code_0_at_16", [Frame(signal(1000, 16, 2, 130), bps_code=0)])
    for ch in range(1, 9):
        add(f"channels_{ch}", [Frame(signal(2048, 16, ch, 140 + ch), subs=[Sub("fixed", order=2, po=2)])])
    po_frames = [Frame(signal(1 << 15, 16, 1, 160), bs_code=15, subs=[Sub("fixed", order=0, po=15, method=1)]),
                 Frame(signal(1 << 14, 16, 1, 161), bs_code=14, subs=[Sub("fixed", order=1, po=12)]) ]
    add("high_partition_orders", po_frames)
    add("po_9_to_11", [Frame(signal(1 << 12, 16, 1, 170 + k), subs=[Sub("fixed", order=1, po=9 + k)]) for k in range(3)], variable=True)
    add("po_13_14", [Frame(signal(1 << 14, 16, 1, 175 + k), bs_code=14, subs=[Sub("fixed", order=1, po=13 + k)]) for k in range(2)])
    x = signal(4096, 16, 2, 9)
    add("metadata_all_blocks_id3", [Frame(x)], blocks=(1, 2, 3, 4, 5, 6), id3v2_tag=id3v2(40), id3v1=True)
    add("metadata_id3v2_footer", [Frame(x)], blocks=(4,), id3v2_tag=id3v2(17, footer=True))
    return out
