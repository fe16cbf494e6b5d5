"""CPU: the WAV / RF64 / AIFF / AIFF-C container parser and bit-depth rules of b200/pcm_reader.py on every stream of tests/pcm_writer.py, the
numpy restatement of the decoder's conversion table against hand values, and the errors of malformed and compressed files."""
import struct

import numpy as np
import pytest

import pcm_writer as W


@pytest.fixture(scope="module")
def pcm(lib_built):
    from audio_separator.separator.b200 import pcm_reader

    return pcm_reader


@pytest.mark.parametrize("name,blob,want", W.cases(), ids=[c[0] for c in W.cases()])
def test_parse_writer_streams(pcm, name, blob, want):
    info = pcm.parse(blob)
    for k in ("format", "channels", "sample_rate", "block_align", "n_frames"):
        assert info[k] == want[k], (k, info[k], want[k])
    assert info["end"] - info["begin"] == want["nbytes"]
    # the span is the writer's payload: it ends where the data / SSND body ends and starts after the SSND offset filler
    if info["container"] in ("AIFF", "AIFC"):
        assert blob[info["begin"] - want.get("offset", 0):info["begin"]] == b"\x5a" * want.get("offset", 0)
    assert info["warnings"] == []


def test_every_format_and_channel_count_is_written(pcm):
    seen = {(c[2]["format"], c[2]["channels"]) for c in W.cases()}
    assert {f for f, _ in seen} == set(range(12))
    assert {c for _, c in seen} == {1, 2, 3, 6}
    names = [c[0] for c in W.cases()]
    assert any(n.startswith("rf64") for n in names) and any("streamed" in n for n in names) and any("aiff_rate" in n for n in names)


def test_payload_span_is_the_data(pcm):
    x = W.ints(40, 2, 16, seed=2)
    d = W.payload(x, W.S16LE)
    blob = W.wav(d, 1, 2, 44100, 4, 16, before=(W.chunk(b"JUNK", b"abc"),), after=(W.chunk(b"LIST", b"tail"),))
    info = pcm.parse(blob)
    assert blob[info["begin"]:info["end"]] == d
    blob = W.aiff(W.payload(x, W.S16BE), 2, 44100, 16, compression=b"twos", name=b"big endian", offset=7, block_size=8)
    info = pcm.parse(blob)
    assert blob[info["begin"]:info["end"]] == W.payload(x, W.S16BE) and info["block_size"] == 8 and info["compression"] == "twos"


def test_conversion_table_hand_values():
    def one(fmt, raw):
        return float(W.restate(bytes(raw), 1, len(raw), 1, fmt, 1)[0, 0])

    assert one(W.S16LE, [0x00, 0x80]) == -1.0
    assert one(W.S16BE, [0x80, 0x00]) == -1.0
    assert one(W.S16LE, [0xFF, 0x7F]) == 32767 / 32768
    assert one(W.U8, [0x80]) == 0.0 and one(W.U8, [0x00]) == -1.0 and one(W.U8, [0xFF]) == 127 / 128
    assert one(W.S8, [0x80]) == -1.0 and one(W.S8, [0x7F]) == 127 / 128
    assert one(W.S24LE, [0x00, 0x00, 0x80]) == -1.0 and one(W.S24BE, [0x7F, 0xFF, 0xFF]) == (2 ** 23 - 1) / 2 ** 23
    assert one(W.S32LE, [0xFF, 0xFF, 0xFF, 0x7F]) == 1.0  # INT32_MAX rounds up to 2^31
    assert one(W.S32BE, [0x80, 0, 0, 0]) == -1.0
    assert one(W.S32LE, [0x41, 0, 0, 0]) == np.float32(65 / 2 ** 31)
    big = (1 << 24) + 3  # 25 significant bits: rounds to nearest even in float32
    assert one(W.S32LE, list(struct.pack("<i", big))) == float(np.float32((1 << 24) + 4)) / 2 ** 31
    # F32: the bits as they are, NaN payloads and infinities included
    for bits in (0x7FC12345, 0xFF800000, 0x7F800001, 0x00000001, 0x40490FDB):
        got = W.restate(struct.pack("<I", bits), 1, 4, 1, W.F32LE, 1).view(np.uint32)[0, 0]
        assert got == bits and W.restate(struct.pack(">I", bits), 1, 4, 1, W.F32BE, 1).view(np.uint32)[0, 0] == bits
    # F64: round to nearest (a double halfway between two floats goes to the even one)
    halfway = 1.0 + 2.0 ** -24
    assert one(W.F64LE, list(struct.pack("<d", halfway))) == 1.0
    assert one(W.F64BE, list(struct.pack(">d", 1.0 + 3 * 2.0 ** -24))) == 1.0 + 2.0 ** -22
    assert one(W.F64LE, list(struct.pack("<d", 1e300))) == np.inf


def test_input_bit_depth_table(pcm):
    want = {W.U8: (16, "PCM_U8"), W.S8: (16, "PCM_S8"), W.S16LE: (16, "PCM_16"), W.S16BE: (16, "PCM_16"), W.S24LE: (24, "PCM_24"),
            W.S24BE: (24, "PCM_24"), W.S32LE: (32, "PCM_32"), W.S32BE: (32, "PCM_32"), W.F32LE: (32, "FLOAT"), W.F32BE: (32, "FLOAT"),
            W.F64LE: (32, "DOUBLE"), W.F64BE: (32, "DOUBLE")}
    for fmt, depth in want.items():
        assert pcm.input_bit_depth({"format": fmt}) == depth


def test_extended_rate(pcm):
    from fractions import Fraction

    for rate in (1, 2, 3, 11025, 44100, 48000, 96000, 192000, (1 << 32) - 1):
        assert pcm.extended_to_rate(W.extended(rate)) == rate
    assert W.extended(44100) == bytes.fromhex("400eac44000000000000")
    assert pcm.extended_to_rate(W.extended(Fraction(44100 * (1 << 48) + 1, 1 << 48))) == 44100  # uses the lowest mantissa bits
    for bad in ("00000000000000000000", "c00eac44000000000000", "7fff8000000000000000", "7fffc000000000000000"):
        with pytest.raises(ValueError, match="sample rate"):
            pcm.extended_to_rate(bytes.fromhex(bad))


def test_size_beyond_the_file_is_cut_with_a_warning(pcm):
    d = W.payload(W.ints(100, 2, 16), W.S16LE)
    info = pcm.parse(W.wav(d, 1, 2, 44100, 4, 16, data_size=len(d) + 40))
    assert info["n_frames"] == 100 and len(info["warnings"]) == 1 and "declares 440 bytes" in info["warnings"][0]
    info = pcm.parse(W.wav(d, 1, 2, 44100, 4, 16)[:-3])  # a partial last frame is dropped
    assert info["n_frames"] == 99
    info = pcm.parse(W.wav(d, 1, 2, 44100, 4, 16, rf64=True, data_size=len(d) * 2))
    assert info["n_frames"] == 100 and len(info["warnings"]) == 1
    a = W.payload(W.ints(100, 2, 16), W.S16BE)
    info = pcm.parse(W.aiff(a, 2, 44100, 16, n_frames=150))
    assert info["n_frames"] == 100 and info["warnings"] == ["'COMM' declares 150 sample frames, 'SSND' holds 100"]
    info = pcm.parse(W.aiff(a, 2, 44100, 16)[:-10])
    assert info["n_frames"] == 97 and len(info["warnings"]) == 2


def test_malformed_containers_raise_value_error(pcm):
    d = W.payload(W.ints(10, 2, 16), W.S16LE)
    good = W.wav(d, 1, 2, 44100, 4, 16)
    bad = {
        "truncated header": good[:10],
        "not a RIFF": b"RIFX" + good[4:],
        "truncated 'fmt '": good[:12] + W.chunk(b"fmt ", bytes(10)),
        "before any 'fmt ' chunk": good[:12] + W.chunk(b"data", d),
        "runs past the end": good[:12] + W.chunk(b"LIST", bytes(4), size=1000) + good[12:],
        "no 'data' chunk": good[:36],
        "impossible block align 3": W.wav(d, 1, 2, 44100, 3, 16),
        "impossible block align 0": W.wav(d, 1, 2, 44100, 0, 16),
        "'fmt ' chunk at byte 12: 0 channels": W.wav(d, 1, 0, 44100, 4, 16),
        "sample rate 0": W.wav(d, 1, 2, 0, 4, 16),
        "16-bit IEEE float": W.wav(d, 3, 2, 44100, 4, 16),
        "40-bit integer PCM": W.wav(d, 1, 1, 44100, 5, 40),
        "without a 'ds64'": b"RF64" + good[4:12] + good[12:36] + W.chunk(b"data", d, size=0xFFFFFFFF),
    }
    a = W.payload(W.ints(10, 2, 16), W.S16BE)
    aiff = W.aiff(a, 2, 44100, 16)
    bad.update({
        "no 'COMM' chunk": aiff[:12] + aiff[12 + 26:],
        "no 'SSND' chunk": aiff[:12 + 26],
        "truncated 'COMM'": aiff[:12] + W.chunk(b"COMM", bytes(10), endian=">"),
        "offset 4 beyond its 2 bytes": W.aiff(a, 2, 44100, 16, offset=4, ssnd_size=10),
        "invalid sample rate": W.aiff(a, 2, bytes(10), 16),
        "33-bit PCM": W.aiff(a, 1, 44100, 33),
        "'COMM' chunk at byte 12: 0 channels": W.aiff(a, 0, 44100, 16, n_frames=10),
    })
    for what, blob in bad.items():  # key: a part of the message
        with pytest.raises(ValueError) as e:
            pcm.parse(blob)
        assert what in str(e.value), (what, str(e.value))
    with pytest.raises(ValueError, match=r"'fmt ' chunk at byte 12"):
        pcm.parse(W.wav(d, 1, 2, 44100, 3, 16))
    with pytest.raises(ValueError, match=r"'LIST' chunk at byte 12 runs past"):
        pcm.parse(good[:12] + W.chunk(b"LIST", bytes(4), size=1000) + good[12:])


def test_compressed_payloads_raise_not_implemented(pcm):
    d = bytes(64)
    for tag in (2, 6, 7, 0x11, 0x55):  # ADPCM, A-law, mu-law, IMA ADPCM, MP3
        with pytest.raises(NotImplementedError, match="format tag"):
            pcm.parse(W.wav(d, tag, 2, 44100, 2, 8))
    ambisonic = W.wav(d, 1, 2, 44100, 4, 16, extensible=True).replace(W._GUID_TAIL, bytes(14))
    with pytest.raises(NotImplementedError, match="sub-format"):
        pcm.parse(ambisonic)
    for comp in (b"ulaw", b"ULAW", b"alaw", b"ALAW", b"ima4", b"MAC3", b"GSM ", b"in24"):
        with pytest.raises(NotImplementedError, match="compression type"):
            pcm.parse(W.aiff(d, 2, 44100, 16, compression=comp))
    with pytest.raises(NotImplementedError, match="raw"):
        pcm.parse(W.aiff(d, 2, 44100, 16, compression=b"raw "))


def test_content_sniffing(pcm):
    assert pcm.is_pcm_container(W.wav(bytes(4), 1, 1, 44100, 2, 16)[:12])
    assert pcm.is_pcm_container(W.wav(bytes(4), 1, 1, 44100, 2, 16, rf64=True)[:12])
    assert pcm.is_pcm_container(W.aiff(bytes(4), 1, 44100, 16)[:12]) and pcm.is_pcm_container(W.aiff(bytes(4), 1, 44100, 16, compression=b"sowt")[:12])
    assert not pcm.is_pcm_container(b"fLaC" + bytes(8)) and not pcm.is_pcm_container(b"RIFF\0\0\0\0AVI ") and not pcm.is_pcm_container(b"FORM")


def test_writer_riff_streams_read_by_scipy():
    """An independent reader of the writer's RIFF / RF64 streams: scipy.io.wavfile gives the same samples as the restatement."""
    import io
    import warnings

    from scipy.io import wavfile

    checked = 0
    for name, blob, want in W.cases():
        if not name.startswith(("wav", "rf64")) or "streamed" in name or "padded" in name:
            continue
        with warnings.catch_warnings():
            warnings.simplefilter("ignore", wavfile.WavFileWarning)  # the writer's unknown chunks
            rate, x = wavfile.read(io.BytesIO(blob))
        x = x.reshape(len(x), -1)
        if x.dtype.kind == "f":
            y = x.astype(np.float32)
        else:
            y = (x.astype(np.float64) - (128 if x.dtype == np.uint8 else 0)) / float(1 << (8 * x.dtype.itemsize - 1))
        data = blob[blob.index(b"data") + 8:]
        ref = W.restate(data, want["n_frames"], want["block_align"], want["channels"], want["format"], want["channels"])
        assert rate == want["sample_rate"] and np.array_equal(y.astype(np.float32).T, ref), name
        checked += 1
    assert checked >= 10
