"""Uncompressed PCM input (WAV, RF64, AIFF, AIFF-C) decoded on the GPU.

The host parses the container and uploads only the payload bytes (the data / SSND chunk), once, from a page-locked buffer; csrc/pcm_decode.cu
converts them into the planar float mix as libsndfile's sf_read_float with normalisation on does, which is what the reference's
librosa.load(path, mono=False, sr=44100) returns (common_separator.py:217-282).  DESIGN.md section 26.

Container rules follow libsndfile: the container sample size governs (wBitsPerSample / the COMM sample size rounded up to whole bytes), so a
24-in-32 extensible WAV reads as PCM_32 and a 20-bit AIFF as PCM_24.  A declared payload size that runs past the end of the file is cut to the
whole frames present, with a warning in info["warnings"].
"""
import struct

import numpy as np

import torch

from ._lib import check, lib

# sample formats of b200sep_pcm_decode_f32 (include/b200sep.h)
U8, S8, S16LE, S16BE, S24LE, S24BE, S32LE, S32BE, F32LE, F32BE, F64LE, F64BE = range(12)
SAMPLE_BYTES = (1, 1, 2, 2, 3, 3, 4, 4, 4, 4, 8, 8)
# the libsndfile subtype of each format, and the bit depth the reference maps it to (common_separator.py:236-245)
SUBTYPE = ("PCM_U8", "PCM_S8", "PCM_16", "PCM_16", "PCM_24", "PCM_24", "PCM_32", "PCM_32", "FLOAT", "FLOAT", "DOUBLE", "DOUBLE")
BIT_DEPTH = {"PCM_U8": 16, "PCM_S8": 16, "PCM_16": 16, "PCM_24": 24, "PCM_32": 32, "FLOAT": 32, "DOUBLE": 32}
MAX_FRAME_BYTES = 65535  # the kernel's limit: WAV's nBlockAlign field

# WAVE_FORMAT_EXTENSIBLE sub-format GUIDs: the format tag in the first two bytes, then this fixed tail
_GUID_TAIL = bytes.fromhex("000000001000800000aa00389b71")
# AIFF-C compression types -> (format by container bytes 1..4, or one fixed format)
_AIFC_INT_BE = (S8, S16BE, S24BE, S32BE)
_AIFC_INT_LE = (S8, S16LE, S24LE, S32LE)
_AIFC = {b"NONE": _AIFC_INT_BE, b"twos": _AIFC_INT_BE, b"sowt": _AIFC_INT_LE, b"fl32": F32BE, b"FL32": F32BE, b"fl64": F64BE, b"FL64": F64BE,
         b"raw ": U8}


def is_pcm_container(head: bytes) -> bool:
    """Content sniffing on the first 12 bytes: RIFF / RF64 with WAVE, or FORM with AIFF / AIFC."""
    return (head[:4] in (b"RIFF", b"RF64") and head[8:12] == b"WAVE") or (head[:4] == b"FORM" and head[8:12] in (b"AIFF", b"AIFC"))


def _chunks(data: bytes, p: int, endian: str, payload: bytes):
    """Yield (id, offset of the chunk header, body start, declared body size) for the chunks from byte p on; bodies are padded to even length.
    Only the payload chunk may run past the end of the file (it is cut by the caller); any other such chunk ends the walk, and the caller reports
    what it has not found by then."""
    while p + 8 <= len(data):
        cid, size = data[p:p + 4], struct.unpack_from(endian + "I", data, p + 4)[0]
        if cid != payload and p + 8 + size > len(data):
            return
        yield cid, p, p + 8, size
        p += 8 + size + (size & 1)


def _need(cid: bytes, at: int, body: int, size: int, want: int, data: bytes):
    if size < want or body + want > len(data):
        raise ValueError(f"truncated {cid.decode('latin-1')!r} chunk at byte {at}: {want} bytes needed")


def _missing(cid: str, data: bytes, p: int, endian: str):
    """ValueError for a required chunk that was not found: names the chunk whose declared size ran past the end of the file, if one did."""
    while p + 8 <= len(data):
        size = struct.unpack_from(endian + "I", data, p + 4)[0]
        if p + 8 + size > len(data):
            return ValueError(f"no {cid} chunk: the {data[p:p + 4].decode('latin-1')!r} chunk at byte {p} runs past the end of the file")
        p += 8 + size + (size & 1)
    if p < len(data):
        return ValueError(f"no {cid} chunk: truncated chunk header at byte {p}")
    return ValueError(f"no {cid} chunk")


def _parse_wav(data: bytes):
    rf64 = data[:4] == b"RF64"
    info = dict(container="RF64" if rf64 else "WAV", warnings=[])
    ds64_data = fmt = None
    for cid, at, body, size in _chunks(data, 12, "<", b"data"):
        if cid == b"ds64":
            _need(cid, at, body, size, 24, data)
            ds64_data = struct.unpack_from("<Q", data, body + 8)[0]
        elif cid == b"fmt ":
            _need(cid, at, body, size, 16, data)
            tag, channels, rate, _, align, bits = struct.unpack_from("<HHIIHH", data, body)
            if tag == 0xFFFE:
                _need(cid, at, body, size, 40, data)
                guid = data[body + 24:body + 40]
                if guid[2:] != _GUID_TAIL:
                    raise NotImplementedError(f"WAVE_FORMAT_EXTENSIBLE sub-format {guid.hex()} is not PCM or IEEE float")
                tag = struct.unpack_from("<H", guid)[0]
            fmt = (tag, channels, rate, align, bits, at)
        elif cid == b"data" and "begin" not in info:
            if fmt is None:
                raise ValueError(f"'data' chunk at byte {at} before any 'fmt ' chunk")
            if rf64 and size == 0xFFFFFFFF:
                if ds64_data is None:
                    raise ValueError(f"RF64 'data' chunk at byte {at} without a 'ds64' chunk")
                size = ds64_data
            streamed = size in (0, 0xFFFFFFFF)
            end = len(data) if streamed else body + size
            info["begin"] = body
            if end > len(data):
                info["warnings"].append(f"'data' chunk at byte {at} declares {size} bytes, the file holds {len(data) - body}")
                end = len(data)
            info["end"] = end
            if streamed or end == len(data):
                break
    if fmt is None:
        raise _missing("'fmt '", data, 12, "<")
    if "begin" not in info:
        raise _missing("'data'", data, 12, "<")
    tag, channels, rate, align, bits, at = fmt
    if tag == 1:
        if not 1 <= bits <= 32:
            raise ValueError(f"'fmt ' chunk at byte {at}: {bits}-bit integer PCM has no libsndfile subtype")
        fmt_code = (U8, S16LE, S24LE, S32LE)[(bits + 7) // 8 - 1]
    elif tag == 3:
        if bits not in (32, 64):
            raise ValueError(f"'fmt ' chunk at byte {at}: {bits}-bit IEEE float")
        fmt_code = F32LE if bits == 32 else F64LE
    else:
        raise NotImplementedError(f"WAV format tag 0x{tag:04x} is compressed or not PCM (only PCM and IEEE float are decoded)")
    info.update(format=fmt_code, channels=channels, sample_rate=rate, block_align=align)
    _check_frame(info, f"'fmt ' chunk at byte {at}")
    return info


def extended_to_rate(b: bytes) -> int:
    """The 80-bit IEEE 754 extended sample rate of a COMM chunk, as libsndfile's integer rate (the value truncated toward zero).
    Raises ValueError for zero, negative, infinite or NaN values."""
    se, mant = struct.unpack(">HQ", b)
    exp = se & 0x7FFF
    if se & 0x8000 or exp == 0x7FFF or mant == 0:
        raise ValueError(f"invalid sample rate {b.hex()}")
    shift = exp - 16383 - 63
    return mant << shift if shift >= 0 else mant >> -shift


def _parse_aiff(data: bytes):
    aifc = data[8:12] == b"AIFC"
    info = dict(container="AIFC" if aifc else "AIFF", warnings=[])
    comm = ssnd = None
    for cid, at, body, size in _chunks(data, 12, ">", b"SSND"):
        if cid == b"COMM":
            _need(cid, at, body, size, 22 if aifc else 18, data)
            channels, frames, bits = struct.unpack_from(">HIH", data, body)
            comp = data[body + 18:body + 22] if aifc else b"NONE"
            comm = (channels, frames, bits, extended_to_rate(data[body + 8:body + 18]), comp, at)
        elif cid == b"SSND" and ssnd is None:
            _need(cid, at, body, size, 8, data)
            offset, block = struct.unpack_from(">II", data, body)
            if offset > size - 8:
                raise ValueError(f"'SSND' chunk at byte {at}: offset {offset} beyond its {size - 8} bytes")
            ssnd = (body + 8 + offset, body + size, at, block)
    if comm is None:
        raise _missing("'COMM'", data, 12, ">")
    if ssnd is None:
        raise _missing("'SSND'", data, 12, ">")
    channels, frames, bits, rate, comp, at = comm
    kind = _AIFC.get(comp)
    if kind is None:
        raise NotImplementedError(f"AIFF-C compression type {comp!r} is not decoded (only uncompressed PCM and float)")
    if kind == U8 and bits != 8:
        raise NotImplementedError(f"AIFF-C 'raw ' at {bits} bits: only 8-bit unsigned PCM is decoded")
    if isinstance(kind, tuple):
        if not 1 <= bits <= 32:
            raise ValueError(f"'COMM' chunk at byte {at}: {bits}-bit PCM has no libsndfile subtype")
        kind = kind[(bits + 7) // 8 - 1]
    begin, end, ssnd_at, block = ssnd
    if end > len(data):
        begin, end = min(begin, len(data)), len(data)
        info["warnings"].append(f"'SSND' chunk at byte {ssnd_at} declares {ssnd[1] - ssnd[0]} sample bytes, the file holds {end - begin}")
    info.update(format=kind, channels=channels, sample_rate=rate, block_align=channels * SAMPLE_BYTES[kind], begin=begin, end=end, block_size=block,
                compression=comp.decode("latin-1"))
    _check_frame(info, f"'COMM' chunk at byte {at}")
    if info["n_frames"] != frames:
        info["warnings"].append(f"'COMM' declares {frames} sample frames, 'SSND' holds {info['n_frames']}")
    return info


def _check_frame(info, where):
    ch, align, b = info["channels"], info["block_align"], SAMPLE_BYTES[info["format"]]
    if ch < 1:
        raise ValueError(f"{where}: {ch} channels")
    if info["sample_rate"] < 1:
        raise ValueError(f"{where}: sample rate {info['sample_rate']}")
    if align < ch * b or align > MAX_FRAME_BYTES:
        raise ValueError(f"{where}: impossible block align {align} for {ch} channels of {b} bytes")
    info["n_frames"] = (info["end"] - info["begin"]) // align


def parse(data: bytes) -> dict:
    """Container of a WAV / RF64 / AIFF / AIFF-C file -> info: format (a b200sep_pcm_decode_f32 code), channels, sample_rate, block_align, the
    payload's byte range [begin, end) and n_frames (whole frames in it), the container, and warnings (a declared size the file does not hold).  Raises ValueError naming the chunk and byte offset for a malformed container, NotImplementedError for a
    compressed payload."""
    if len(data) < 12:
        raise ValueError(f"truncated header: {len(data)} bytes")
    if not is_pcm_container(data[:12]):
        raise ValueError("not a RIFF/WAVE, RF64 or FORM/AIFF container")
    return _parse_wav(data) if data[:4] != b"FORM" else _parse_aiff(data)


def input_bit_depth(info):
    """(input_bit_depth, input_subtype): the subtype libsndfile reports and the bit depth the reference maps it to; PCM_U8 is not in the reference's
    table and gets its 16-bit default."""
    sub = SUBTYPE[info["format"]]
    return BIT_DEPTH[sub], sub


def decode(data: bytes, device="cuda"):
    """Whole file -> ((min(channels, 2), N) float32 tensor on `device`, info).  Only the payload is uploaded, once, from a page-locked buffer;
    one kernel converts it (b200sep_pcm_decode_f32)."""
    info = parse(data)
    n, align = info["n_frames"], info["block_align"]
    nbytes = n * align
    dev = torch.device(device)
    host = torch.empty(max(16, (nbytes + 15) // 16 * 16), dtype=torch.uint8, pin_memory=True)
    h = host.numpy()
    h[:nbytes] = np.frombuffer(data, np.uint8, nbytes, info["begin"])
    h[nbytes:] = 0
    buf = host.to(dev, non_blocking=True)
    oc = min(info["channels"], 2)
    out = torch.empty((oc, n), dtype=torch.float32, device=dev)
    check(lib.b200sep_pcm_decode_f32(buf.data_ptr(), n, align, info["channels"], info["format"], oc, out.data_ptr(), n,
                                     torch.cuda.current_stream(dev).cuda_stream), "pcm_decode_f32")
    info["bytes_uploaded"] = nbytes
    return out, info
