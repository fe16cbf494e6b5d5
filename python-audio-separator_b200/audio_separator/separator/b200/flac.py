"""FLAC (RFC 9639) output of a normalised stereo stem, and FLAC input decoded on the GPU.

Output: the frames are encoded on the GPU (csrc/flac.cu: predictor search, residuals, Rice coding, bit packing and CRCs per 4096-sample block), so only the
compressed bytes cross to the host, in one copy.  This module adds the `fLaC` marker and one STREAMINFO block in front of them; no Vorbis comment,
seek table or padding.  The STREAMINFO MD5 is written as zero, which RFC 9639 defines as "not computed": the MD5 of the PCM is one serial chain over
the whole track, which would need the PCM on the host or a serial GPU kernel (DESIGN.md section 23).

Input: the host parses the container (an optional ID3v2 tag, `fLaC`, the metadata blocks, a trailing ID3v1 tag) and uploads only the frame bytes;
csrc/flac_decode.cu finds the frames and decodes them into the planar float mix (DESIGN.md section 24).
"""
import struct

import numpy as np

import torch

from ._lib import B200SepError, check, lib

BLOCK_SIZE = 4096


def stream_bps(bits: int, use_soundfile: bool):
    """Sample size of the FLAC stream the reference's writers store for output at `bits` bits (common_separator.py:302-451), or None when the writer
    cannot store it.  pydub / ffmpeg (the default): 16 -> 16, 24 -> 24, and 32 -> 24, because ffmpeg's FLAC encoder stores s32 input at 24 bits.
    libsndfile: 16 -> 16, 24 -> 24, and no 32-bit FLAC (the reference logs the error and writes no file)."""
    if bits in (16, 24):
        return bits
    if bits == 32:
        return None if use_soundfile else 24
    raise ValueError(f"no FLAC rule for {bits}-bit output")


def streaminfo(sample_rate: int, bps: int, total_samples: int, min_frame: int, max_frame: int, channels: int = 2) -> bytes:
    """The 34-byte STREAMINFO body: fixed block size BLOCK_SIZE (a shorter last block is allowed), the frame sizes in bytes, MD5 all zero."""
    if not (0 < sample_rate < 1 << 20 and 4 <= bps <= 32 and 0 <= total_samples < 1 << 36 and 0 <= min_frame < 1 << 24 and 0 <= max_frame < 1 << 24):
        raise ValueError("STREAMINFO field out of range")
    packed = (sample_rate << 44) | ((channels - 1) << 41) | ((bps - 1) << 36) | total_samples
    return struct.pack(">HH", BLOCK_SIZE, BLOCK_SIZE) + min_frame.to_bytes(3, "big") + max_frame.to_bytes(3, "big") + packed.to_bytes(8, "big") + bytes(16)


def stream_header(sample_rate: int, bps: int, total_samples: int, min_frame: int, max_frame: int) -> bytes:
    """`fLaC` + the STREAMINFO metadata block with the last-metadata-block flag set."""
    body = streaminfo(sample_rate, bps, total_samples, min_frame, max_frame)
    return b"fLaC" + bytes([0x80]) + len(body).to_bytes(3, "big") + body


def encode(x: torch.Tensor, bits: int, via_int16: bool, bps: int, sample_rate: int) -> bytes:
    """Whole FLAC file of the normalised (N, 2) float32 CUDA stem `x`.  Samples are quantised like the WAV writer at `bits` bits
    (b200sep_to_pcm_bytes with the same via_int16) and stored at `bps` bits."""
    if not (x.is_cuda and x.dtype == torch.float32 and x.dim() == 2 and x.shape[1] == 2):
        raise ValueError("FLAC encoding takes a (N, 2) float32 CUDA stem")
    x = x.contiguous()
    n = int(x.shape[0])
    stream = torch.cuda.current_stream(x.device).cuda_stream
    work = torch.empty(max(1, lib.b200sep_flac_work_bytes(n)), dtype=torch.uint8, device=x.device)
    out = torch.empty(max(1, lib.b200sep_flac_max_bytes(n, bps)), dtype=torch.uint8, device=x.device)
    result = torch.empty(4, dtype=torch.int64, device=x.device)
    check(lib.b200sep_flac_encode(x.data_ptr(), n, bits, int(via_int16), bps, sample_rate, work.data_ptr(), out.data_ptr(), result.data_ptr(), stream), "flac_encode")
    total, min_frame, max_frame, bad = result.tolist()
    if bad:
        raise B200SepError(f"flac_encode: {bad} frame(s) packed to a different size than planned")
    return stream_header(sample_rate, bps, n, min_frame, max_frame) + out[:total].cpu().numpy().tobytes()


# ---- input ---------------------------------------------------------------------------------------------------------------------------

# result[2] codes of b200sep_flac_locate / _decode (include/b200sep.h)
DECODE_ERRORS = {
    1: "no valid frame header where a frame must start",
    2: "no frame end with a matching CRC-16 (damaged or truncated)",
    3: "frame or sample number out of sequence",
    4: "reserved or invalid subframe, predictor or residual code",
    5: "the subframes do not end at the frame's CRC-16",
}


def id3v2_length(head: bytes) -> int:
    """Bytes of an ID3v2 tag at the start of `head` (header, syncsafe size, footer when its flag is set), 0 when there is none."""
    if len(head) < 10 or head[:3] != b"ID3":
        return 0
    size = head[6:10]
    if any(b & 0x80 for b in size):
        raise ValueError("malformed ID3v2 tag: size is not syncsafe")
    n = (size[0] << 21) | (size[1] << 14) | (size[2] << 7) | size[3]
    return 10 + n + (10 if head[5] & 0x10 else 0)


def is_flac(path) -> bool:
    """Content sniffing: `fLaC` at the start of the file, or after an ID3v2 tag."""
    with open(path, "rb") as f:
        head = f.read(10)
        try:
            skip = id3v2_length(head)
        except ValueError:
            return False
        if skip:
            f.seek(skip)
            return f.read(4) == b"fLaC"
    return head[:4] == b"fLaC"


def parse_streaminfo(body: bytes) -> dict:
    if len(body) != 34:
        raise ValueError(f"STREAMINFO is 34 bytes, got {len(body)}")
    x = int.from_bytes(body[10:18], "big")
    return dict(min_block=int.from_bytes(body[0:2], "big"), max_block=int.from_bytes(body[2:4], "big"), min_frame=int.from_bytes(body[4:7], "big"),
                max_frame=int.from_bytes(body[7:10], "big"), sample_rate=x >> 44, channels=((x >> 41) & 7) + 1, bps=((x >> 36) & 31) + 1,
                total_samples=x & ((1 << 36) - 1), md5=bytes(body[18:34]))


def parse(data: bytes):
    """Container of a FLAC file -> (STREAMINFO dict with the list of metadata block types under "blocks", first frame byte, end of the frames).
    Every metadata block up to the last-block flag is walked; a trailing 128-byte ID3v1 tag is excluded from the frames."""
    p = id3v2_length(data)
    if data[p:p + 4] != b"fLaC":
        raise ValueError("not a FLAC stream: no fLaC marker")
    p += 4
    info, blocks = None, []
    while True:
        if p + 4 > len(data):
            raise ValueError(f"truncated FLAC metadata at byte {p}")
        h, length = data[p], int.from_bytes(data[p + 1:p + 4], "big")
        kind = h & 0x7F
        if kind == 127:
            raise ValueError(f"invalid FLAC metadata block type 127 at byte {p}")
        if p + 4 + length > len(data):
            raise ValueError(f"truncated FLAC metadata: block type {kind} at byte {p} needs {length} bytes")
        if kind == 0:
            if info is not None:
                raise ValueError("more than one STREAMINFO block")
            info = parse_streaminfo(data[p + 4:p + 4 + length])
        blocks.append(kind)
        p += 4 + length
        if h & 0x80:
            break
    if info is None:
        raise ValueError("FLAC stream without STREAMINFO")
    end = len(data)
    if end - p >= 128 and data[end - 128:end - 125] == b"TAG":
        end -= 128
    info["blocks"] = blocks
    return info, p, end


def input_bit_depth(bps: int):
    """(input_bit_depth, input_subtype) of a FLAC stream: libsndfile reports PCM_S8 / PCM_16 / PCM_24 and the reference maps them to 16 / 16 / 24
    (common_separator.py:236-245)."""
    if not 4 <= bps <= 24:
        raise ValueError(f"no libsndfile subtype for {bps}-bit FLAC")
    return (16, "PCM_S8") if bps <= 8 else (16, "PCM_16") if bps <= 16 else (24, "PCM_24")


def _raise_on_error(r, begin):
    code = int(r[2])
    if code:
        raise ValueError(f"FLAC frame {int(r[3])} at byte {begin + int(r[4])}: {DECODE_ERRORS.get(code, f'error {code}')}")


def decode(data: bytes, device="cuda"):
    """Whole FLAC file -> ((min(channels, 2), N) float32 tensor on `device`, info).  mix[c, n] = sample[n, c] * 2^-(bps-1), exact for bps <= 24.
    N is what the frames hold (info["n_samples"]); STREAMINFO's total (info["total_samples"]) may be 0 or differ.  Only the frame bytes are uploaded,
    from a page-locked buffer.  Raises ValueError naming the frame and byte offset for a damaged or malformed stream, NotImplementedError above
    24 bits."""
    info, begin, end = parse(data)
    bps, ch, rate = info["bps"], info["channels"], info["sample_rate"]
    if bps > 24:
        raise NotImplementedError(f"{bps}-bit FLAC is not supported: libsndfile has no FLAC subtype above 24 bits")
    if bps < 4:
        raise ValueError(f"invalid FLAC sample size {bps}")
    if not 0 < rate < 1 << 20:
        raise ValueError(f"invalid FLAC sample rate {rate}")
    n = end - begin
    dev = torch.device(device)
    host = torch.empty(max(16, (n + 15) // 16 * 16), dtype=torch.uint8, pin_memory=True)
    h = host.numpy()
    h[:n] = np.frombuffer(data, np.uint8, n, begin)
    h[n:] = 0
    buf = host.to(dev, non_blocking=True)
    variable = int(data[begin + 1] & 1) if n >= 2 else 0
    work = torch.empty(max(8, lib.b200sep_flac_decode_work_bytes(n)), dtype=torch.uint8, device=dev)
    result = torch.empty(8, dtype=torch.int64, device=dev)
    stream = torch.cuda.current_stream(dev).cuda_stream
    check(lib.b200sep_flac_locate(buf.data_ptr(), n, rate, bps, ch, variable, work.data_ptr(), result.data_ptr(), stream), "flac_locate")
    r = result.tolist()
    _raise_on_error(r, begin)
    n_frames, n_samples, max_frame = r[0], r[1], r[5]
    out = torch.empty((min(ch, 2), n_samples), dtype=torch.float32, device=dev)
    check(lib.b200sep_flac_decode(buf.data_ptr(), n, work.data_ptr(), n_frames, max_frame, out.data_ptr(), n_samples, result.data_ptr(), stream),
          "flac_decode")
    _raise_on_error(result.tolist(), begin)
    info.update(n_samples=n_samples, frames=n_frames, first_number=r[6], variable_blocking=variable, bytes_uploaded=n)
    return out, info
