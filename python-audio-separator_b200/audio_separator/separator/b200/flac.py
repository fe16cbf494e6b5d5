"""FLAC output (RFC 9639) of a normalised stereo stem.

The frames are encoded on the GPU (csrc/flac.cu: predictor search, residuals, Rice coding, bit packing and CRCs per 4096-sample block), so only the
compressed bytes cross to the host, in one copy.  This module adds the `fLaC` marker and one STREAMINFO block in front of them; no Vorbis comment,
seek table or padding.  The STREAMINFO MD5 is written as zero, which RFC 9639 defines as "not computed": the MD5 of the PCM is one serial chain over
the whole track, which would need the PCM on the host or a serial GPU kernel (DESIGN.md section 23).
"""
import struct

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
