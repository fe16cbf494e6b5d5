"""File-level chunking rules of `Separator(chunk_duration=...)` (the reference's AudioChunker and Separator._process_with_chunking,
audio_chunking.py, separator.py:1003-1012, :1047-1156).  Host arithmetic only (stdlib), so the CPU tests import it.

The reference cuts the file with pydub, whose slicing works in milliseconds: `len(seg)` is round(1000 * (frames / rate)), a millisecond
position maps to frame int(ms * (rate / 1000.0)), and a slice that ends past the data is padded with silence.  pydub is not pinned here
(DESIGN §28), these rules restate its published source.
"""
import re


def chunk_ms(chunk_duration) -> int:
    """AudioChunker.chunk_duration_ms."""
    return int(chunk_duration * 1000)


def should_chunk(n_frames: int, sample_rate: int, chunk_duration) -> bool:
    """AudioChunker.should_chunk(duration) with duration = frames / rate (librosa.get_duration)."""
    return n_frames / sample_rate > chunk_ms(chunk_duration) / 1000


def total_ms(n_frames: int, sample_rate: int) -> int:
    """pydub AudioSegment.__len__."""
    return round(1000 * (float(n_frames) / sample_rate))


def ms_to_frame(ms: int, sample_rate: int) -> int:
    """pydub AudioSegment._parse_position (frame_count(ms) truncated)."""
    return int(ms * (sample_rate / 1000.0))


def chunk_bounds(n_frames: int, sample_rate: int, chunk_duration) -> list:
    """[(start_frame, end_frame)] of every chunk, as AudioChunker.split_audio slices the file.  end_frame may exceed n_frames by less than
    a millisecond of frames: those frames are silence (pydub pads a short slice)."""
    cm, t = chunk_ms(chunk_duration), total_ms(n_frames, sample_rate)
    bounds = []
    for i in range((t + cm - 1) // cm):
        start = i * cm
        end = min(start + cm, t)
        bounds.append((ms_to_frame(start, sample_rate), ms_to_frame(end, sample_rate)))
    return bounds


def stem_key(filename: str):
    """The stem name a chunk's output file is grouped under: the text inside `_(...)` of its name (None when there is none)."""
    m = re.search(r"_\(([^)]+)\)", filename)
    return m.group(1) if m else None


def joined_name(base: str, key: str, ext: str, custom_output_names=None) -> str:
    """File name of a joined stem: `{base}_({key}).{ext}`, or `{custom_output_names[key]}.{ext}` (exact key match)."""
    name = custom_output_names[key] if custom_output_names and key in custom_output_names else f"{base}_({key})"
    return f"{name}.{ext}"

