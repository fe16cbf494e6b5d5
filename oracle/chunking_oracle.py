"""Plain-function restatement of the reference's file-level chunking (audio_chunking.AudioChunker and Separator._process_with_chunking) over
pydub's millisecond slicing, written from pydub's published source: AudioSegment.__len__, _parse_position / frame_count, __getitem__ (pads
up to 2 ms of missing frames with silence) and `+` (append with crossfade=0).  oracle/make_golden_chunking.py pins it against the unmodified
reference code run on a restated pydub.AudioSegment."""
import math
import re


def chunk_ms(chunk_duration):
    return int(chunk_duration * 1000)


def should_chunk(n, sr, chunk_duration):
    return n / sr > chunk_ms(chunk_duration) / 1000


def pydub_len(n, sr):
    return round(1000 * (float(n) / sr))


def frame_at(ms, sr):
    return int(ms * (sr / 1000.0))


def boundaries(n, sr, chunk_duration):
    """[(start_ms, end_ms, start_frame, end_frame)] of every chunk."""
    cm, total = chunk_ms(chunk_duration), pydub_len(n, sr)
    out = []
    for i in range(math.ceil(total / cm)):
        s = i * cm
        e = min(s + cm, total)
        out.append((s, e, frame_at(s, sr), frame_at(e, sr)))
    return out


def group_and_name(chunk_outputs, base, ext, custom_output_names=None):
    """chunk_outputs: per chunk, the stem file names its separation returned.  -> [(output file name, [chunk index, ...])] in write order."""
    groups = {}
    for i, names in enumerate(chunk_outputs):
        for f in names:
            m = re.search(r"_\(([^)]+)\)", f)
            groups.setdefault(m.group(1), []).append(i)
    out = []
    for key in sorted(groups):
        name = custom_output_names[key] if custom_output_names and key in custom_output_names else f"{base}_({key})"
        out.append((f"{name}.{ext}", groups[key]))
    return out
