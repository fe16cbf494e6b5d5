"""Pin oracle/chunking_oracle.py against the UNMODIFIED reference AudioChunker and Separator._process_with_chunking and write
tests/golden/chunking.npz.

pydub is not installed, so `pydub.AudioSegment` is a restatement of the parts the reference uses (len, millisecond slicing with silence
padding, `+`, from_file / export over in-memory sample arrays); the pydub semantics themselves stay unpinned.  The separation of each chunk is
a stub `_separate_file` that returns named stems, one of them missing for one chunk (a near-silent stem the reference does not write)."""
import json
import logging
import os
import sys
import tempfile
import types

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import chunking_oracle as C  # noqa: E402

GOLD = os.path.join(os.path.dirname(HERE), "tests", "golden")
_STORE = {}  # path -> (frames, channels) int array: the "files" the restated AudioSegment reads and writes


class AudioSegment:
    """pydub.AudioSegment over (frames, channels) integer sample arrays (pydub/audio_segment.py)."""

    def __init__(self, samples, frame_rate):
        self.samples, self.frame_rate = np.asarray(samples), frame_rate

    def frame_count(self, ms=None):
        return ms * (self.frame_rate / 1000.0) if ms is not None else float(len(self.samples))

    def __len__(self):
        return round(1000 * (self.frame_count() / self.frame_rate))

    def _parse_position(self, val):
        if val < 0:
            val = len(self) - abs(val)
        return int(self.frame_count(ms=len(self)) if val == float("inf") else self.frame_count(ms=val))

    def __getitem__(self, ms):
        start = ms.start if ms.start is not None else 0
        end = ms.stop if ms.stop is not None else len(self)
        start, end = min(start, len(self)), min(end, len(self))
        start, end = self._parse_position(start), self._parse_position(end)
        data = self.samples[start:end]
        missing = (end - start) - len(data)
        if missing:
            if missing > self.frame_count(ms=2):
                raise ValueError(f"too many missing frames: {missing}")
            data = np.concatenate([data, np.zeros((missing, self.samples.shape[1]), self.samples.dtype)])
        return AudioSegment(data, self.frame_rate)

    def __add__(self, other):
        return AudioSegment(np.concatenate([self.samples, other.samples]), other.frame_rate if not len(self.samples) else self.frame_rate)

    @classmethod
    def empty(cls):
        return cls(np.zeros((0, 2), np.int32), 1)

    @classmethod
    def from_file(cls, path, *a, **k):
        return cls(*_STORE[path])

    def export(self, path, format=None, **k):
        _STORE[path] = (self.samples, self.frame_rate)
        open(path, "wb").close()


STEMS = ("Vocals", "Instrumental", "Other")


def run_reference(sep_cls, n, sr, chunk_duration, missing=(), custom=None):
    """_process_with_chunking on an n-frame 'file' whose samples are their own frame indices; stems are the chunk times 1 / 2 / 3, with
    (chunk, stem) pairs in `missing` not written.  -> ([(output name, samples)], [chunk sample ranges as seen by the stub])."""
    with tempfile.TemporaryDirectory() as out_dir:
        src = os.path.join(out_dir, "long mix.wav")
        AudioSegment(np.stack([np.arange(n), -np.arange(n)], axis=1).astype(np.int64), sr).export(src)
        sep = sep_cls.__new__(sep_cls)
        sep.logger, sep.chunk_duration, sep.output_dir, sep.output_format, sep.model_instance = logging.getLogger("ref"), chunk_duration, out_dir, "WAV", None
        seen = []

        def separate_file(chunk_path, custom_output_names=None):
            samples, rate = _STORE[chunk_path]
            i = len(seen)
            seen.append(samples[:, 0].copy())
            names = []
            for k, stem in enumerate(STEMS):
                if (i, stem) in missing:
                    continue
                name = f"{os.path.splitext(os.path.basename(chunk_path))[0]}_({stem})_model.wav"
                AudioSegment(samples * (k + 1), rate).export(os.path.join(sep.output_dir, name))
                names.append(name)
            return names

        sep._separate_file = separate_file
        paths = sep._process_with_chunking(src, custom)
        return [(os.path.basename(p), _STORE[p][0]) for p in paths], seen


def main():
    sys.modules["pydub"] = types.SimpleNamespace(AudioSegment=AudioSegment)
    import ref_shim

    ref_shim.install()
    chunker_mod = ref_shim.ref_module("audio_separator.separator.audio_chunking")
    sep_cls = ref_shim.ref_module("audio_separator.separator.separator").Separator
    # (frames, rate, chunk_duration): fractional durations, 1-frame remainders, int(ms * sr / 1000.0) rounding down, padded last slices
    table = [(44100 * 10, 44100, 3), (44100 * 10 + 1, 44100, 3), (44100 * 9, 44100, 3), (44100 * 9 + 1, 44100, 3), (44100 * 9 - 1, 44100, 3),
             (123457, 44100, 0.7), (123457, 44100, 1.2345), (100003, 48000, 0.5), (88200 + 22, 44100, 1), (88200 + 23, 44100, 1),
             (99999, 44100, 0.333), (70001, 32000, 0.25), (44100 * 2 + 7, 44100, 0.1), (1000, 44100, 0.01), (220501, 44100, 2.5)]
    bounds, counts = [], []
    for n, sr, cd in table:
        ch = chunker_mod.AudioChunker(cd, logging.getLogger("ref"))
        assert ch.should_chunk(n / sr) == C.should_chunk(n, sr, cd), (n, sr, cd)
        outs, seen = run_reference(sep_cls, n, sr, cd)
        ours = C.boundaries(n, sr, cd)
        assert len(seen) == len(ours), (n, sr, cd, len(seen), len(ours))
        for (s_ms, e_ms, a, b), got in zip(ours, seen):
            want = np.concatenate([np.arange(a, min(b, n)), np.zeros(max(0, b - n), np.int64)])
            assert np.array_equal(got, want), (n, sr, cd, a, b)
        for _, samples in outs:  # plain concatenation of the chunk stems
            assert len(samples) == sum(b - a for _, _, a, b in ours)
        bounds.append(np.array([[a, b] for _, _, a, b in ours], np.int64).reshape(-1, 2))
        counts.append(len(ours))
    # should_chunk at the boundary: duration == chunk_duration does not chunk
    for n, sr, cd in ((44100 * 3, 44100, 3), (44100 * 3 + 1, 44100, 3), (48000, 48000, 1.0), (22050, 44100, 0.5)):
        assert chunker_mod.AudioChunker(cd).should_chunk(n / sr) == C.should_chunk(n, sr, cd)
    # grouping, sorted order, names (custom names included), a missing chunk stem
    cases = [dict(missing=(), custom=None), dict(missing=((1, "Other"),), custom=None), dict(missing=((0, "Vocals"), (2, "Vocals")), custom={"Vocals": "lead", "other": "x"})]
    names = []
    n, sr, cd = 44100 * 3 + 500, 44100, 1
    for case in cases:
        outs, seen = run_reference(sep_cls, n, sr, cd, missing=case["missing"], custom=case["custom"])
        ours = C.group_and_name([[f"chunk_{i:04d}_({s})_model.wav" for s in STEMS if (i, s) not in case["missing"]] for i in range(len(seen))],
                                "long mix", "wav", case["custom"])
        assert [o[0] for o in outs] == [o[0] for o in ours], (outs, ours)
        b = C.boundaries(n, sr, cd)
        for (name, samples), (_, members) in zip(outs, ours):
            assert len(samples) == sum(b[i][3] - b[i][2] for i in members)
        names.append([[nm, members] for nm, members in ours])
    np.savez_compressed(os.path.join(GOLD, "chunking.npz"), table=np.array(table, dtype=np.float64), counts=np.array(counts, np.int64),
                        bounds=np.concatenate(bounds), names=np.array(json.dumps({"n": n, "sr": sr, "chunk_duration": cd, "cases": cases, "out": names},
                                                                                   default=list)))
    print("wrote tests/golden/chunking.npz; oracle pinned: OK")


if __name__ == "__main__":
    main()
