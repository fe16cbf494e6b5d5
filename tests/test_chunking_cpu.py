"""File-level chunking rules (b200/chunking.py) against the golden of the reference's AudioChunker / _process_with_chunking
(oracle/make_golden_chunking.py), and the `chunk_duration` / `ensemble_preset` arguments of Separator."""
import json
import os
import re

import numpy as np
import pytest

from audio_separator.separator.b200 import chunking
from audio_separator.separator.separator import Separator

GOLD = os.path.join(os.path.dirname(__file__), "golden", "chunking.npz")


@pytest.fixture(scope="module")
def gold():
    with np.load(GOLD) as z:
        return {k: z[k] for k in z.files}


def test_bounds_match_golden(gold):
    bounds = iter(gold["bounds"].tolist())
    for (n, sr, cd), count in zip(gold["table"].tolist(), gold["counts"].tolist()):
        n, sr = int(n), int(sr)
        got = chunking.chunk_bounds(n, sr, cd)
        assert len(got) == count, (n, sr, cd)
        assert [list(b) for b in got] == [next(bounds) for _ in range(count)], (n, sr, cd)
        # contiguous, and the padding past the data never exceeds pydub's 2 ms
        assert all(a1 == b0 for (_, b0), (a1, _) in zip(got, got[1:]))
        assert got[-1][1] - n <= 2 * sr / 1000


def test_grouping_and_names_match_golden(gold):
    spec = json.loads(str(gold["names"]))
    n, sr, cd = spec["n"], spec["sr"], spec["chunk_duration"]
    k = len(chunking.chunk_bounds(n, sr, cd))
    for case, want in zip(spec["cases"], spec["out"]):
        missing = {tuple(m) for m in case["missing"]}
        groups = {}
        for i in range(k):
            for stem in ("Vocals", "Instrumental", "Other"):
                if (i, stem) not in missing:
                    groups.setdefault(chunking.stem_key(f"chunk_{i:04d}_({stem})_model.wav"), []).append(i)
        got = [[chunking.joined_name("long mix", key, "wav", case["custom"]), groups[key]] for key in sorted(groups)]
        assert got == want


def test_should_chunk_boundary():
    assert not chunking.should_chunk(44100 * 3, 44100, 3)  # duration == chunk_duration: the normal path
    assert chunking.should_chunk(44100 * 3 + 1, 44100, 3)
    assert chunking.should_chunk(44100 * 3 + 1, 44100, 3.0009)  # chunk_ms truncates 3000.9 to 3000
    assert chunking.should_chunk(44100, 44100, 0.9999)  # 999 ms


def test_stem_key_and_names():
    assert chunking.stem_key("mix_(Vocals)_UVR-MDX-NET-Inst_HQ_3.wav") == "Vocals"
    assert chunking.stem_key("lead.wav") is None
    assert chunking.joined_name("song", "Vocals", "flac") == "song_(Vocals).flac"
    assert chunking.joined_name("song", "Vocals", "wav", {"Vocals": "v"}) == "v.wav"
    assert chunking.joined_name("song", "Vocals", "wav", {"vocals": "v"}) == "song_(Vocals).wav"  # exact key, as the reference


@pytest.mark.parametrize("value", [0, -1, -0.5])
def test_chunk_duration_must_be_positive(value):
    with pytest.raises(ValueError, match=re.escape("chunk_duration must be greater than 0")):
        Separator(chunk_duration=value, info_only=True)


def test_chunk_duration_accepted_and_ensemble_preset_raises():
    assert Separator(chunk_duration=600, info_only=True).chunk_duration == 600
    assert Separator(info_only=True).chunk_duration is None
    with pytest.raises(NotImplementedError):
        Separator(ensemble_preset="vocal_balanced", info_only=True)
