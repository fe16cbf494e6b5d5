"""CPU: the FLAC oracle (oracle/flac_oracle.py) against the frames of real encoders (tests/golden/flac_frames.npz, oracle/make_golden_flac.py),
STREAMINFO packing of b200/flac.py, and the sample-size rules of the FLAC writers."""
import os

import numpy as np
import pytest

import flac_oracle as F

TAGS = ("libflac16", "ffmpeg16", "ffmpeg24")


@pytest.fixture(scope="module")
def golden(golden_dir):
    return dict(np.load(os.path.join(golden_dir, "flac_frames.npz")))


@pytest.mark.parametrize("tag", TAGS)
def test_oracle_decodes_golden_frames(golden, tag):
    d = F.decode_frames(golden[f"{tag}_streaminfo"].tobytes(), golden[f"{tag}_frames"].tobytes())  # raises on any CRC mismatch
    want = golden[f"{tag}_samples"]
    assert np.array_equal(d.samples, want)
    assert sum(f[1] for f in d.frames) == int(golden[f"{tag}_encoder_bytes"]) == golden[f"{tag}_frames"].size
    assert {"LPC", "RICE"} <= d.seen
    if tag == "ffmpeg24":
        assert "wasted" in d.seen and np.all(want % 256 == 0)


def test_flipped_byte_is_a_crc_error(golden):
    si, frames = golden["libflac16_streaminfo"].tobytes(), golden["libflac16_frames"].tobytes()
    d = F.decode_frames(si, frames)
    start, length, _ = d.frames[1]
    base = start - (4 + 4 + 34)  # offsets in d.frames count the marker and the STREAMINFO block
    for pos, kind in ((base + 4, "CRC-8"), (base + length - 1, "CRC-16"), (base + length - 2, "CRC-16")):
        bad = bytearray(frames)
        bad[pos] ^= 0x10
        with pytest.raises(F.CRCError, match=kind):
            F.decode_frames(si, bytes(bad))
    bad = bytearray(frames)
    bad[base + length // 2] ^= 0x01  # inside the residual: either the frame no longer parses or its CRC-16 fails
    with pytest.raises(F.FlacError):
        F.decode_frames(si, bytes(bad))


def test_streaminfo_roundtrip(lib_built):
    from audio_separator.separator.b200 import flac

    for rate, bps, total, mn, mx in ((44100, 16, 882000, 14, 16403), (48000, 24, 1, 20, 20), (1048575, 24, (1 << 36) - 1, 0, (1 << 24) - 1)):
        head = flac.stream_header(rate, bps, total, mn, mx)
        assert head[:4] == b"fLaC" and head[4] == 0x80 and int.from_bytes(head[5:8], "big") == 34 and len(head) == 42
        info = F.parse_streaminfo(head[8:])
        assert info == dict(min_block=4096, max_block=4096, min_frame=mn, max_frame=mx, sample_rate=rate, channels=2, bps=bps, total_samples=total,
                            md5=bytes(16))
    with pytest.raises(ValueError):
        flac.streaminfo(44100, 16, 1 << 36, 0, 0)


def test_writer_sample_size_rules(lib_built):
    """The reference's writers: pydub/ffmpeg stores 16 -> 16, 24 -> 24 and 32 -> 24 bits; libsndfile 16 -> 16, 24 -> 24 and has no 32-bit FLAC."""
    from audio_separator.separator.b200 import flac

    table = {(16, False): 16, (24, False): 24, (32, False): 24, (16, True): 16, (24, True): 24, (32, True): None}
    for (bits, use_sf), want in table.items():
        assert flac.stream_bps(bits, use_sf) == want
    with pytest.raises(ValueError):
        flac.stream_bps(8, False)


def test_make_golden_flac_reruns(tmp_path, golden):
    import make_golden_flac as G

    if not G.present():
        pytest.skip("reference inputs not present")
    out = G.build(str(tmp_path / "flac_frames.npz"), verbose=False)
    assert sorted(out) == sorted(golden)
    for k, v in out.items():
        assert np.array_equal(np.asarray(v), golden[k]), k
