"""CPU: the FLAC container parser and bit-depth rules of b200/flac.py, the stream oracle (oracle/flac_stream_oracle.py) against flac_oracle, the
test writer (tests/flac_writer.py) checked by the stream oracle, and the decoder fixture (tests/golden/flac_decode.npz, oracle/make_golden_flac_decode.py)."""
import os

import numpy as np
import pytest

import flac_oracle as F
import flac_stream_oracle as S
import flac_writer as W


@pytest.fixture(scope="module")
def flac(lib_built):
    from audio_separator.separator.b200 import flac

    return flac


def _stream(**kw):
    return W.stream([W.Frame(W.signal(1000, 16, 2, 0))], 44100, 16, **kw)[0]


@pytest.mark.parametrize("footer", (False, True))
def test_parser_id3v2_and_every_block_type(flac, tmp_path, footer):
    data = _stream(blocks=(1, 2, 3, 4, 5, 6), id3v2_tag=W.id3v2(33, footer=footer), id3v1=True)
    info, begin, end = flac.parse(data)
    tag = 10 + 33 + (10 if footer else 0)
    assert data[tag:tag + 4] == b"fLaC" and flac.id3v2_length(data) == tag
    assert info["blocks"] == [0, 1, 2, 3, 4, 5, 6]
    assert (info["sample_rate"], info["bps"], info["channels"], info["total_samples"]) == (44100, 16, 2, 1000)
    assert data[begin:begin + 2] == b"\xff\xf8" and end == len(data) - 128 and data[end:end + 3] == b"TAG"
    (tmp_path / "x.bin").write_bytes(data)
    assert flac.is_flac(str(tmp_path / "x.bin"))
    (tmp_path / "y.bin").write_bytes(data[:tag] + b"RIFF" + data[tag + 4:])
    assert not flac.is_flac(str(tmp_path / "y.bin"))


def test_parser_rejects_truncated_or_unmarked_streams(flac):
    data = _stream(blocks=(4,))
    info, begin, _ = flac.parse(data)
    for cut in range(4, begin):
        with pytest.raises(ValueError, match="truncated FLAC metadata"):
            flac.parse(data[:cut])
    with pytest.raises(ValueError, match="no fLaC marker"):
        flac.parse(b"RIFF" + data[4:])
    with pytest.raises(ValueError, match="no fLaC marker"):
        flac.parse(W.id3v2(5) + b"fLa")
    no_si = b"fLaC" + W.metadata_block(1, bytes(10), True)
    with pytest.raises(ValueError, match="without STREAMINFO"):
        flac.parse(no_si)


def test_bit_depth_table(flac):
    want = {**{b: (16, "PCM_S8") for b in range(4, 9)}, **{b: (16, "PCM_16") for b in range(9, 17)}, **{b: (24, "PCM_24") for b in range(17, 25)}}
    for bps, v in want.items():
        assert flac.input_bit_depth(bps) == v
    for bps in (3, 25, 32):
        with pytest.raises(ValueError):
            flac.input_bit_depth(bps)


def _bare(data):
    """The stream without the ID3 tags around it (the oracle reads from `fLaC` to the end)."""
    if data[:3] == b"ID3":
        ss = data[6:10]
        data = data[10 + ((ss[0] << 21) | (ss[1] << 14) | (ss[2] << 7) | ss[3]) + (10 if data[5] & 0x10 else 0):]
    return data[:-128] if data[-128:-125] == b"TAG" else data


def test_writer_streams_decode_with_the_oracle():
    seen = set()
    for name, (data, want, tools) in W.cases().items():
        d = S.decode(_bare(data), first_anywhere=True)
        assert np.array_equal(d.samples, want), name
        seen |= tools
    assert W.REQUIRED_TOOLS <= seen, sorted(W.REQUIRED_TOOLS - seen)


def test_stream_oracle_agrees_with_flac_oracle(golden_dir):
    g = dict(np.load(os.path.join(golden_dir, "flac_frames.npz")))
    for tag in ("libflac16", "ffmpeg16", "ffmpeg24"):
        si, frames = g[f"{tag}_streaminfo"].tobytes(), g[f"{tag}_frames"].tobytes()
        a, b = F.decode_frames(si, frames), S.decode_frames(si, frames)
        assert np.array_equal(a.samples, b.samples) and a.frames == b.frames and a.seen <= b.seen, tag
        assert b.streaminfo["first_number"] == 0 and not b.streaminfo["variable"]
    bad = bytearray(frames)
    bad[len(bad) // 2] ^= 0x01
    with pytest.raises(F.FlacError):
        S.decode_frames(si, bytes(bad))


def test_decode_fixture_with_the_oracle(golden_dir):
    g = dict(np.load(os.path.join(golden_dir, "flac_decode.npz")))
    for tag in ("clocks", "levee", "mardy_mid", "fallen"):
        d = S.decode_frames(g[f"{tag}_streaminfo"].tobytes(), g[f"{tag}_frames"].tobytes(), first_anywhere=True)
        assert np.array_equal(d.samples, g[f"{tag}_samples"]), tag
    assert F.parse_streaminfo(g["fallen_streaminfo"].tobytes())["sample_rate"] == 96000


def test_make_golden_flac_decode_reruns(tmp_path, golden_dir):
    import make_golden_flac_decode as G

    if not G.present():
        pytest.skip("reference inputs not present")
    golden = dict(np.load(os.path.join(golden_dir, "flac_decode.npz")))
    out = G.build(str(tmp_path / "flac_decode.npz"), verbose=False)
    assert sorted(out) == sorted(golden)
    for k, v in out.items():
        assert np.array_equal(np.asarray(v), golden[k]), k
