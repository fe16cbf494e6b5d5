"""CPU: the steps every architecture plugin shares live once in CommonSeparator / b200.engine -- device setup, checkpoint loading, stem output
and the peak-normalisation scale rule."""
import glob
import logging
import os

import numpy as np
import pytest
import torch

import mdx_oracle as O
from conftest import ROOT

PKG = os.path.join(ROOT, "python-audio-separator_b200", "audio_separator")


def _sources():
    return {os.path.relpath(p, PKG): open(p).read() for p in glob.glob(os.path.join(PKG, "**", "*.py"), recursive=True)}


def test_shared_steps_have_one_copy():
    src = _sources()
    assert sorted(f for f, s in src.items() if '"b200_sharded"' in s) == [os.path.join("separator", "common_separator.py")]
    assert sum(s.count("lib.b200sep_normalize(") for s in src.values()) == 1
    plugins = {f: s for f, s in src.items() if f.startswith(os.path.join("separator", "architectures", ""))}
    assert len(plugins) == 5  # __init__ + MDX, MDXC, VR, Demucs
    for f, s in plugins.items():
        for step in ("dist.is_initialized", "torch.load", "np.load(", "get_stem_output_path"):
            assert step not in s, f"{f} has its own copy of {step}"


@pytest.mark.parametrize("peak,max_peak,min_peak,scale", [
    (1.8, 0.9, 0.0, 0.5),      # above max_peak: attenuate to max_peak
    (1.8, 0.9, None, 0.5),
    (0.25, 0.9, 0.5, 2.0),     # below min_peak: amplify to min_peak
    (0.25, 0.9, None, 1.0),    # min_peak None: never amplify
    (0.25, 0.9, 0.0, 1.0),
    (0.9, 0.9, 0.5, 1.0),      # at max_peak: unchanged
    (0.5, 0.9, 0.5, 1.0),      # at min_peak: unchanged
    (0.0, 0.9, 0.5, 1.0),      # silent with min_peak > 0: left as it is (no division by a zero peak)
    (0.0, 0.9, None, 1.0),
])
def test_normalize_scale(lib_built, peak, max_peak, min_peak, scale):
    from audio_separator.separator.b200.engine import normalize_scale

    assert normalize_scale(peak, max_peak, min_peak) == scale
    if peak > 0:  # the factor the numpy normalize applies to a host array of that peak
        x = np.array([peak, -peak / 2], dtype=np.float64)
        assert np.allclose(O.normalize(x.copy(), max_peak, min_peak), x * scale, rtol=1e-12)


def _common(tmp_path, **kw):
    from audio_separator.separator.common_separator import CommonSeparator

    cfg = dict(logger=logging.getLogger("t"), log_level=20, model_name="tiny", model_path="/x/tiny.npz", model_data={"primary_stem": "Vocals"},
               output_dir=str(tmp_path), output_format="WAV", normalization_threshold=0.9, amplification_threshold=0.0, sample_rate=44100)
    cfg.update(kw)
    cs = CommonSeparator(cfg)
    cs.audio_file_base = "song"
    return cs


def test_write_stems(tmp_path, lib_built):
    stems = [(name, (O.synth_music(2000, seed=i) * (0.3 + 0.2 * i)).T.copy()) for i, name in enumerate(("Instrumental", "Drums", "Vocals"))]
    cs = _common(tmp_path / "a")
    paths = cs.write_stems(stems, None)
    assert paths == ["song_(Instrumental)_tiny.wav", "song_(Drums)_tiny.wav", "song_(Vocals)_tiny.wav"]  # the caller's order
    assert (cs.primary_stem_output_path, cs.secondary_stem_output_path) == (paths[2], paths[0])
    ref = _common(tmp_path / "ref")
    for (name, src), path in zip(stems, paths):  # the bytes write_audio writes
        ref.write_audio(path, src)
        assert open(tmp_path / "a" / path, "rb").read() == open(tmp_path / "ref" / path, "rb").read()

    one = _common(tmp_path / "b", output_single_stem="drUMs")
    assert one.write_stems(stems, {"DRUMS": "kit", "vocals": "v"}) == ["kit.wav"]  # the filter and the custom names ignore case
    assert sorted(os.listdir(tmp_path / "b")) == ["kit.wav"]
    assert (one.primary_stem_output_path, one.secondary_stem_output_path) == (None, None)
    assert _common(tmp_path / "c", output_single_stem="Guitar").write_stems(stems, None) == []


def test_load_checkpoint(tmp_path):
    from audio_separator.separator.common_separator import load_checkpoint

    w = {"a.weight": np.arange(6, dtype=np.float32).reshape(2, 3) / 8, "a.num_batches_tracked": np.array(3, dtype=np.int64)}
    np.savez(tmp_path / "w.npz", **w)
    got = load_checkpoint(str(tmp_path / "w.npz"))  # as stored
    assert got.keys() == w.keys() and all(got[k].dtype == w[k].dtype and np.array_equal(got[k], w[k]) for k in w)
    sd = {k: torch.from_numpy(v) for k, v in w.items()}
    sd["a.weight"] = sd["a.weight"].half()  # fp16 -> fp32 is exact
    torch.save(sd, tmp_path / "plain.pth")
    torch.save({"state_dict": sd, "epoch": 7}, tmp_path / "train.ckpt")  # a training checkpoint: its state_dict entry
    for name in ("plain.pth", "train.ckpt"):
        got = load_checkpoint(str(tmp_path / name))
        assert got.keys() == w.keys() and all(got[k].dtype == np.float32 and np.array_equal(got[k], w[k]) for k in w)
