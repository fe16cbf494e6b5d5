"""Pin the reference's resampling glue and write tests/golden/pitch_small.npz and tests/golden/vr_rates_small.npz (build container only;
see oracle/ref_shim.py).

  * MDXC pitch_shift: the reference's own MDXCSeparator.demix with pitch_shift in {-3, +2}, for a tiny TFC_TDF_net (two stems) and a tiny
    BS-Roformer (single target + residual) -- change_pitch_semitones, the chunk loop on the pitched length, pitch_fix, match_array_shapes,
    the residual (mdxc_separator.py:230-244, :268-270, :406-468).
  * VR at 32 / 48 kHz: the reference's VRSeparator.loading_mix / inference_vr / spec_to_wav and the final resample to 44.1 kHz
    (vr_separator.py:221-222, :239-240, :255-293) for tiny nets on 2band_32000, 2band_48000 and 1band_sr32000_hl512.

librosa is absent here: librosa.resample / librosa.load are served by oracle/resample_oracle.py, dispatched on res_type (polyphase =
scipy.signal.resample_poly), the way make_golden_vr.py injects its resampler; the synthesis-side band up-sampling of cmb_spectrogram_to_wave
runs the Kaiser polyphase stand-in (vr_oracle.upsample), as the product does.  Each reference result is asserted equal to the oracle
composition.  These goldens pin the reference's glue (order, lengths, match_array_shapes, residual, band chain); the resampler itself is
pinned only to its own restatement (no soxr / libsamplerate here)."""
import json
import logging
import math
import os
import sys
import types

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import mdx_oracle as M  # noqa: E402
import mdxc_oracle as X  # noqa: E402
import ref_shim  # noqa: E402
import resample_oracle as RO  # noqa: E402
import roformer_oracle as R  # noqa: E402
import vr_oracle as V  # noqa: E402
from make_golden_mdxc import SMALL as MDXC_SMALL, ref_cfg, ref_net as mdxc_ref_net  # noqa: E402
from make_golden_roformer import SMALL as RF_SMALL, ref_model as rf_ref_model  # noqa: E402
from make_golden_vr import check, librosa_stub, ref_net as vr_ref_net, ref_separator  # noqa: E402

GOLD = os.path.join(os.path.dirname(HERE), "tests", "golden")
PITCHES = (-3, 2)
VR_PARAMS = ("2band_32000", "2band_48000", "1band_sr32000_hl512")
REF_PARAMS = os.path.join(ref_shim.REF_ROOT, "audio_separator", "separator", "uvr_lib_v5", "vr_network", "modelparams")


class AD(dict):
    __getattr__ = dict.__getitem__


def pcm_wave(n, seed):
    """a 16-bit-exact stereo test signal: what a plugin reads back from the PCM_16 WAV the GPU test writes"""
    return (np.round(M.synth_music(n, seed=seed) * 32767).astype(np.int16).astype(np.float32) / 32768.0).astype(np.float32)


def rf_cfg(**kw):
    return R.BSRoformerConfig(**dict(RF_SMALL, **kw))


# ------------------------------------------------------------------------------------------------ oracle compositions (also run by the CPU test)
def pitch_demix(mix, s, demix_fn, n_stems_out):
    """MDXCSeparator.demix with pitch_shift = s: pitched mix -> chunk loop -> every stem pitched back and fitted to N -> (rows, 2, N)."""
    (a, b), (c, d) = RO.pitch_rates(44100, s)
    stems = demix_fn(RO.resample(mix, a, b, "sinc_fastest"))[:n_stems_out]
    return np.stack([RO.match_array_shapes(RO.resample(st, c, d, "sinc_fastest"), mix.shape[1]) for st in stems])


def vr_param(name):
    """the product's built-in copy of modelparams/<name>.json (main() checks it against the reference's file)"""
    import importlib.util

    spec = importlib.util.spec_from_file_location("b200_vr_params", os.path.join(os.path.dirname(HERE), "python-audio-separator_b200", "audio_separator", "separator",
                                                                                  "b200", "vr_params.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod.normalise(mod.BUILTIN[name])


def vr_loading_mix(wave44, p):
    """librosa.load(sr=top band) + VRSeparator.loading_mix with every band's res_type -> (2, bins+1, frames) c64"""
    n = len(p["band"])
    waves, specs = {}, {}
    for d in range(n, 0, -1):
        bp = p["band"][d]
        waves[d] = RO.resample(wave44, 44100, bp["sr"], bp["res_type"]) if d == n else RO.resample(waves[d + 1], p["band"][d + 1]["sr"], bp["sr"], bp["res_type"])
        specs[d] = V.wave_to_spectrogram(waves[d], bp["hl"], bp["n_fft"], p, False, d)
    return V.combine_spectrograms(specs, p)


def vr_stem(spec, p):
    """spec_to_wav (stand-in band up-sampler) + librosa.resample(model sr -> 44100, soxr_hq)"""
    return RO.resample(V.cmb_spectrogram_to_wave(np.nan_to_num(spec), p).astype(np.float32), p["sr"], 44100, "soxr_hq")


def vr_cfg(p):
    return V.VRConfig(param=p, nn_architecture=31191, window_size=272, aggression=5, primary_stem="Instrumental")


def vr_separate(wave44, p, w):
    """VRSeparator.separate of a 44.1 kHz mix with a model at p["sr"]: loading_mix, inference_vr, both stems back at 44.1 kHz -> (primary, secondary)"""
    cfg = vr_cfg(p)
    y, v = V.inference_vr(vr_loading_mix(wave44, p), cfg, lambda b: V.predict_mask(w, cfg, b), batch_size=2)
    return vr_stem(y, p), vr_stem(v, p)


# ------------------------------------------------------------------------------------------------ reference runs
def mdxc_pitch(out):
    ms = ref_shim.ref_module("audio_separator.separator.architectures.mdxc_separator")
    su = ref_shim.ref_module("audio_separator.separator.uvr_lib_v5.spec_utils")
    assert su.wav_resolution_float_resampling == "sinc_fastest"
    su.librosa = types.SimpleNamespace(resample=lambda y, orig_sr, target_sr, res_type="soxr_hq": RO.resample(y, orig_sr, target_sr, res_type))
    mix = M.normalize(pcm_wave(9000, 77), 0.9, 0.0)
    out.update(mix_seed=77, n_samples=9000)
    # TFC_TDF_net, two stems, no target instrument
    cfg = X.MDXCConfig(**MDXC_SMALL)
    gain = float(np.load(os.path.join(GOLD, "mdxc_small.npz"))["out_gain"])
    w = X.make_weights(cfg, seed=3, out_gain=gain)
    net = mdxc_ref_net(cfg, w)
    # Roformer, single target (Vocals) with the residual
    rcfg = rf_cfg(overlap=2)
    rw = R.make_weights(rcfg, seed=3)
    rmodel = rf_ref_model(rcfg, rw)
    out.update(tfc_weights_seed=3, tfc_out_gain=np.float64(gain), rf_weights_seed=3, rf_overlap=2)
    for s in PITCHES:
        sep = object.__new__(ms.MDXCSeparator)
        sep.logger = logging.getLogger("ref")
        sep.is_roformer, sep.model_run, sep.override_model_segment_size = False, net, False
        sep.model_data_cfgdict = ref_cfg(cfg)
        sep.overlap, sep.batch_size, sep.torch_device, sep.sample_rate = cfg.overlap, 2, torch.device("cpu"), 44100
        sep.pitch_shift, sep.is_primary_stem_main_target = s, False
        sep.primary_stem_name, sep.secondary_stem_name = "Vocals", "Instrumental"
        src = sep.demix(mix.copy())
        ref = np.stack([src[k] for k in cfg.instruments])
        orc = pitch_demix(mix, s, lambda m: X.demix(m, cfg, lambda x: X.net_forward(w, cfg, x)), 2)
        check(f"MDXC TFC demix pitch_shift={s:+d}", ref, orc, 2e-5)
        out[f"tfc_pitch{s:+d}"] = ref.astype(np.float32)

        sep = object.__new__(ms.MDXCSeparator)
        sep.logger = logging.getLogger("ref")
        sep.pitch_shift, sep.is_roformer, sep.override_model_segment_size = s, True, False
        sep.overlap, sep.sample_rate = rcfg.overlap, 44100
        sep.model_run = rmodel
        sep.model_data_cfgdict = AD(inference=AD(dim_t=rcfg.dim_t), model=AD(stft_hop_length=rcfg.stft_hop_length), audio=AD(sample_rate=44100, hop_length=rcfg.stft_hop_length),
                                    training=AD(instruments=["Vocals", "Instrumental"], target_instrument="Vocals"))
        sep.is_primary_stem_main_target = True
        sep.primary_stem_name, sep.secondary_stem_name = "Vocals", "Instrumental"
        src = sep.demix(mix.copy())
        ref = np.stack([src["Vocals"], src["Instrumental"]])
        prim = pitch_demix(mix, s, lambda m: R.demix(m, rcfg, lambda c: R.forward(rw, rcfg, c), n_instruments=2), 1)[0]
        check(f"MDXC BS-Roformer demix pitch_shift={s:+d} (primary, residual)", ref, np.stack([prim, mix - prim]), 2e-5)
        out[f"rf_pitch{s:+d}"] = ref.astype(np.float32)


def vr_rates(out):
    librosa_stub()
    su = ref_shim.ref_module("audio_separator.separator.uvr_lib_v5.spec_utils")
    vs = ref_shim.ref_module("audio_separator.separator.architectures.vr_separator")
    # vr_separator's librosa (load / resample of the analysis bands / the final resample): the resampler oracle; spec_utils' librosa (band
    # up-sampling of cmb_spectrogram_to_wave): the Kaiser polyphase stand-in the product runs there
    lib_vr = sys.modules["librosa"]
    lib_vr.resample = lambda y, orig_sr, target_sr, res_type="soxr_hq": RO.resample(y, orig_sr, target_sr, res_type)
    su.librosa = types.SimpleNamespace(stft=lib_vr.stft, istft=lib_vr.istft, resample=lambda y, orig_sr, target_sr, res_type: V.upsample(y, orig_sr, target_sr))
    wave = pcm_wave(8000, 61)
    out.update(wave_seed=61, n_samples=8000)
    arch = 31191
    for i, name in enumerate(VR_PARAMS):
        p = vr_param(name)
        with open(os.path.join(REF_PARAMS, f"{name}.json")) as f:
            ref_p = json.load(f)
        assert p == {**p, **{k: v for k, v in ref_p.items() if k != "band"}} and p["band"] == {int(k): v for k, v in ref_p["band"].items()}, name
        w = V.make_weights(arch, seed=11 + i)
        net = vr_ref_net(arch, p["bins"] * 2, w)
        sep = ref_separator(vr_cfg(p), net, wave)
        sep.model_samplerate = p["sr"]
        vs.librosa.load = lambda f, sr, mono, dtype, res_type: (RO.resample(wave, 44100, sr, res_type), sr)
        X_ref = sep.loading_mix()
        check(f"VR {name}: loading_mix (load at {p['sr']} Hz + band chain)", X_ref, vr_loading_mix(wave, p), 1e-4)
        y_ref, v_ref = sep.inference_vr(X_ref.copy(), "cpu", sep.aggressiveness)
        stems = []
        for spec in (y_ref, v_ref):  # vr_separator.py:217-222 / :235-240
            st = sep.spec_to_wav(spec).T
            st = vs.librosa.resample(st.T, orig_sr=sep.model_samplerate, target_sr=44100).T
            stems.append(st.T)
        for k, (st, st_orc) in enumerate(zip(stems, vr_separate(wave, p, w))):
            check(f"VR {name}: {'primary' if k == 0 else 'secondary'} stem at 44.1 kHz", st, st_orc, 2e-5)
            assert st.shape == (2, math.ceil(p["band"][len(p["band"])]["hl"] * (y_ref.shape[2] - 1) * 44100 / p["sr"])), st.shape
        # only the stems are stored (the spectrograms would make the file several times larger); the CPU test recomputes them from the seeds
        out.update({f"{name}_weights_seed": 11 + i, f"{name}_frames": y_ref.shape[2], f"{name}_primary": stems[0].astype(np.float32),
                    f"{name}_secondary": stems[1].astype(np.float32)})


def main():
    ref_shim.install()
    pitch, vr = {}, {}
    mdxc_pitch(pitch)
    vr_rates(vr)
    np.savez_compressed(os.path.join(GOLD, "pitch_small.npz"), **pitch)
    np.savez_compressed(os.path.join(GOLD, "vr_rates_small.npz"), **vr)
    print("wrote tests/golden/pitch_small.npz and tests/golden/vr_rates_small.npz; reference glue pinned: OK (resampler: pinned to its restatement only)")


if __name__ == "__main__":
    main()
