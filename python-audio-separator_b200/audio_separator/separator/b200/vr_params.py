"""Model-parameter tables of the VR architecture (the values ModelParameters reads from uvr_lib_v5/vr_network/modelparams/<name>.json,
vr_network/model_param_init.py:40-71).  A few common layouts are built in; any other `<name>.json` is looked up next to the model file
(or in a `modelparams/` directory beside it) and normalised the same way."""
import json
import os


def _band(sr, hl, n_fft, crop_start, crop_stop, res_type, **kw):
    return dict(sr=sr, hl=hl, n_fft=n_fft, crop_start=crop_start, crop_stop=crop_stop, res_type=res_type, **kw)


def _four_band_v2(reduction_bins):
    return {"bins": 672, "unstable_bins": 8, "reduction_bins": reduction_bins, "sr": 44100, "pre_filter_start": 668, "pre_filter_stop": 672,
            "band": {1: _band(7350, 80, 640, 0, 85, "polyphase", lpf_start=25, lpf_stop=53),
                     2: _band(7350, 80, 320, 4, 87, "polyphase", hpf_start=25, hpf_stop=12, lpf_start=31, lpf_stop=62),
                     3: _band(14700, 160, 512, 17, 216, "polyphase", hpf_start=48, hpf_stop=24, lpf_start=139, lpf_stop=210),
                     4: _band(44100, 480, 960, 78, 383, "kaiser_fast", hpf_start=130, hpf_stop=86)}}


def _two_band(sr, hl, n_fft, lpf_stop, hpf_start, hpf_stop):
    """modelparams/2band_32000.json, 2band_48000.json: a 6 kHz band under the model-rate band."""
    return {"bins": 768, "unstable_bins": 7, "reduction_bins": 705, "sr": sr, "pre_filter_start": 710, "pre_filter_stop": 731,
            "band": {1: _band(6000, 66, 512, 0, 240, "sinc_fastest", lpf_start=60, lpf_stop=lpf_stop),
                     2: _band(sr, hl, n_fft, 22, 505, "sinc_medium", hpf_start=hpf_start, hpf_stop=hpf_stop)}}


def _one_band(sr, hl, res_type, pre_filter_start, pre_filter_stop):
    return {"bins": 1024, "unstable_bins": 0, "reduction_bins": 0, "sr": sr, "pre_filter_start": pre_filter_start, "pre_filter_stop": pre_filter_stop,
            "band": {1: _band(sr, hl, 2048, 0, 1024, res_type, hpf_start=-1)}}


BUILTIN = {
    "4band_v2": _four_band_v2(637),
    "4band_v3": _four_band_v2(530),
    "1band_sr44100_hl512": {"bins": 1024, "unstable_bins": 0, "reduction_bins": 0, "sr": 44100, "pre_filter_start": 1023, "pre_filter_stop": 1024,
                            "band": {1: _band(44100, 512, 2048, 0, 1024, "sinc_best", hpf_start=-1)}},
    "1band_sr44100_hl1024": {"bins": 1024, "unstable_bins": 0, "reduction_bins": 0, "sr": 44100, "pre_filter_start": 1023, "pre_filter_stop": 1024,
                             "band": {1: _band(44100, 1024, 2048, 0, 1024, "sinc_best", hpf_start=-1)}},
    # models at other rates: VRSeparator resamples the mix to the top band's rate and the stems back to 44.1 kHz
    "2band_32000": _two_band(32000, 352, 1024, 118, 44, 23),
    "2band_48000": _two_band(48000, 528, 1536, 240, 82, 22),
    "1band_sr32000_hl512": _one_band(32000, 512, "kaiser_fast", 1000, 1021),
    "1band_sr16000_hl512": _one_band(16000, 512, "sinc_best", 1023, 1024),
    "1band_sr33075_hl384": _one_band(33075, 384, "sinc_best", 1000, 1021),
}


def normalise(param: dict) -> dict:
    """ModelParameters.__init__: integer band keys, missing stereo-mode switches default to False, n_bins alias."""
    p = dict(param)
    p["band"] = {int(k): dict(v) for k, v in param["band"].items()}
    for k in ("mid_side", "mid_side_b", "mid_side_b2", "stereo_w", "stereo_n", "reverse"):
        p.setdefault(k, False)
    if "n_bins" in p:
        p["bins"] = p["n_bins"]
    return p


def load(name: str, model_dir: str) -> dict:
    for cand in (os.path.join(model_dir, f"{name}.json"), os.path.join(model_dir, "modelparams", f"{name}.json")):
        if os.path.exists(cand):
            with open(cand, encoding="utf-8") as f:
                return normalise(json.load(f))
    if name in BUILTIN:
        return normalise(BUILTIN[name])
    raise FileNotFoundError(f"VR model parameters '{name}' are not built in: put {name}.json next to the model file")
