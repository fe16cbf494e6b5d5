"""CPU: the band-limited resampler's oracle (oracle/resample_oracle.py) against scipy.signal.upfirdn with exactly evaluated taps, the filter
sets' passband / stopband figures, librosa's lengths, and the pitch / VR-rate goldens (oracle/make_golden_resample.py) reproduced by the
oracle composition."""
import math
import os

import numpy as np
import pytest
import scipy.signal

import mdx_oracle as M
import mdxc_oracle as X
import resample_oracle as RO
import roformer_oracle as R
import vr_oracle as V
from make_golden_resample import MDXC_SMALL, PITCHES, VR_PARAMS, pcm_wave, pitch_demix, rf_cfg, vr_param, vr_separate

DESIGNS = ("soxr_hq", "sinc_medium", "sinc_fastest", "kaiser_fast")


def exact_filter(res_type, x):
    """the continuous filter h(x) in float64, no table"""
    nz, beta, ro = RO.FILTERS[res_type]
    x = np.abs(x)
    win = (np.i0(beta * np.sqrt(np.clip(1 - (x / nz) ** 2, 0, None))) - 1) / (np.i0(beta) - 1)
    return np.where(x < nz, ro * np.sinc(ro * x) * win, 0.0)


@pytest.mark.parametrize("res_type", DESIGNS)
@pytest.mark.parametrize("orig_sr,target_sr", [(48000, 44100), (44100, 32000), (32000, 6000), (32000, 44100)])
def test_oracle_vs_upfirdn_exact_taps(res_type, orig_sr, target_sr):
    g_ = math.gcd(orig_sr, target_sr)
    up, down = target_sr // g_, orig_sr // g_
    g = min(1.0, up / down)
    nz = RO.FILTERS[res_type][0]
    J = -(-(int(math.ceil(nz * up / g)) + 1) // down) * down  # half length, a multiple of `down` so the delay is a whole output
    taps = g * exact_filter(res_type, g * (np.arange(2 * J + 1) - J) / up)
    x = np.random.default_rng(orig_sr + target_sr).standard_normal((2, 3000)) * 0.5
    n_out = -(-3000 * up // down)
    want = scipy.signal.upfirdn(taps, x, up, down)[:, J // down : J // down + n_out]
    got = RO.sinc_resample(x, target_sr / orig_sr, *RO.table(res_type))
    assert got.shape == want.shape == (2, n_out)
    assert np.abs(got - want).max() <= 5e-6  # the table-interpolation bound at 512 points per zero crossing


def test_oracle_tables_are_the_products(lib_built):
    from audio_separator.separator.b200 import resample

    assert resample.PER_ZERO == RO.PER_ZERO and resample.FILTERS == RO.FILTERS
    for res_type in RO.FILTERS:
        tab = resample.sinc_table(*resample.filter_design(res_type))
        assert tab.dtype == np.float32 and np.array_equal(tab, RO.table(res_type)[0])
    with pytest.raises(NotImplementedError, match="soxr_vhq"):
        resample.filter_design("soxr_vhq")


# (passband |H-1| bound, up to), (-6 dB frequency), (stopband dB, from): fractions of the lower rate's Nyquist (b200/resample.py docstring)
FIGURES = {
    "soxr_hq": ((1e-7, 0.85), 0.9475937167399596, (-140.0, 1.05)),
    "sinc_medium": ((2e-6, 0.80), 0.90, (-115.0, 1.0)),
    "sinc_fastest": ((2e-5, 0.70), 0.80, (-95.0, 0.90)),
    "kaiser_fast": ((2e-3, 0.70), 0.85, (-80.0, 1.05)),
}


@pytest.mark.parametrize("res_type", DESIGNS)
def test_filter_set_figures(res_type):
    (pb, f_pass), f6, (sb, f_stop) = FIGURES[res_type]
    nz = RO.FILTERS[res_type][0]
    P = 64  # samples of h per unit: the spectrum is the continuous filter's far beyond 4x Nyquist
    h = exact_filter(res_type, np.arange(-nz * P, nz * P + 1) / P)
    nfft = 1 << 22
    H = np.abs(np.fft.rfft(h, nfft)) / P
    f = np.fft.rfftfreq(nfft, 1.0 / P) / 0.5
    assert np.abs(H[f <= f_pass] - 1).max() <= pb
    assert abs(20 * np.log10(np.interp(f6, f, H)) + 6.02) <= 0.1
    assert 20 * np.log10(H[(f >= f_stop) & (f < 4)].max()) <= sb
    if res_type == "soxr_hq":
        assert abs(20 * np.log10(np.interp(0.90, f, H)) + 0.04) <= 0.005


def test_librosa_lengths(lib_built):
    from audio_separator.separator.b200 import resample

    for n, a, b in ((1, 44100, 32000), (7, 32000, 44100), (10007, 48000, 44100), (44100 * 300, 44100, 32000), (10007, 32000, 6000)):
        assert resample.out_length(n, a, b) == math.ceil(n * b / a)
        if n < 20000:
            assert RO.sinc_resample(np.zeros((1, n)), b / a, *RO.table("kaiser_fast")).shape[1] == math.ceil(n * b / a)
    for s in (-12, -3, -1, 1, 2, 12):  # the two-way pitch lengths: librosa's ceil(N * float(target) / orig) on float rates
        (a, b), (c, d) = RO.pitch_rates(44100, s)
        for n in (1, 9000, 44100 * 10 + 3):
            n_p = resample.out_length(n, a, b)
            assert n_p == int(np.ceil(n * (float(b) / a)))
            n_back = resample.out_length(n_p, c, d)
            assert n_back == int(np.ceil(n_p * (float(d) / c))) and abs(n_back - n) <= 2
    x = np.arange(10, dtype=np.float32).reshape(2, 5)
    assert np.array_equal(RO.match_array_shapes(x, 3), x[:, :3])
    assert np.array_equal(RO.match_array_shapes(x, 7), np.pad(x, ((0, 0), (0, 2))))
    assert RO.resample(x, 44100, 44100, "soxr_hq") is x


def test_pitch_golden_reproduced_by_oracle(golden_dir):
    z = np.load(os.path.join(golden_dir, "pitch_small.npz"))
    mix = M.normalize(pcm_wave(int(z["n_samples"]), int(z["mix_seed"])), 0.9, 0.0)
    cfg = X.MDXCConfig(**MDXC_SMALL)
    w = X.make_weights(cfg, seed=int(z["tfc_weights_seed"]), out_gain=float(z["tfc_out_gain"]))
    rcfg = rf_cfg(overlap=int(z["rf_overlap"]))
    rw = R.make_weights(rcfg, seed=int(z["rf_weights_seed"]))
    for s in PITCHES:
        tfc = pitch_demix(mix, s, lambda m: X.demix(m, cfg, lambda x: X.net_forward(w, cfg, x)), 2)
        assert tfc.shape == z[f"tfc_pitch{s:+d}"].shape == (2, 2, mix.shape[1])
        assert np.abs(tfc - z[f"tfc_pitch{s:+d}"]).max() <= 2e-5
        prim = pitch_demix(mix, s, lambda m: R.demix(m, rcfg, lambda c: R.forward(rw, rcfg, c), n_instruments=2), 1)[0]
        assert np.abs(np.stack([prim, mix - prim]) - z[f"rf_pitch{s:+d}"]).max() <= 2e-5


@pytest.mark.parametrize("name", VR_PARAMS)
def test_vr_rates_golden_reproduced_by_oracle(golden_dir, name):
    z = np.load(os.path.join(golden_dir, "vr_rates_small.npz"))
    p = vr_param(name)
    wave = pcm_wave(int(z["n_samples"]), int(z["wave_seed"]))
    got = vr_separate(wave, p, V.make_weights(31191, seed=int(z[f"{name}_weights_seed"])))
    for g, stem in zip(got, ("primary", "secondary")):
        want = z[f"{name}_{stem}"]
        assert g.shape == want.shape == (2, math.ceil(p["band"][len(p["band"])]["hl"] * (int(z[f"{name}_frames"]) - 1) * 44100 / p["sr"]))
        assert np.abs(g - want).max() <= 2e-5
