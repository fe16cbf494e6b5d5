"""CPU oracle of the band-limited resampler (b200sep_resample_sinc_f32) -- TEST INFRASTRUCTURE, not product code.

A float64 numpy restatement of the kernel's arithmetic over the same float32 tables (audio_separator/separator/b200/resample.py):
  y[c][n] = g * sum_k x[c][k] * h(g * |n*step - k|),  step = 1 / ratio,  g = min(1, ratio),  n = 0 .. ceil(N * ratio) - 1,
h = the table linearly interpolated at u = g * per_zero * |n*step - k|, zero from u >= n_zeros * per_zero on, x zero outside [0, N).
`resample` dispatches on res_type like librosa.resample: "polyphase" is scipy.signal.resample_poly, the sinc res_types run the
restatement.  No soxr / libsamplerate / resampy is available to compare against: the sinc sets are pinned only to this restatement.
"""
from __future__ import annotations

import math

import numpy as np

PER_ZERO = 512
_HQ = (64, 14.769656459379492, 0.9475937167399596)
FILTERS = {"soxr_hq": _HQ, "sinc_best": _HQ, "kaiser_best": _HQ, "sinc_medium": (48, 12.0, 0.90), "sinc_fastest": (32, 10.0, 0.80), "kaiser_fast": (16, 8.555, 0.85)}


def table(res_type: str) -> tuple[np.ndarray, int, int]:
    """(float32 table, n_zeros, per_zero) of a sinc res_type: rolloff * sinc(rolloff * x) * (Kaiser(beta) - edge) over x = i / per_zero in [0, n_zeros],
    evaluated in float64 and rounded once (tests/test_resample_cpu.py checks these are the product's tables, bit for bit)."""
    n_zeros, beta, rolloff = FILTERS[res_type]
    x = np.arange(n_zeros * PER_ZERO + 1, dtype=np.float64) / PER_ZERO
    win = (np.i0(beta * np.sqrt(np.clip(1.0 - (x / n_zeros) ** 2, 0.0, None))) - 1.0) / (np.i0(beta) - 1.0)
    return (rolloff * np.sinc(rolloff * x) * win).astype(np.float32), n_zeros, PER_ZERO


def sinc_resample(x: np.ndarray, ratio: float, tab: np.ndarray, n_zeros: int, per_zero: int, idx=None, block=1 << 22) -> np.ndarray:
    """The kernel's arithmetic in float64: x (C, N) -> (C, ceil(N * ratio)), or only the outputs `idx` when given."""
    x = np.asarray(x, dtype=np.float64)
    C, n_in = x.shape
    n_out = int(np.ceil(n_in * ratio))
    idx = np.arange(n_out, dtype=np.int64) if idx is None else np.asarray(idx, dtype=np.int64)
    step, g = 1.0 / ratio, min(1.0, ratio)
    n_tab = n_zeros * per_zero
    tab = np.asarray(tab, dtype=np.float64)
    reach = int(math.ceil(n_zeros / g)) + 1
    offs = np.arange(-reach, reach + 1, dtype=np.int64)
    out = np.zeros((C, idx.size), np.float64)
    rows = max(1, block // offs.size)
    for a in range(0, idx.size, rows):
        t = idx[a : a + rows].astype(np.float64) * step
        k = np.floor(t).astype(np.int64)[:, None] + offs[None, :]
        u = g * per_zero * np.abs(t[:, None] - k)
        i = np.minimum(np.floor(u).astype(np.int64), n_tab - 1)
        fr = u - i
        h = np.where(u < n_tab, tab[i] + fr * (tab[i + 1] - tab[i]), 0.0)
        ok = (k >= 0) & (k < n_in)
        h = np.where(ok, h, 0.0)
        kc = np.clip(k, 0, n_in - 1)
        for c in range(C):
            out[c, a : a + rows] = g * (x[c][kc] * h).sum(axis=1)
    return out


def resample(y: np.ndarray, orig_sr, target_sr, res_type: str = "soxr_hq") -> np.ndarray:
    """librosa.resample(y, orig_sr=, target_sr=, res_type=) on a 1-D or (C, N) array, float32 out (librosa keeps the input dtype)."""
    if orig_sr == target_sr:
        return y
    y = np.asarray(y)
    if res_type == "polyphase":
        import scipy.signal

        g = math.gcd(int(orig_sr), int(target_sr))
        return scipy.signal.resample_poly(y, int(target_sr) // g, int(orig_sr) // g, axis=-1).astype(np.float32)
    tab, n_zeros, per_zero = table(res_type)
    x2 = y.reshape(-1, y.shape[-1])
    out = sinc_resample(x2, float(target_sr) / orig_sr, tab, n_zeros, per_zero)
    return out.reshape(y.shape[:-1] + (out.shape[-1],)).astype(np.float32)


def match_array_shapes(a: np.ndarray, n: int) -> np.ndarray:
    """spec_utils.match_array_shapes(a, like) with n = like.shape[1]."""
    if a.shape[1] > n:
        return a[:, :n]
    if a.shape[1] < n:
        return np.pad(a, ((0, 0), (0, n - a.shape[1])))
    return a


def pitch_rates(sr, semitones):
    """The two rate pairs of the MDXC pitch path, computed as the reference does: mix sr -> sr * 2**(-s/12), stems back by 2**(s/12)."""
    sr_pitched = sr * 2 ** (-semitones / 12)
    return (sr, sr_pitched), (sr_pitched, sr_pitched * 2 ** (semitones / 12))
