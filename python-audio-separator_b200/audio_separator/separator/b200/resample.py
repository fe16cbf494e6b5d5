"""librosa.resample on the GPU: the one module that knows the resampling filters.

`resample(x, orig_sr, target_sr, res_type)` follows librosa 0.11's conventions for a (C, N) float32 CUDA tensor: ratio = float(target_sr) / orig_sr,
the input itself when the rates are equal, ceil(N * ratio) output samples, no `scale`.  Rates may be floats (the MDXC pitch path).

res_type "polyphase" is scipy.signal.resample_poly (Kaiser(5.0) FIR, integer rates), exactly as librosa calls it.  Every other supported
res_type runs the band-limited interpolator b200sep_resample_sinc_f32 (any ratio in [1/16, 16]) with a Kaiser-windowed sinc
h(x) = rolloff * sinc(rolloff * x) * (I0(beta * sqrt(1 - (x / n_zeros)^2)) - 1) / (I0(beta) - 1) on |x| <= n_zeros, in units of the lower
rate's sample period, tabulated at PER_ZERO points per zero crossing in float32 and linearly interpolated.  The Kaiser window is lowered by
its edge value so h reaches zero at n_zeros: with no step at the edge of the support, an output does not depend on which side of the edge a
tap's rounded position falls (at rational ratios taps land on it exactly).  The sets are this project's
stand-ins for the libraries librosa would call (soxr, libsamplerate, resampy).  They approximate those libraries' bandwidths; they are not a
measured match.  Frequencies below are fractions of the lower rate's Nyquist frequency; figures are of the continuous filter's
spectrum (tests/test_resample_cpu.py holds them):

  res_type                         (n_zeros, beta, rolloff)                      passband                                -6 dB   stopband
  soxr_hq, sinc_best, kaiser_best  (64, 14.769656459379492, 0.9475937167399596)  |H-1| <= 1e-7 to 0.85, -0.04 dB at 0.90  0.95    <= -140 dB from 1.05
  sinc_medium                      (48, 12.0, 0.90)                              |H-1| <= 2e-6 to 0.80                   0.90    <= -115 dB from 1.0
  sinc_fastest                     (32, 10.0, 0.80)                              |H-1| <= 2e-5 to 0.70                   0.80    <= -95 dB from 0.90
  kaiser_fast                      (16, 8.555, 0.85)                             |H-1| <= 2e-3 to 0.70                   0.85    <= -80 dB from 1.05
"""
from __future__ import annotations

import math

import numpy as np
import torch

from ._lib import check, lib

PER_ZERO = 512  # table points per zero crossing: the linear interpolation error is ~2e-6 of full scale
_HQ = (64, 14.769656459379492, 0.9475937167399596)
FILTERS = {  # res_type -> (n_zeros, kaiser_beta, rolloff)
    "soxr_hq": _HQ,
    "sinc_best": _HQ,
    "kaiser_best": _HQ,
    "sinc_medium": (48, 12.0, 0.90),
    "sinc_fastest": (32, 10.0, 0.80),
    "kaiser_fast": (16, 8.555, 0.85),
}
_tables: dict = {}  # ((n_zeros, beta, rolloff), device) -> float32 CUDA table
_taps: dict = {}  # (up, down, device) -> (taps float32 CUDA, n_pre_remove)


def filter_design(res_type: str):
    """(n_zeros, kaiser_beta, rolloff) of a sinc res_type."""
    if res_type not in FILTERS:
        raise NotImplementedError(f"res_type={res_type!r} is not covered: use one of polyphase, {', '.join(FILTERS)}")
    return FILTERS[res_type]


def sinc_table(n_zeros: int, beta: float, rolloff: float, per_zero: int = PER_ZERO) -> np.ndarray:
    """h at x = i / per_zero, i = 0 .. n_zeros * per_zero, evaluated in float64 and rounded once to float32 (the kernel and the oracle index
    the same values)."""
    x = np.arange(n_zeros * per_zero + 1, dtype=np.float64) / per_zero
    win = (np.i0(beta * np.sqrt(np.clip(1.0 - (x / n_zeros) ** 2, 0.0, None))) - 1.0) / (np.i0(beta) - 1.0)
    return (rolloff * np.sinc(rolloff * x) * win).astype(np.float32)


def resample_poly_design(up: int, down: int):
    """The FIR scipy.signal.resample_poly designs (window=("kaiser", 5.0)) and the alignment of its output:
    -> (taps float32 zero-padded in front and scaled by `up`, n_pre_remove, up, down) for the gcd-reduced ratio."""
    g = math.gcd(up, down)
    up, down = up // g, down // g
    max_rate = max(up, down)
    f_c = 1.0 / max_rate
    half_len = 10 * max_rate
    n = 2 * half_len + 1
    m = np.arange(n, dtype=np.float64) - half_len
    h = f_c * np.sinc(f_c * m) * np.kaiser(n, 5.0)  # firwin: windowed ideal low-pass, unit gain at DC
    h = h / h.sum() * up
    n_pre_pad = down - half_len % down
    n_pre_remove = (half_len + n_pre_pad) // down
    return np.concatenate([np.zeros(n_pre_pad), h]).astype(np.float32), n_pre_remove, up, down


def out_length(n_in: int, orig_sr, target_sr) -> int:
    """librosa.resample's output length: ceil(n_in * target_sr / orig_sr) (exact integer arithmetic for integer rates, as resample_poly)."""
    if float(orig_sr).is_integer() and float(target_sr).is_integer():
        return -(-n_in * int(target_sr) // int(orig_sr))
    return int(np.ceil(n_in * (float(target_sr) / orig_sr)))


def resample(x: torch.Tensor, orig_sr, target_sr, res_type: str = "soxr_hq") -> torch.Tensor:
    """librosa.resample(x, orig_sr=orig_sr, target_sr=target_sr, res_type=res_type) for a (C, N) float32 CUDA tensor, on its device."""
    if orig_sr == target_sr:
        return x
    assert x.dim() == 2 and x.dtype == torch.float32 and x.is_cuda, "resample takes a (C, N) float32 CUDA tensor"
    x = x.contiguous()
    C, n_in = x.shape
    stream = torch.cuda.current_stream(x.device).cuda_stream
    if res_type == "polyphase":
        if not (float(orig_sr).is_integer() and float(target_sr).is_integer()):
            raise ValueError(f"polyphase resampling needs integer rates, got {orig_sr} -> {target_sr}")
        g = math.gcd(int(orig_sr), int(target_sr))
        key = (int(target_sr) // g, int(orig_sr) // g, x.device)
        if key not in _taps:
            taps, pre, _, _ = resample_poly_design(key[0], key[1])
            _taps[key] = (torch.from_numpy(taps).to(x.device), pre)
        taps, pre = _taps[key]
        y = torch.empty((C, out_length(n_in, orig_sr, target_sr)), dtype=torch.float32, device=x.device)
        check(lib.b200sep_resample_poly_f32(x.data_ptr(), taps.data_ptr(), taps.numel(), key[0], key[1], pre, C, n_in, y.shape[1], y.data_ptr(), stream),
              "resample_poly_f32")
        return y
    design = filter_design(res_type)
    key = (design, x.device)
    if key not in _tables:
        _tables[key] = torch.from_numpy(sinc_table(*design)).to(x.device)
    ratio = float(target_sr) / orig_sr
    y = torch.empty((C, int(np.ceil(n_in * ratio))), dtype=torch.float32, device=x.device)
    check(lib.b200sep_resample_sinc_f32(x.data_ptr(), C, n_in, _tables[key].data_ptr(), design[0], PER_ZERO, ratio, y.shape[1], y.data_ptr(), stream),
          "resample_sinc_f32")
    return y


def match_length(x: torch.Tensor, n: int) -> torch.Tensor:
    """spec_utils.match_array_shapes(x, like) for a (C, M) tensor and n = like.shape[1]: cut to n columns or pad with zeros."""
    if x.shape[1] == n:
        return x
    if x.shape[1] > n:
        return x[:, :n].contiguous()
    return torch.nn.functional.pad(x, (0, n - x.shape[1]))
