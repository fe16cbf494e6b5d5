"""H100 mirror of the reference's `STFT` helper (audio_separator/separator/uvr_lib_v5/stft.py:4-126).

Same constructor, `__call__` and `inverse` contract -- (B, C, T) <-> (B, 2C, dim_f, T//hop+1), planes
[L_re, L_im, R_re, R_im] -- but both directions are single launches of the hand-written sm_90a FFT kernels
(csrc/stft.cu) instead of torch.stft / torch.istft.  CUDA tensors in, CUDA tensors out; anything else raises.
"""
import torch

from ..b200.engine import LAYOUT_CFT, StftPlan


class STFT:
    def __init__(self, logger, n_fft, hop_length, dim_f, device):
        self.logger, self.n_fft, self.hop_length, self.dim_f, self.device = logger, n_fft, hop_length, dim_f, device
        self._plan = StftPlan(n_fft, hop_length)

    def _on_device(self, t):
        if not isinstance(t, torch.Tensor):
            raise TypeError("STFT expects a torch.Tensor")
        if not t.is_cuda:
            raise RuntimeError("the H100 STFT only runs on CUDA tensors (no CPU fallback); move the input to the GPU")
        return t.to(torch.float32)

    def __call__(self, input_tensor):
        x = self._on_device(input_tensor)
        lead, (c, t) = x.shape[:-2], x.shape[-2:]
        rows = x.reshape(-1, t)
        n = rows.shape[0]
        if n % 2:  # the kernel transforms channel PAIRS as one complex FFT; pad an odd row count with silence
            rows = torch.cat([rows, torch.zeros_like(rows[:1])], 0)
        spec = self._plan.forward(rows.reshape(-1, 2, t), self.dim_f, zero_bins=0, layout=LAYOUT_CFT)
        frames = spec.shape[-1]
        spec = spec.reshape(-1, 2, self.dim_f, frames)[:n]  # (rows, {re,im}, F, frames)
        return spec.reshape(*lead, c * 2, self.dim_f, frames)

    def inverse(self, input_tensor):
        s = self._on_device(input_tensor)
        lead, (c2, f, t) = s.shape[:-3], s.shape[-3:]
        if c2 % 2:
            raise ValueError(f"STFT.inverse expects (..., 2*C, dim_f, frames); got {c2} planes")
        rows = s.reshape(-1, 2, f, t)
        n = rows.shape[0]
        if n % 2:
            rows = torch.cat([rows, torch.zeros_like(rows[:1])], 0)
        wave = self._plan.inverse(rows.reshape(-1, 4, f, t), layout=LAYOUT_CFT)
        wave = wave.reshape(-1, wave.shape[-1])[:n]
        return wave.reshape(*lead, 2, -1) if c2 == 4 else wave.reshape(*lead, c2 // 2, -1)
