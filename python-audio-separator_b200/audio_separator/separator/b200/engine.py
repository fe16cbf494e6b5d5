"""Python handles over the C-ABI engine (libb200sep.so).  PyTorch is used only for device memory and streams.

MdxEngine is the device-resident replacement of the reference's per-chunk loop
(architectures/mdx_separator.py:293-450): the padded mixture, every chunk's spectrogram, the network
activations, the iSTFT frames and the overlap-add accumulators all stay in HBM; the host sees one upload of the
mix and one download of the stems.
"""
from __future__ import annotations

import ctypes as C

import numpy as np
import torch

from . import _lib
from ._lib import LAYOUT_CFT, LAYOUT_CTF, check, lib


def _require_cuda():
    if not torch.cuda.is_available():
        raise RuntimeError("the H100 engine needs a CUDA device (sm_90a); there is no CPU fallback")


def _ptr(t: torch.Tensor) -> int:
    assert t.is_cuda and t.is_contiguous(), "engine buffers must be contiguous CUDA tensors"
    return t.data_ptr()


def _stream() -> int:
    return torch.cuda.current_stream().cuda_stream


class StftPlan:
    """b200sep_stft_plan handle (replaces STFT.__init__, uvr_lib_v5/stft.py:11-18)."""

    def __init__(self, n_fft: int, hop: int):
        _require_cuda()
        self.n_fft, self.hop = int(n_fft), int(hop)
        h = C.c_void_p()
        check(lib.b200sep_stft_plan_create(C.byref(h), self.n_fft, self.hop), "stft_plan_create")
        self.handle = h

    def __del__(self):
        h = getattr(self, "handle", None)
        if h and lib is not None:  # `lib` may already be torn down at interpreter exit
            lib.b200sep_stft_plan_destroy(h)
            self.handle = None

    def forward(self, wave: torch.Tensor, dim_f: int, zero_bins: int = 0, layout: int = LAYOUT_CFT) -> torch.Tensor:
        """wave (B,2,T) float32 cuda -> (B,4,dim_f,frames) [CFT] or (B,4,frames,dim_f) [CTF]."""
        assert wave.dim() == 3 and wave.shape[1] == 2 and wave.dtype == torch.float32
        wave = wave.contiguous()
        B, _, T = wave.shape
        frames = T // self.hop + 1
        shape = (B, 4, dim_f, frames) if layout == LAYOUT_CFT else (B, 4, frames, dim_f)
        spec = torch.empty(shape, dtype=torch.float32, device=wave.device)
        check(lib.b200sep_stft_forward(self.handle, _ptr(wave), 2 * T, T, 0, B, T, dim_f, zero_bins, layout, _ptr(spec), _stream()), "stft_forward")
        return spec

    def inverse(self, spec: torch.Tensor, layout: int = LAYOUT_CFT) -> torch.Tensor:
        """spec (B,4,dim_f,frames) [CFT] / (B,4,frames,dim_f) [CTF] -> wave (B,2,hop*(frames-1))."""
        assert spec.dim() == 4 and spec.shape[1] == 4 and spec.dtype == torch.float32
        spec = spec.contiguous()
        B = spec.shape[0]
        dim_f, frames = (spec.shape[2], spec.shape[3]) if layout == LAYOUT_CFT else (spec.shape[3], spec.shape[2])
        wave = torch.empty((B, 2, self.hop * (frames - 1)), dtype=torch.float32, device=spec.device)
        nwork = lib.b200sep_stft_inverse_work_floats(self.handle, B, frames, dim_f, layout)
        work = torch.empty(nwork, dtype=torch.float32, device=spec.device)
        check(lib.b200sep_stft_inverse(self.handle, _ptr(spec), B, frames, dim_f, layout, _ptr(wave), _ptr(work), _stream()), "stft_inverse")
        return wave


class MdxNet:
    """b200sep_mdxnet handle: ConvTDFNet weights + activation arena on the device."""

    def __init__(self, params_flat: np.ndarray, dim_c, dim_f, dim_t, num_blocks, l, g, k, bn, max_batch=1, precision=0):
        _require_cuda()
        self.cfg = _lib.MdxNetConfig(dim_c, dim_f, dim_t, num_blocks, l, g, k, bn, max_batch, precision)
        params_flat = np.ascontiguousarray(params_flat, dtype=np.float32)
        expect = lib.b200sep_mdxnet_param_count(C.byref(self.cfg))
        if expect != params_flat.size:
            raise ValueError(f"ConvTDFNet config expects {expect} parameters, blob has {params_flat.size}")
        h = C.c_void_p()
        check(lib.b200sep_mdxnet_create(C.byref(h), C.byref(self.cfg), params_flat.ctypes.data_as(C.c_void_p), params_flat.size), "mdxnet_create")
        self.handle = h
        self.max_batch = max_batch
        self.dim_c, self.dim_f, self.dim_t = dim_c, dim_f, dim_t

    def __del__(self):
        h = getattr(self, "handle", None)
        if h and lib is not None:
            lib.b200sep_mdxnet_destroy(h)
            self.handle = None

    @property
    def device_bytes(self) -> int:
        return int(lib.b200sep_mdxnet_device_bytes(self.handle))

    def profile(self, enable: bool):
        check(lib.b200sep_mdxnet_profile_enable(self.handle, int(enable)), "mdxnet_profile_enable")

    def profile_read(self) -> dict:
        """{category: {"ms", "launches", "flops", "bytes"}} summed over the forwards since profile(True)."""
        n = 8
        ms, ln, fl, by = (C.c_float * n)(), (C.c_int64 * n)(), (C.c_double * n)(), (C.c_double * n)()
        k = lib.b200sep_mdxnet_profile_read(self.handle, n, ms, ln, fl, by)
        if k < 0:
            check(k, "mdxnet_profile_read")
        return {lib.b200sep_mdxnet_profile_name(i).decode(): {"ms": float(ms[i]), "launches": int(ln[i]), "flops": float(fl[i]), "bytes": float(by[i])} for i in range(k)}

    def forward(self, spec: torch.Tensor, layout: int = LAYOUT_CFT) -> torch.Tensor:
        """spec (B,4,dim_f,dim_t) [CFT, the ONNX graph's input layout] or (B,4,dim_t,dim_f) [CTF] -> same shape."""
        spec = spec.contiguous()
        want = (self.dim_c, self.dim_f, self.dim_t) if layout == LAYOUT_CFT else (self.dim_c, self.dim_t, self.dim_f)
        if tuple(spec.shape[1:]) != want or spec.dtype != torch.float32:
            raise ValueError(f"ConvTDFNet input must be float32 (B,{want}), got {tuple(spec.shape)} {spec.dtype}")
        out = torch.empty_like(spec)
        B = spec.shape[0]
        for b0 in range(0, B, self.max_batch):
            nb = min(self.max_batch, B - b0)
            check(lib.b200sep_mdxnet_forward(self.handle, _ptr(spec[b0 : b0 + nb]), _ptr(out[b0 : b0 + nb]), nb, layout, _stream()), "mdxnet_forward")
        return out


class MdxEngine:
    """Device-resident MDX separation: chunk grid, run_model batches, windowed overlap-add, stem arithmetic."""

    def __init__(self, net: MdxNet | None, n_fft, hop_length, dim_f, segment_size, overlap, compensate=1.0, enable_denoise=False, batch_size=None):
        _require_cuda()
        self.net = net
        self.n_fft, self.hop, self.dim_f = int(n_fft), int(hop_length), int(dim_f)
        self.segment_size = int(segment_size)
        self.overlap = float(overlap)
        self.compensate = float(compensate)
        self.enable_denoise = bool(enable_denoise)
        self.trim = self.n_fft // 2  # mdx_separator.py:217
        self.chunk_size = self.hop * (self.segment_size - 1)  # :220
        self.gen_size = self.chunk_size - 2 * self.trim  # :223
        self.plan = StftPlan(self.n_fft, self.hop)
        self.batch = int(batch_size or (net.max_batch if net is not None else 8))
        if net is not None:
            self.batch = min(self.batch, net.max_batch)
        self._work = None
        self.device = torch.device("cuda", torch.cuda.current_device())

    # ---- chunk grid (mdx_separator.py:307-348)
    def grid(self, n_samples: int, is_match_mix=False):
        overlap = 0.02 if is_match_mix else self.overlap
        gen = self.chunk_size - 2 * self.trim
        pad = gen + self.trim - (n_samples % gen)
        L = self.trim + n_samples + pad
        step = int((1 - overlap) * self.chunk_size)
        n_chunks = (L + step - 1) // step
        return L, step, n_chunks, overlap

    def _workspace(self, batch):
        need = lib.b200sep_mdx_run_model_work_floats(self.plan.handle, batch, self.chunk_size, self.dim_f)
        if self._work is None or self._work.numel() < need:
            self._work = torch.empty(need, dtype=torch.float32, device=self.device)
        return self._work

    def run_model(self, mix: torch.Tensor, is_match_mix=False) -> torch.Tensor:
        """MDXSeparator.run_model (mdx_separator.py:414-450) on a contiguous (B,2,chunk) CUDA tensor."""
        mix = mix.contiguous()
        B, _, T = mix.shape
        assert T == self.chunk_size, (T, self.chunk_size)
        out = torch.empty_like(mix)
        net = None if is_match_mix else self.net.handle
        for b0 in range(0, B, self.batch):
            nb = min(self.batch, B - b0)
            work = self._workspace(nb)
            check(
                lib.b200sep_mdx_run_model(self.plan.handle, net, _ptr(mix[b0 : b0 + nb]), 2 * T, T, 0, nb, T, self.dim_f, int(self.enable_denoise), _ptr(out[b0 : b0 + nb]), _ptr(work), _stream()),
                "mdx_run_model",
            )
        return out

    def demix_device(self, mix_dev: torch.Tensor, is_match_mix=False, out_scale=1.0, with_secondary=False, interleave=False):
        """MDXSeparator.demix (mdx_separator.py:293-412) with everything resident in HBM.

        mix_dev: (2,N) float32 CUDA (already peak-normalised by the caller).  Returns primary (2,N) [or (N,2) when
        interleave] and, with_secondary, secondary = mix - compensate*primary (mdx_separator.py:182).
        """
        assert mix_dev.is_cuda and mix_dev.dtype == torch.float32 and mix_dev.shape[0] == 2
        mix_dev = mix_dev.contiguous()
        N = mix_dev.shape[1]
        L, step, n_chunks, overlap = self.grid(N, is_match_mix)
        T = self.chunk_size
        mixture = torch.zeros((2, L), dtype=torch.float32, device=self.device)  # [0]*trim + mix + [0]*pad, :329
        mixture[:, self.trim : self.trim + N] = mix_dev
        chunks = torch.empty((n_chunks, 2, T), dtype=torch.float32, device=self.device)
        net = None if is_match_mix else self.net.handle
        esz = 4
        for b0 in range(0, n_chunks, self.batch):
            nb = min(self.batch, n_chunks - b0)
            work = self._workspace(nb)
            check(
                lib.b200sep_mdx_run_model(
                    self.plan.handle, net, mixture.data_ptr() + b0 * step * esz, step, L, L - b0 * step, nb, T, self.dim_f, int(self.enable_denoise), _ptr(chunks[b0 : b0 + nb]), _ptr(work), _stream()
                ),
                "mdx_run_model",
            )
        shape = (N, 2) if interleave else (2, N)
        primary = torch.empty(shape, dtype=torch.float32, device=self.device)
        secondary = torch.empty(shape, dtype=torch.float32, device=self.device) if with_secondary else None
        check(
            lib.b200sep_demix_overlap_add(
                _ptr(chunks), n_chunks, T, step, L, self.trim, N, int(overlap != 0), float(out_scale), _ptr(mix_dev) if with_secondary else None, self.compensate, int(interleave), _ptr(primary), _ptr(secondary) if with_secondary else None, _stream()
            ),
            "demix_overlap_add",
        )
        return (primary, secondary) if with_secondary else primary

    # ---- array-level body of MDXSeparator.separate (mdx_separator.py:152-182)
    def separate_device(self, mix_dev: torch.Tensor, normalization_threshold=0.9, amplification_threshold=0.0):
        """mix_dev (2,N) float32 CUDA as loaded -> (primary (N,2), secondary (N,2)) CUDA float32."""
        n = mix_dev.numel()
        peak = torch.empty(1, dtype=torch.float32, device=self.device)
        check(lib.b200sep_absmax(_ptr(mix_dev), n, _ptr(peak), _stream()), "absmax")  # :155
        mixn = torch.empty_like(mix_dev)
        min_peak = -1.0 if amplification_threshold is None else float(amplification_threshold)
        check(lib.b200sep_normalize(_ptr(mix_dev), n, _ptr(peak), float(normalization_threshold), min_peak, _ptr(mixn), _stream()), "normalize")  # :156
        # `source = demix(mix) * peak` (:159): out_scale is a host float in the C ABI; read the peak back (4 bytes)
        peak_h = float(peak.item())
        return self.demix_device(mixn, out_scale=peak_h, with_secondary=True, interleave=True)

    def to_pcm16(self, stem: torch.Tensor, normalization_threshold=0.9, amplification_threshold=0.0):
        """write_audio_pydub's sample path on the device (common_separator.py:310-339): returns int16 (N*2,) or None."""
        stem = stem.contiguous()
        n = stem.numel()
        peak = torch.empty(1, dtype=torch.float32, device=self.device)
        check(lib.b200sep_absmax(_ptr(stem), n, _ptr(peak), _stream()), "absmax")
        norm = torch.empty_like(stem)
        min_peak = -1.0 if amplification_threshold is None else float(amplification_threshold)
        check(lib.b200sep_normalize(_ptr(stem), n, _ptr(peak), float(normalization_threshold), min_peak, _ptr(norm), _stream()), "normalize")
        pk = float(peak.item())
        s = 1.0
        if pk > normalization_threshold:
            s = normalization_threshold / pk
        elif min_peak >= 0 and pk < min_peak:
            s = min_peak / pk
        if pk * s < 1e-6:
            return None
        out = torch.empty(n, dtype=torch.int16, device=self.device)
        check(lib.b200sep_to_pcm16(_ptr(norm), n, _ptr(out), _stream()), "to_pcm16")
        return out


# =========================================================================================================
# MDXC (MDX23C / TFC_TDF_net) -- architectures/mdxc_separator.py non-Roformer branch
def tfcnet_param_names(dim_f, num_subbands, audio_channels, num_scales, l, c, g, bn, num_targets):
    """Ordered (name, shape) of TFC_TDF_net's state_dict (uvr_lib_v5/tfc_tdf_v3.py:110-214)."""
    out = []
    dim_c = num_subbands * audio_channels * 2
    f = dim_f // num_subbands

    def norm(prefix, ch):
        out.append((f"{prefix}.weight", (ch,)))
        out.append((f"{prefix}.bias", (ch,)))

    def block(prefix, in_c, ch, ff):
        for i in range(l):
            b = f"{prefix}.blocks.{i}"
            norm(f"{b}.tfc1.0", in_c)
            out.append((f"{b}.tfc1.2.weight", (ch, in_c, 3, 3)))
            norm(f"{b}.tdf.0", ch)
            out.append((f"{b}.tdf.2.weight", (ff // bn, ff)))
            norm(f"{b}.tdf.3", ch)
            out.append((f"{b}.tdf.5.weight", (ff, ff // bn)))
            norm(f"{b}.tfc2.0", ch)
            out.append((f"{b}.tfc2.2.weight", (ch, ch, 3, 3)))
            out.append((f"{b}.shortcut.weight", (ch, in_c, 1, 1)))
            in_c = ch

    out.append(("first_conv.weight", (c, dim_c, 1, 1)))
    ch = c
    for i in range(num_scales):
        block(f"encoder_blocks.{i}.tfc_tdf", ch, ch, f)
        norm(f"encoder_blocks.{i}.downscale.conv.0", ch)
        out.append((f"encoder_blocks.{i}.downscale.conv.2.weight", (ch + g, ch, 2, 2)))
        f //= 2
        ch += g
    block("bottleneck_block", ch, ch, f)
    for i in range(num_scales):
        norm(f"decoder_blocks.{i}.upscale.conv.0", ch)
        out.append((f"decoder_blocks.{i}.upscale.conv.2.weight", (ch, ch - g, 2, 2)))
        f *= 2
        ch -= g
        block(f"decoder_blocks.{i}.tfc_tdf", 2 * ch, ch, f)
    out.append(("final_conv.0.weight", (ch, ch + dim_c, 1, 1)))
    out.append(("final_conv.2.weight", (num_targets * dim_c, ch, 1, 1)))
    return out


class TfcNet:
    """b200sep_tfcnet handle (TFC_TDF_net weights + arena).  `state`: name -> array in the reference's state_dict naming."""

    def __init__(self, state: dict, dim_f, dim_t, num_subbands=4, audio_channels=2, num_scales=5, l=2, c=128, g=128, bn=4, num_targets=2, max_batch=1):
        _require_cuda()
        names = tfcnet_param_names(dim_f, num_subbands, audio_channels, num_scales, l, c, g, bn, num_targets)
        parts = []
        for name, shape in names:
            a = np.asarray(state[name], dtype=np.float32)
            if tuple(a.shape) != tuple(shape):
                raise ValueError(f"parameter {name}: expected shape {shape}, got {a.shape}")
            parts.append(a.reshape(-1))
        flat = np.ascontiguousarray(np.concatenate(parts))
        self.cfg = _lib.TfcNetConfig(dim_f, dim_t, num_subbands, audio_channels, num_scales, l, c, g, bn, num_targets, max_batch)
        expect = lib.b200sep_tfcnet_param_count(C.byref(self.cfg))
        if expect != flat.size:
            raise ValueError(f"TFC_TDF_net config expects {expect} parameters, state has {flat.size}")
        h = C.c_void_p()
        check(lib.b200sep_tfcnet_create(C.byref(h), C.byref(self.cfg), flat.ctypes.data_as(C.c_void_p), flat.size), "tfcnet_create")
        self.handle = h
        self.max_batch, self.dim_f, self.dim_t, self.num_targets = max_batch, dim_f, dim_t, num_targets

    def __del__(self):
        h = getattr(self, "handle", None)
        if h and lib is not None:
            lib.b200sep_tfcnet_destroy(h)
            self.handle = None

    @property
    def device_bytes(self) -> int:
        return int(lib.b200sep_tfcnet_device_bytes(self.handle))

    def forward_spec(self, spec: torch.Tensor) -> torch.Tensor:
        """spec (B,4,dim_t,dim_f) float32 CUDA [layout CTF] -> (B, S, 4, dim_t, dim_f)."""
        spec = spec.contiguous()
        assert tuple(spec.shape[1:]) == (4, self.dim_t, self.dim_f) and spec.dtype == torch.float32, spec.shape
        B = spec.shape[0]
        out = torch.empty((B, self.num_targets, 4, self.dim_t, self.dim_f), dtype=torch.float32, device=spec.device)
        for b0 in range(0, B, self.max_batch):
            nb = min(self.max_batch, B - b0)
            check(lib.b200sep_tfcnet_forward(self.handle, _ptr(spec[b0 : b0 + nb]), _ptr(out[b0 : b0 + nb]), nb, _stream()), "tfcnet_forward")
        return out


class MdxcEngine:
    """Device-resident MDXCSeparator.demix, non-Roformer branch (mdxc_separator.py:345-404): unfold -> batches ->
    STFT -> TFC_TDF_net -> iSTFT -> rectangular overlap-add / overlap.

    With `dist` (torch.distributed, nccl, one process per GPU) the chunk grid is time-sharded (SURVEY.md section 8e, MDXC row): rank r finalises the
    output samples [N*r/W, N*(r+1)/W), computes the chunks that start there and receives from its left neighbour the chunks that reach into its range
    (`overlap - 1` of them: 228 480 samples of halo at the MDX23C sizes), b200/sharded.py."""

    def __init__(self, net: TfcNet, n_fft, hop_length, dim_f, dim_t, overlap, dist=None, group=None):
        _require_cuda()
        from .sharded import ShardRunner

        self.net, self.n_fft, self.hop, self.dim_f, self.dim_t, self.overlap = net, int(n_fft), int(hop_length), int(dim_f), int(dim_t), int(overlap)
        self.chunk_size = self.hop * (self.dim_t - 1)  # :361
        self.hop_size = self.chunk_size // self.overlap  # :364
        self.plan = StftPlan(self.n_fft, self.hop)
        self.batch = net.max_batch
        self.device = torch.device("cuda", torch.cuda.current_device())
        self.runner = ShardRunner(dist, group)
        self.rank, self.world = self.runner.rank, self.runner.world

    def grid(self, n_samples):
        chunk, hop = self.chunk_size, self.hop_size
        pad = hop - (n_samples - chunk) % hop  # :367
        front = chunk - hop
        Lp = front + n_samples + pad + front
        return Lp, front, pad, (Lp - chunk) // hop + 1

    def model_run(self, wave: torch.Tensor) -> torch.Tensor:
        """TFC_TDF_net.forward (tfc_tdf_v3.py:230-267): (B,2,chunk) CUDA -> (B,S,2,chunk)."""
        B, _, T = wave.shape
        S = self.net.num_targets
        out = torch.empty((B, S, 2, T), dtype=torch.float32, device=wave.device)
        for b0 in range(0, B, self.batch):
            nb = min(self.batch, B - b0)
            spec = self.plan.forward(wave[b0 : b0 + nb], self.dim_f, 0, LAYOUT_CTF)
            y = self.net.forward_spec(spec)  # (nb, S, 4, frames, dim_f)
            w = self.plan.inverse(y.reshape(nb * S, 4, y.shape[-2], y.shape[-1]), LAYOUT_CTF)
            out[b0 : b0 + nb] = w.reshape(nb, S, 2, T)
        return out

    def out_range(self, N):
        return N * self.rank // self.world, N * (self.rank + 1) // self.world

    def demix_device(self, mix_dev: torch.Tensor) -> torch.Tensor:
        """mix (2,N) float32 CUDA -> (S, 2, q1 - q0): this rank's output range (the whole (S, 2, N) on a single GPU)."""
        from .sharded import plan_range_shards

        mix_dev = mix_dev.contiguous()
        N = mix_dev.shape[1]
        Lp, front, pad, n_chunks = self.grid(N)
        T, hop, S = self.chunk_size, self.hop_size, self.net.num_targets
        sh = plan_range_shards(N, self.world, n_chunks, hop, T, front)[self.rank]
        # this rank's part of the padded mixture (:371): positions [c0*hop, (c1-1)*hop + chunk)
        p0 = sh.c0 * hop
        p1 = (sh.c1 - 1) * hop + T if sh.n_own else p0 + 1
        padded = torch.zeros((2, p1 - p0), dtype=torch.float32, device=self.device)
        a, b = max(p0, front), min(p1, front + N)
        if b > a:
            padded[:, a - p0 : b - p0] = mix_dev[:, a - front : b - front]
        Ls = padded.shape[1]
        local = torch.empty((sh.halo + sh.n_own, S * 2, T), dtype=torch.float32, device=self.device)

        def compute(buf, slot0, unit0, nb):
            spec = torch.empty((nb, 4, self.dim_t, self.dim_f), dtype=torch.float32, device=self.device)
            off = unit0 * hop - p0
            # chunks are read straight out of the padded mixture (mix.unfold(1, chunk, hop), :374)
            check(lib.b200sep_stft_forward(self.plan.handle, padded.data_ptr() + off * 4, hop, Ls, Ls - off, nb, T, self.dim_f, 0, LAYOUT_CTF, _ptr(spec), _stream()), "stft_forward")
            y = self.net.forward_spec(spec)
            w = self.plan.inverse(y.reshape(nb * S, 4, self.dim_t, self.dim_f), LAYOUT_CTF)  # (nb*S, 2, T)
            buf[slot0 : slot0 + nb] = w.reshape(nb, S * 2, T)

        self.runner.wait_all(self.runner.run_units(sh, local, compute, self.batch))
        n_q = sh.q1 - sh.q0
        out = torch.empty((S * 2, n_q), dtype=torch.float32, device=self.device)
        if n_q:
            check(lib.b200sep_rect_overlap_add_range(_ptr(local), sh.c0 - sh.halo, sh.halo + sh.n_own, n_chunks, S * 2, T, hop, front, N, sh.q0, sh.q1, float(self.overlap),
                                                     _ptr(out), n_q, sh.q0, _stream()), "rect_overlap_add_range")  # :395-402
        return out.reshape(S, 2, n_q)

    def gather(self, part: torch.Tensor, N: int):
        """Rank 0: the full (S, 2, N) stems from every rank's demix_device slice (None elsewhere); identity on a single GPU."""
        if self.world == 1:
            return part
        return self.runner.gather_cols(part, [(N * r // self.world, N * (r + 1) // self.world) for r in range(self.world)], N)
