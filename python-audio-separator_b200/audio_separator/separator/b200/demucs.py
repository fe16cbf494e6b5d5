"""HTDemucs (Demucs v4) on the fp32 operator kernels of libb200sep.so.

HTDemucsNet.forward replaces HTDemucs.forward (uvr_lib_v5/demucs/htdemucs.py:483-620) for the structure of the released htdemucs
checkpoints (depth 4, no GroupNorm in the encoder/decoder layers, DConv in both, complex-as-channels, sin embeddings, norm_first +
layer-scale + norm_out cross-transformer).  DemucsEngine replaces apply_model (demucs/apply.py:124-260) and
DemucsSeparator.demix_demucs (architectures/demucs_separator.py:162-195).

This file is the graph builder only: it owns device buffers (torch tensors = device memory, nothing else) and the ORDER of the
operator launches; every arithmetic step is a kernel behind the C ABI (include/b200sep.h).  No CPU / ATen compute fallback.
"""
from __future__ import annotations

import math
from dataclasses import dataclass
from fractions import Fraction

import numpy as np
import torch

from ._lib import LAYOUT_CFT, MATH_BF16X3, check, lib
from .engine import StftPlan, _ptr, _require_cuda, _stream, _window
from .ops import (ACT_GELU, ACT_NONE, _new, block_conv_weight, block_convtr_weight, conv2d, conv_transpose, ew, gemm, glu, groupnorm1, layernorm, linear,
                  to_device)
from .sharded import ShardRunner, plan_range_shards

# Code written against this module imports the operator wrappers from it: they stay importable here, defined once in ops.py.
from .ops import ACT_RELU, _packed_conv, _packed_linear  # noqa: F401
from .ops import gemm as _gemm_raw  # noqa: F401

_DCONV_FUSED_HID = (4, 6, 8, 12, 16, 24, 32, 48)  # hidden widths b200sep_dconv_f32 is instantiated for


@dataclass
class HTDemucsConfig:
    """Constructor arguments of HTDemucs that shape the graph (htdemucs.py:36-98); defaults = the released htdemucs models."""

    sources: tuple = ("drums", "bass", "other", "vocals")
    audio_channels: int = 2
    channels: int = 48
    growth: int = 2
    nfft: int = 4096
    depth: int = 4
    kernel_size: int = 8
    stride: int = 4
    context: int = 1
    dconv_depth: int = 2
    dconv_comp: int = 8
    bottom_channels: int = 512
    t_layers: int = 5
    t_heads: int = 8
    t_hidden_scale: float = 4.0
    freq_emb: float = 0.2
    emb_scale: float = 10.0
    samplerate: int = 44100
    segment: Fraction = Fraction(39, 5)
    max_period: float = 10000.0

    @property
    def hop(self):
        return self.nfft // 4

    @property
    def seg_len(self):  # int(self.segment * self.samplerate), htdemucs.py:486
        return int(Fraction(self.segment) * self.samplerate)

    def valid_length(self, length):  # HTDemucs.valid_length (htdemucs.py:469-481): every input runs at the training segment
        return self.seg_len

    def validate(self):
        if self.audio_channels != 2:
            raise ValueError("the H100 HTDemucs path handles stereo models only")
        if self.kernel_size != 8 or self.stride != 4 or self.context != 1:
            raise ValueError("the H100 HTDemucs path needs kernel_size 8, stride 4, context 1 (the released htdemucs geometry)")
        if self.dconv_depth != 2:
            raise ValueError("the H100 HTDemucs path needs dconv_depth 2 (dilations 1 and 2)")
        if self.nfft // 2 != self.stride**self.depth * (self.nfft // 2 // self.stride**self.depth):
            raise ValueError("nfft/2 must be divisible by stride**depth")


def sin_embedding_1d(length: int, dim: int, max_period: float) -> np.ndarray:
    """create_sin_embedding (transformer.py:19-26) as (length, dim): [cos(phase) | sin(phase)]."""
    half = dim // 2
    pos = np.arange(length, dtype=np.float32)[:, None]
    expo = np.arange(half, dtype=np.float32)[None, :] / np.float32(half - 1)
    phase = pos / np.power(np.float32(max_period), expo, dtype=np.float32)
    return np.concatenate([np.cos(phase), np.sin(phase)], axis=1).astype(np.float32)


def sin_embedding_2d_tokens(dim: int, height: int, width: int, max_period: float) -> np.ndarray:
    """create_2d_sin_embedding (transformer.py:29-49) already rearranged "c fr t -> (t fr) c": (width*height, dim).
    First half of the channels encodes the width (time) position, second half the height (frequency) position, sin/cos interleaved."""
    half = dim // 2
    div = np.exp(np.arange(0, half, 2, dtype=np.float32) * np.float32(-(math.log(max_period) / half))).astype(np.float32)
    pw = np.arange(width, dtype=np.float32)[:, None] * div[None, :]   # (width, half/2)
    ph = np.arange(height, dtype=np.float32)[:, None] * div[None, :]  # (height, half/2)
    pe = np.zeros((width, height, dim), np.float32)
    pe[:, :, 0:half:2] = np.sin(pw)[:, None, :]
    pe[:, :, 1:half:2] = np.cos(pw)[:, None, :]
    pe[:, :, half::2] = np.sin(ph)[None, :, :]
    pe[:, :, half + 1 :: 2] = np.cos(ph)[None, :, :]
    return pe.reshape(width * height, dim)


# --------------------------------------------------------------------------------------------------------- the networks
class DemucsNetBase:
    """What every Demucs net shares: device, math mode, device weights and the plain DConv branch."""

    def __init__(self, cfg, device=None, math=MATH_BF16X3):
        """math: MATH_BF16X3 (default, ~fp32) or MATH_FP16 (torch.autocast precision) for every tensor-core GEMM, convolution and attention of
        this net, fixed for its lifetime (the graphs GraphedForward captures record the mode of each launch)."""
        _require_cuda()
        cfg.validate()
        self.cfg = cfg
        self.math = int(math)
        self.device = torch.device(device) if device is not None else torch.device("cuda", torch.cuda.current_device())  # one process per GPU: the rank's own device
        self.S = len(cfg.sources)
        self.W = {}

    def _put(self, name, a):
        self.W[name] = to_device(a, self.device)

    def _dconv(self, x, prefix):
        """DConv.forward (demucs.py:166-168) on x (B,C,Fr,T): conv1d k3 dilated -> GroupNorm(1)+GELU -> 1x1 -> GroupNorm(1) -> GLU, LayerScale residual."""
        W = self.W
        C_ = x.shape[1]
        if f"{prefix}.dconv.layers.0.0.weight" not in W:  # dconv_mode without DConv on this side (hdemucs.py:83-84, :268-269)
            return x
        B, _, Fr, L = x.shape
        for d in range(self.cfg.dconv_depth):
            p = f"{prefix}.dconv.layers.{d}"
            dil = 2**d
            hid = W[f"{p}.0.bias"].numel()
            if hid in _DCONV_FUSED_HID and C_ * 2 * (-(-hid // 4) * 4 + 4) * 4 <= 200 * 1024:
                # one fused residual layer (csrc/dconv_fused.cu); the C -> hid convolution of the widest layers stays on the tensor cores
                u_in = None
                if 3 * C_ * (-(-hid // 4) * 4) * 4 > 200 * 1024:
                    u_in = conv2d(x, W[f"{p}.0.weight"], W[f"{p}.0.bias"], hid, (1, 3), p=(0, dil), dw=dil, math=self.math)
                work = _new((lib.b200sep_dconv_work_floats(B, C_, Fr, L, hid),), x)
                check(lib.b200sep_dconv_f32(_ptr(x), _ptr(x), _ptr(W[f"{p}.0.weight:raw"]), _ptr(W[f"{p}.0.bias"]), _ptr(W[f"{p}.1.weight"]), _ptr(W[f"{p}.1.bias"]),
                                            _ptr(W[f"{p}.3.weight:raw"]), _ptr(W[f"{p}.3.bias"]), _ptr(W[f"{p}.4.weight"]), _ptr(W[f"{p}.4.bias"]), _ptr(W[f"{p}.6.scale"]),
                                            B, C_, Fr, L, hid, dil, _ptr(u_in) if u_in is not None else None, _ptr(work), _stream()), "dconv_f32")
                continue
            h = conv2d(x, W[f"{p}.0.weight"], W[f"{p}.0.bias"], hid, (1, 3), p=(0, dil), dw=dil, math=self.math)
            groupnorm1(h, W[f"{p}.1.weight"], W[f"{p}.1.bias"], ACT_GELU)
            h = conv2d(h, W[f"{p}.3.weight"], W[f"{p}.3.bias"], 2 * C_, (1, 1), math=self.math)
            groupnorm1(h, W[f"{p}.4.weight"], W[f"{p}.4.bias"])
            x = glu(h, res=x, scale=W[f"{p}.6.scale"])
        return x


class HybridDemucsNet(DemucsNetBase):
    """The spectral front and back ends of the hybrid (spectrogram + waveform) Demucs forwards and their STFT plan.  HTDemucsNet and HDemucsNet add
    their layers and launch order."""

    def __init__(self, cfg, device=None, math=MATH_BF16X3):
        super().__init__(cfg, device, math)
        self.stft = StftPlan(cfg.nfft, cfg.hop)

    def spec_in(self, mix, pad_mode):
        """_spec + _magnitude and the input normalisation (htdemucs.py:383-403, :415-424, :501-510; hdemucs.py:529-548, :570-579) on mix
        (B, 2, L) contiguous: the normalised STFT, frames 2 .. 2+le of the (3*hop/2, 3*hop/2 + le*hop - L)-padded signal (pad_mode 0 reflect, 1 zero),
        bins 0 .. nfft/2-1.  -> x (B, 4, nfft/2, le) and xt (B, 2, 1, L), standardised per sample, and stats (B, 4): per sample the mean and std of
        the spectrogram, then of the waveform."""
        B, _, length = mix.shape
        hl, nfft = self.cfg.hop, self.cfg.nfft
        le = -(-length // hl)
        Fq = nfft // 2
        spec = _new((B, 4, Fq, le), mix)
        check(lib.b200sep_stft_forward_ex(self.stft.handle, _ptr(mix), 2 * length, length, 0, B, length, le, hl // 2 * 3, 1.0 / math.sqrt(nfft), Fq, 0, LAYOUT_CFT,
                                          pad_mode, _ptr(spec), _stream()), "stft_forward_ex")
        stats = _new((B, 4), mix)
        x = _new(spec.shape, mix)
        xt = _new((B, 2, 1, length), mix)
        fs = 4
        mswork = _new((lib.b200sep_meanstd_work_floats(B),), mix)
        check(lib.b200sep_meanstd_batch_f32(_ptr(spec), spec[0].numel(), B, spec[0].numel(), _ptr(stats), 4, _ptr(mswork), _stream()), "meanstd_batch_f32")
        check(lib.b200sep_meanstd_batch_f32(_ptr(mix), mix[0].numel(), B, mix[0].numel(), stats.data_ptr() + 2 * fs, 4, _ptr(mswork), _stream()), "meanstd_batch_f32")
        for b in range(B):
            check(lib.b200sep_ew_f32(_ptr(spec[b]), stats.data_ptr() + (4 * b) * fs, _ptr(x[b]), spec[b].numel(), 1.0, 0.0, 2, _stream()), "ew_f32")
            check(lib.b200sep_ew_f32(_ptr(mix[b]), stats.data_ptr() + (4 * b + 2) * fs, _ptr(xt[b]), mix[b].numel(), 1.0, 0.0, 2, _stream()), "ew_f32")
        return x, xt, stats

    def spec_out(self, x, xt, stats, length, ola_offset):
        """The output end (htdemucs.py:405-413; hdemucs.py:550-568): x (B, S*4, nfft/2, le) * std + mean -> _mask (cac) -> _ispec, an
        iSTFT with the Nyquist bin and two frames per side zero whose overlap-add starts at sample ola_offset, plus the time branch xt * std + mean
        -> (B, S, 2, length).  De-normalises x and xt in place."""
        S = self.S
        B, _, Fq, le = x.shape
        out = _new((B, S, 2, length), x)
        nwork = lib.b200sep_stft_inverse_work_floats(self.stft.handle, S, le, Fq, LAYOUT_CFT)
        work = _new((nwork,), x)
        xi = _new((S, 2, length), x)
        fs = 4
        for b in range(B):
            check(lib.b200sep_ew_f32(_ptr(x[b]), stats.data_ptr() + (4 * b) * fs, _ptr(x[b]), x[b].numel(), 1.0, 0.0, 3, _stream()), "ew_f32")
            check(lib.b200sep_stft_inverse_ex(self.stft.handle, _ptr(x[b]), S, le, Fq, LAYOUT_CFT, length, ola_offset, 2, math.sqrt(self.cfg.nfft), _ptr(xi), _ptr(work),
                                              _stream()), "stft_inverse_ex")
            check(lib.b200sep_ew_f32(_ptr(xt[b]), stats.data_ptr() + (4 * b + 2) * fs, _ptr(out[b]), xt[b].numel(), 1.0, 0.0, 3, _stream()), "ew_f32")
            ew(out[b], xi, out[b])
        return out


class HTDemucsNet(HybridDemucsNet):
    """Device-resident HTDemucs weights (re-blocked for the conv kernel) + the launch sequence of one forward."""

    def __init__(self, cfg: HTDemucsConfig, state: dict, device=None, math=MATH_BF16X3):
        super().__init__(cfg, device, math)
        st = {k: np.asarray(v, dtype=np.float32) for k, v in state.items()}
        self._check_structure(st)
        for name, a in st.items():
            if ".dconv.layers." in name and name.endswith((".0.weight", ".3.weight")):  # the fused DConv kernel takes the plain (out, in[, k]) matrices
                self._put(name + ":raw", a.reshape(a.shape[0], -1) if name.endswith(".3.weight") else a)
            if name.endswith("conv_tr.weight"):
                a = block_convtr_weight(a.reshape(a.shape[0], a.shape[1], cfg.kernel_size), cfg.stride)
            elif name.endswith(".weight") and a.ndim >= 3 and "crosstransformer" not in name:
                if name.startswith(("encoder.", "decoder.")) and a.ndim == 4:
                    a = block_conv_weight(a)  # (co, ci, K, 1) freq conv / (co, ci, 3, 3) rewrite / (co, ci, 1, 1)
                else:  # Conv1d (co, ci, k) -> kernel (1, k)
                    a = block_conv_weight(a.reshape(a.shape[0], a.shape[1], 1, a.shape[2]))
            if name.endswith("in_proj_weight") or name.endswith("in_proj_bias"):  # nn.MultiheadAttention packs q, k, v: keep three persistent tensors
                D = a.shape[0] // 3
                kind = "weight" if name.endswith("weight") else "bias"
                for j, nm in enumerate("qkv"):
                    self._put(name.replace(f"in_proj_{kind}", f"{nm}_{kind}"), a[j * D : (j + 1) * D])
                continue
            self._put(name, a)
        # ScaledEmbedding.forward * freq_emb weight (hdemucs.py:62-64, htdemucs.py:539-541): added after encoder 0, shape (C, Fr)
        emb = st["freq_emb.embedding.weight"] * np.float32(cfg.emb_scale)  # (Fr, C)
        self.freq_emb_t = to_device((np.float32(cfg.freq_emb) * emb).T, self.device)
        self._pe_cache = {}
        self._emb_cache = {}
        from .graphs import GraphedForward

        self.graphed = GraphedForward(self.forward)

    def _check_structure(self, st):
        cfg = self.cfg
        need = ["encoder.0.conv.weight", "tencoder.0.conv.weight", "decoder.0.conv_tr.weight", "tdecoder.0.conv_tr.weight", "freq_emb.embedding.weight",
                "encoder.0.rewrite.weight", "decoder.0.rewrite.weight"]
        if cfg.t_layers:
            need += ["crosstransformer.norm_in.weight", "crosstransformer.layers.0.norm_out.weight", "crosstransformer.layers.0.gamma_1.scale"]
        for n in need:
            if n not in st:
                raise ValueError(f"state dict lacks {n}: not an htdemucs-v4 checkpoint of the supported structure")
        for n in st:
            if ".norm1.weight" in n and n.startswith(("encoder", "decoder", "tencoder", "tdecoder")):
                raise ValueError("encoder/decoder GroupNorm layers (norm_starts < depth) are not supported")
        if f"encoder.{cfg.depth - 1}.conv.weight" not in st or f"encoder.{cfg.depth}.conv.weight" in st:
            raise ValueError(f"state dict does not have depth {cfg.depth}")
        if st["encoder.0.conv.weight"].shape[0] != cfg.channels:
            raise ValueError("config.channels does not match the checkpoint")
        if any(".dconv.layers.0.3.weight" in n for n in st) and f"encoder.0.dconv.layers.{cfg.dconv_depth - 1}.0.weight" not in st and \
                f"decoder.0.dconv.layers.{cfg.dconv_depth - 1}.0.weight" not in st:
            raise ValueError("config.dconv_depth does not match the checkpoint")
        if any(".dconv.layers.0.0.weight" in n and st[n].shape[-1] != 3 for n in st) or any(".lstm." in n or ".attn." in n for n in st):
            raise ValueError("DConv with LSTM / attention or a kernel other than 3 is not supported")
        if bool(cfg.bottom_channels) != ("channel_upsampler.weight" in st):
            raise ValueError("config.bottom_channels does not match the checkpoint")

    # ---- sub-graphs --------------------------------------------------------------------------------------------
    def _enc(self, x, prefix, freq):
        """HEncLayer.forward (hdemucs.py:119-153), norm = Identity, empty = False."""
        W, cfg = self.W, self.cfg
        co = W[f"{prefix}.conv.bias"].numel()
        if freq:
            y = conv2d(x, W[f"{prefix}.conv.weight"], W[f"{prefix}.conv.bias"], co, (cfg.kernel_size, 1), s=(cfg.stride, 1), p=(cfg.kernel_size // 4, 0), act=ACT_GELU, math=self.math)
        else:
            le = x.shape[-1]
            y = conv2d(x, W[f"{prefix}.conv.weight"], W[f"{prefix}.conv.bias"], co, (1, cfg.kernel_size), s=(1, cfg.stride), p=(0, cfg.kernel_size // 4), act=ACT_GELU,
                       out_hw=(1, -(-le // cfg.stride)), math=self.math)  # F.pad to a multiple of the stride == implicit zero columns on the right
        y = self._dconv(y, prefix)
        z = conv2d(y, W[f"{prefix}.rewrite.weight"], W[f"{prefix}.rewrite.bias"], 2 * co, (1, 1), math=self.math)
        return glu(z)

    def _dec(self, x, skip, length, prefix, freq, last):
        """HDecLayer.forward (hdemucs.py:299-330), norm = Identity, empty = False."""
        W, cfg = self.W, self.cfg
        ci = x.shape[1]
        x = ew(x, skip, _new(x.shape, x))
        if freq:
            y = glu(conv2d(x, W[f"{prefix}.rewrite.weight"], W[f"{prefix}.rewrite.bias"], 2 * ci, (3, 3), p=(1, 1), math=self.math))
        else:
            y = glu(conv2d(x, W[f"{prefix}.rewrite.weight"], W[f"{prefix}.rewrite.bias"], 2 * ci, (1, 3), p=(0, 1), math=self.math))
        y = self._dconv(y, prefix)
        co = W[f"{prefix}.conv_tr.bias"].numel()
        act = ACT_NONE if last else ACT_GELU
        if freq:
            return conv_transpose(y, W[f"{prefix}.conv_tr.weight"], W[f"{prefix}.conv_tr.bias"], co, 1, cfg.stride, cfg.kernel_size // 4, y.shape[2] * cfg.stride, act, math=self.math)
        return conv_transpose(y, W[f"{prefix}.conv_tr.weight"], W[f"{prefix}.conv_tr.bias"], co, 2, cfg.stride, cfg.kernel_size // 4, length, act, math=self.math)

    def _mha(self, q_in, kv_in, p, res, res_scale):
        """nn.MultiheadAttention(batch_first) + the layer-scaled residual: res + gamma * out_proj(softmax(QK^T/sqrt(hd)) V).  q_in (B,Lq,D), kv_in (B,Lk,D)."""
        W = self.W
        B, Lq, D = q_in.shape
        Lk = kv_in.shape[1]
        H = self.cfg.t_heads
        hd = D // H
        q = linear(q_in.view(B * Lq, D), W[f"{p}.q_weight"], W[f"{p}.q_bias"], math=self.math)
        k = linear(kv_in.view(B * Lk, D), W[f"{p}.k_weight"], W[f"{p}.k_bias"], math=self.math)
        # V^T per batch: (D, Lk) = Wv (D,D) @ kv^T, bias per row
        vt = _new((B, D, Lk), q_in)
        wv, bv = W[f"{p}.v_weight"], W[f"{p}.v_bias"]
        gemm(_ptr(wv), _ptr(kv_in), _ptr(vt), D, Lk, D, D, D, Lk, B, 0, Lk * D, D * Lk, bias_m=_ptr(bv), math=self.math)
        o = _new((B, Lq, D), q_in)
        if hd == 64:  # one kernel, the (H, Lq, Lk) scores stay on chip
            work = _new((lib.b200sep_attention_work_floats_math(B, H, Lq, Lk, self.math),), q_in)  # tile images of Q, K, V^T (split once, not once per consumer)
            check(lib.b200sep_attention_f32_math(_ptr(q), _ptr(k), _ptr(vt), _ptr(o), B, H, Lq, Lk, hd, Lq * D, D, Lk * D, D, D * Lk, Lk, Lq * D, D, 1.0 / math.sqrt(hd),
                                                 0, _ptr(work), self.math, _stream()), "attention_f32")
            y = linear(o.view(B * Lq, D), W[f"{p}.out_proj.weight"], W[f"{p}.out_proj.bias"], res=res.view(B * Lq, D), res_scale=res_scale, math=self.math)
            return y.view(B, Lq, D)
        sc = _new((H, Lq, Lk), q_in)
        fs = 4  # bytes per float
        for b in range(B):
            gemm(q.data_ptr() + b * Lq * D * fs, k.data_ptr() + b * Lk * D * fs, _ptr(sc), Lq, Lk, hd, D, D, Lk, H, hd, hd, Lq * Lk, alpha=1.0 / math.sqrt(hd), math=self.math)
            check(lib.b200sep_softmax_rows_f32(_ptr(sc), H * Lq, Lk, Lk, _stream()), "softmax_rows_f32")
            gemm(_ptr(sc), vt.data_ptr() + b * D * Lk * fs, o.data_ptr() + b * Lq * D * fs, Lq, hd, Lk, Lk, Lk, D, H, Lq * Lk, hd * Lk, hd, math=self.math)
        y = linear(o.view(B * Lq, D), W[f"{p}.out_proj.weight"], W[f"{p}.out_proj.bias"], res=res.view(B * Lq, D), res_scale=res_scale, math=self.math)
        return y.view(B, Lq, D)

    def _ffn(self, x_norm, x, p):
        W = self.W
        B, L, D = x.shape
        h = linear(x_norm.view(B * L, D), W[f"{p}.linear1.weight"], W[f"{p}.linear1.bias"], act=ACT_GELU, math=self.math)
        return linear(h, W[f"{p}.linear2.weight"], W[f"{p}.linear2.bias"], res=x.view(B * L, D), res_scale=W[f"{p}.gamma_2.scale"], math=self.math).view(B, L, D)

    def _self_layer(self, x, p):  # MyTransformerEncoderLayer.forward, norm_first (transformer.py:268-274)
        W = self.W
        n1 = layernorm(x, W[f"{p}.norm1.weight"], W[f"{p}.norm1.bias"])
        x = self._mha(n1, n1, f"{p}.self_attn", x, W[f"{p}.gamma_1.scale"])
        x = self._ffn(layernorm(x, W[f"{p}.norm2.weight"], W[f"{p}.norm2.bias"]), x, p)
        return groupnorm1(x, W[f"{p}.norm_out.weight"], W[f"{p}.norm_out.bias"], channel_last=True)

    def _cross_layer(self, q, k, p):  # CrossTransformerEncoderLayer.forward, norm_first (transformer.py:385-390)
        W = self.W
        x = self._mha(layernorm(q, W[f"{p}.norm1.weight"], W[f"{p}.norm1.bias"]), layernorm(k, W[f"{p}.norm2.weight"], W[f"{p}.norm2.bias"]), f"{p}.cross_attn", q,
                      W[f"{p}.gamma_1.scale"])
        x = self._ffn(layernorm(x, W[f"{p}.norm3.weight"], W[f"{p}.norm3.bias"]), x, p)
        return groupnorm1(x, W[f"{p}.norm_out.weight"], W[f"{p}.norm_out.bias"], channel_last=True)

    def _pos(self, kind, *dims):
        key = (kind,) + dims
        if key not in self._pe_cache:
            a = sin_embedding_2d_tokens(*dims, self.cfg.max_period) if kind == "2d" else sin_embedding_1d(*dims, self.cfg.max_period)
            self._pe_cache[key] = torch.from_numpy(a).to(self.device)
        return self._pe_cache[key]

    def _transformer(self, x, xt):
        """channel up-samplers + CrossTransformerEncoder.forward + channel down-samplers (htdemucs.py:546-560, transformer.py:529-560)."""
        W, cfg = self.W, self.cfg
        B, c0, Fr, T1 = x.shape
        if cfg.bottom_channels:
            D = cfg.bottom_channels
            x = conv2d(x.view(B, c0, 1, Fr * T1), W["channel_upsampler.weight"], W["channel_upsampler.bias"], D, (1, 1), math=self.math).view(B, D, Fr, T1)
            xt = conv2d(xt, W["channel_upsampler_t.weight"], W["channel_upsampler_t.bias"], D, (1, 1), math=self.math)
        D = x.shape[1]
        T2 = xt.shape[-1]
        xs = _new((B, T1, Fr, D), x)  # "b c fr t1 -> b (t1 fr) c"
        check(lib.b200sep_permute4_f32(_ptr(x), _ptr(xs), B, D, Fr, T1, 0, 3, 2, 1, _stream()), "permute4_f32")
        xs = layernorm(xs.view(B, T1 * Fr, D), W["crosstransformer.norm_in.weight"], W["crosstransformer.norm_in.bias"])
        pe2 = self._pos("2d", D, Fr, T1)
        for b in range(B):
            ew(xs[b], pe2, xs[b])
        xts = _new((B, T2, 1, D), x)  # "b c t2 -> b t2 c"
        check(lib.b200sep_permute4_f32(_ptr(xt), _ptr(xts), B, D, 1, T2, 0, 3, 2, 1, _stream()), "permute4_f32")
        xts = layernorm(xts.view(B, T2, D), W["crosstransformer.norm_in_t.weight"], W["crosstransformer.norm_in_t.bias"])
        pe1 = self._pos("1d", T2, D)
        for b in range(B):
            ew(xts[b], pe1, xts[b])
        for li in range(cfg.t_layers):
            pf, pt = f"crosstransformer.layers.{li}", f"crosstransformer.layers_t.{li}"
            if li % 2 == 0:
                xs = self._self_layer(xs, pf)
                xts = self._self_layer(xts, pt)
            else:
                old = xs
                xs = self._cross_layer(xs, xts, pf)
                xts = self._cross_layer(xts, old, pt)
        x = _new((B, D, Fr, T1), xs)
        check(lib.b200sep_permute4_f32(_ptr(xs), _ptr(x), B, T1, Fr, D, 0, 3, 2, 1, _stream()), "permute4_f32")
        xt = _new((B, D, 1, T2), xs)
        check(lib.b200sep_permute4_f32(_ptr(xts), _ptr(xt), B, T2, 1, D, 0, 3, 2, 1, _stream()), "permute4_f32")
        if cfg.bottom_channels:
            x = conv2d(x.view(B, D, 1, Fr * T1), W["channel_downsampler.weight"], W["channel_downsampler.bias"], c0, (1, 1), math=self.math).view(B, c0, Fr, T1)
            xt = conv2d(xt, W["channel_downsampler_t.weight"], W["channel_downsampler_t.bias"], c0, (1, 1), math=self.math)
        return x, xt

    # ---- forward ---------------------------------------------------------------------------------------------------
    def forward(self, mix: torch.Tensor) -> torch.Tensor:
        """mix (B, 2, L <= seg_len) float32 cuda -> (B, S, 2, L).  (eval mode, use_train_segment: shorter inputs are zero-padded
        to the training segment and the output is cut back, htdemucs.py:486-493, :614-618.)"""
        cfg = self.cfg
        assert mix.dim() == 3 and mix.shape[1] == 2 and mix.dtype == torch.float32 and mix.is_cuda
        B, _, L0 = mix.shape
        T_len = cfg.seg_len
        if L0 > T_len:
            raise ValueError(f"segment of {L0} samples exceeds the training segment {T_len}")
        if L0 < T_len:
            mp = torch.zeros((B, 2, T_len), dtype=torch.float32, device=mix.device)
            mp[..., :L0].copy_(mix)
        else:
            mp = mix.contiguous()
        x, xt, stats = self.spec_in(mp, 0)  # reflect-padded
        saved, saved_t, lengths_t = [], [], []
        for i in range(cfg.depth):  # htdemucs.py:520-544 (every time encoder runs: no "empty" layers at depth 4)
            lengths_t.append(xt.shape[-1])
            xt = self._enc(xt, f"tencoder.{i}", False)
            saved_t.append(xt)
            x = self._enc(x, f"encoder.{i}", True)
            if i == 0:
                Bc, Cc, Fr, Tt = x.shape
                emb = self._freq_emb_full(Fr, Tt, Cc)
                for b in range(B):
                    ew(x[b], emb, x[b])
            saved.append(x)
        if cfg.t_layers:
            x, xt = self._transformer(x, xt)
        for j in range(cfg.depth):  # :562-580
            last = j == cfg.depth - 1
            x = self._dec(x, saved.pop(-1), 0, f"decoder.{j}", True, last)
            xt = self._dec(xt, saved_t.pop(-1), lengths_t.pop(-1), f"tdecoder.{j}", False, last)
        out = self.spec_out(x, xt, stats, T_len, cfg.hop // 2 * 3)
        return out[..., :L0] if L0 < T_len else out

    def _freq_emb_full(self, Fr, Tt, Cc):
        """freq_emb * emb broadcast over time, (C, Fr, T) -- materialised once per shape so the add is a plain element-wise kernel."""
        key = (Fr, Tt, Cc)
        if key not in self._emb_cache:
            self._emb_cache[key] = self.freq_emb_t[:, :, None].expand(Cc, Fr, Tt).contiguous()
        return self._emb_cache[key]

    __call__ = forward


# --------------------------------------------------------------------------------------------------------- apply_model / demix
def group_units(clens, seg, pads):
    """Consecutive units (segments of one apply_model pass) that can share a forward: -> [(j0, j1, input width)].  A model that pads every chunk to its training
    segment (HTDemucs.valid_length, htdemucs.py:469-481) takes all of them at width `seg`; otherwise `clens` are the input widths (the chunk lengths for HDemucs,
    which has no valid_length, apply.py:252-257; their valid lengths for Demucs), and only runs of equal width batch -- in practice all full segments, then the
    shorter last one."""
    if pads:
        return [(0, len(clens), seg)] if clens else []
    groups, j0 = [], 0
    while j0 < len(clens):
        j1 = j0 + 1
        while j1 < len(clens) and clens[j1] == clens[j0]:
            j1 += 1
        groups.append((j0, j1, clens[j0]))
        j0 = j1
    return groups


class DemucsEngine:
    """apply_model(shifts, split=True, overlap) over a bag of HTDemucs models + DemucsSeparator.demix_demucs, device resident.

    With `dist` (torch.distributed, backend nccl, one process per GPU) the segments of every (model, shift) pass are time-sharded
    (SURVEY.md section 8e, Demucs row, option A): rank r finalises the output samples [N*r/W, N*(r+1)/W) of EVERY pass, computes the
    segments that start in that range and receives from its left neighbour the one or two segments that reach into it (b200/sharded.py).
    Per output sample the passes accumulate in the single-GPU order, so the sharded result is the single-GPU result."""

    def __init__(self, nets, bag_weights=None, overlap=0.25, batch_size=4, dist=None, group=None, split=True):
        """nets: the bag's members, each run at its own segment and padding rule (cfg.seg_len, cfg.valid_length); self.cfg (the first member's)
        supplies only what a bag shares: sources and sample rate (apply.py:46-50)."""
        _require_cuda()
        self.nets = list(nets)
        cfg = self.nets[0].cfg
        self.cfg = cfg
        S = len(cfg.sources)
        if bag_weights is None:
            bag_weights = [[1.0] * S for _ in self.nets]  # BagOfModels default (apply.py:52-57)
        assert len(bag_weights) == len(self.nets) and all(len(w) == S for w in bag_weights)
        self.bag_weights = [list(map(float, w)) for w in bag_weights]
        self.overlap = float(overlap)
        self.batch_size = int(batch_size)
        self.device = self.nets[0].device
        self.runner = ShardRunner(dist, group)
        self.split = bool(split)  # apply_model(split=...): False = segments_enabled False, ONE forward over the whole (shifted) track (apply.py:251-260)
        if not self.split and self.runner.world > 1:
            raise ValueError("split=False is one forward over the whole track: nothing to shard across ranks")

    def out_range(self, N):
        """Output samples [q0, q1) this rank finalises (everything on a single GPU)."""
        return self.runner.out_range(N)

    def _apply_split(self, net, tensor, offset, length, out, q0, n_out, scale, chan_scale, accumulate):
        """apply_model's split branch on TensorChunk(tensor, offset, length) (apply.py:215-250); the weighted result's samples
        [q0, q0 + n_out) -- this rank's part [r0, r1) of them -- are scaled and written / accumulated into out (S*2, r1 - r0)."""
        cfg = net.cfg
        seg = cfg.seg_len
        S = len(cfg.sources)
        stride = int((1 - self.overlap) * seg)
        offs = list(range(0, length, stride))
        sh = plan_range_shards(n_out, self.runner.world, len(offs), stride, seg, q0)[self.runner.rank]
        assert tuple(out.shape) == (S * 2, sh.q1 - sh.q0), (out.shape, sh)
        # TensorChunk.padded zero-fills outside the tensor (apply.py:97-113): only the part this rank's segments read is materialised
        lo = offset + sh.c0 * stride - seg
        hi = offset + (sh.c1 - 1) * stride + 2 * seg if sh.n_own else lo + 1
        ext = _window(tensor, lo, hi)
        local = torch.empty((sh.halo + sh.n_own, S * 2, seg), dtype=torch.float32, device=tensor.device)

        def compute(buf, slot0, unit0, n):
            clens = [min(length - offs[unit0 + j], seg) for j in range(n)]
            # chunk.padded(model.valid_length(chunk length)) (apply.py:252-257): HTDemucs the training segment, HDemucs the chunk itself, Demucs the nearest
            # length its convolutions consume whole -- centred, real neighbouring samples where the tensor has them
            widths = [cfg.valid_length(c) for c in clens]
            for j0, j1, width in group_units(widths, seg, False):  # units of one input width form one forward (only the last segment of a pass is shorter)
                batch = _new((j1 - j0, 2, width), tensor)
                for j in range(j0, j1):
                    start = offset + offs[unit0 + j] - (width - clens[j]) // 2 - lo
                    assert 0 <= start and start + width <= ext.shape[-1], (start, width, ext.shape)
                    batch[j - j0].copy_(ext[:, start : start + width])
                y = net.graphed(batch)  # (n, S, 2, width): the launch list of the forward (HTDemucs: replayed as one CUDA graph per batch size)
                for j in range(j0, j1):  # center_trim to the chunk length (apply.py:258), stored from sample 0
                    d = (width - clens[j]) // 2
                    buf[slot0 + j, :, : clens[j]].copy_(y[j - j0].reshape(S * 2, width)[:, d : d + clens[j]])

        self.runner.wait_all(self.runner.run_units(sh, local, compute, self.batch_size))
        if sh.q1 > sh.q0:
            check(lib.b200sep_triangle_overlap_add_range(_ptr(local), sh.c0 - sh.halo, sh.halo + sh.n_own, len(offs), S * 2, seg, stride, length, q0 + sh.q0, sh.q1 - sh.q0,
                                                         scale, _ptr(chan_scale) if chan_scale is not None else None, int(accumulate), _ptr(out), sh.q1 - sh.q0, 0,
                                                         _stream()), "triangle_overlap_add_range")

    def _apply_whole(self, net, tensor, offset, length, out, q0, n_out, scale, chan_scale, accumulate):
        """apply_model's leaf (apply.py:251-260) on TensorChunk(tensor, offset, length): the chunk zero-padded (centred) to model.valid_length(length) -- the training
        segment for HTDemucs, which REFUSES anything longer (htdemucs.py:469-481); the length itself for models without valid_length -- one forward, center_trim."""
        cfg = net.cfg
        S = len(cfg.sources)
        valid = cfg.valid_length(length)
        if valid < length:
            raise ValueError(f"Given length {length} is longer than training length {valid}")
        delta = valid - length
        start = offset - delta // 2
        batch = _window(tensor, start, start + valid)[None]
        y = net.forward(batch).reshape(S * 2, valid)
        d = delta // 2  # center_trim (utils.py:53-70): delta // 2 off the left
        cs = chan_scale.cpu().tolist() if chan_scale is not None else [1.0] * (S * 2)
        for c in range(S * 2):
            src = y[c, d + q0 : d + q0 + n_out]
            ew(src, out[c] if accumulate else None, out[c], scale * cs[c], 1.0 if accumulate else 0.0)

    def apply_model(self, mix: torch.Tensor, shift_offsets, net_index=0, out=None, chan_scale=None, accumulate=False):
        """mix (2, N) cuda -> (S*2, q1 - q0): this rank's output range (the whole (S*2, N) on a single GPU).
        shift_offsets: the `random.randint(0, max_shift)` draws of apply.py:207 (empty = shifts 0)."""
        net = self.nets[net_index]
        S = len(self.cfg.sources)
        N = mix.shape[-1]
        r0, r1 = self.out_range(N)
        if out is None:
            out = _new((S * 2, r1 - r0), mix)
        one = self._apply_split if self.split else self._apply_whole
        if not shift_offsets:
            one(net, mix, 0, N, out, 0, N, 1.0, chan_scale, accumulate)
            return out
        ms = int(0.5 * net.cfg.samplerate)
        pm = torch.zeros((2, N + 2 * ms), dtype=torch.float32, device=mix.device)
        pm[:, ms : ms + N].copy_(mix)
        for i, o in enumerate(shift_offsets):
            one(net, pm, o, N + ms - o, out, ms - o, N, 1.0 / len(shift_offsets), chan_scale, accumulate or i > 0)
        return out

    def demix_device(self, mix_d: torch.Tensor, shift_offsets) -> torch.Tensor:
        """DemucsSeparator.demix_demucs (demucs_separator.py:162-195) on a (2, N) CUDA mix -> this rank's (S, 2, q1 - q0) slice of the sources
        (sources 0/1 swapped like the reference; the whole (S, 2, N) on a single GPU).  shift_offsets: one list of shift draws per model of the bag."""
        S = len(self.cfg.sources)
        N = mix_d.shape[1]
        ref = ew(mix_d[0], mix_d[1], _new((N,), mix_d), 0.5, 0.5)
        stats = _new((2,), mix_d)
        check(lib.b200sep_meanstd_f32(_ptr(ref), N, _ptr(stats), _stream()), "meanstd_f32")
        mean, std = (float(v) for v in stats.cpu())
        mn = ew(mix_d, None, _new(mix_d.shape, mix_d), 1.0 / std, -mean / std)
        tot = np.sum(np.asarray(self.bag_weights, np.float64), axis=0)
        r0, r1 = self.out_range(N)
        out = _new((S * 2, r1 - r0), mix_d)
        for mi in range(len(self.nets)):
            cs = torch.tensor(np.repeat(np.asarray(self.bag_weights[mi]) / tot, 2).astype(np.float32), device=self.device)
            self.apply_model(mn, list(shift_offsets[mi]), mi, out, cs, accumulate=mi > 0)
        ew(out, None, out, std, mean)
        src = out.view(S, 2, r1 - r0)
        return torch.cat([src[1:2], src[0:1], src[2:]], dim=0) if S >= 2 else src

    def gather(self, part: torch.Tensor, N: int):
        """Rank 0: the full (S, 2, N) sources from every rank's demix_device slice (None elsewhere); identity on a single GPU."""
        return self.runner.gather(part, N)

    def demix_host(self, mix_host: torch.Tensor, out_host: torch.Tensor, shift_offsets):
        """End-to-end entry point on page-locked host tensors: mix_host (2, N) -> out_host (S, 2, N).  Sharded runs map the SAME two buffers in every rank:
        each rank uploads the mix over its own PCIe link and downloads only the (S, 2, q1 - q0) slice it finalised -- no gather.  Returns this rank's (h2d, d2h) bytes."""
        mix_d = mix_host.to(self.device, non_blocking=True)
        N = mix_d.shape[1]
        part = self.demix_device(mix_d, shift_offsets)
        r0, r1 = self.out_range(N)
        S = part.shape[0]
        for s_ in range(S if r1 > r0 else 0):
            for c in range(2):
                out_host[s_, c, r0:r1].copy_(part[s_, c], non_blocking=True)  # contiguous row slices: true async copies
        torch.cuda.current_stream().synchronize()
        return int(mix_host.numel() * 4), int(part.numel() * 4)

    def demix(self, mix: np.ndarray, shift_offsets) -> np.ndarray:
        """Host arrays in and out: mix (2, N) -> sources (S, 2, N) (rank 0; None on the other ranks of a sharded run)."""
        mix_d = torch.from_numpy(np.ascontiguousarray(mix, dtype=np.float32)).to(self.device)
        full = self.gather(self.demix_device(mix_d, shift_offsets), mix_d.shape[1])
        return None if full is None else full.cpu().numpy()
