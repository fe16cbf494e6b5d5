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
import os
from dataclasses import dataclass
from fractions import Fraction

import numpy as np
import torch

from ._lib import LAYOUT_CFT, check, lib
from .engine import StftPlan, _ptr, _require_cuda, _stream

ACT_NONE, ACT_RELU, ACT_GELU = 0, 1, 2
_FUSED_ATTENTION = os.environ.get("B200SEP_FUSED_ATTN", "1") != "0"  # 0: the unfused scores / softmax / P V launches (A/B measurements)
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

    def validate(self):
        if self.audio_channels != 2:
            raise ValueError("the H100 HTDemucs path handles stereo models only")
        if self.kernel_size != 8 or self.stride != 4 or self.context != 1:
            raise ValueError("the H100 HTDemucs path needs kernel_size 8, stride 4, context 1 (the released htdemucs geometry)")
        if self.dconv_depth != 2:
            raise ValueError("the H100 HTDemucs path needs dconv_depth 2 (dilations 1 and 2)")
        if self.nfft // 2 != self.stride**self.depth * (self.nfft // 2 // self.stride**self.depth):
            raise ValueError("nfft/2 must be divisible by stride**depth")


# --------------------------------------------------------------------------------------------------------- host-side weight prep
def _ceil48(n):
    return -(-n // 48) * 48


def block_conv_weight(w: np.ndarray) -> np.ndarray:
    """(Cout, Cin, KH, KW) -> [Cin][KH*KW][ceil48(Cout)], the layout b200sep_conv2d_f32 streams through shared memory."""
    co, ci, kh, kw = w.shape
    out = np.zeros((ci, kh * kw, _ceil48(co)), np.float32)
    out[:, :, :co] = w.transpose(1, 2, 3, 0).reshape(ci, kh * kw, co)
    return out


def block_convtr_weight(w: np.ndarray, stride: int) -> np.ndarray:
    """ConvTranspose weight (Cin, Cout, K) with K = 2*stride -> the 2-tap convolution over the coarse index q whose GEMM column
    r*Cout + co produces output sample q*stride + r:   y[q*s + r] = x[q-1] . W[:, :, r + s] + x[q] . W[:, :, r]."""
    ci, co, k = w.shape
    assert k == 2 * stride
    out = np.zeros((ci, 2, _ceil48(stride * co)), np.float32)
    for r in range(stride):
        out[:, 0, r * co : (r + 1) * co] = w[:, :, r + stride]
        out[:, 1, r * co : (r + 1) * co] = w[:, :, r]
    return out


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


# --------------------------------------------------------------------------------------------------------- operator wrappers
def _new(shape, like=None, device=None):
    return torch.empty(shape, dtype=torch.float32, device=like.device if like is not None else device)


def _packed_conv(wb, cin, taps, cout):
    """The tensor-core image of a blocked convolution weight (bf16 hi/lo planes in the kernel's shared-memory layout), built once per tensor."""
    pk = getattr(wb, "_b200_packed", None)
    if pk is None and cin * taps >= 32 and cout >= 16:
        cin8 = -(-cin // 8) * 8
        pk = _new((lib.b200sep_tc_packed_floats(cout, cin8 * taps),), wb)
        check(lib.b200sep_tc_pack_conv_weights(_ptr(wb), cin, taps, cout, _ptr(pk), _stream()), "tc_pack_conv_weights")
        wb._b200_packed = pk
    return pk


def _packed_linear(w):
    pk = getattr(w, "_b200_packed", None)
    if pk is None and w.shape[0] >= 32 and w.shape[1] >= 32:
        pk = _new((lib.b200sep_tc_packed_floats(w.shape[0], w.shape[1]),), w)
        check(lib.b200sep_tc_pack_linear_weights(_ptr(w), w.shape[0], w.shape[1], w.shape[1], _ptr(pk), _stream()), "tc_pack_linear_weights")
        w._b200_packed = pk
    return pk


def conv2d(x, wb, bias, cout, k, s=(1, 1), p=(0, 0), dw=1, act=ACT_NONE, add=None, add_before_act=False, out_hw=None, out=None, out_c_off=0, dh=1):
    """x (B,Cin,H,W) -> (B,cout,Ho,Wo);  out_hw overrides the implied output size (right/bottom zero padding is implicit);
    out/out_c_off: write into channels [out_c_off, out_c_off + cout) of an existing (B, C_total, Ho, Wo) tensor (a fused torch.cat)."""
    B, cin, H, W = x.shape
    if out_hw is None:
        Ho = (H + 2 * p[0] - dh * (k[0] - 1) - 1) // s[0] + 1
        Wo = (W + 2 * p[1] - dw * (k[1] - 1) - 1) // s[1] + 1
    else:
        Ho, Wo = out_hw
    if out is None:
        y, ct = _new((B, cout, Ho, Wo), x), 0
    else:
        assert out.shape[0] == B and tuple(out.shape[2:]) == (Ho, Wo), (out.shape, (B, cout, Ho, Wo))
        y, ct = out, out.shape[1]
    pk = _packed_conv(wb, cin, k[0] * k[1], cout)
    check(lib.b200sep_conv2d_f32(_ptr(x), _ptr(wb), _ptr(bias) if bias is not None else None, _ptr(add) if add is not None else None, _ptr(y), B, cin, H, W, cout,
                                 Ho, Wo, k[0], k[1], s[0], s[1], p[0], p[1], dh, dw, act, int(add_before_act), 0, 1, 0, 0, ct, out_c_off,
                                 _ptr(pk) if pk is not None else None, _stream()), "conv2d_f32")
    return y


def conv_transpose(x, wb, bias, cout, axis, stride, trim, out_len, act=ACT_NONE):
    """nn.ConvTranspose1d/2d with kernel 2*stride along `axis` (1 = H, 2 = W), output cropped to [trim, trim + out_len)."""
    B, cin, H, W = x.shape
    if axis == 1:
        y = _new((B, cout, out_len, W), x)
        k, p, hw = (2, 1), (1, 0), (H + 1, W)
    else:
        y = _new((B, cout, H, out_len), x)
        k, p, hw = (1, 2), (0, 1), (H, W + 1)
    pk = _packed_conv(wb, cin, 2, stride * cout)
    check(lib.b200sep_conv2d_f32(_ptr(x), _ptr(wb), _ptr(bias), None, _ptr(y), B, cin, H, W, stride * cout, hw[0], hw[1], k[0], k[1], 1, 1, p[0], p[1], 1, 1, act, 0,
                                 axis, stride, trim, out_len, 0, 0, _ptr(pk) if pk is not None else None, _stream()), "conv2d_f32(transposed)")
    return y


def groupnorm1(x, gamma, beta, act=ACT_NONE, channel_last=False):
    """in place; x (B,C,Fr,L) channel-first (one sample per (b, fr)) or (B,L,C) channel_last."""
    if channel_last:
        B, L, Cc = x.shape
        Fr = 1
    else:
        B, Cc, Fr, L = x.shape
    work = _new((lib.b200sep_groupnorm1_work_floats(B, Cc, Fr, L),), x)
    check(lib.b200sep_groupnorm1_f32(_ptr(x), _ptr(gamma), _ptr(beta), _ptr(x), B, Cc, Fr, L, act, int(channel_last), _ptr(work), _stream()), "groupnorm1_f32")
    return x


def glu(a, res=None, scale=None):
    B, c2, H, W = a.shape
    y = _new((B, c2 // 2, H, W), a)
    check(lib.b200sep_glu_f32(_ptr(a), _ptr(res) if res is not None else None, _ptr(scale) if scale is not None else None, _ptr(y), B, c2 // 2, H * W, _stream()), "glu_f32")
    return y


def layernorm(x, gamma, beta):
    y = torch.empty_like(x)
    check(lib.b200sep_layernorm_f32(_ptr(x), _ptr(gamma), _ptr(beta), _ptr(y), x.numel() // x.shape[-1], x.shape[-1], _stream()), "layernorm_f32")
    return y


def ew(a, b, out, alpha=1.0, beta=1.0, op=0):
    check(lib.b200sep_ew_f32(_ptr(a), _ptr(b) if b is not None else None, _ptr(out), a.numel(), alpha, beta, op, _stream()), "ew_f32")
    return out


def linear(x2d, w, bias, act=ACT_NONE, res=None, res_scale=None):
    """(M,K) @ w(N,K)^T + bias -> (M,N); optional res + res_scale[n] * (.)"""
    M, K = x2d.shape
    N = w.shape[0]
    y = _new((M, N), x2d)
    pk = _packed_linear(w)
    check(lib.b200sep_gemm_f32(_ptr(x2d), _ptr(w), _ptr(y), M, N, K, K, K, N, 1, 0, 0, 0, 1.0, _ptr(bias) if bias is not None else None, None, act,
                               _ptr(res) if res is not None else None, _ptr(res_scale) if res_scale is not None else None, _ptr(pk) if pk is not None else None,
                               _stream()), "gemm_f32")
    return y


def _gemm_raw(a_ptr, b_ptr, c_ptr, M, N, K, lda, ldb, ldc, batch, sA, sB, sC, alpha=1.0, bias_n=None, bias_m=None):
    check(lib.b200sep_gemm_f32(a_ptr, b_ptr, c_ptr, M, N, K, lda, ldb, ldc, batch, sA, sB, sC, alpha, bias_n, bias_m, 0, None, None, None, _stream()), "gemm_f32")


# --------------------------------------------------------------------------------------------------------- the network
class HTDemucsNet:
    """Device-resident HTDemucs weights (re-blocked for the conv kernel) + the launch sequence of one forward."""

    def __init__(self, cfg: HTDemucsConfig, state: dict, device=None):
        _require_cuda()
        cfg.validate()
        self.cfg = cfg
        self.device = torch.device(device) if device is not None else torch.device("cuda", torch.cuda.current_device())  # one process per GPU: the rank's own device
        self.S = len(cfg.sources)
        self.stft = StftPlan(cfg.nfft, cfg.hop)
        self.W = {}
        st = {k: np.asarray(v, dtype=np.float32) for k, v in state.items()}
        self._check_structure(st)
        for name, a in st.items():
            if ".dconv.layers." in name and name.endswith((".0.weight", ".3.weight")):  # the fused DConv kernel takes the plain (out, in[, k]) matrices
                self.W[name + ":raw"] = torch.from_numpy(np.ascontiguousarray(a.reshape(a.shape[0], -1) if name.endswith(".3.weight") else a)).to(self.device)
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
                    self.W[name.replace(f"in_proj_{kind}", f"{nm}_{kind}")] = torch.from_numpy(np.ascontiguousarray(a[j * D : (j + 1) * D])).to(self.device)
                continue
            self.W[name] = torch.from_numpy(np.ascontiguousarray(a)).to(self.device)
        # ScaledEmbedding.forward * freq_emb weight (hdemucs.py:62-64, htdemucs.py:539-541): added after encoder 0, shape (C, Fr)
        emb = st["freq_emb.embedding.weight"] * np.float32(cfg.emb_scale)  # (Fr, C)
        self.freq_emb_t = torch.from_numpy(np.ascontiguousarray((np.float32(cfg.freq_emb) * emb).T)).to(self.device)
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
                    u_in = conv2d(x, W[f"{p}.0.weight"], W[f"{p}.0.bias"], hid, (1, 3), p=(0, dil), dw=dil)
                work = _new((lib.b200sep_dconv_work_floats(B, C_, Fr, L, hid),), x)
                check(lib.b200sep_dconv_f32(_ptr(x), _ptr(x), _ptr(W[f"{p}.0.weight:raw"]), _ptr(W[f"{p}.0.bias"]), _ptr(W[f"{p}.1.weight"]), _ptr(W[f"{p}.1.bias"]),
                                            _ptr(W[f"{p}.3.weight:raw"]), _ptr(W[f"{p}.3.bias"]), _ptr(W[f"{p}.4.weight"]), _ptr(W[f"{p}.4.bias"]), _ptr(W[f"{p}.6.scale"]),
                                            B, C_, Fr, L, hid, dil, _ptr(u_in) if u_in is not None else None, _ptr(work), _stream()), "dconv_f32")
                continue
            h = conv2d(x, W[f"{p}.0.weight"], W[f"{p}.0.bias"], hid, (1, 3), p=(0, dil), dw=dil)
            groupnorm1(h, W[f"{p}.1.weight"], W[f"{p}.1.bias"], ACT_GELU)
            h = conv2d(h, W[f"{p}.3.weight"], W[f"{p}.3.bias"], 2 * C_, (1, 1))
            groupnorm1(h, W[f"{p}.4.weight"], W[f"{p}.4.bias"])
            x = glu(h, res=x, scale=W[f"{p}.6.scale"])
        return x

    def _enc(self, x, prefix, freq):
        """HEncLayer.forward (hdemucs.py:119-153), norm = Identity, empty = False."""
        W, cfg = self.W, self.cfg
        co = W[f"{prefix}.conv.bias"].numel()
        if freq:
            y = conv2d(x, W[f"{prefix}.conv.weight"], W[f"{prefix}.conv.bias"], co, (cfg.kernel_size, 1), s=(cfg.stride, 1), p=(cfg.kernel_size // 4, 0), act=ACT_GELU)
        else:
            le = x.shape[-1]
            y = conv2d(x, W[f"{prefix}.conv.weight"], W[f"{prefix}.conv.bias"], co, (1, cfg.kernel_size), s=(1, cfg.stride), p=(0, cfg.kernel_size // 4), act=ACT_GELU,
                       out_hw=(1, -(-le // cfg.stride)))  # F.pad to a multiple of the stride == implicit zero columns on the right
        y = self._dconv(y, prefix)
        z = conv2d(y, W[f"{prefix}.rewrite.weight"], W[f"{prefix}.rewrite.bias"], 2 * co, (1, 1))
        return glu(z)

    def _dec(self, x, skip, length, prefix, freq, last):
        """HDecLayer.forward (hdemucs.py:299-330), norm = Identity, empty = False."""
        W, cfg = self.W, self.cfg
        ci = x.shape[1]
        x = ew(x, skip, _new(x.shape, x))
        if freq:
            y = glu(conv2d(x, W[f"{prefix}.rewrite.weight"], W[f"{prefix}.rewrite.bias"], 2 * ci, (3, 3), p=(1, 1)))
        else:
            y = glu(conv2d(x, W[f"{prefix}.rewrite.weight"], W[f"{prefix}.rewrite.bias"], 2 * ci, (1, 3), p=(0, 1)))
        y = self._dconv(y, prefix)
        co = W[f"{prefix}.conv_tr.bias"].numel()
        act = ACT_NONE if last else ACT_GELU
        if freq:
            return conv_transpose(y, W[f"{prefix}.conv_tr.weight"], W[f"{prefix}.conv_tr.bias"], co, 1, cfg.stride, cfg.kernel_size // 4, y.shape[2] * cfg.stride, act)
        return conv_transpose(y, W[f"{prefix}.conv_tr.weight"], W[f"{prefix}.conv_tr.bias"], co, 2, cfg.stride, cfg.kernel_size // 4, length, act)

    def _mha(self, q_in, kv_in, p, res, res_scale):
        """nn.MultiheadAttention(batch_first) + the layer-scaled residual: res + gamma * out_proj(softmax(QK^T/sqrt(hd)) V).  q_in (B,Lq,D), kv_in (B,Lk,D)."""
        W = self.W
        B, Lq, D = q_in.shape
        Lk = kv_in.shape[1]
        H = self.cfg.t_heads
        hd = D // H
        q = linear(q_in.view(B * Lq, D), W[f"{p}.q_weight"], W[f"{p}.q_bias"])
        k = linear(kv_in.view(B * Lk, D), W[f"{p}.k_weight"], W[f"{p}.k_bias"])
        # V^T per batch: (D, Lk) = Wv (D,D) @ kv^T, bias per row
        vt = _new((B, D, Lk), q_in)
        wv, bv = W[f"{p}.v_weight"], W[f"{p}.v_bias"]
        _gemm_raw(_ptr(wv), _ptr(kv_in), _ptr(vt), D, Lk, D, D, D, Lk, B, 0, Lk * D, D * Lk, bias_m=_ptr(bv))
        o = _new((B, Lq, D), q_in)
        if hd == 64 and _FUSED_ATTENTION:  # one kernel, the (H, Lq, Lk) scores stay on chip
            work = _new((lib.b200sep_attention_work_floats(B, H, Lq, Lk),), q_in)  # bf16 hi / lo tile images of Q, K, V^T (split once, not once per consumer)
            check(lib.b200sep_attention_f32(_ptr(q), _ptr(k), _ptr(vt), _ptr(o), B, H, Lq, Lk, hd, Lq * D, D, Lk * D, D, D * Lk, Lk, Lq * D, D, 1.0 / math.sqrt(hd),
                                            0, _ptr(work), _stream()), "attention_f32")
            y = linear(o.view(B * Lq, D), W[f"{p}.out_proj.weight"], W[f"{p}.out_proj.bias"], res=res.view(B * Lq, D), res_scale=res_scale)
            return y.view(B, Lq, D)
        sc = _new((H, Lq, Lk), q_in)
        fs = 4  # bytes per float
        for b in range(B):
            _gemm_raw(q.data_ptr() + b * Lq * D * fs, k.data_ptr() + b * Lk * D * fs, _ptr(sc), Lq, Lk, hd, D, D, Lk, H, hd, hd, Lq * Lk, alpha=1.0 / math.sqrt(hd))
            check(lib.b200sep_softmax_rows_f32(_ptr(sc), H * Lq, Lk, Lk, _stream()), "softmax_rows_f32")
            _gemm_raw(_ptr(sc), vt.data_ptr() + b * D * Lk * fs, o.data_ptr() + b * Lq * D * fs, Lq, hd, Lk, Lk, Lk, D, H, Lq * Lk, hd * Lk, hd)
        y = linear(o.view(B * Lq, D), W[f"{p}.out_proj.weight"], W[f"{p}.out_proj.bias"], res=res.view(B * Lq, D), res_scale=res_scale)
        return y.view(B, Lq, D)

    def _ffn(self, x_norm, x, p):
        W = self.W
        B, L, D = x.shape
        h = linear(x_norm.view(B * L, D), W[f"{p}.linear1.weight"], W[f"{p}.linear1.bias"], act=ACT_GELU)
        return linear(h, W[f"{p}.linear2.weight"], W[f"{p}.linear2.bias"], res=x.view(B * L, D), res_scale=W[f"{p}.gamma_2.scale"]).view(B, L, D)

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
            x = conv2d(x.view(B, c0, 1, Fr * T1), W["channel_upsampler.weight"], W["channel_upsampler.bias"], D, (1, 1)).view(B, D, Fr, T1)
            xt = conv2d(xt, W["channel_upsampler_t.weight"], W["channel_upsampler_t.bias"], D, (1, 1))
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
            x = conv2d(x.view(B, D, 1, Fr * T1), W["channel_downsampler.weight"], W["channel_downsampler.bias"], c0, (1, 1)).view(B, c0, Fr, T1)
            xt = conv2d(xt, W["channel_downsampler_t.weight"], W["channel_downsampler_t.bias"], c0, (1, 1))
        return x, xt

    # ---- forward ---------------------------------------------------------------------------------------------------
    def forward(self, mix: torch.Tensor) -> torch.Tensor:
        """mix (B, 2, L <= seg_len) float32 cuda -> (B, S, 2, L).  (eval mode, use_train_segment: shorter inputs are zero-padded
        to the training segment and the output is cut back, htdemucs.py:486-493, :614-618.)"""
        cfg, S = self.cfg, self.S
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
        hl, nfft = cfg.hop, cfg.nfft
        le = -(-T_len // hl)
        Fq = nfft // 2
        # _spec + _magnitude (htdemucs.py:383-403, :415-424): normalized STFT, frames 2..2+le of the 3*hop/2-reflect-padded signal, bins 0..nfft/2-1
        spec = _new((B, 4, Fq, le), mp)
        check(lib.b200sep_stft_forward_ex(self.stft.handle, _ptr(mp), 2 * T_len, T_len, 0, B, T_len, le, hl // 2 * 3, 1.0 / math.sqrt(nfft), Fq, 0, LAYOUT_CFT,
                                          0, _ptr(spec), _stream()), "stft_forward_ex")
        stats = _new((B, 4), mp)  # per sample: mean, std of the spectrogram; mean, std of the waveform
        x = _new(spec.shape, mp)
        xt = _new((B, 2, 1, T_len), mp)
        fs = 4
        mswork = _new((lib.b200sep_meanstd_work_floats(B),), mp)
        check(lib.b200sep_meanstd_batch_f32(_ptr(spec), spec[0].numel(), B, spec[0].numel(), _ptr(stats), 4, _ptr(mswork), _stream()), "meanstd_batch_f32")
        check(lib.b200sep_meanstd_batch_f32(_ptr(mp), mp[0].numel(), B, mp[0].numel(), stats.data_ptr() + 2 * fs, 4, _ptr(mswork), _stream()), "meanstd_batch_f32")
        for b in range(B):
            check(lib.b200sep_ew_f32(_ptr(spec[b]), stats.data_ptr() + (4 * b) * fs, _ptr(x[b]), spec[b].numel(), 1.0, 0.0, 2, _stream()), "ew_f32")
            check(lib.b200sep_ew_f32(_ptr(mp[b]), stats.data_ptr() + (4 * b + 2) * fs, _ptr(xt[b]), mp[b].numel(), 1.0, 0.0, 2, _stream()), "ew_f32")
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
        # x (B, S*4, Fq, le) * std + mean -> _mask (cac) -> _ispec (:405-413): iSTFT with the Nyquist bin and two frames per side zero
        out = _new((B, S, 2, T_len), mp)
        nwork = lib.b200sep_stft_inverse_work_floats(self.stft.handle, S, le, Fq, LAYOUT_CFT)
        work = _new((nwork,), mp)
        xi = _new((S, 2, T_len), mp)
        for b in range(B):
            check(lib.b200sep_ew_f32(_ptr(x[b]), stats.data_ptr() + (4 * b) * fs, _ptr(x[b]), x[b].numel(), 1.0, 0.0, 3, _stream()), "ew_f32")
            check(lib.b200sep_stft_inverse_ex(self.stft.handle, _ptr(x[b]), S, le, Fq, LAYOUT_CFT, T_len, hl // 2 * 3, 2, math.sqrt(nfft), _ptr(xi), _ptr(work), _stream()),
                  "stft_inverse_ex")
            check(lib.b200sep_ew_f32(_ptr(xt[b]), stats.data_ptr() + (4 * b + 2) * fs, _ptr(out[b]), xt[b].numel(), 1.0, 0.0, 3, _stream()), "ew_f32")
            ew(out[b], xi, out[b])
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
    segment (HTDemucs.valid_length, htdemucs.py:469-481) takes all of them at width `seg`; a model without valid_length (HDemucs) runs every chunk at its own
    length (apply.py:252-257), so only runs of equal length batch -- in practice all full segments, then the shorter last one."""
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
        _require_cuda()
        from .sharded import ShardRunner

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
        self.rank, self.world = self.runner.rank, self.runner.world
        self.split = bool(split)  # apply_model(split=...): False = segments_enabled False, ONE forward over the whole (shifted) track (apply.py:251-260)
        if not self.split and self.world > 1:
            raise ValueError("split=False is one forward over the whole track: nothing to shard across ranks")

    def out_range(self, N):
        """Output samples [q0, q1) this rank finalises (everything on a single GPU)."""
        return N * self.rank // self.world, N * (self.rank + 1) // self.world

    def _apply_split(self, net, tensor, offset, length, out, q0, n_out, scale, chan_scale, accumulate):
        """apply_model's split branch on TensorChunk(tensor, offset, length) (apply.py:215-250); the weighted result's samples
        [q0, q0 + n_out) -- this rank's part [r0, r1) of them -- are scaled and written / accumulated into out (S*2, r1 - r0)."""
        from .sharded import plan_range_shards

        cfg = self.cfg
        seg = cfg.seg_len
        S = len(cfg.sources)
        stride = int((1 - self.overlap) * seg)
        total = tensor.shape[-1]
        offs = list(range(0, length, stride))
        sh = plan_range_shards(n_out, self.world, len(offs), stride, seg, q0)[self.rank]
        assert tuple(out.shape) == (S * 2, sh.q1 - sh.q0), (out.shape, sh)
        # TensorChunk.padded zero-fills outside the tensor (apply.py:97-113): only the part this rank's segments read is materialised
        lo = offset + sh.c0 * stride - seg
        hi = offset + (sh.c1 - 1) * stride + 2 * seg if sh.n_own else lo + 1
        ext = torch.zeros((2, hi - lo), dtype=torch.float32, device=tensor.device)
        a, b = max(lo, 0), min(hi, total)
        if b > a:
            ext[:, a - lo : b - lo].copy_(tensor[:, a:b])
        local = torch.empty((sh.halo + sh.n_own, S * 2, seg), dtype=torch.float32, device=tensor.device)

        pads = getattr(cfg, "pads_to_segment", True)  # HTDemucs: chunk.padded(valid_length = training segment); HDemucs: every chunk at its own length (apply.py:252-257)

        def compute(buf, slot0, unit0, n):
            clens = [min(length - offs[unit0 + j], seg) for j in range(n)]
            for j0, j1, width in group_units(clens, seg, pads):  # units of one input length form one forward (only the last segment of a pass is shorter)
                batch = _new((j1 - j0, 2, width), tensor)
                for j in range(j0, j1):
                    start = offset + offs[unit0 + j] - ((seg - clens[j]) // 2 if pads else 0)
                    batch[j - j0].copy_(ext[:, start - lo : start - lo + width])
                y = net.graphed(batch)  # (n, S, 2, width): the launch list of the forward (HTDemucs: replayed as one CUDA graph per batch size)
                for j in range(j0, j1):  # center_trim to the chunk's valid length (apply.py:258), stored from sample 0
                    d = (seg - clens[j]) // 2 if pads else 0
                    buf[slot0 + j, :, : clens[j]].copy_(y[j - j0].reshape(S * 2, width)[:, d : d + clens[j]])

        self.runner.wait_all(self.runner.run_units(sh, local, compute, self.batch_size))
        if sh.q1 > sh.q0:
            check(lib.b200sep_triangle_overlap_add_range(_ptr(local), sh.c0 - sh.halo, sh.halo + sh.n_own, len(offs), S * 2, seg, stride, length, q0 + sh.q0, sh.q1 - sh.q0,
                                                         scale, _ptr(chan_scale) if chan_scale is not None else None, int(accumulate), _ptr(out), sh.q1 - sh.q0, 0,
                                                         _stream()), "triangle_overlap_add_range")

    def _apply_whole(self, net, tensor, offset, length, out, q0, n_out, scale, chan_scale, accumulate):
        """apply_model's leaf (apply.py:251-260) on TensorChunk(tensor, offset, length): the chunk zero-padded (centred) to model.valid_length(length) -- the training
        segment for HTDemucs, which REFUSES anything longer (htdemucs.py:469-481); the length itself for models without valid_length -- one forward, center_trim."""
        cfg = self.cfg
        S = len(cfg.sources)
        seg = cfg.seg_len
        valid = seg if getattr(cfg, "pads_to_segment", True) else length
        if valid < length:
            raise ValueError(f"Given length {length} is longer than training length {valid}")
        delta = valid - length
        start = offset - delta // 2
        batch = torch.zeros((1, 2, valid), dtype=torch.float32, device=tensor.device)
        a, b = max(start, 0), min(start + valid, tensor.shape[-1])
        if b > a:
            batch[0, :, a - start : b - start].copy_(tensor[:, a:b])
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
        ms = int(0.5 * self.cfg.samplerate)
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
        if self.world == 1:
            return part
        return self.runner.gather_cols(part, [(N * r // self.world, N * (r + 1) // self.world) for r in range(self.world)], N)

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
