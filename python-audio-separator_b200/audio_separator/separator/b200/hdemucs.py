"""Hybrid Demucs v3 (HDemucs: the conv + BiLSTM + LocalState model behind hdemucs_mmi / mdx_extra) on the fp32 operator kernels of libb200sep.so.

HDemucsNet.forward replaces HDemucs.forward (uvr_lib_v5/demucs/hdemucs.py:665-783) for hybrid, complex-as-channels models without
multi_freqs: frequency and time encoders with GroupNorm from `norm_starts` on, the "empty" time layer whose output is injected into the
frequency branch at the layer where one frequency is left, DConv branches with a 2-layer bidirectional LSTM over overlapping 200-step
frames and the LocalState attention (demucs.py:19-67, :99-231), decoders that mirror it.  The model runs at the length it is given
(HDemucs has no valid_length: apply.py:252-257); DemucsEngine drives it through the same apply_model logic as HTDemucs.

Graph builder only: device buffers and the ORDER of the operator launches; every arithmetic step is a kernel behind the C ABI.
"""
from __future__ import annotations

from dataclasses import dataclass

import numpy as np
import torch

from ._lib import MATH_BF16X3, check, lib
from .demucs import DemucsNetBase, HybridDemucsNet
from .engine import _ptr, _stream
from .ops import (ACT_GELU, ACT_NONE, _new, block_conv_weight, block_convtr_weight, conv2d, conv_transpose, ew, glu, groupnorm, groupnorm1, linear, lstm_bidir,
                  lstm_bidir_weights)


@dataclass
class HDemucsConfig:
    """Constructor arguments of HDemucs that shape the graph (hdemucs.py:360-400); defaults = the constructor's."""

    sources: tuple = ("drums", "bass", "other", "vocals")
    audio_channels: int = 2
    channels: int = 48
    growth: int = 2
    nfft: int = 4096
    depth: int = 6
    hybrid_old: bool = False
    freq_emb: float = 0.2
    emb_scale: float = 10.0
    kernel_size: int = 8
    time_stride: int = 2
    stride: int = 4
    context: int = 1
    context_enc: int = 0
    norm_starts: int = 4
    norm_groups: int = 4
    dconv_mode: int = 1
    dconv_depth: int = 2
    dconv_comp: int = 4
    dconv_attn: int = 4
    dconv_lstm: int = 4
    samplerate: int = 44100
    segment: float = 40.0
    attn_heads: int = 4      # DConv's LocalState(hidden, heads=4, ndecay=4) and BLSTM(hidden, layers=2, max_steps=200) (demucs.py:99, :152-155)
    attn_ndecay: int = 4
    lstm_layers: int = 2
    lstm_max_steps: int = 200

    @property
    def hop(self):
        return self.nfft // 4

    @property
    def seg_len(self):  # int(model.samplerate * model.segment), apply.py:218
        return int(self.samplerate * self.segment)

    pads_to_segment = False  # apply_model runs every chunk at its own length (no valid_length)

    def valid_length(self, length):  # HDemucs has no valid_length: apply_model runs a chunk at its own length (apply.py:252-257)
        return length

    def validate(self):
        if self.audio_channels != 2:
            raise ValueError("the H100 HDemucs path handles stereo models only")
        if self.kernel_size != 2 * self.stride:
            raise ValueError("the H100 HDemucs path needs kernel_size == 2 * stride (the transposed convolutions are 2-tap over the coarse index)")
        if self.dconv_depth != 2:
            raise ValueError("the H100 HDemucs path needs dconv_depth 2 (dilations 1 and 2)")


def layer_plan(cfg: HDemucsConfig):
    """The geometry HDemucs.__init__ derives per layer index (hdemucs.py:455-527): dicts for the frequency encoder / decoder and, while the
    frequency axis is longer than one, the time encoder / decoder (`empty`: the merge layer that is just its convolution)."""
    S, C = len(cfg.sources), cfg.audio_channels
    chin, chin_z, chout, chout_z = C, 2 * C, cfg.channels, cfg.channels
    freqs = cfg.nfft // 2
    plan = []
    for index in range(cfg.depth):
        common = dict(norm=index >= cfg.norm_starts, lstm=index >= cfg.dconv_lstm, attn=index >= cfg.dconv_attn)
        freq = freqs > 1
        ker, stri = (cfg.kernel_size, cfg.stride) if freq else (cfg.time_stride * 2, cfg.time_stride)
        pad, last_freq = True, False
        if freq and freqs <= cfg.kernel_size:
            ker, pad, last_freq = freqs, False, True
        if last_freq:
            chout_z = max(chout, chout_z)
            chout = chout_z
        enc = dict(common, chin=chin_z, chout=chout_z, k=ker, s=stri, freq=freq, pad=ker // 4 if pad else 0, dconv=bool(cfg.dconv_mode & 1), context=cfg.context_enc, empty=False)
        tenc = dict(common, chin=chin, chout=chout, k=cfg.kernel_size, s=cfg.stride, freq=False, pad=cfg.kernel_size // 4, dconv=bool(cfg.dconv_mode & 1),
                    context=cfg.context_enc, empty=last_freq) if freq else None
        if index == 0:
            chin = C * S
            chin_z = 2 * chin
        dec = dict(common, chin=chout_z, chout=chin_z, k=ker, s=stri, freq=freq, pad=ker // 4 if pad else 0, dconv=bool(cfg.dconv_mode & 2), context=cfg.context, empty=False,
                   last=index == 0)
        tdec = dict(common, chin=chout, chout=chin, k=cfg.kernel_size, s=cfg.stride, freq=False, pad=cfg.kernel_size // 4, dconv=bool(cfg.dconv_mode & 2), context=cfg.context,
                    empty=last_freq, last=index == 0) if freq else None
        plan.append(dict(enc=enc, tenc=tenc, dec=dec, tdec=tdec))
        chin, chin_z = chout, chout_z
        chout, chout_z = int(cfg.growth * chout), int(cfg.growth * chout_z)
        if freq:
            freqs = 1 if freqs <= cfg.kernel_size else freqs // cfg.stride
    return plan


class DemucsLayers(DemucsNetBase):
    """The encoder and decoder layers of the v3 models (HEncLayer / HDecLayer, hdemucs.py:67-330, with the DConv branch and its BLSTM / LocalState)
    and the device layout of their weights, under the HEncLayer / HDecLayer parameter names.  HDemucsNet runs them in both branches of the hybrid
    model; DemucsNet (demucs_v3.py) runs them as the whole time-domain Demucs, whose layers are the time branch's."""

    def _load_weights(self, st):
        """Host arrays (float32) of the layer parameters -> device tensors in the layouts the operators take."""
        cfg = self.cfg
        for name, a in st.items():
            if ".lstm." in name:
                continue  # repacked below
            if ".dconv.layers." in name and name.endswith((".0.weight", ".3.weight")) and a.ndim == 3 and a.shape[-1] in (1, 3):
                # the fused plain DConv kernel takes the (out, in[, k]) matrices as they are (layers without LSTM / LocalState: index 3 is the 1x1)
                self._put(name + ":raw", a.reshape(a.shape[0], -1) if name.endswith(".3.weight") else a)
            if name.endswith("conv_tr.weight"):
                a = block_convtr_weight(a.reshape(a.shape[0], a.shape[1], -1), a.reshape(a.shape[0], a.shape[1], -1).shape[2] // 2)
            elif name.endswith(".linear.weight"):
                pass  # BLSTM.linear: a plain (out, in) matrix for gemm_f32
            elif name.endswith(".weight") and a.ndim >= 3:
                a = block_conv_weight(a if a.ndim == 4 else a.reshape(a.shape[0], a.shape[1], 1, a.shape[2]))
            self._put(name, a)
        for name in st:  # nn.LSTM parameters, per layer
            if name.endswith(".lstm.weight_ih_l0"):
                p = name[: -len(".weight_ih_l0")]
                for layer in range(cfg.lstm_layers):
                    self.W[f"{p}.{layer}"] = lstm_bidir_weights(st, p, layer, self.device)

    # ---- DConv with BLSTM / LocalState ----------------------------------------------------------------------------------------
    def _blstm(self, h, p):
        """BLSTM(hidden, layers=2, max_steps=200, skip=True).forward (demucs.py:34-67) on h (B, C, 1, T) -> (B, C, 1, T)."""
        W, cfg = self.W, self.cfg
        B, C, _, T = h.shape
        width = cfg.lstm_max_steps
        if width is not None and T > width:
            stride = width // 2
            nf = -(-T // stride)
        else:
            width, stride, nf = T, T, 1
        N = B * nf
        fr = _new((width, N, C), h)
        check(lib.b200sep_lstm_frames_gather_f32(_ptr(h), _ptr(fr), B, C, T, nf, width, stride, _stream()), "lstm_frames_gather_f32")
        x2 = fr.view(width * N, C)
        for layer in range(cfg.lstm_layers):
            x2 = lstm_bidir(x2, N, W[f"{p}.lstm.{layer}"], self.math)
        lin = linear(x2, W[f"{p}.linear.weight"], W[f"{p}.linear.bias"], math=self.math)
        y = _new(h.shape, h)
        check(lib.b200sep_lstm_frames_scatter_f32(_ptr(lin), _ptr(h), _ptr(y), B, C, T, nf, width, stride if nf > 1 else 2, _stream()), "lstm_frames_scatter_f32")
        return y

    def _local_state(self, h, p):
        """LocalState(hidden, heads=4, ndecay=4).forward (demucs.py:197-231) on h (B, C, 1, T)."""
        W, cfg = self.W, self.cfg
        B, C, _, T = h.shape
        q = conv2d(h, W[f"{p}.query.weight"], W[f"{p}.query.bias"], C, (1, 1), math=self.math)
        k = conv2d(h, W[f"{p}.key.weight"], W[f"{p}.key.bias"], C, (1, 1), math=self.math)
        ct = conv2d(h, W[f"{p}.content.weight"], W[f"{p}.content.bias"], C, (1, 1), math=self.math)
        nd = cfg.attn_heads * cfg.attn_ndecay
        dq = conv2d(h, W[f"{p}.query_decay.weight"], W[f"{p}.query_decay.bias"], nd, (1, 1), math=self.math)
        res = _new(h.shape, h)
        check(lib.b200sep_local_state_attn_f32(_ptr(q), _ptr(k), _ptr(ct), _ptr(dq), _ptr(res), B, C, T, cfg.attn_heads, cfg.attn_ndecay, _stream()), "local_state_attn_f32")
        return conv2d(res, W[f"{p}.proj.weight"], W[f"{p}.proj.bias"], C, (1, 1), add=h, math=self.math)

    def _dconv_layer(self, x, prefix, L):
        """DConv.forward (demucs.py:166-168) for the layer kinds of this model: the plain branch (DemucsNetBase._dconv), or conv -> GroupNorm+GELU ->
        BLSTM -> LocalState -> 1x1 -> GroupNorm -> GLU with the LayerScale residual."""
        if not (L["lstm"] or L["attn"]):
            return self._dconv(x, prefix)
        W = self.W
        B, C_, Fr, T = x.shape
        if Fr != 1:
            raise NotImplementedError("BLSTM / LocalState DConv branches on a layer with more than one frequency row")
        for d in range(self.cfg.dconv_depth):
            p = f"{prefix}.dconv.layers.{d}"
            dil = 2**d
            hid = W[f"{p}.0.bias"].numel()
            h = conv2d(x, W[f"{p}.0.weight"], W[f"{p}.0.bias"], hid, (1, 3), p=(0, dil), dw=dil, math=self.math)
            groupnorm1(h, W[f"{p}.1.weight"], W[f"{p}.1.bias"], ACT_GELU)
            i = 3
            if L["lstm"]:
                h = self._blstm(h, f"{p}.{i}")
                i += 1
            if L["attn"]:
                h = self._local_state(h, f"{p}.{i}")
                i += 1
            h = conv2d(h, W[f"{p}.{i}.weight"], W[f"{p}.{i}.bias"], 2 * C_, (1, 1), math=self.math)
            groupnorm1(h, W[f"{p}.{i + 1}.weight"], W[f"{p}.{i + 1}.bias"])
            x = glu(h, res=x, scale=W[f"{p}.{i + 3}.scale"])
        return x

    # ---- encoder / decoder layers --------------------------------------------------------------------------------------------
    def _enc_layer(self, x, prefix, L, inject=None):
        """HEncLayer.forward (hdemucs.py:119-153) on x (B, C, Fr, T) (time branch and merged layers: Fr = 1)."""
        W, G = self.W, self.cfg.norm_groups
        co, k, s, pad = L["chout"], L["k"], L["s"], L["pad"]
        fused_act = ACT_NONE if (L["empty"] or L["norm"]) else ACT_GELU
        if L["freq"]:
            y = conv2d(x, W[f"{prefix}.conv.weight"], W[f"{prefix}.conv.bias"], co, (k, 1), s=(s, 1), p=(pad, 0), act=fused_act, add=inject, add_before_act=inject is not None, math=self.math)
        else:
            if x.shape[2] != 1:
                raise ValueError(f"{prefix}: a time layer needs one frequency row, got {tuple(x.shape)}")
            le = -(-x.shape[-1] // s) * s  # F.pad to a multiple of the stride == implicit zero columns on the right
            y = conv2d(x, W[f"{prefix}.conv.weight"], W[f"{prefix}.conv.bias"], co, (1, k), s=(1, s), p=(0, pad), act=fused_act, add=inject, add_before_act=inject is not None,
                       out_hw=(1, (le + 2 * pad - k) // s + 1), math=self.math)
        if L["empty"]:
            return y
        if L["norm"]:
            groupnorm(y, G, W[f"{prefix}.norm1.weight"], W[f"{prefix}.norm1.bias"], ACT_GELU)
        if L["dconv"]:
            y = self._dconv_layer(y, prefix, L)
        ctx = L["context"]
        kk = 1 + 2 * ctx
        if L["freq"]:
            z = conv2d(y, W[f"{prefix}.rewrite.weight"], W[f"{prefix}.rewrite.bias"], 2 * co, (kk, kk), p=(ctx, ctx), math=self.math)
        else:
            z = conv2d(y, W[f"{prefix}.rewrite.weight"], W[f"{prefix}.rewrite.bias"], 2 * co, (1, kk), p=(0, ctx), math=self.math)
        if L["norm"]:
            groupnorm(z, G, W[f"{prefix}.norm2.weight"], W[f"{prefix}.norm2.bias"])
        return glu(z)

    def _dec_layer(self, x, skip, length, prefix, L):
        """HDecLayer.forward (hdemucs.py:299-330) -> (z, y).  x None = the all-zero tensor the decoder starts from (hdemucs.py:719-723)."""
        W, G = self.W, self.cfg.norm_groups
        ci, co, s, pad = L["chin"], L["chout"], L["s"], L["pad"]
        if not L["empty"]:
            x = skip if x is None else ew(x, skip, _new(x.shape, x))
            ctx = L["context"]
            kk = 1 + 2 * ctx
            if L["freq"]:
                y = conv2d(x, W[f"{prefix}.rewrite.weight"], W[f"{prefix}.rewrite.bias"], 2 * ci, (kk, kk), p=(ctx, ctx), math=self.math)
            else:
                y = conv2d(x, W[f"{prefix}.rewrite.weight"], W[f"{prefix}.rewrite.bias"], 2 * ci, (1, kk), p=(0, ctx), math=self.math)
            if L["norm"]:
                groupnorm(y, G, W[f"{prefix}.norm1.weight"], W[f"{prefix}.norm1.bias"])
            y = glu(y)
            if L["dconv"]:
                y = self._dconv_layer(y, prefix, L)
        else:
            y = x
        act = ACT_NONE if L["last"] else ACT_GELU
        axis = 1 if L["freq"] else 2
        n_in = y.shape[2] if L["freq"] else y.shape[3]
        full = (n_in + 1) * s  # (n_in - 1) * s + kernel, kernel = 2 * s
        target = full - 2 * pad if L["freq"] else length
        wt, bt = W[f"{prefix}.conv_tr.weight"], W[f"{prefix}.conv_tr.bias"]
        if not L.get("norm_tr", L["norm"]):  # norm_tr: the time-domain Demucs, whose outermost decoder has no GroupNorm after its transposed convolution
            return conv_transpose(y, wt, bt, co, axis, s, pad, target, act, math=self.math), y
        # GroupNorm sees the UNtrimmed transposed convolution (hdemucs.py:322-328: norm2, then the crop, then GELU)
        z = conv_transpose(y, wt, bt, co, axis, s, 0, full, ACT_NONE, math=self.math)
        groupnorm(z, G, W[f"{prefix}.norm2.weight"], W[f"{prefix}.norm2.bias"], act)
        if target != full:
            z = (z[:, :, pad : pad + target, :] if L["freq"] else z[:, :, :, pad : pad + target]).contiguous()  # a strided device copy
        return z, y


class HDemucsNet(HybridDemucsNet, DemucsLayers):
    """Device-resident HDemucs weights + the launch sequence of one forward."""

    def __init__(self, cfg: HDemucsConfig, state: dict, device=None, math=MATH_BF16X3):
        super().__init__(cfg, device, math)
        self.plan = layer_plan(cfg)
        self.encs = [(f"encoder.{i}", P["enc"]) for i, P in enumerate(self.plan)]
        self.decs = [(f"decoder.{j}", P["dec"]) for j, P in enumerate(self.plan[::-1])]
        tencs = [P["tenc"] for P in self.plan if P["tenc"] is not None]
        tdecs = [P["tdec"] for P in self.plan if P["tdec"] is not None][::-1]
        self.tencs = [(f"tencoder.{i}", L) for i, L in enumerate(tencs)]
        self.tdecs = [(f"tdecoder.{j}", L) for j, L in enumerate(tdecs)]
        st = {k: np.asarray(v, dtype=np.float32) for k, v in state.items()}
        self._check_structure(st)
        self._load_weights(st)
        if cfg.freq_emb:
            # ScaledEmbedding.forward * freq_emb_scale (hdemucs.py:62-64, :708-713) as one value per (channel, frequency) row
            emb = st["freq_emb.embedding.weight"] * np.float32(cfg.emb_scale)  # (Fr, C)
            self._put("freq_emb:rows", (np.float32(cfg.freq_emb) * emb).T.reshape(-1))
        self.graphed = self.forward  # variable lengths: launched directly

    def _check_structure(self, st):
        cfg = self.cfg
        for prefix, L in self.encs + self.tencs:
            w = st.get(f"{prefix}.conv.weight")
            if w is None or w.shape[0] != L["chout"] or w.shape[1] != L["chin"] or w.shape[2] != L["k"]:
                raise ValueError(f"{prefix}.conv.weight {None if w is None else w.shape} does not match the configured HDemucs structure {L}")
            if (f"{prefix}.norm1.weight" in st) != (L["norm"] and not L["empty"]):
                raise ValueError(f"{prefix}: GroupNorm presence does not match norm_starts={cfg.norm_starts}")
        if f"encoder.{cfg.depth}.conv.weight" in st:
            raise ValueError(f"state dict is deeper than depth {cfg.depth}")
        if any(".query_freqs." in n for n in st):
            raise ValueError("LocalState with nfreqs > 0 is not supported")
        for prefix, L in self.encs + self.tencs + self.decs + self.tdecs:
            if L["empty"] or not L["dconv"]:
                continue
            if L["freq"] and L["k"] != cfg.kernel_size and (L["lstm"] or L["attn"]):
                pass  # the merge layer: one frequency row after its convolution
            has_lstm = f"{prefix}.dconv.layers.0.3.lstm.weight_ih_l0" in st
            if has_lstm != L["lstm"]:
                raise ValueError(f"{prefix}: BLSTM presence does not match dconv_lstm={cfg.dconv_lstm}")

    # ---- forward -------------------------------------------------------------------------------------------------------------
    def forward(self, mix: torch.Tensor) -> torch.Tensor:
        """mix (B, 2, L) float32 cuda -> (B, S, 2, L)."""
        cfg, W = self.cfg, self.W
        assert mix.dim() == 3 and mix.shape[1] == 2 and mix.dtype == torch.float32 and mix.is_cuda
        mp = mix.contiguous()
        B, _, length = mp.shape
        x, xt, stats = self.spec_in(mp, 1 if cfg.hybrid_old else 0)  # hybrid_old: zero- instead of reflect-padded
        saved, saved_t, lengths, lengths_t = [], [], [], []
        for idx, (prefix, L) in enumerate(self.encs):  # hdemucs.py:697-716
            lengths.append(x.shape[-1])
            inject = None
            if idx < len(self.tencs):
                tp, Lt = self.tencs[idx]
                lengths_t.append(xt.shape[-1])
                xt = self._enc_layer(xt, tp, Lt)
                if not Lt["empty"]:
                    saved_t.append(xt)
                else:
                    inject = xt
            x = self._enc_layer(x, prefix, L, inject)
            if idx == 0 and cfg.freq_emb:
                check(lib.b200sep_add_rowvec_f32(_ptr(x), _ptr(W["freq_emb:rows"]), B, x.shape[1] * x.shape[2], x.shape[3], _stream()), "add_rowvec_f32")
            saved.append(x)
        x = None
        offset = cfg.depth - len(self.tdecs)
        for idx, (prefix, L) in enumerate(self.decs):  # hdemucs.py:724-749
            x, pre = self._dec_layer(x, saved.pop(-1), lengths.pop(-1), prefix, L)
            if idx >= offset:
                tp, Lt = self.tdecs[idx - offset]
                length_t = lengths_t.pop(-1)
                if Lt["empty"]:
                    assert pre.shape[2] == 1, pre.shape
                    xt, _ = self._dec_layer(pre, None, length_t, tp, Lt)
                else:
                    xt, _ = self._dec_layer(xt, saved_t.pop(-1), length_t, tp, Lt)
        assert not saved and not saved_t and not lengths_t
        return self.spec_out(x, xt, stats, length, 0 if cfg.hybrid_old else cfg.hop // 2 * 3)

    __call__ = forward
