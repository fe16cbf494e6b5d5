"""The time-domain Demucs v3 network (uvr_lib_v5/demucs/demucs.py:234-453, class Demucs: the waveform members of the v3 bags mdx / mdx_extra) on the
fp32 operator kernels of libb200sep.so.

Its encoder and decoder layers are the time-branch layers of HDemucs -- strided convolution, GroupNorm from `norm_starts` on, GELU, the DConv
branch with BLSTM / LocalState, the GLU rewrite, the 2-tap transposed convolution -- so DemucsNet runs them through DemucsLayers (hdemucs.py) under
the HEncLayer / HDecLayer parameter names its `nn.Sequential` indices map onto.  What is its own: the mono normalisation, the centred zero pad to
valid_length and julius.resample_frac x2 / /2 around the layers (csrc/demucs_ops.cu), and no padding in the strided convolutions.

Graph builder only: device buffers and the ORDER of the operator launches; every arithmetic step is a kernel behind the C ABI.
"""
from __future__ import annotations

import math
from dataclasses import dataclass

import numpy as np
import torch

from ._lib import MATH_BF16X3, check, lib
from .engine import _ptr, _stream
from .hdemucs import DemucsLayers
from .ops import _new, to_device


@dataclass
class DemucsConfig:
    """Constructor arguments of Demucs that shape the graph (demucs.py:236-272); defaults = the constructor's."""

    sources: tuple = ("drums", "bass", "other", "vocals")
    audio_channels: int = 2
    channels: int = 64
    growth: float = 2.0
    depth: int = 6
    kernel_size: int = 8
    stride: int = 4
    context: int = 1
    norm_starts: int = 4
    norm_groups: int = 4
    dconv_mode: int = 1
    dconv_depth: int = 2
    dconv_comp: int = 4
    dconv_attn: int = 4
    dconv_lstm: int = 4
    samplerate: int = 44100
    segment: float = 40.0
    attn_heads: int = 4      # DConv's LocalState(hidden, heads=4, ndecay=4) and BLSTM(hidden, layers=2, max_steps=200) (demucs.py:158-161)
    attn_ndecay: int = 4
    lstm_layers: int = 2
    lstm_max_steps: int = 200

    @property
    def seg_len(self):  # int(model.samplerate * model.segment), apply.py:218
        return int(self.samplerate * self.segment)

    def valid_length(self, length):
        """Demucs.valid_length (demucs.py:382-403): the nearest length whose x2-resampled signal every strided convolution consumes whole."""
        length *= 2
        for _ in range(self.depth):
            length = max(1, math.ceil((length - self.kernel_size) / self.stride) + 1)
        for _ in range(self.depth):
            length = (length - 1) * self.stride + self.kernel_size
        return int(math.ceil(length / 2))

    def validate(self):
        if self.audio_channels != 2:
            raise ValueError("the H100 Demucs path handles stereo models only")
        if self.kernel_size != 2 * self.stride or self.stride % 2:
            raise ValueError("the H100 Demucs path needs kernel_size == 2 * stride with an even stride (2-tap transposed convolutions, even resampled lengths)")
        if self.dconv_depth != 2:
            raise ValueError("the H100 Demucs path needs dconv_depth 2 (dilations 1 and 2)")


def layer_plan(cfg: DemucsConfig):
    """The geometry Demucs.__init__ derives per layer index (demucs.py:340-371), as the dicts of hdemucs.layer_plan for time layers: unpadded strided
    convolutions, an encoder rewrite without context, decoder outputs untrimmed, and index 0's decoder without GroupNorm or GELU after its
    transposed convolution (`norm_tr`)."""
    plan = []
    chin, ch = cfg.audio_channels, cfg.channels
    for index in range(cfg.depth):
        common = dict(norm=index >= cfg.norm_starts, lstm=index >= cfg.dconv_lstm, attn=index >= cfg.dconv_attn, k=cfg.kernel_size, s=cfg.stride, freq=False,
                      pad=0, empty=False)
        enc = dict(common, chin=chin, chout=ch, dconv=bool(cfg.dconv_mode & 1), context=0)
        dec = dict(common, chin=ch, chout=chin if index > 0 else len(cfg.sources) * cfg.audio_channels, dconv=bool(cfg.dconv_mode & 2), context=cfg.context,
                   last=index == 0, norm_tr=index > 0 and index >= cfg.norm_starts)
        plan.append(dict(enc=enc, dec=dec))
        chin, ch = ch, int(cfg.growth * ch)
    return plan


def layer_names(cfg: DemucsConfig, state: dict) -> dict:
    """Demucs state-dict keys (`encoder.{i}.{Sequential index}...`, decoders in forward order) -> the HEncLayer / HDecLayer names DemucsLayers reads.
    Applies Demucs.load_state_dict's rename of the previous generation's `.2.` rewrite keys to `.3.` (demucs.py:444-453) first."""
    st = dict(state)
    for idx in range(cfg.depth):
        for a in ("encoder", "decoder"):
            for b in ("bias", "weight"):
                new, old = f"{a}.{idx}.3.{b}", f"{a}.{idx}.2.{b}"
                if old in st and new not in st:
                    st[new] = st.pop(old)
    e = 1 if cfg.dconv_mode & 1 else 0  # a DConv shifts the rewrite / transposed convolution one Sequential slot on
    d = 1 if cfg.dconv_mode & 2 else 0
    slots = {"encoder": {0: "conv", 1: "norm1", 3 + e: "rewrite", 4 + e: "norm2"}, "decoder": {0: "rewrite", 1: "norm1", 3 + d: "conv_tr", 4 + d: "norm2"}}
    if e:
        slots["encoder"][3] = "dconv"
    if d:
        slots["decoder"][3] = "dconv"
    out = {}
    for key, v in st.items():
        parts = key.split(".")
        name = slots.get(parts[0], {}).get(int(parts[2])) if len(parts) > 3 and parts[1].isdigit() and parts[2].isdigit() else None
        if name is None:
            raise ValueError(f"state key {key} is not part of the configured Demucs structure (lstm_layers > 0, rewrite / glu off, or another dconv_mode)")
        out[".".join([parts[0], parts[1], name] + parts[3:])] = v
    return out


def julius_taps(old: int, new: int, zeros: int = 24, rolloff: float = 0.945):
    """The filters of julius.ResampleFrac(old, new, zeros, rolloff) (julius/resample.py, _init_kernels) in float64: -> (taps (new, 2 * width + old), width)."""
    sr = min(old, new) * rolloff
    width = math.ceil(zeros * old / sr)
    idx = np.arange(-width, width + old, dtype=np.float64)
    rows = []
    for i in range(new):
        t = np.clip((-i / new + idx / old) * sr, -zeros, zeros) * math.pi
        k = np.where(t == 0, 1.0, np.sin(t) / np.where(t == 0, 1.0, t)) * np.cos(t / zeros / 2) ** 2
        rows.append(k / k.sum())
    return np.stack(rows), width


class DemucsNet(DemucsLayers):
    """Device-resident Demucs v3 weights + the launch sequence of one forward."""

    def __init__(self, cfg: DemucsConfig, state: dict, device=None, math=MATH_BF16X3):
        super().__init__(cfg, device, math)
        self.plan = layer_plan(cfg)
        self.encs = [(f"encoder.{i}", P["enc"]) for i, P in enumerate(self.plan)]
        self.decs = [(f"decoder.{j}", P["dec"]) for j, P in enumerate(self.plan[::-1])]
        st = layer_names(cfg, {k: np.asarray(v, dtype=np.float32) for k, v in state.items()})
        self._check_structure(st)
        self._load_weights(st)
        up, self.up_width = julius_taps(1, 2)
        down, self.down_width = julius_taps(2, 1)
        self.up_taps, self.down_taps = to_device(up, self.device), to_device(down, self.device)
        self.graphed = self.forward  # chunk widths vary with the chunk length: launched directly

    def _check_structure(self, st):
        cfg = self.cfg
        want = set()
        for prefix, L in self.encs + self.decs:
            enc = prefix.startswith("encoder")
            conv = f"{prefix}.conv.weight" if enc else f"{prefix}.conv_tr.weight"
            shape = (L["chout"], L["chin"], L["k"]) if enc else (L["chin"], L["chout"], L["k"])
            w = st.get(conv)
            if w is None or tuple(w.shape) != shape:
                raise ValueError(f"{conv} {None if w is None else tuple(w.shape)} does not match the configured Demucs structure (expected {shape})")
            rw = st.get(f"{prefix}.rewrite.weight")
            rshape = (2 * L["chout"], L["chout"], 1) if enc else (2 * L["chin"], L["chin"], 2 * L["context"] + 1)
            if rw is None or tuple(rw.shape) != rshape:
                raise ValueError(f"{prefix}.rewrite.weight {None if rw is None else tuple(rw.shape)} does not match the configured Demucs structure (expected {rshape})")
            want |= {f"{conv[: -len('weight')]}{b}" for b in ("weight", "bias")} | {f"{prefix}.rewrite.{b}" for b in ("weight", "bias")}
            norms = ["norm1", "norm2"] if enc else ["norm1"] + (["norm2"] if L["norm_tr"] else [])
            if L["norm"]:
                want |= {f"{prefix}.{n}.{b}" for n in norms for b in ("weight", "bias")}
            if L["dconv"]:
                if f"{prefix}.dconv.layers.{cfg.dconv_depth - 1}.0.weight" not in st:
                    raise ValueError(f"{prefix}: the DConv branch of dconv_mode={cfg.dconv_mode}, dconv_depth={cfg.dconv_depth} is missing")
                if (f"{prefix}.dconv.layers.0.3.lstm.weight_ih_l0" in st) != L["lstm"]:
                    raise ValueError(f"{prefix}: BLSTM presence does not match dconv_lstm={cfg.dconv_lstm}")
                has_attn = any(n.startswith(f"{prefix}.dconv.layers.0.") and ".query_decay." in n for n in st)
                if has_attn != L["attn"]:
                    raise ValueError(f"{prefix}: LocalState presence does not match dconv_attn={cfg.dconv_attn}")
                want |= {n for n in st if n.startswith(f"{prefix}.dconv.")}
        extra, missing = sorted(set(st) - want), sorted(want - set(st))
        if extra or missing:
            raise ValueError(f"state dict does not match the configured Demucs structure: unexpected {extra[:4]}, missing {missing[:4]}")
        if any(".query_freqs." in n for n in st):
            raise ValueError("LocalState with nfreqs > 0 is not supported")

    def forward(self, mix: torch.Tensor) -> torch.Tensor:
        """Demucs.forward (demucs.py:405-442): mix (B, 2, L) float32 cuda -> (B, S, 2, L)."""
        cfg = self.cfg
        assert mix.dim() == 3 and mix.shape[1] == 2 and mix.dtype == torch.float32 and mix.is_cuda
        mp = mix.contiguous()
        B, _, length = mp.shape
        valid = cfg.valid_length(length)
        x = _new((B, 2, 1, 2 * valid), mp)
        stats = _new((B, 2), mp)
        work = _new((lib.b200sep_meanstd_work_floats(B),), mp)
        check(lib.b200sep_demucs_upsample2_f32(_ptr(mp), B, length, valid, _ptr(self.up_taps), self.up_width, _ptr(stats), _ptr(x), _ptr(work), _stream()),
              "demucs_upsample2_f32")
        saved, lengths = [], []
        for prefix, L in self.encs:
            lengths.append(x.shape[-1])
            x = self._enc_layer(x, prefix, L)
            saved.append(x)
        x = None
        for prefix, L in self.decs:  # the first decoder sees x + center_trim(x, x) = 2 x (demucs.py:432-435); valid lengths make every trim empty
            x, _ = self._dec_layer(saved[-1] if x is None else x, saved.pop(-1), lengths.pop(-1), prefix, L)
        assert x.shape[-1] == 2 * valid, (x.shape, valid)
        out = _new((B, self.S, 2, length), mp)
        check(lib.b200sep_demucs_downsample2_f32(_ptr(x), B, self.S * 2, valid, length, _ptr(self.down_taps), self.down_width, _ptr(stats), _ptr(out), _stream()),
              "demucs_downsample2_f32")
        return out

    __call__ = forward
