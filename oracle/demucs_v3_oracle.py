"""CPU oracle for the time-domain Demucs v3 network -- TEST INFRASTRUCTURE, not product code.

Functional torch-CPU restatement of
  * Demucs.__init__ parameter layout / valid_length / forward   uvr_lib_v5/demucs/demucs.py:234-442 (nn.Sequential encoder / decoder layers)
  * julius.resample_frac(x, old, new) with ResampleFrac's defaults (zeros=24, rolloff=0.945): julius is not a dependency of this project, so the
    filter is restated from its definition (replicate-padded input, stride-`old` convolution with `new` windowed-sinc phase filters, phases
    interleaved) -- the same restatement is injected into the reference when it is pinned, so this step is "parity unpinned"
  * apply_model for a member with valid_length and a BagOfModels of members with their own segments   demucs/apply.py:124-260
The DConv branch reuses hdemucs_oracle's BLSTM / LocalState restatements.  Pinned against the unmodified reference by
oracle/make_golden_demucs_v3.py.
"""
from __future__ import annotations

import math
from dataclasses import dataclass

import numpy as np

import hdemucs_oracle as H
from demucs_oracle import center_trim, padded


@dataclass
class V3Config:
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
    # LocalState / BLSTM constants of DConv (demucs.py:158-161)
    attn_heads: int = 4
    attn_ndecay: int = 4
    lstm_layers: int = 2
    lstm_max_steps: int = 200

    @property
    def seg_len(self):  # apply.py:218
        return int(self.samplerate * self.segment)

    def kwargs(self):  # what the reference constructor receives
        return dict(sources=list(self.sources), audio_channels=self.audio_channels, channels=self.channels, growth=self.growth, depth=self.depth,
                    kernel_size=self.kernel_size, stride=self.stride, context=self.context, norm_starts=self.norm_starts, norm_groups=self.norm_groups,
                    dconv_mode=self.dconv_mode, dconv_depth=self.dconv_depth, dconv_comp=self.dconv_comp, dconv_attn=self.dconv_attn, dconv_lstm=self.dconv_lstm,
                    samplerate=self.samplerate, segment=self.segment)

    def valid_length(self, length):  # demucs.py:382-403 (resample=True)
        length *= 2
        for _ in range(self.depth):
            length = max(1, math.ceil((length - self.kernel_size) / self.stride) + 1)
        for _ in range(self.depth):
            length = (length - 1) * self.stride + self.kernel_size
        return int(math.ceil(length / 2))


def param_shapes(cfg: V3Config):
    """state_dict names (nn.Sequential indices) and shapes of Demucs(**cfg.kwargs()), encoders then decoders (decoder 0 = the deepest layer)."""
    S, C = len(cfg.sources), cfg.audio_channels
    enc, dec = [], []

    def dconv(p, ch, lstm, attn, out):
        hid = int(ch / cfg.dconv_comp)
        for d in range(cfg.dconv_depth):
            q = f"{p}.layers.{d}"
            out.extend([(f"{q}.0.weight", (hid, ch, 3)), (f"{q}.0.bias", (hid,)), (f"{q}.1.weight", (hid,)), (f"{q}.1.bias", (hid,))])
            i = 3
            if lstm:
                for layer in range(cfg.lstm_layers):
                    for sfx in ("", "_reverse"):
                        nin = hid if layer == 0 else 2 * hid
                        out.extend([(f"{q}.{i}.lstm.weight_ih_l{layer}{sfx}", (4 * hid, nin)), (f"{q}.{i}.lstm.weight_hh_l{layer}{sfx}", (4 * hid, hid)),
                                    (f"{q}.{i}.lstm.bias_ih_l{layer}{sfx}", (4 * hid,)), (f"{q}.{i}.lstm.bias_hh_l{layer}{sfx}", (4 * hid,))])
                out.extend([(f"{q}.{i}.linear.weight", (hid, 2 * hid)), (f"{q}.{i}.linear.bias", (hid,))])
                i += 1
            if attn:
                for nm, co in (("content", hid), ("query", hid), ("key", hid), ("query_decay", cfg.attn_heads * cfg.attn_ndecay), ("proj", hid)):
                    out.extend([(f"{q}.{i}.{nm}.weight", (co, hid, 1)), (f"{q}.{i}.{nm}.bias", (co,))])
                i += 1
            out.extend([(f"{q}.{i}.weight", (2 * ch, hid, 1)), (f"{q}.{i}.bias", (2 * ch,)), (f"{q}.{i + 1}.weight", (2 * ch,)), (f"{q}.{i + 1}.bias", (2 * ch,)),
                        (f"{q}.{i + 3}.scale", (ch,))])

    chin, ch = C, cfg.channels
    for index in range(cfg.depth):
        norm, lstm, attn = index >= cfg.norm_starts, index >= cfg.dconv_lstm, index >= cfg.dconv_attn
        p = f"encoder.{index}"
        e = [(f"{p}.0.weight", (ch, chin, cfg.kernel_size)), (f"{p}.0.bias", (ch,))]
        if norm:
            e += [(f"{p}.1.weight", (ch,)), (f"{p}.1.bias", (ch,))]
        r = 3
        if cfg.dconv_mode & 1:
            dconv(f"{p}.3", ch, lstm, attn, e)
            r = 4
        e += [(f"{p}.{r}.weight", (2 * ch, ch, 1)), (f"{p}.{r}.bias", (2 * ch,))]
        if norm:
            e += [(f"{p}.{r + 1}.weight", (2 * ch,)), (f"{p}.{r + 1}.bias", (2 * ch,))]
        enc.append(e)
        co = chin if index > 0 else S * C
        p = f"decoder.{cfg.depth - 1 - index}"
        d = [(f"{p}.0.weight", (2 * ch, ch, 2 * cfg.context + 1)), (f"{p}.0.bias", (2 * ch,))]
        if norm:
            d += [(f"{p}.1.weight", (2 * ch,)), (f"{p}.1.bias", (2 * ch,))]
        t = 3
        if cfg.dconv_mode & 2:
            dconv(f"{p}.3", ch, lstm, attn, d)
            t = 4
        d += [(f"{p}.{t}.weight", (ch, co, cfg.kernel_size)), (f"{p}.{t}.bias", (co,))]
        if norm and index > 0:
            d += [(f"{p}.{t + 1}.weight", (co,)), (f"{p}.{t + 1}.bias", (co,))]
        dec.insert(0, d)
        chin, ch = ch, int(cfg.growth * ch)
    return [x for e in enc for x in e] + [x for d in dec for x in d]


def make_weights(cfg: V3Config, seed=0):
    rng = np.random.default_rng(seed)
    w = {}
    for name, shape in param_shapes(cfg):
        if name.endswith(".scale"):
            a = rng.uniform(0.05, 0.3, shape)
        elif ".lstm." in name:
            a = rng.uniform(-1.0, 1.0, shape) / math.sqrt(shape[0] // 4)
        elif "query_decay.bias" in name:
            a = rng.normal(-2.0, 0.3, shape)
        elif "query_decay.weight" in name:
            a = rng.normal(0.0, 0.3 / math.sqrt(shape[1]), shape)
        elif len(shape) == 1 and name.endswith(".weight"):
            a = rng.uniform(0.7, 1.3, shape)
        elif len(shape) == 1:
            a = rng.normal(0.0, 0.05, shape)
        else:
            fan_in = int(np.prod(shape[1:]))
            a = rng.normal(0.0, math.sqrt(1.5 / fan_in), shape)
        w[name] = a.astype(np.float32)
    return w


# ---------------------------------------------------------------------------------------------------------
def julius_taps(old: int, new: int, zeros: int = 24, rolloff: float = 0.945):
    """ResampleFrac._init_kernels in float64: -> (kernel (new, 2 * width + old), width)."""
    sr = min(old, new) * rolloff
    width = math.ceil(zeros * old / sr)
    idx = np.arange(-width, width + old, dtype=np.float64)
    rows = []
    for i in range(new):
        t = np.clip((-i / new + idx / old) * sr, -zeros, zeros) * math.pi
        k = np.where(t == 0, 1.0, np.sin(t) / np.where(t == 0, 1.0, t)) * np.cos(t / zeros / 2) ** 2
        rows.append(k / k.sum())
    return np.stack(rows), width


def resample_frac(x, old_sr: int, new_sr: int, output_length=None, full=False, zeros: int = 24, rolloff: float = 0.945):
    """julius.resample_frac (ResampleFrac.forward) on a torch tensor (..., L); the taps are rounded once to float32 (as the kernels take them)."""
    import torch
    import torch.nn.functional as F

    if old_sr == new_sr:
        return x
    k, width = julius_taps(old_sr, new_sr, zeros, rolloff)
    shape, length = x.shape, x.shape[-1]
    xp = F.pad(x.reshape(-1, length)[:, None], (width, width + old_sr), mode="replicate")
    ys = F.conv1d(xp, torch.from_numpy(k.astype(np.float32)).to(x.dtype)[:, None, :], stride=old_sr)
    y = ys.transpose(1, 2).reshape(list(shape[:-1]) + [-1])
    n = new_sr * length / old_sr
    n = output_length if output_length is not None else (math.ceil(n) if full else int(math.floor(n)))
    return y[..., :n]


def resample_in(x, valid: int):
    """The input end of Demucs.forward (demucs.py:409-422) on a torch tensor (B, 2, L): -> (julius x2 of the normalised, centred-zero-padded
    input (B, 2, 2 * valid), mean (B, 1, 1), std (B, 1, 1)) -- the contract of b200sep_demucs_upsample2_f32."""
    import torch.nn.functional as F

    mono = x.mean(dim=1, keepdim=True)
    mean = mono.mean(dim=-1, keepdim=True)
    std = mono.std(dim=-1, keepdim=True)
    x = (x - mean) / (1e-5 + std)
    delta = valid - x.shape[-1]
    return resample_frac(F.pad(x, (delta // 2, delta - delta // 2)), 1, 2), mean, std


def resample_out(x, mean, std, length: int):
    """The output end (demucs.py:437-441): julius /2, de-normalisation, center_trim -- the contract of b200sep_demucs_downsample2_f32."""
    return center_trim(resample_frac(x, 2, 1) * std + mean, length)


def forward(weights, cfg: V3Config, mix: np.ndarray, dtype="float32", taps=None) -> np.ndarray:
    """Demucs.forward in eval mode: mix (B, 2, L) -> (B, S, 2, L).  `taps` (a dict) receives every encoder / decoder output."""
    import torch
    import torch.nn.functional as F

    td = torch.float64 if dtype == "float64" else torch.float32
    W = {k: torch.from_numpy(np.asarray(v)).to(td) for k, v in weights.items()}
    x = torch.from_numpy(np.ascontiguousarray(mix)).to(td)
    B, _, length = x.shape
    G = cfg.norm_groups

    def tap(name, t):
        if taps is not None:
            taps[name] = t.to(torch.float32).numpy().copy()

    def norm(y, p, on):
        return F.group_norm(y, G, W[f"{p}.weight"], W[f"{p}.bias"], 1e-5) if on else y

    def dconv(y, prefix, lstm, attn):  # demucs.py:149-168
        for d in range(cfg.dconv_depth):
            p = f"{prefix}.layers.{d}"
            dil = 2**d
            h = F.conv1d(y, W[f"{p}.0.weight"], W[f"{p}.0.bias"], dilation=dil, padding=dil)
            h = F.gelu(F.group_norm(h, 1, W[f"{p}.1.weight"], W[f"{p}.1.bias"]))
            i = 3
            if lstm:
                h = H.blstm(h, W, f"{p}.{i}", cfg)
                i += 1
            if attn:
                h = H.local_state(h, W, f"{p}.{i}", cfg)
                i += 1
            h = F.conv1d(h, W[f"{p}.{i}.weight"], W[f"{p}.{i}.bias"])
            h = F.glu(F.group_norm(h, 1, W[f"{p}.{i + 1}.weight"], W[f"{p}.{i + 1}.bias"]), dim=1)
            y = y + W[f"{p}.{i + 3}.scale"][:, None] * h
        return y

    with torch.no_grad():
        x, mean, std = resample_in(x, cfg.valid_length(length))
        saved = []
        for index in range(cfg.depth):  # demucs.py:347-355
            p = f"encoder.{index}"
            on, lstm, attn = index >= cfg.norm_starts, index >= cfg.dconv_lstm, index >= cfg.dconv_attn
            x = F.gelu(norm(F.conv1d(x, W[f"{p}.0.weight"], W[f"{p}.0.bias"], stride=cfg.stride), f"{p}.1", on))
            r = 3
            if cfg.dconv_mode & 1:
                x = dconv(x, f"{p}.3", lstm, attn)
                r = 4
            x = F.glu(norm(F.conv1d(x, W[f"{p}.{r}.weight"], W[f"{p}.{r}.bias"]), f"{p}.{r + 1}", on), dim=1)
            tap(f"enc{index}", x)
            saved.append(x)
        for j in range(cfg.depth):  # demucs.py:357-369, :432-435
            index = cfg.depth - 1 - j
            p = f"decoder.{j}"
            on, lstm, attn = index >= cfg.norm_starts, index >= cfg.dconv_lstm, index >= cfg.dconv_attn
            x = x + center_trim(saved.pop(-1), x.shape[-1])
            x = F.glu(norm(F.conv1d(x, W[f"{p}.0.weight"], W[f"{p}.0.bias"], padding=cfg.context), f"{p}.1", on), dim=1)
            t = 3
            if cfg.dconv_mode & 2:
                x = dconv(x, f"{p}.3", lstm, attn)
                t = 4
            x = F.conv_transpose1d(x, W[f"{p}.{t}.weight"], W[f"{p}.{t}.bias"], stride=cfg.stride)
            if index > 0:
                x = F.gelu(norm(x, f"{p}.{t + 1}", on))
            tap(f"dec{j}", x)
        out = resample_out(x, mean, std, length).reshape(B, len(cfg.sources), cfg.audio_channels, length)
    return out.to(torch.float32).numpy()


# ---------------------------------------------------------------------------------------------------------
def _valid(cfg, length):  # model.valid_length where the model has one (apply.py:252-255); HDemucs has none
    return cfg.valid_length(length) if hasattr(cfg, "valid_length") else length


def apply_chunk(model_fn, cfg, tensor: np.ndarray, offset: int, length: int):
    """apply_model's leaf (apply.py:251-260): TensorChunk(tensor, offset, length).padded(valid_length) -- real neighbouring samples, zeros only
    outside `tensor` -- one forward, center_trim back to `length`."""
    return center_trim(model_fn(padded(tensor, offset, length, _valid(cfg, length))), length)


def apply_split(model_fn, cfg, tensor: np.ndarray, offset: int, length: int, overlap=0.25):
    """apply_model(split=True) (apply.py:215-250) with the member's own segment."""
    S = len(cfg.sources)
    seg = cfg.seg_len
    stride = int((1 - overlap) * seg)
    out = np.zeros((1, S, tensor.shape[1], length), np.float32)
    sw = np.zeros(length, np.float32)
    weight = np.concatenate([np.arange(1, seg // 2 + 1), np.arange(seg - seg // 2, 0, -1)]).astype(np.float32)
    weight = weight / weight.max()
    for off in range(0, length, stride):
        clen = min(length - off, seg)
        out[..., off : off + seg] += weight[:clen] * apply_chunk(model_fn, cfg, tensor, offset + off, clen)
        sw[off : off + seg] += weight[:clen]
    return out / sw


def apply_model(model_fn, cfg, mix: np.ndarray, shift_offsets, split=True, overlap=0.25):
    """apply_model(shifts=len(shift_offsets), split) (apply.py:197-260), offsets injected: mix (1, C, N) -> (1, S, C, N)."""
    N = mix.shape[-1]
    one = (lambda t, o, n: apply_split(model_fn, cfg, t, o, n, overlap)) if split else (lambda t, o, n: apply_chunk(model_fn, cfg, t, o, n))
    if not shift_offsets:
        return one(mix, 0, N)
    max_shift = int(0.5 * cfg.samplerate)
    pm = padded(mix, 0, N, N + 2 * max_shift)
    out = 0
    for o in shift_offsets:
        out = out + one(pm, o, N + max_shift - o)[..., max_shift - o :]
    return out / len(shift_offsets)


def apply_bag(members, bag_weights, mix: np.ndarray, shift_offsets, split=True, overlap=0.25):
    """apply_model on a BagOfModels (apply.py:169-195): members [(model_fn, cfg)], per-source weights, one list of shift draws per member."""
    S = len(members[0][1].sources)
    est, totals = 0, [0.0] * S
    for (fn, cfg), wts, offs in zip(members, bag_weights, shift_offsets):
        out = apply_model(fn, cfg, mix, offs, split, overlap)
        for k, wk in enumerate(wts):
            out[:, k] *= wk
            totals[k] += wk
        est = est + out
    for k in range(S):
        est[:, k] /= totals[k]
    return est
