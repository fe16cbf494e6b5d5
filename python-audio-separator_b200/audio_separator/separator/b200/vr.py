"""VR architecture (CascadedASPPNet, "VR arch" v4 / v5.0 models) on the operator kernels of libb200sep.so.

VRNet.predict_mask replaces CascadedASPPNet.predict_mask (uvr_lib_v5/vr_network/nets.py:96-175, layers.py:8-294); VREngine replaces
VRSeparator.loading_mix / inference_vr / spec_to_wav (architectures/vr_separator.py:255-375) with the multi-band STFT, the band
resampling, the patch loop, the mask post-processing and the band synthesis all on the GPU.
This file is the graph builder: device buffers + launch order.  All arithmetic is behind the C ABI (include/b200sep.h).

VR 5.1 models (nets_new.CascadedNet, LSTM branch) run through VRNet51.  enable_tta, enable_post_process and high_end_process are supported, and so are models whose parameters run at
another rate than the file's (e.g. 32 / 48 kHz): the mix and the analysis bands are resampled with each band's res_type (b200/resample.py)
and the stems are resampled back to 44.1 kHz.  Not covered (raises): `reverse` model parameters, a top band whose rate is not the model's, a
res_type b200/resample.py has no filter for.  The band UP-sampling of the synthesis side uses the Kaiser polyphase design of res_type
"polyphase" (the reference calls libsamplerate "sinc_fastest" there; see DESIGN.md: parity unpinned for that step).

VREngine(dist=...) splits the patches of one track over the GPUs of a box (b200/sharded.py `plan_patch_shards`): the patches do not overlap, so
there is no halo; rank 0 gathers the mask and runs the mask post-processing and the synthesis.
"""
from __future__ import annotations

import math

import numpy as np
import torch

from ._lib import LAYOUT_CFT, MATH_BF16X3, check, lib
from .engine import StftPlan, _ptr, _require_cuda, _stream
from .ops import ACT_LEAKY, ACT_RELU, ACT_SIGMOID, _new, block_conv_weight, conv2d, ew, linear, lstm_bidir, lstm_bidir_weights, to_device
from .resample import resample, resample_poly_design  # noqa: F401  (resample_poly_design: the polyphase FIR, re-exported)
from .sharded import ShardRunner, shard_patches
NON_ACCOM_STEMS = ("Vocals", "Other", "Bass", "Drums", "Guitar", "Piano", "Synthesizer", "Strings", "Woodwinds", "Brass", "Wind Inst")  # common_separator.py:55
NN_ARCH_SIZES = (31191, 33966, 56817, 123821, 123812, 129605, 218409, 537238, 537227)  # vr_separator.py:166
VR_51_SIZES = (56817, 218409)


def copy_view(src: torch.Tensor, dst: torch.Tensor):
    """dst[...] = src[...] for two (possibly strided / broadcast) 4-D views of float32 CUDA storage: one strided-copy kernel."""
    assert src.dim() == 4 and tuple(src.shape) == tuple(dst.shape), (src.shape, dst.shape)
    d = src.shape
    check(lib.b200sep_copy4_f32(src.data_ptr(), dst.data_ptr(), d[0], d[1], d[2], d[3], *src.stride(), *dst.stride(), _stream()), "copy4_f32")


def lp_gain(n_bins, start, stop):
    """fft_lp_filter as a per-bin gain (spec_utils.py:410-418)."""
    g = np.ones(n_bins, np.float64)
    v = 1.0
    for b in range(start, stop):
        v -= 1 / (stop - start)
        g[b] = v
    g[stop:] = 0
    return g


def hp_gain(n_bins, start, stop):
    """fft_hp_filter as a per-bin gain (spec_utils.py:421-429)."""
    g = np.ones(n_bins, np.float64)
    v = 1.0
    for b in range(start, stop, -1):
        v -= 1 / (start - stop)
        g[b] = v
    g[0 : stop + 1] = 0
    return g


def lp_filter_mask(n_bins, start, stop):
    """get_lp_filter_mask (spec_utils.py:398-401, the VR 5.1 filters): ones, a linear ramp 1 -> 0 over [start-1, stop], zeros."""
    return np.concatenate([np.ones(start - 1), np.linspace(1, 0, stop - start + 1), np.zeros(n_bins - stop)])


def hp_filter_mask(n_bins, start, stop):
    """get_hp_filter_mask (spec_utils.py:404-407): zeros up to `stop`, a linear ramp 0 -> 1 up to `start`, ones."""
    return np.concatenate([np.zeros(stop + 1), np.linspace(0, 1, 1 + start - stop), np.ones(n_bins - start - 2)])


def merge_weights(frame_min: np.ndarray, thres: float, min_range=64, fade_size=32):
    """The per-frame weight merge_artifacts builds (spec_utils.py:180-212): runs of more than `min_range` consecutive frames whose smallest mask value
    exceeds `thres` get weight 1 with `fade_size`-frame linear ramps (none at the very start / end of the track; a run that starts closer than one
    fade after the previous one is merged into it).  Returns None where the reference's code raises and leaves the mask untouched (no such frame)."""
    if min_range < fade_size * 2:
        return None
    n = len(frame_min)
    hot = np.flatnonzero(frame_min > thres)
    if hot.size == 0:
        return None
    breaks = np.flatnonzero(np.diff(hot) != 1)
    starts, ends = np.concatenate([[hot[0]], hot[breaks + 1]]), np.concatenate([hot[breaks], [hot[-1]]])
    w = np.zeros(n, np.float32)
    prev_end = None
    up, down = np.linspace(0, 1, fade_size).astype(np.float32), np.linspace(1, 0, fade_size).astype(np.float32)
    for s, e in zip(starts, ends):
        if e - s <= min_range:
            continue
        s, e = int(s), int(e)
        if prev_end is not None and s - prev_end < fade_size:
            s = prev_end - fade_size * 2
        if s != 0:
            w[s : s + fade_size] = up[: max(0, min(fade_size, n - s))] if s >= 0 else w[s : s + fade_size]
        else:
            s -= fade_size
        if e != n:
            w[e - fade_size : e] = down
        else:
            e += fade_size
        w[s + fade_size : e - fade_size] = 1
        prev_end = e
    return w


def capacity(nn_architecture: int):
    """determine_model_capacity (nets.py:67-93)."""
    if nn_architecture in (31191, 33966, 129605):
        return 16, 8, 16, 32
    if nn_architecture in (123821, 123812):
        return 32, 16, 32, 64
    if nn_architecture in (537238, 537227):
        return 64, 32, 64, 128
    raise NotImplementedError(f"nn_architecture {nn_architecture}: only CascadedASPPNet sizes are covered (VR 5.1 CascadedNet is not)")


class VRNetBase:
    """What the VR networks share (VRNet, VRNet51): eval mode with BatchNorm folded into the preceding (bias-free) convolution, Dropout =
    identity; the convolution + BatchNorm + activation block, the decoder step and the cropping of predict_mask."""

    def __init__(self, n_fft_bins: int, offset: int, device=None, math=MATH_BF16X3):
        """math: MATH_BF16X3 (default, ~fp32) or MATH_FP16 (torch.autocast precision) for every tensor-core convolution / GEMM of this net."""
        _require_cuda()
        self.math = int(math)
        self.max_bin, self.output_bin, self.offset = n_fft_bins // 2, n_fft_bins // 2 + 1, offset
        self.device = torch.device(device) if device is not None else torch.device("cuda", torch.cuda.current_device())  # one process per GPU: the rank's own device
        self.W = {}

    def _load(self, state):
        """Uploads the folded convolutions and the output convolution; returns the state as host arrays for what a net adds."""
        st = {k: np.asarray(v) for k, v in state.items()}
        self._fold_all(st)
        self._put("out.w", block_conv_weight(st["out.weight"].astype(np.float32)))
        return st

    def _fold_all(self, st):
        for name in st:
            if not name.endswith(".conv.0.weight"):
                continue
            p = name[: -len(".conv.0.weight")]
            if p + ".conv.2.running_var" in st:  # SeperableConv2DBNActiv: depthwise (C,1,3,3), pointwise (nout,C,1,1), BatchNorm at index 2
                self._put(p + ".dw", st[name].reshape(st[name].shape[0], 9).astype(np.float32))
                self._fold(p, st[p + ".conv.1.weight"], st, p + ".conv.2")
            elif p + ".conv.1.running_var" in st:  # Conv2DBNActiv
                self._fold(p, st[name], st, p + ".conv.1")

    def _put(self, name, a):
        self.W[name] = to_device(a, self.device)

    def _fold(self, p, w, st, bn):
        inv = st[bn + ".weight"].astype(np.float64) / np.sqrt(st[bn + ".running_var"].astype(np.float64) + 1e-5)
        wf = (w.astype(np.float64) * inv[:, None, None, None]).astype(np.float32)
        self._put(p + ".w", block_conv_weight(wf))
        self._put(p + ".b", (st[bn + ".bias"].astype(np.float64) - st[bn + ".running_mean"].astype(np.float64) * inv).astype(np.float32))
        self.W[p + ".k"] = int(w.shape[-1])

    # ---- sub-graphs
    def _cba(self, x, p, stride=1, act=ACT_RELU, out=None, out_c_off=0, dil=(1, 1)):
        k = self.W[p + ".k"]
        cout = self.W[p + ".b"].numel()
        pad = (dil[0] * (k // 2), dil[1] * (k // 2))  # Conv2DBNActiv(..., pad=dilation, dilation=dilation) in the ASPP modules
        return conv2d(x, self.W[p + ".w"], self.W[p + ".b"], cout, (k, k), s=(stride, stride), p=pad, dw=dil[1], dh=dil[0], act=act, out=out, out_c_off=out_c_off,
                      math=self.math)

    def _dec(self, x, skip, conv):
        """Decoder: x up-sampled 2x (bilinear, align_corners), the skip cropped to its width concatenated on the channels, then the block `conv`."""
        B, C, H, W = x.shape
        Cs, Hs, Ws = skip.shape[1:]
        if Hs != 2 * H or Ws < 2 * W:
            raise ValueError(f"decoder skip {tuple(skip.shape)} does not fit the up-sampled {(B, C, 2 * H, 2 * W)} (the reference fails here too)")
        cat = _new((B, C + Cs, 2 * H, 2 * W), x)
        check(lib.b200sep_upsample2x_bilinear_f32(_ptr(x), _ptr(cat), B, C, H, W, C + Cs, 0, _stream()), "upsample2x_bilinear_f32")
        d = (Ws - 2 * W) // 2  # crop_center: time axis (spec_utils.py:50-71)
        copy_view(skip[:, :, :, d : d + 2 * W], cat[:, C:])
        return self._cba(cat, conv)

    def predict_mask(self, x: torch.Tensor) -> torch.Tensor:
        m = self.forward(x)
        if self.offset > 0:
            B, _, nb, Wd = m.shape
            out = _new((B, 2, nb, Wd - 2 * self.offset), m)
            copy_view(m[:, :, :, self.offset : Wd - self.offset], out)
            return out
        return m


class VRNet(VRNetBase):
    """CascadedASPPNet in eval mode."""

    def __init__(self, nn_architecture: int, n_fft_bins: int, state: dict, device=None, math=MATH_BF16X3):
        super().__init__(n_fft_bins, 128, device, math)
        self.arch = int(nn_architecture)
        self.c1, self.cb, self.c2, self.c3 = capacity(self.arch)
        self.n_enc = 5 if self.arch == 129605 else 4
        self.n_extra = 1 if self.arch == 129605 else (2 if self.arch in (537238, 537227, 33966) else 0)
        self._load(state)
        need = ["stg1_low_band_net.enc1.conv1.w", "stg3_full_band_net.dec1.conv.w", "stg2_bridge.w", "out.w", "stg1_low_band_net.aspp.conv3.dw"]
        for n in need:
            if n not in self.W:
                raise ValueError(f"state dict lacks {n.rsplit('.', 1)[0]}: not a CascadedASPPNet checkpoint")
        if self.W["stg1_low_band_net.enc1.conv1.b"].numel() != self.c1:
            raise ValueError("checkpoint width does not match the capacity of its nn_architecture size")

    def _sep(self, x, p, dil, out, out_c_off):
        B, C, H, W = x.shape
        y = _new(x.shape, x)
        check(lib.b200sep_dwconv3x3_f32(_ptr(x), _ptr(self.W[p + ".dw"]), _ptr(y), B, C, H, W, dil, _stream()), "dwconv3x3_f32")
        return self._cba(y, p, out=out, out_c_off=out_c_off)

    def _aspp(self, x, p):
        B, C, H, W = x.shape
        n_feat = 5 + self.n_extra
        cat = _new((B, C * n_feat, H, W), x)
        pooled = _new((B, C, 1, W), x)
        check(lib.b200sep_mean_h_f32(_ptr(x), _ptr(pooled), B * C, H, W, _stream()), "mean_h_f32")
        f1 = self._cba(pooled, p + ".conv1.1")  # (B,C,1,W); bilinear resize of a height-1 map (align_corners) = broadcast over H
        copy_view(f1.expand(B, C, H, W), cat[:, :C])
        self._cba(x, p + ".conv2", out=cat, out_c_off=C)
        for i, dil in ((3, 4), (4, 8), (5, 16)):
            self._sep(x, f"{p}.conv{i}", dil, cat, C * (i - 1))
        for i in range(self.n_extra):  # conv6 / conv7 are one shared module in the reference: the same weights under both names
            self._sep(x, f"{p}.conv{6 + i}", 16, cat, C * (5 + i))
        return self._cba(cat, p + ".bottleneck.0")

    def _base(self, x, p):
        skips = []
        for i in range(1, self.n_enc + 1):
            s = self._cba(x, f"{p}.enc{i}.conv1", act=ACT_LEAKY)
            x = self._cba(s, f"{p}.enc{i}.conv2", stride=2, act=ACT_LEAKY)
            skips.append(s)
        x = self._aspp(x, f"{p}.aspp")
        for i in range(self.n_enc, 0, -1):
            x = self._dec(x, skips[i - 1], f"{p}.dec{i}.conv")
        return x

    def forward(self, x: torch.Tensor) -> torch.Tensor:
        """x (B, 2, >= max_bin, W) magnitudes -> mask (B, 2, output_bin, W) (CascadedASPPNet.forward, eval)."""
        assert x.dim() == 4 and x.shape[1] == 2 and x.dtype == torch.float32 and x.is_cuda
        B, _, _, Wd = x.shape
        mb, c1, c2 = self.max_bin, self.c1, self.c2
        bw = mb // 2
        h2 = _new((B, 2 + c1 + c2, mb, Wd), x)  # cat([x, aux1, aux2], 1); its first 2 + c1 channels are stage 2's input
        copy_view(x[:, :, :mb], h2[:, :2])
        lo, hi = _new((B, 2, bw, Wd), x), _new((B, 2, mb - bw, Wd), x)
        copy_view(x[:, :, :bw], lo)
        copy_view(x[:, :, bw:mb], hi)
        copy_view(self._base(lo, "stg1_low_band_net"), h2[:, 2 : 2 + c1, :bw])
        copy_view(self._base(hi, "stg1_high_band_net"), h2[:, 2 : 2 + c1, bw:])
        h1 = _new((B, 2 + c1, mb, Wd), x)
        copy_view(h2[:, : 2 + c1], h1)
        self_aux2 = self._base(self._cba(h1, "stg2_bridge"), "stg2_full_band_net")
        copy_view(self_aux2, h2[:, 2 + c1 :])
        h = self._base(self._cba(h2, "stg3_bridge"), "stg3_full_band_net")
        m = conv2d(h, self.W["out.w"], None, 2, (1, 1), act=ACT_SIGMOID, math=self.math)
        mask = _new((B, 2, self.output_bin, Wd), x)
        copy_view(m, mask[:, :, :mb])
        copy_view(m[:, :, mb - 1 : mb].expand(B, 2, self.output_bin - mb, Wd), mask[:, :, mb:])  # F.pad(mode="replicate") on the bin axis
        return mask


class VRNet51(VRNetBase):
    """CascadedNet of VR 5.1 (vr_network/nets_new.py:52-160, layers_new.py): five band nets with stride-2 encoders, an ASPP of dilated 3x3 convolutions
    (dilations (4,2), (8,4), (12,6)) and a bidirectional-LSTM branch over the time axis in front of the last decoder; eval mode (BatchNorm folded)."""

    def __init__(self, n_fft_bins: int, nout: int, nout_lstm: int, state: dict, nn_arch_size: int = 56817, device=None, math=MATH_BF16X3):
        super().__init__(n_fft_bins, 64, device, math)
        self.arch = int(nn_arch_size)
        self.nout = 64 if self.arch == 218409 else int(nout)
        st = self._load(state)
        for name in st:  # LSTMModule: the bidirectional LSTM, dense + BatchNorm1d folded
            if not name.endswith(".lstm.weight_ih_l0"):
                continue
            p = name[: -len(".lstm.weight_ih_l0")]
            self.W[f"{p}.lstm"] = lstm_bidir_weights(st, f"{p}.lstm", 0, self.device)
            inv = st[f"{p}.dense.1.weight"].astype(np.float64) / np.sqrt(st[f"{p}.dense.1.running_var"].astype(np.float64) + 1e-5)
            self._put(f"{p}.dense.w", (st[f"{p}.dense.0.weight"].astype(np.float64) * inv[:, None]).astype(np.float32))
            self._put(f"{p}.dense.b", ((st[f"{p}.dense.0.bias"].astype(np.float64) - st[f"{p}.dense.1.running_mean"].astype(np.float64)) * inv
                                       + st[f"{p}.dense.1.bias"].astype(np.float64)).astype(np.float32))
        for n in ("stg1_low_band_net.0.enc1.w", "stg1_low_band_net.1.w", "stg3_full_band_net.lstm_dec2.lstm", "stg3_full_band_net.dec1.conv1.w", "out.w"):
            if n not in self.W:
                raise ValueError(f"state dict lacks {n.rsplit('.', 1)[0]}: not a VR 5.1 CascadedNet checkpoint")
        if self.W["stg3_full_band_net.enc1.b"].numel() != self.nout:
            raise ValueError("model_data nout does not match the checkpoint")

    def _enc(self, x, p, stride):
        return self._cba(self._cba(x, f"{p}.conv1", stride=stride, act=ACT_LEAKY), f"{p}.conv2", act=ACT_LEAKY)

    def _aspp51(self, x, p):
        B, C, H, W = x.shape
        co = self.W[f"{p}.conv2.b"].numel()
        cat = _new((B, co * 5, H, W), x)
        pooled = _new((B, C, 1, W), x)
        check(lib.b200sep_mean_h_f32(_ptr(x), _ptr(pooled), B * C, H, W, _stream()), "mean_h_f32")
        f1 = self._cba(pooled, f"{p}.conv1.1")
        copy_view(f1.expand(B, co, H, W), cat[:, :co])
        self._cba(x, f"{p}.conv2", out=cat, out_c_off=co)
        for i, dil in ((3, (4, 2)), (4, (8, 4)), (5, (12, 6))):
            self._cba(x, f"{p}.conv{i}", out=cat, out_c_off=co * (i - 1), dil=dil)
        return self._cba(cat, f"{p}.bottleneck")

    def _lstm(self, x, p, out, out_c_off):
        """LSTMModule.forward (layers_new.py:130-149): (N, C, nbins, nframes) -> one channel (N, 1, nbins, nframes) written into `out`."""
        W = self.W
        N, _, nb, nf = x.shape
        hc = self._cba(x, f"{p}.conv")  # (N, 1, nbins, nframes)
        seq = _new((nf, N, nb, 1), x)
        copy_view(hc.permute(3, 0, 2, 1), seq)  # "N 1 bins frames -> frames N bins"
        hs = lstm_bidir(seq.view(nf * N, nb), N, W[f"{p}.lstm"], self.math)
        dn = linear(hs, W[f"{p}.dense.w"], W[f"{p}.dense.b"], act=ACT_RELU, math=self.math)  # Linear + BatchNorm1d (folded) + ReLU: (frames*N, bins)
        copy_view(dn.view(nf, N, nb, 1).permute(1, 3, 2, 0), out[:, out_c_off : out_c_off + 1])

    def _base51(self, x, p):
        e1 = self._cba(x, f"{p}.enc1")
        e2 = self._enc(e1, f"{p}.enc2", 2)
        e3 = self._enc(e2, f"{p}.enc3", 2)
        e4 = self._enc(e3, f"{p}.enc4", 2)
        e5 = self._enc(e4, f"{p}.enc5", 2)
        h = self._aspp51(e5, f"{p}.aspp")
        h = self._dec(h, e4, f"{p}.dec4.conv1")
        h = self._dec(h, e3, f"{p}.dec3.conv1")
        h = self._dec(h, e2, f"{p}.dec2.conv1")
        B, C, H, W = h.shape
        hl = _new((B, C + 1, H, W), h)  # torch.cat([bottleneck, lstm_dec2(bottleneck)], dim=1)
        copy_view(h, hl[:, :C])
        self._lstm(h, f"{p}.lstm_dec2", hl, C)
        return self._dec(hl, e1, f"{p}.dec1.conv1")

    def forward(self, x: torch.Tensor) -> torch.Tensor:
        assert x.dim() == 4 and x.shape[1] == 2 and x.dtype == torch.float32 and x.is_cuda
        B, _, _, Wd = x.shape
        mb = self.max_bin
        bw = mb // 2
        no = self.nout
        xin = _new((B, 2, mb, Wd), x)
        copy_view(x[:, :, :mb], xin)
        lo, hi = _new((B, 2, bw, Wd), x), _new((B, 2, mb - bw, Wd), x)
        copy_view(x[:, :, :bw], lo)
        copy_view(x[:, :, bw:mb], hi)
        l1 = self._cba(self._base51(lo, "stg1_low_band_net.0"), "stg1_low_band_net.1")  # (B, no/4, bw, W)
        h1 = self._base51(hi, "stg1_high_band_net")
        c4 = no // 4
        l2_in, h2_in = _new((B, 2 + c4, bw, Wd), x), _new((B, 2 + c4, mb - bw, Wd), x)
        copy_view(lo, l2_in[:, :2]); copy_view(l1, l2_in[:, 2:])
        copy_view(hi, h2_in[:, :2]); copy_view(h1, h2_in[:, 2:])
        l2 = self._cba(self._base51(l2_in, "stg2_low_band_net.0"), "stg2_low_band_net.1")  # (B, no/2, bw, W)
        h2 = self._base51(h2_in, "stg2_high_band_net")
        c2 = no // 2
        f3_in = _new((B, 2 + c4 + c2, mb, Wd), x)  # cat([x, aux1, aux2], 1) with aux_i = cat([l_i, h_i], 2)
        copy_view(xin, f3_in[:, :2])
        copy_view(l1, f3_in[:, 2 : 2 + c4, :bw]); copy_view(h1, f3_in[:, 2 : 2 + c4, bw:])
        copy_view(l2, f3_in[:, 2 + c4 :, :bw]); copy_view(h2, f3_in[:, 2 + c4 :, bw:])
        f3 = self._base51(f3_in, "stg3_full_band_net")
        m = conv2d(f3, self.W["out.w"], None, 2, (1, 1), act=ACT_SIGMOID, math=self.math)
        mask = _new((B, 2, self.output_bin, Wd), x)
        copy_view(m, mask[:, :, :mb])
        copy_view(m[:, :, mb - 1 : mb].expand(B, 2, self.output_bin - mb, Wd), mask[:, :, mb:])
        return mask


class VREngine:
    """The VRSeparator hot path between reading the file and final_process, device resident."""

    def __init__(self, net: VRNet, param: dict, window_size=512, aggression=5, primary_stem="Instrumental", batch_size=1, dist=None, group=None):
        """dist / group: torch.distributed (backend nccl, one process per GPU) -- every rank is given the same track, runs the front end on all of
        it and predicts its own run of patches (b200/sharded.py `plan_patch_shards`); rank 0 gathers the mask and runs the back end, the other
        ranks get None from `inference` and `separate`.  Without dist the same code runs as one rank predicting every patch."""
        self.net, self.p = net, param
        self.runner = ShardRunner(dist, group)
        self.is_51 = isinstance(net, VRNet51)  # is_v51_model: filter masks instead of the running-gain filters, per-band convert_channels
        self.window_size, self.batch_size = int(window_size), max(1, int(batch_size))
        self.aggression, self.primary_stem = int(aggression), primary_stem
        self.device = net.device
        p = param
        if p.get("reverse"):
            raise NotImplementedError("model parameters with reverse=true are not covered")
        self.n_bands = len(p["band"])
        if net.output_bin != p["bins"] + 1:
            raise ValueError("network bin count does not match the model parameters")
        self.plans = {d: StftPlan(bp["n_fft"], bp["hl"]) for d, bp in p["band"].items()}
        # pre-filter of combine_spectrograms (spec_utils.py:266-277) as a per-bin gain
        g = np.ones(p["bins"] + 1, np.float64)
        if p["pre_filter_start"] > 0:
            if self.is_51:
                g = lp_filter_mask(p["bins"] + 1, p["pre_filter_start"], p["pre_filter_stop"])
            elif self.n_bands == 1:
                g = lp_gain(p["bins"] + 1, p["pre_filter_start"], p["pre_filter_stop"])
            else:
                gp = 1.0
                for b in range(p["pre_filter_start"] + 1, p["pre_filter_stop"]):
                    gp = math.pow(10, -(b - p["pre_filter_start"]) * (3.5 - gp) / 20.0)
                    g[b] = gp
        self.pre_gain = torch.from_numpy(g.astype(np.float32)).to(self.device)
        # synthesis-side band filters of cmb_spectrogram_to_wave (spec_utils.py:341-395)
        self.syn_gain = {}
        for d in range(1, self.n_bands + 1):
            bp = p["band"][d]
            nb = bp["n_fft"] // 2 + 1
            g = np.ones(nb, np.float64)
            hp_f, lp_f = (hp_filter_mask, lp_filter_mask) if self.is_51 else (hp_gain, lp_gain)
            if d == self.n_bands:
                if bp.get("hpf_start", -1) > 0:
                    g = hp_f(nb, bp["hpf_start"], bp["hpf_stop"] - 1)
            elif d == 1:
                g = lp_f(nb, bp["lpf_start"], bp["lpf_stop"])
            else:
                g = hp_f(nb, bp["hpf_start"], bp["hpf_stop"] - 1) * lp_f(nb, bp["lpf_start"], bp["lpf_stop"])
            self.syn_gain[d] = torch.from_numpy(g.astype(np.float32)).to(self.device)
        from .graphs import GraphedForward

        self.graphed = GraphedForward(self.net.predict_mask)

    # ---- analysis
    def _wave_to_spec(self, wave: torch.Tensor, d: int) -> torch.Tensor:
        """wave_to_spectrogram (spec_utils.py:282-312): (2, n) -> planes (4, n_fft/2+1, 1 + n//hop)."""
        p, bp = self.p, self.p["band"][d]
        if self.is_51:
            pass  # wave_to_spectrogram(is_v51_model=True): plain L/R transform, convert_channels afterwards
        elif p.get("mid_side"):
            w2 = _new(wave.shape, wave)
            ew(wave[0], wave[1], w2[0], 0.5, 0.5)
            ew(wave[0], wave[1], w2[1], 1.0, -1.0)
            wave = w2
        elif p.get("mid_side_b2"):
            w2 = _new(wave.shape, wave)
            ew(wave[1], wave[0], w2[0], 1.0, 0.5)
            ew(wave[0], wave[1], w2[1], 1.0, -0.5)
            wave = w2
        n = wave.shape[1]
        n_fft, hop = bp["n_fft"], bp["hl"]
        frames = 1 + n // hop
        spec = _new((4, n_fft // 2 + 1, frames), wave)
        check(lib.b200sep_stft_forward_ex(self.plans[d].handle, _ptr(wave), 2 * n, n, 0, 1, n, frames, n_fft // 2, 1.0, n_fft // 2 + 1, 0, LAYOUT_CFT, 1, _ptr(spec),
                                          _stream()), "stft_forward_ex")
        cc = bp.get("convert_channels") if self.is_51 else None
        if cc in ("mid_side_c", "mid_side", "stereo_n"):  # convert_channels (spec_utils.py:232-247): a real 2x2 mix of the L / R spectrograms
            (a, b), (c, e) = {"mid_side_c": ((1.0, 0.25), (-0.25, 1.0)), "mid_side": ((0.5, 0.5), (1.0, -1.0)), "stereo_n": ((1 / 0.9375, 0.25 / 0.9375), (0.25 / 0.9375, 1 / 0.9375))}[cc]
            mixed = _new(spec.shape, spec)
            L, R = spec[0:2], spec[2:4]  # (re, im) planes of the two channels
            ew(L, R, mixed[0:2], a, b)
            ew(L, R, mixed[2:4], c, e)
            spec = mixed
        return spec

    def loading_mix(self, wave: torch.Tensor, keep_high_end=False) -> torch.Tensor:
        """VRSeparator.loading_mix + combine_spectrograms: (2, N) at the top band's rate -> planes (4, bins + 1, frames)."""
        p, n = self.p, self.n_bands
        if p["band"][n]["sr"] != p["sr"]:
            raise NotImplementedError("the top band must be read at the model sample rate")
        waves, specs = {}, {}
        for d in range(n, 0, -1):
            bp = p["band"][d]
            if d == n:
                waves[d] = wave.contiguous()
            else:
                waves[d] = resample(waves[d + 1], p["band"][d + 1]["sr"], bp["sr"], bp["res_type"])
            specs[d] = self._wave_to_spec(waves[d], d)
        if keep_high_end:  # high_end_process (vr_separator.py:287-289): the top band's bins above its crop, as loaded
            bp = p["band"][n]
            self.high_end_h = (bp["n_fft"] // 2 - bp["crop_stop"]) + (p["pre_filter_stop"] - p["pre_filter_start"])
            mb = bp["n_fft"] // 2
            self.high_end = specs[n][:, mb - self.high_end_h : mb, :].contiguous()
        l = min(s.shape[2] for s in specs.values())
        out = torch.zeros((4, p["bins"] + 1, l), dtype=torch.float32, device=self.device)
        off = 0
        for d in range(1, n + 1):
            bp = p["band"][d]
            h = bp["crop_stop"] - bp["crop_start"]
            copy_view(specs[d][None, :, bp["crop_start"] : bp["crop_stop"], :l], out[None, :, off : off + h])
            off += h
        if off > p["bins"]:
            raise ValueError("Too much bins")
        if p["pre_filter_start"] > 0:
            check(lib.b200sep_bin_gain_f32(_ptr(out), _ptr(self.pre_gain), 4, p["bins"] + 1, l, _stream()), "bin_gain_f32")
        return out

    # ---- inference
    def _exponents(self):
        """adjust_aggr (spec_utils.py:472-492): exponent below / above the split bin, per channel."""
        aggr = float(int(self.aggression) / 100) * 2
        if aggr == 0:
            return 1.0, 1.0, 1.0, 1.0
        if self.primary_stem in NON_ACCOM_STEMS:
            aggr = 1 - aggr
        a = [aggr, aggr]
        corr = self.p.get("aggr_correction")
        if corr is not None:
            a[0] += corr["left"]
            a[1] += corr["right"]
        return 1 + a[0] / 3, 1 + a[0], 1 + a[1] / 3, 1 + a[1]

    def _execute(self, spec, pad_l, pad_r, roi):
        """_execute of inference_vr (vr_separator.py:296-327): zero-pad the magnitudes, normalise by the maximum, run every patch -> mask (2, bins, patches*roi).
        Sharded: every rank pads and normalises the whole track, predicts its own patches, and rank 0 gets the gathered mask (the other ranks None)."""
        nb, n_frame = spec.shape[1], spec.shape[2]
        off = self.net.offset
        n_pad = pad_l + n_frame + pad_r
        mag = torch.zeros((2, nb, n_pad), dtype=torch.float32, device=self.device)
        check(lib.b200sep_vr_magnitude_pad(_ptr(spec), _ptr(mag), nb, n_frame, n_pad, pad_l, _stream()), "vr_magnitude_pad")
        mx = _new((1,), mag)
        check(lib.b200sep_absmax(_ptr(mag), mag.numel(), _ptr(mx), _stream()), "absmax")
        peak = float(mx.cpu())
        if self.runner.world > 1:  # the ranks normalise independently: a rank given a different track must fail here, not write a wrong mask
            dist = self.runner.dist
            pk = torch.tensor([peak, -peak], dtype=torch.float32, device=self.device)
            dist.all_reduce(pk, op=dist.ReduceOp.MAX, group=self.runner.group)
            if float(pk[0]) != peak or float(pk[1]) != -peak:
                raise RuntimeError(f"VREngine: the ranks disagree on the normalisation peak ({peak} here, {-float(pk[1])}..{float(pk[0])} over the group): "
                                   "every rank must be given the same track")
        ew(mag, None, mag, 1.0 / peak if peak > 0 else float("nan"), 0.0)  # X_mag_pad /= X_mag_pad.max()
        patches = (n_pad - 2 * off) // roi
        if patches <= 0 or self.window_size - 2 * off <= 0:
            raise ValueError("Window size error: h1_shape[3] must be greater than h2_shape[3]")

        def predict(p0, p1):
            part = _new((2, nb, (p1 - p0) * roi), mag)
            self._predict(mag, p0, p1, roi, part)
            return part

        return shard_patches(self.runner, patches, roi, self.batch_size, predict)

    def _predict(self, mag, p0, p1, roi, out):
        """The patches [p0, p1) of the normalised padded magnitude, in forwards of batch_size from p0 -> out (2, bins, (p1 - p0) * roi)."""
        nb, n_pad = mag.shape[1], mag.shape[2]
        m4 = out.view(2, nb, p1 - p0, roi)
        for i in range(p0, p1, self.batch_size):
            b = min(self.batch_size, p1 - i)
            batch = _new((b, 2, nb, self.window_size), mag)
            src = torch.as_strided(mag, (b, 2, nb, self.window_size), (roi, nb * n_pad, n_pad, 1), storage_offset=i * roi)
            copy_view(src, batch)
            pred = self.graphed(batch)  # (b, 2, nb, roi): CascadedASPPNet.predict_mask, its launch list replayed as one CUDA graph per batch size
            copy_view(pred, m4[:, :, i - p0 : i - p0 + b].permute(2, 0, 1, 3))

    def _post_process(self, mask, n_frame, thres):
        """merge_artifacts (spec_utils.py:180-223) on the aggressiveness-adjusted mask (2, bins, stride): the min over (channel, bin) per frame is reduced
        on the device, the run detection works on that frames-long vector on the host, the merge runs on the device."""
        nb, stride = mask.shape[1], mask.shape[2]
        fm = _new((n_frame,), mask)
        check(lib.b200sep_vr_frame_min(_ptr(mask), stride, 2 * nb, n_frame, _ptr(fm), _stream()), "vr_frame_min")
        w = merge_weights(fm.cpu().numpy(), float(thres))
        if w is not None:
            wd = torch.from_numpy(w).to(self.device)
            check(lib.b200sep_vr_mask_merge(_ptr(mask), _ptr(wd), stride, 2 * nb, n_frame, _stream()), "vr_mask_merge")

    def masks(self, spec: torch.Tensor, enable_tta=False):
        """The network part of inference_vr (vr_separator.py:296-359): planes (4, bins+1, frames) -> mask (2, bins+1, >= frames), averaged over
        both passes with enable_tta.  Sharded: rank 0 gets the mask, the other ranks None."""
        nb, n_frame = spec.shape[1], spec.shape[2]
        off = self.net.offset
        roi = self.window_size - 2 * off
        if roi == 0:
            roi = self.window_size
        pad_l, pad_r = off, roi - (n_frame % roi) + off  # make_padding (spec_utils.py:85-96)
        mask = self._execute(spec, pad_l, pad_r, roi)
        if enable_tta:  # second pass shifted by half a region of interest; (mask + mask_tta[roi/2:]) / 2 on the first n_frame columns (:351-359)
            m2 = self._execute(spec, pad_l + roi // 2, pad_r + roi // 2, roi)
            if mask is None:
                return None
            avg = _new((2, nb, n_frame), mask)
            a_c, b_c = _new((2, nb, n_frame), mask), _new((2, nb, n_frame), mask)
            copy_view(mask[None, :, :, :n_frame], a_c[None])
            copy_view(m2[None, :, :, roi // 2 : roi // 2 + n_frame], b_c[None])
            mask = ew(a_c, b_c, avg, 0.5, 0.5)
        return mask

    def inference(self, spec: torch.Tensor, enable_tta=False, post_process_threshold=None):
        """VRSeparator.inference_vr (vr_separator.py:295-366): planes (4, bins+1, frames) -> (y planes, v planes); None on the ranks other than 0 of a
        sharded run."""
        mask = self.masks(spec, enable_tta)
        if mask is None:
            return None
        return self.apply_mask(spec, mask, post_process_threshold)

    def apply_mask(self, spec: torch.Tensor, mask: torch.Tensor, post_process_threshold=None):
        """The mask side of inference_vr (vr_separator.py:329-366): adjust_aggr, merge_artifacts (post_process_threshold), the products -> (y, v)
        planes.  Updates `mask` in place when post-processing."""
        nb, n_frame = spec.shape[1], spec.shape[2]
        y, v = _new(spec.shape, spec), _new(spec.shape, spec)
        e = self._exponents()
        if post_process_threshold is not None:  # enable_post_process: adjust_aggr first, then merge_artifacts, then the products (vr_separator.py:329-343)
            check(lib.b200sep_vr_mask_pow(_ptr(mask), mask.shape[2], nb, n_frame, self.p["band"][1]["crop_stop"], e[0], e[1], e[2], e[3], _stream()), "vr_mask_pow")
            self._post_process(mask, n_frame, post_process_threshold)
            e = (1.0, 1.0, 1.0, 1.0)
        check(lib.b200sep_vr_apply_mask(_ptr(mask), mask.shape[2], _ptr(spec), nb, n_frame, self.p["band"][1]["crop_stop"], e[0], e[1], e[2], e[3], _ptr(y), _ptr(v),
                                        _stream()), "vr_apply_mask")
        return y, v

    # ---- synthesis
    def _spec_to_wave(self, s: torch.Tensor, d: int) -> torch.Tensor:
        """spectrogram_to_wave (spec_utils.py:315-338): planes (4, n_fft/2+1, frames) -> (2, hop*(frames-1))."""
        bp, p = self.p["band"][d], self.p
        frames, nb = s.shape[2], s.shape[1]
        out_len = bp["hl"] * (frames - 1)
        wave = _new((2, out_len), s)
        work = _new((lib.b200sep_stft_inverse_work_floats(self.plans[d].handle, 1, frames, nb, LAYOUT_CFT),), s)
        check(lib.b200sep_stft_inverse_ex(self.plans[d].handle, _ptr(s), 1, frames, nb, LAYOUT_CFT, out_len, bp["n_fft"] // 2, 0, 1.0, _ptr(wave), _ptr(work), _stream()),
              "stft_inverse_ex")
        if self.is_51:
            cc = bp.get("convert_channels")
            if cc in ("mid_side_c", "mid_side", "stereo_n"):  # spectrogram_to_wave(is_v51_model=True) (spec_utils.py:322-330)
                (a, b), (c, e) = {"mid_side_c": ((1 / 1.0625, -1 / 4.25), (1 / 4.25, 1 / 1.0625)), "mid_side": ((1.0, 0.5), (1.0, -0.5)), "stereo_n": ((1.0, -0.25), (-0.25, 1.0))}[cc]
                w2 = _new(wave.shape, wave)
                ew(wave[0], wave[1], w2[0], a, b)
                ew(wave[0], wave[1], w2[1], c, e)
                return w2
            return wave
        if p.get("mid_side"):
            w2 = _new(wave.shape, wave)
            ew(wave[0], wave[1], w2[0], 1.0, 0.5)
            ew(wave[0], wave[1], w2[1], 1.0, -0.5)
            return w2
        if p.get("mid_side_b2"):
            w2 = _new(wave.shape, wave)
            ew(wave[1], wave[0], w2[0], 1 / 1.25, 0.4)
            ew(wave[0], wave[1], w2[1], 1 / 1.25, -0.4)
            return w2
        return wave

    def spec_to_wav(self, spec_m: torch.Tensor, high_end=False) -> torch.Tensor:
        """cmb_spectrogram_to_wave (spec_utils.py:341-395): planes (4, bins+1, frames) -> (2, hop_top*(frames-1)).  high_end: mirror the kept input high end
        into the top band (VRSeparator.spec_to_wav with high_end_process, vr_separator.py:368-372)."""
        p, n = self.p, self.n_bands
        frames = spec_m.shape[2]
        off = 0
        wave = None
        for d in range(1, n + 1):
            bp = p["band"][d]
            nb = bp["n_fft"] // 2 + 1
            s = torch.zeros((4, nb, frames), dtype=torch.float32, device=self.device)
            h = bp["crop_stop"] - bp["crop_start"]
            copy_view(spec_m[None, :, off : off + h], s[None, :, bp["crop_start"] : bp["crop_stop"]])
            off += h
            if d == n and high_end:
                he = self.high_end
                check(lib.b200sep_vr_mirror_high_end(_ptr(spec_m), spec_m.shape[1], _ptr(he), he.shape[1], he.shape[2], _ptr(s), nb, frames, self.high_end_h, bp["n_fft"] // 2,
                                                     p["pre_filter_start"], _stream()), "vr_mirror_high_end")
            filtered = (d == n and bp.get("hpf_start", -1) > 0) or d < n
            if filtered:
                check(lib.b200sep_bin_gain_f32(_ptr(s), _ptr(self.syn_gain[d]), 4, nb, frames, _stream()), "bin_gain_f32")
            w_d = self._spec_to_wave(s, d)
            if d == n:
                wave = w_d if n == 1 else ew(wave, w_d, wave)
            else:
                if d > 1:
                    w_d = ew(wave, w_d, w_d)
                wave = resample(w_d, bp["sr"], p["band"][d + 1]["sr"], "polyphase")  # the stand-in for the reference's sinc_fastest up-sampling
        return wave

    def separate(self, wave: np.ndarray, enable_tta=False, post_process_threshold=None, high_end_process=False, sr=None):
        """(2, N) host -> primary (2, M), secondary (2, M) host float32, M = hop_top * (frames - 1); None on the ranks other than 0 of a sharded run.
        sr: the rate of `wave` when it is not the model's (VRSeparator passes 44100).  The mix is then resampled to the top band's rate with that
        band's res_type, as librosa.load(sr=band sr) does (vr_separator.py:273), and both stems are resampled back to `sr` with librosa's default
        soxr_hq (:221-222, :239-240), M = ceil(M_model * sr / model sr).  Sharded: every rank resamples the mix, rank 0 the stems."""
        wd = torch.from_numpy(np.ascontiguousarray(wave, dtype=np.float32)).to(self.device)
        top = self.p["band"][self.n_bands]
        model_sr = self.p["sr"]
        if sr is not None:
            wd = resample(wd, sr, top["sr"], top["res_type"])
        spec = self.loading_mix(wd, keep_high_end=high_end_process)
        yv = self.inference(spec, enable_tta, post_process_threshold)
        if yv is None:
            return None
        out = []
        for s in yv:
            w = self.spec_to_wav(s, high_end_process)
            if sr is not None:
                w = resample(w, model_sr, sr, "soxr_hq")
            out.append(w.cpu().numpy())
        return tuple(out)
