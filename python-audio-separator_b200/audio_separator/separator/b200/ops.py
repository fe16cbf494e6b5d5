"""The operator layer of the network graph builders (demucs.py, hdemucs.py, roformer.py, vr.py): one thin wrapper per C-ABI operator
(include/b200sep.h) on float32 torch device buffers, the host-side weight layouts those operators take, and the cache of tensor-core
weight images.  Nothing here knows a network.
"""
from __future__ import annotations

import numpy as np
import torch

from ._lib import MATH_BF16X3, check, lib
from .engine import _ptr, _stream

# the `act` codes of conv2d_f32 and gemm_f32
ACT_NONE, ACT_RELU, ACT_GELU, ACT_LEAKY, ACT_SIGMOID, ACT_TANH = 0, 1, 2, 3, 4, 5


# --------------------------------------------------------------------------------------------------------- host-side weight prep
def to_device(a, device) -> torch.Tensor:
    """A host array as a contiguous float32 device tensor."""
    return torch.from_numpy(np.ascontiguousarray(a, dtype=np.float32)).to(device)


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


def lstm_bidir_weights(st, p, layer, device):
    """The parameters `{p}.*_l{layer}` / `{p}.*_l{layer}_reverse` of one nn.LSTM(bidirectional=True) layer (host arrays) -> the device tensors
    lstm_bidir takes: per direction the input weight (4*hid, in) and b_ih + b_hh summed in float64, and the recurrent matrices of both
    directions stacked, (2, 4*hid, hid) for lstm_bidir_f32 (hid <= 96) or transposed (2, hid, 4*hid) for lstm_bidir_wide_f32."""
    wih, bias, whh = [], [], []
    for sfx in ("", "_reverse"):
        wih.append(to_device(st[f"{p}.weight_ih_l{layer}{sfx}"], device))
        bias.append(to_device(st[f"{p}.bias_ih_l{layer}{sfx}"].astype(np.float64) + st[f"{p}.bias_hh_l{layer}{sfx}"].astype(np.float64), device))
        whh.append(st[f"{p}.weight_hh_l{layer}{sfx}"])
    if whh[0].shape[1] > 96:
        whh = [w.T for w in whh]
    return wih, bias, to_device(np.stack(whh), device)


# --------------------------------------------------------------------------------------------------------- operator wrappers
def _new(shape, like=None, device=None):
    return torch.empty(shape, dtype=torch.float32, device=like.device if like is not None else device)


def _packed_cache(w):
    """{math mode: packed image} of one weight tensor"""
    cache = getattr(w, "_b200_packed", None)
    if cache is None:
        cache = w._b200_packed = {}
    return cache


def _packed_conv(wb, cin, taps, cout, math=MATH_BF16X3):
    """The tensor-core image of a blocked convolution weight (bf16 hi/lo planes, or one fp16 plane, in the kernel's shared-memory layout), built once
    per tensor and math mode."""
    cache = _packed_cache(wb)
    pk = cache.get(math)
    if pk is None and cin * taps >= 32 and cout >= 16:
        cin8 = -(-cin // 8) * 8
        pk = _new((lib.b200sep_tc_packed_floats_math(cout, cin8 * taps, math),), wb)
        check(lib.b200sep_tc_pack_conv_weights_math(_ptr(wb), cin, taps, cout, _ptr(pk), math, _stream()), "tc_pack_conv_weights")
        cache[math] = pk
    return pk


def _packed_linear(w, math=MATH_BF16X3):
    cache = _packed_cache(w)
    pk = cache.get(math)
    if pk is None and w.shape[0] >= 32 and w.shape[1] >= 32:
        pk = _new((lib.b200sep_tc_packed_floats_math(w.shape[0], w.shape[1], math),), w)
        check(lib.b200sep_tc_pack_linear_weights_math(_ptr(w), w.shape[0], w.shape[1], w.shape[1], _ptr(pk), math, _stream()), "tc_pack_linear_weights")
        cache[math] = pk
    return pk


def conv2d(x, wb, bias, cout, k, s=(1, 1), p=(0, 0), dw=1, act=ACT_NONE, add=None, add_before_act=False, out_hw=None, out=None, out_c_off=0, dh=1, math=MATH_BF16X3):
    """x (B,Cin,H,W) -> (B,cout,Ho,Wo);  out_hw overrides the implied output size (right/bottom zero padding is implicit);
    out/out_c_off: write into channels [out_c_off, out_c_off + cout) of an existing (B, C_total, Ho, Wo) tensor (a fused torch.cat).
    math: MATH_BF16X3 or MATH_FP16 (tensor-core arithmetic; the SIMT fallback for small shapes is fp32 either way)."""
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
    pk = _packed_conv(wb, cin, k[0] * k[1], cout, math)
    check(lib.b200sep_conv2d_f32_math(_ptr(x), _ptr(wb), _ptr(bias) if bias is not None else None, _ptr(add) if add is not None else None, _ptr(y), B, cin, H, W, cout,
                                      Ho, Wo, k[0], k[1], s[0], s[1], p[0], p[1], dh, dw, act, int(add_before_act), 0, 1, 0, 0, ct, out_c_off,
                                      _ptr(pk) if pk is not None else None, math, _stream()), "conv2d_f32")
    return y


def conv_transpose(x, wb, bias, cout, axis, stride, trim, out_len, act=ACT_NONE, math=MATH_BF16X3):
    """nn.ConvTranspose1d/2d with kernel 2*stride along `axis` (1 = H, 2 = W), output cropped to [trim, trim + out_len)."""
    B, cin, H, W = x.shape
    if axis == 1:
        y = _new((B, cout, out_len, W), x)
        k, p, hw = (2, 1), (1, 0), (H + 1, W)
    else:
        y = _new((B, cout, H, out_len), x)
        k, p, hw = (1, 2), (0, 1), (H, W + 1)
    pk = _packed_conv(wb, cin, 2, stride * cout, math)
    check(lib.b200sep_conv2d_f32_math(_ptr(x), _ptr(wb), _ptr(bias), None, _ptr(y), B, cin, H, W, stride * cout, hw[0], hw[1], k[0], k[1], 1, 1, p[0], p[1], 1, 1, act,
                                      0, axis, stride, trim, out_len, 0, 0, _ptr(pk) if pk is not None else None, math, _stream()), "conv2d_f32(transposed)")
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


def groupnorm(x, groups, gamma, beta, act=ACT_NONE):
    """nn.GroupNorm(groups, C) in place on contiguous channel-first x (B, C, ...)."""
    B, C = x.shape[:2]
    X = x[0, 0].numel()
    work = _new((lib.b200sep_groupnorm_work_floats(B, C, groups, X),), x)
    check(lib.b200sep_groupnorm_f32(_ptr(x), _ptr(gamma), _ptr(beta), _ptr(x), B, C, groups, X, act, _ptr(work), _stream()), "groupnorm_f32")
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


def gemm(a, b, c, M, N, K, lda, ldb, ldc, batch=1, sA=0, sB=0, sC=0, alpha=1.0, bias_n=None, bias_m=None, act=ACT_NONE, res=None, res_scale=None, packed=None,
         math=MATH_BF16X3):
    """b200sep_gemm_f32 on device addresses: C[z] = act(alpha * A[z] (M,K; lda) @ B[z] (N,K; ldb)^T + bias_n[n] + bias_m[m]), then
    res + res_scale[n] * (.) with res at the strides of C; batch strides sA / sB / sC in floats.  packed: the tensor-core image of a static B
    (_packed_linear), or None."""
    check(lib.b200sep_gemm_f32_math(a, b, c, M, N, K, lda, ldb, ldc, batch, sA, sB, sC, alpha, bias_n, bias_m, act, res, res_scale, packed, math, _stream()), "gemm_f32")


def linear(x2d, w, bias, act=ACT_NONE, res=None, res_scale=None, math=MATH_BF16X3, out=None):
    """(M,K) @ w(N,K)^T + bias -> (M,N); optional res + res_scale[n] * (.).  x2d and out (allocated when None) may be row-strided views, such
    as a column slice of a wider matrix; res has the strides of out."""
    M, K = x2d.shape
    N = w.shape[0]
    y = _new((M, N), x2d) if out is None else out
    assert x2d.is_cuda and x2d.stride(1) == 1 and tuple(y.shape) == (M, N) and y.stride(1) == 1
    pk = _packed_linear(w, math)
    gemm(x2d.data_ptr(), _ptr(w), y.data_ptr(), M, N, K, x2d.stride(0), K, y.stride(0), bias_n=_ptr(bias) if bias is not None else None, act=act,
         res=_ptr(res) if res is not None else None, res_scale=_ptr(res_scale) if res_scale is not None else None, packed=_ptr(pk) if pk is not None else None,
         math=math)
    return y


def lstm_bidir(x2d, N, weights, math=MATH_BF16X3):
    """One bidirectional nn.LSTM layer over x2d (T*N, in), rows time-major, weights from lstm_bidir_weights: the input projections of both
    directions (gemm_f32, biases fused), then the recurrence -> (T*N, 2*hid) = [forward h_t | reverse h_t]."""
    wih, bias, whh = weights
    hid = wih[0].shape[0] // 4
    M, K = x2d.shape
    xp = _new((2, M, 4 * hid), x2d)
    for d in range(2):
        gemm(_ptr(x2d), _ptr(wih[d]), xp[d].data_ptr(), M, 4 * hid, K, K, K, 4 * hid, bias_n=_ptr(bias[d]), math=math)
    out = _new((M, 2 * hid), x2d)
    if hid <= 96:
        check(lib.b200sep_lstm_bidir_f32(_ptr(xp), _ptr(whh), _ptr(out), M // N, N, hid, _stream()), "lstm_bidir_f32")
    else:
        check(lib.b200sep_lstm_bidir_wide_f32(_ptr(xp), _ptr(whh), _ptr(out), M // N, N, hid, _stream()), "lstm_bidir_wide_f32")
    return out
