"""Operand-rounding restatement of the fp16 tensor-core mode (MATH_FP16) for the oracles.

Inside `fp16_operands()` every contraction that the library sends to the tensor cores gets both operands rounded to fp16 (`x.half()`, so
|x| > 65504 becomes +-inf like autocast's cast) and is then contracted in float64.  Biases, norms, softmax, STFTs and the contractions the
library runs on its fp32 SIMT kernels are left alone.  This is what the kernels compute, up to the order of the fp32 accumulation, so a
forward of the unmodified oracle at dtype="float64" under this context is the reference the fp16 mode is held to.

Which launches run on the tensor cores is a shape rule of the library (tc_gemm_usable / tc_conv_usable in csrc/tc_f32.cu); `tc_gemm_usable`
and `tc_conv_usable` restate it, and tests/test_autocast_ops_gpu.py::test_shape_rule_matches_the_library holds the two copies together (on
either side of each threshold, MATH_FP16 changes the result exactly when the restated rule says tensor core).  The patch covers:
  * F.linear (gemm_f32) and the two attention einsums of the Roformer oracles (the fused attention kernel for head dimension 64; otherwise the
    scores are a gemm_f32 and P V is the fp32 gemm_kn_f32);
  * F.conv1d / F.conv2d / F.conv_transpose1d / F.conv_transpose2d of the HTDemucs oracle (conv2d_f32; a transposed convolution is a 2-tap
    convolution with stride * Cout columns, on the tensor cores only when Cout is a multiple of 16).  DConv layers whose hidden width the fused
    fp32 DConv kernel handles (demucs.py `_DCONV_FUSED_HID`) stay unrounded: pass `dconv_fused_hid` to enable that rule.
"""
import contextlib

import torch
import torch.nn.functional as F


def r16(x: torch.Tensor) -> torch.Tensor:
    return x.to(torch.float16).to(torch.float64)


def tc_gemm_usable(M, N, K, batch=1):
    return K >= 32 and N >= 32 and M * N * batch >= 128 * 128


def tc_conv_usable(cin, cout, kh, kw, ho, wo, b):
    return cin * kh * kw >= 32 and cout >= 16 and ho * wo * b >= 512


def _dconv_fused(cin, cout, k, fused_hid):
    """True for the two convolutions of a DConv layer that HTDemucsNet._dconv runs inside the fused fp32 kernel (b200sep_dconv_f32)."""
    if not fused_hid:
        return False
    if k == 3 and 4 * cout == cin:  # C -> hid, k 3 (hid = C / 4)
        C, hid = cin, cout
        first = True
    elif k == 1 and cout == 8 * cin:  # hid -> 2C, 1x1
        C, hid = cout // 2, cin
        first = False
    else:
        return False
    h4 = -(-hid // 4) * 4
    if hid not in fused_hid or C * 2 * (h4 + 4) * 4 > 200 * 1024:
        return False
    return not (first and 3 * C * h4 * 4 > 200 * 1024)  # the widest layers run their C -> hid convolution on conv2d_f32


@contextlib.contextmanager
def fp16_operands(dconv_fused_hid=()):
    linear0, einsum0 = F.linear, torch.einsum
    conv1d0, conv2d0, convt1d0, convt2d0 = F.conv1d, F.conv2d, F.conv_transpose1d, F.conv_transpose2d

    def linear(x, w, b=None):
        M = x.numel() // x.shape[-1]
        N, K = w.shape
        if not tc_gemm_usable(M, N, K):
            return linear0(x, w, b)
        y = linear0(r16(x), r16(w)).to(x.dtype)
        return y + b if b is not None else y

    def einsum(eq, *ops):
        if eq == "bhid,bhjd->bhij":  # attention scores
            q, k = ops
            B, H, n, dh = q.shape
            if dh == 64 or tc_gemm_usable(n, k.shape[2], dh, B * H):
                return einsum0(eq, r16(q), r16(k)).to(q.dtype)
        elif eq == "bhij,bhjd->bhid":  # P V: fused kernel (dh 64) only
            p, v = ops
            if v.shape[-1] == 64:
                return einsum0(eq, r16(p), r16(v)).to(p.dtype)
        return einsum0(eq, *ops)

    def conv(op, nd):
        def f(x, w, b=None, stride=1, padding=0, dilation=1, groups=1):
            y = op(x, w, None, stride, padding, dilation, groups)
            cout, cin = w.shape[0], w.shape[1]
            taps = w.shape[2] * (w.shape[3] if nd == 2 else 1)
            hw = y.shape[2] * (y.shape[3] if nd == 2 else 1)
            if groups == 1 and tc_conv_usable(cin, cout, taps, 1, hw, 1, x.shape[0]) and not (nd == 1 and _dconv_fused(cin, cout, w.shape[2], dconv_fused_hid)):
                y = op(r16(x), r16(w), None, stride, padding, dilation, groups).to(x.dtype)
            return y + b.view(-1, *([1] * nd)) if b is not None else y
        return f

    def convt(op, nd):
        def f(x, w, b=None, stride=1, padding=0, output_padding=0, groups=1, dilation=1):
            y = op(x, w, None, stride, padding, output_padding, groups, dilation)
            cin, cout = w.shape[0], w.shape[1]
            s = stride if isinstance(stride, int) else max(stride)
            coarse = (x.shape[2] + 1) * x.shape[3] if nd == 2 else x.shape[2] + 1  # the 2-tap convolution runs over the coarse index, one past the input
            if groups == 1 and cout % 16 == 0 and tc_conv_usable(cin, s * cout, 2, 1, coarse, 1, x.shape[0]):
                y = op(r16(x), r16(w), None, stride, padding, output_padding, groups, dilation).to(x.dtype)
            return y + b.view(-1, *([1] * nd)) if b is not None else y
        return f

    F.linear, torch.einsum = linear, einsum
    F.conv1d, F.conv2d, F.conv_transpose1d, F.conv_transpose2d = conv(conv1d0, 1), conv(conv2d0, 2), convt(convt1d0, 1), convt(convt2d0, 2)
    try:
        yield
    finally:
        F.linear, torch.einsum = linear0, einsum0
        F.conv1d, F.conv2d, F.conv_transpose1d, F.conv_transpose2d = conv1d0, conv2d0, convt1d0, convt2d0
