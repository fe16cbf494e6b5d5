// Operators of the VR (CascadedASPPNet) path that are not plain convolutions: depthwise dilated 3x3, bilinear x2 up-sampling
// (align_corners), the frequency-axis average pool of the ASPP module, a strided 4-D copy (crop / concat / broadcast), per-bin
// gains, magnitude of a complex spectrogram, the mask -> two complex spectrograms step of VRSeparator.inference_vr, and the
// polyphase FIR resampler (scipy.signal.resample_poly == librosa.resample(res_type="polyphase")).
#include <math.h>

#include "common.cuh"

namespace b200sep {

// depthwise 3x3, dilation d, padding d (SeperableConv2DBNActiv's first conv, vr_network/layers.py:60-70): y[b][c] = x[b][c] (*) w[c]
__global__ void dwconv3x3_kernel(const float* __restrict__ x, const float* __restrict__ w, float* __restrict__ y, int C, int H, int W, int dil, int64_t n) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const int wq = (int)(i % W);
    const int h = (int)((i / W) % H);
    const int64_t bc = i / ((int64_t)W * H);
    const int c = (int)(bc % C);
    const float* xp = x + bc * H * W;
    const float* wp = w + c * 9;
    float acc = 0.f;
#pragma unroll
    for (int kh = 0; kh < 3; ++kh) {
      const int hi = h + (kh - 1) * dil;
      if (hi < 0 || hi >= H) continue;
#pragma unroll
      for (int kw = 0; kw < 3; ++kw) {
        const int wi = wq + (kw - 1) * dil;
        if (wi < 0 || wi >= W) continue;
        acc = fmaf(__ldg(&xp[(int64_t)hi * W + wi]), __ldg(&wp[kh * 3 + kw]), acc);
      }
    }
    y[i] = acc;
  }
}

// F.interpolate(scale_factor=2, mode="bilinear", align_corners=True) (Decoder, layers.py:175): (B,C,H,W) -> channels [c_off, c_off+C) of
// a (B, c_total, 2H, 2W) tensor.  Source index = dst * (in-1)/(out-1) in float, as ATen's area_pixel_compute_source_index does.
__global__ void upsample2x_kernel(const float* __restrict__ x, float* __restrict__ y, int C, int H, int W, int c_total, int c_off, int64_t n) {
  const int Ho = 2 * H, Wo = 2 * W;
  const float sh = (Ho > 1) ? (float)(H - 1) / (float)(Ho - 1) : 0.f;
  const float sw = (Wo > 1) ? (float)(W - 1) / (float)(Wo - 1) : 0.f;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const int wo = (int)(i % Wo);
    const int ho = (int)((i / Wo) % Ho);
    const int64_t bc = i / ((int64_t)Wo * Ho);
    const int c = (int)(bc % C);
    const int64_t b = bc / C;
    const float fh = sh * ho, fw = sw * wo;
    const int h0 = (int)fh, w0 = (int)fw;
    const int h1 = min(h0 + 1, H - 1), w1 = min(w0 + 1, W - 1);
    const float lh = fh - h0, lw = fw - w0;
    const float* xp = x + bc * H * W;
    const float v00 = __ldg(&xp[(int64_t)h0 * W + w0]), v01 = __ldg(&xp[(int64_t)h0 * W + w1]);
    const float v10 = __ldg(&xp[(int64_t)h1 * W + w0]), v11 = __ldg(&xp[(int64_t)h1 * W + w1]);
    const float v = (1.f - lh) * ((1.f - lw) * v00 + lw * v01) + lh * ((1.f - lw) * v10 + lw * v11);
    y[((b * c_total + c_off + c) * Ho + ho) * Wo + wo] = v;
  }
}

// nn.AdaptiveAvgPool2d((1, None)) (ASPPModule.conv1, layers.py:232): mean over H.  (B*C, H, W) -> (B*C, W)
__global__ void mean_h_kernel(const float* __restrict__ x, float* __restrict__ y, int H, int W, int64_t n) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const int wq = (int)(i % W);
    const int64_t bc = i / W;
    const float* xp = x + bc * H * W + wq;
    float s = 0.f;
    for (int h = 0; h < H; ++h) s += __ldg(&xp[(int64_t)h * W]);
    y[i] = s / (float)H;
  }
}

struct Copy4 {
  int64_t ss[4], ds[4];
  int d[4];
};
__global__ void copy4_kernel(const float* __restrict__ src, float* __restrict__ dst, Copy4 p, int64_t n) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    int64_t r = i;
    const int i3 = (int)(r % p.d[3]); r /= p.d[3];
    const int i2 = (int)(r % p.d[2]); r /= p.d[2];
    const int i1 = (int)(r % p.d[1]); r /= p.d[1];
    const int i0 = (int)r;
    dst[i0 * p.ds[0] + i1 * p.ds[1] + i2 * p.ds[2] + i3 * p.ds[3]] = __ldg(&src[i0 * p.ss[0] + i1 * p.ss[1] + i2 * p.ss[2] + i3 * p.ss[3]]);
  }
}

// x[p][bin][t] *= gain[bin] for `planes` planes of (bins, frames)
__global__ void bin_gain_kernel(float* __restrict__ x, const float* __restrict__ gain, int bins, int frames, int64_t n) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const int b = (int)((i / frames) % bins);
    x[i] *= __ldg(&gain[b]);
  }
}

// planes (L re, L im, R re, R im) of (bins, frames) -> magnitudes (2, bins, frames_out) written at column t + pad_l (the rest is the
// caller's zero fill): spec_utils.preprocess + np.pad of inference_vr (vr_separator.py:345-349)
__global__ void cabs_pad_kernel(const float* __restrict__ spec, float* __restrict__ mag, int bins, int frames, int frames_out, int pad_l, int64_t n) {
  const int64_t plane = (int64_t)bins * frames;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const int t = (int)(i % frames);
    const int64_t cb = i / frames;  // c * bins + bin
    const int c = (int)(cb / bins);
    const int64_t o = (cb % bins) * frames + t;
    const float re = __ldg(&spec[(2 * c) * plane + o]), im = __ldg(&spec[(2 * c + 1) * plane + o]);
    mag[cb * frames_out + pad_l + t] = hypotf(re, im);
  }
}

// adjust_aggr + the two masked spectrograms (spec_utils.py:472-492, vr_separator.py:329-343):
//   m = mask ^ e(c, bin);  y = m * X;  v = (1 - m) * X   (X complex as 4 planes; mask (2, bins, mask_stride) read at column t)
__global__ void vr_mask_kernel(const float* __restrict__ mask, int mask_stride, const float* __restrict__ spec, int bins, int frames, int split_bin, float e_lo0,
                               float e_hi0, float e_lo1, float e_hi1, float* __restrict__ y, float* __restrict__ v, int64_t n) {
  const int64_t plane = (int64_t)bins * frames;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const int t = (int)(i % frames);
    const int64_t cb = i / frames;
    const int c = (int)(cb / bins), bin = (int)(cb % bins);
    float m = __ldg(&mask[cb * mask_stride + t]);
    const float e = (c == 0) ? (bin < split_bin ? e_lo0 : e_hi0) : (bin < split_bin ? e_lo1 : e_hi1);
    if (e != 1.f) m = powf(m, e);
    const int64_t o = (int64_t)bin * frames + t;
    const float re = __ldg(&spec[(2 * c) * plane + o]), im = __ldg(&spec[(2 * c + 1) * plane + o]);
    float yr = m * re, yi = m * im, vr = (1.f - m) * re, vi = (1.f - m) * im;
    // np.nan_to_num(nan=0, posinf=0, neginf=0) (vr_separator.py:187-188).  The reference forms mask * |X| * exp(i angle X): a non-finite
    // component makes |X| non-finite, so both components of that entry are non-finite there and both become 0.
    if (!isfinite(re) || !isfinite(im)) yr = yi = vr = vi = 0.f;
    if (!isfinite(yr)) yr = 0.f;
    if (!isfinite(yi)) yi = 0.f;
    if (!isfinite(vr)) vr = 0.f;
    if (!isfinite(vi)) vi = 0.f;
    y[(2 * c) * plane + o] = yr;
    y[(2 * c + 1) * plane + o] = yi;
    v[(2 * c) * plane + o] = vr;
    v[(2 * c + 1) * plane + o] = vi;
  }
}

// adjust_aggr alone (spec_utils.py:472-492), in place on the mask (2, bins, stride): needed when merge_artifacts runs between it and the products
__global__ void vr_mask_pow_kernel(float* __restrict__ mask, int stride, int bins, int frames, int split_bin, float e_lo0, float e_hi0, float e_lo1, float e_hi1, int64_t n) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const int t = (int)(i % frames);
    const int64_t cb = i / frames;
    const int c = (int)(cb / bins), bin = (int)(cb % bins);
    const float e = (c == 0) ? (bin < split_bin ? e_lo0 : e_hi0) : (bin < split_bin ? e_lo1 : e_hi1);
    if (e != 1.f) mask[cb * stride + t] = powf(mask[cb * stride + t], e);
  }
}

// y_mask.min(axis=(0, 1)) of merge_artifacts (spec_utils.py:187): smallest mask value of every frame
__global__ void vr_frame_min_kernel(const float* __restrict__ mask, int stride, int rows, int frames, float* __restrict__ out) {
  for (int t = blockIdx.x * blockDim.x + threadIdx.x; t < frames; t += gridDim.x * blockDim.x) {
    float m = INFINITY;
    for (int r = 0; r < rows; ++r) m = fminf(m, __ldg(&mask[(int64_t)r * stride + t]));
    out[t] = m;
  }
}

// y_mask += weight * (1 - y_mask) with a per-frame weight (merge_artifacts, spec_utils.py:213-214)
__global__ void vr_mask_merge_kernel(float* __restrict__ mask, const float* __restrict__ w, int stride, int frames, int64_t n) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const int t = (int)(i % frames);
    const int64_t r = i / frames;
    const float m = mask[r * stride + t];
    mask[r * stride + t] = m + __ldg(&w[t]) * (1.f - m);
  }
}

// spec_utils.mirroring("mirroring") (:458-463) written straight into the top band's un-cropped spectrogram: row i of the kept high end (bins
// max_bin-h .. max_bin-1 of the band) takes the magnitude of combined-spectrogram bin (pre_filter_start - 11 - i) with the input's phase, where that is smaller
__global__ void vr_mirror_kernel(const float* __restrict__ spec_m, int bins, const float* __restrict__ high, int high_rows, int high_frames, float* __restrict__ band,
                                 int band_bins, int frames, int h, int max_bin, int pre_filter_start, int64_t n) {
  const int64_t plane_m = (int64_t)bins * frames, plane_h = (int64_t)high_rows * high_frames, plane_b = (int64_t)band_bins * frames;
  for (int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; idx < n; idx += (int64_t)gridDim.x * blockDim.x) {
    const int t = (int)(idx % frames);
    const int i = (int)((idx / frames) % h);
    const int c = (int)(idx / ((int64_t)frames * h));
    const int bm = pre_filter_start - 11 - i;
    const float mr = __ldg(&spec_m[(2 * c) * plane_m + (int64_t)bm * frames + t]), mi = __ldg(&spec_m[(2 * c + 1) * plane_m + (int64_t)bm * frames + t]);
    const float hr = __ldg(&high[(2 * c) * plane_h + (int64_t)i * high_frames + t]), hi = __ldg(&high[(2 * c + 1) * plane_h + (int64_t)i * high_frames + t]);
    const float mag = hypotf(mr, mi), a = hypotf(hr, hi);
    float outr = hr, outi = hi;
    if (!(a <= mag)) {  // |input| > |mirror|: keep the input's phase, take the mirrored magnitude
      const float sc = mag / a;
      outr = hr * sc;
      outi = hi * sc;
    }
    const int64_t o = (int64_t)(max_bin - h + i) * frames + t;
    band[(2 * c) * plane_b + o] = outr;
    band[(2 * c + 1) * plane_b + o] = outi;
  }
}

// scipy.signal.resample_poly / upfirdn: y[k] = sum_i x[i] * h[(k + n_pre_remove) * down - i * up], h = the zero-padded, up-scaled
// Kaiser FIR the host builds (see vr.py).  x (C, n_in) -> y (C, n_out); double accumulation keeps the 1e-7 agreement with scipy.
__global__ void resample_poly_kernel(const float* __restrict__ x, const float* __restrict__ h, int n_taps, int up, int down, int64_t n_pre_remove, int64_t n_in,
                                     int64_t n_out, float* __restrict__ y) {
  const int c = blockIdx.y;
  const float* xc = x + (int64_t)c * n_in;
  for (int64_t k = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; k < n_out; k += (int64_t)gridDim.x * blockDim.x) {
    const int64_t m = (k + n_pre_remove) * down;
    // taps j = m - i*up in [0, n_taps)  ->  i in [ceil((m - n_taps + 1)/up), floor(m/up)]
    int64_t i_hi = m / up;
    int64_t i_lo = (m - n_taps + 1 <= 0) ? 0 : (m - n_taps + 1 + up - 1) / up;
    if (i_hi > n_in - 1) i_hi = n_in - 1;
    double acc = 0.0;
    for (int64_t i = i_lo; i <= i_hi; ++i) acc += (double)__ldg(&xc[i]) * (double)__ldg(&h[m - i * up]);
    y[(int64_t)c * n_out + k] = (float)acc;
  }
}

// One CTA per (batch element, direction): 4*hid threads, thread j owns gate row j of W_hh (kept in shared memory, transposed so the inner
// product reads are conflict-free); h_{t-1} and the four gate pre-activations are exchanged through shared memory, two barriers per step.
__global__ void lstm_bidir_kernel(const float* __restrict__ xp, const float* __restrict__ whh, float* __restrict__ out, int T, int N, int hid) {
  extern __shared__ float lsm[];
  float* wT = lsm;                     // [hid][4*hid]: wT[k][j] = W_hh[j][k]
  float* hbuf = wT + 4 * hid * hid;    // [hid]
  float* gates = hbuf + hid;           // [4*hid]
  const int n = blockIdx.x, dir = blockIdx.y, j = threadIdx.x, G = 4 * hid;
  const float* w = whh + (int64_t)dir * G * hid;
  for (int i = j; i < G * hid; i += G) {
    const int row = i / hid, k = i - row * hid;
    wT[k * G + row] = w[i];
  }
  if (j < hid) hbuf[j] = 0.f;
  float c = 0.f;
  __syncthreads();
  const float* xpd = xp + (int64_t)dir * T * N * G;
  for (int s = 0; s < T; ++s) {
    const int t = dir ? T - 1 - s : s;
    float g = __ldg(&xpd[((int64_t)t * N + n) * G + j]);
    for (int k = 0; k < hid; ++k) g = fmaf(wT[k * G + j], hbuf[k], g);
    gates[j] = g;
    __syncthreads();
    if (j < hid) {
      const float ig = 1.f / (1.f + expf(-gates[j])), fg = 1.f / (1.f + expf(-gates[hid + j]));
      const float gg = tanhf(gates[2 * hid + j]), og = 1.f / (1.f + expf(-gates[3 * hid + j]));
      c = fg * c + ig * gg;
      const float h = og * tanhf(c);
      hbuf[j] = h;
      out[((int64_t)t * N + n) * (2 * hid) + dir * hid + j] = h;
    }
    __syncthreads();
  }
}

static inline int ew_grid(int64_t n) { return (int)std::min<int64_t>(cdiv(n, 256), kNumSMs * 16); }

}  // namespace b200sep

using namespace b200sep;

extern "C" int b200sep_dwconv3x3_f32(const float* x, const float* w, float* y, int B, int C, int H, int W, int dilation, void* stream) {
  B2_CHECK_ARG(x && w && y && B >= 1 && C >= 1 && H >= 1 && W >= 1 && dilation >= 1, "dwconv3x3_f32: bad argument");
  const int64_t n = (int64_t)B * C * H * W;
  dwconv3x3_kernel<<<ew_grid(n), 256, 0, (cudaStream_t)stream>>>(x, w, y, C, H, W, dilation, n);
  B2_LAUNCHED();
  return B200SEP_OK;
}

extern "C" int b200sep_upsample2x_bilinear_f32(const float* x, float* y, int B, int C, int H, int W, int dst_c_total, int dst_c_off, void* stream) {
  B2_CHECK_ARG(x && y && B >= 1 && C >= 1 && H >= 1 && W >= 1 && dst_c_off >= 0 && dst_c_off + C <= dst_c_total, "upsample2x_bilinear_f32: bad argument");
  const int64_t n = (int64_t)B * C * 4 * H * W;
  upsample2x_kernel<<<ew_grid(n), 256, 0, (cudaStream_t)stream>>>(x, y, C, H, W, dst_c_total, dst_c_off, n);
  B2_LAUNCHED();
  return B200SEP_OK;
}

extern "C" int b200sep_mean_h_f32(const float* x, float* y, int BC, int H, int W, void* stream) {
  B2_CHECK_ARG(x && y && BC >= 1 && H >= 1 && W >= 1, "mean_h_f32: bad argument");
  const int64_t n = (int64_t)BC * W;
  mean_h_kernel<<<ew_grid(n), 256, 0, (cudaStream_t)stream>>>(x, y, H, W, n);
  B2_LAUNCHED();
  return B200SEP_OK;
}

extern "C" int b200sep_copy4_f32(const float* src, float* dst, int d0, int d1, int d2, int d3, int64_t ss0, int64_t ss1, int64_t ss2, int64_t ss3, int64_t ds0,
                                 int64_t ds1, int64_t ds2, int64_t ds3, void* stream) {
  B2_CHECK_ARG(src && dst && d0 >= 0 && d1 >= 0 && d2 >= 0 && d3 >= 0, "copy4_f32: bad argument");
  const int64_t n = (int64_t)d0 * d1 * d2 * d3;
  if (n == 0) return B200SEP_OK;
  Copy4 p;
  p.d[0] = d0; p.d[1] = d1; p.d[2] = d2; p.d[3] = d3;
  p.ss[0] = ss0; p.ss[1] = ss1; p.ss[2] = ss2; p.ss[3] = ss3;
  p.ds[0] = ds0; p.ds[1] = ds1; p.ds[2] = ds2; p.ds[3] = ds3;
  copy4_kernel<<<ew_grid(n), 256, 0, (cudaStream_t)stream>>>(src, dst, p, n);
  B2_LAUNCHED();
  return B200SEP_OK;
}

extern "C" int b200sep_bin_gain_f32(float* x, const float* gain, int planes, int bins, int frames, void* stream) {
  B2_CHECK_ARG(x && gain && planes >= 1 && bins >= 1 && frames >= 1, "bin_gain_f32: bad argument");
  const int64_t n = (int64_t)planes * bins * frames;
  bin_gain_kernel<<<ew_grid(n), 256, 0, (cudaStream_t)stream>>>(x, gain, bins, frames, n);
  B2_LAUNCHED();
  return B200SEP_OK;
}

extern "C" int b200sep_vr_magnitude_pad(const float* spec, float* mag, int bins, int frames, int frames_out, int pad_l, void* stream) {
  B2_CHECK_ARG(spec && mag && bins >= 1 && frames >= 1 && pad_l >= 0 && pad_l + frames <= frames_out, "vr_magnitude_pad: bad argument");
  const int64_t n = (int64_t)2 * bins * frames;
  cabs_pad_kernel<<<ew_grid(n), 256, 0, (cudaStream_t)stream>>>(spec, mag, bins, frames, frames_out, pad_l, n);
  B2_LAUNCHED();
  return B200SEP_OK;
}

extern "C" int b200sep_vr_apply_mask(const float* mask, int mask_stride, const float* spec, int bins, int frames, int split_bin, float exp_low_left, float exp_high_left,
                                     float exp_low_right, float exp_high_right, float* y_spec, float* v_spec, void* stream) {
  B2_CHECK_ARG(mask && spec && y_spec && v_spec && bins >= 1 && frames >= 1 && mask_stride >= frames && split_bin >= 0, "vr_apply_mask: bad argument");
  const int64_t n = (int64_t)2 * bins * frames;
  vr_mask_kernel<<<ew_grid(n), 256, 0, (cudaStream_t)stream>>>(mask, mask_stride, spec, bins, frames, split_bin, exp_low_left, exp_high_left, exp_low_right,
                                                             exp_high_right, y_spec, v_spec, n);
  B2_LAUNCHED();
  return B200SEP_OK;
}

extern "C" int b200sep_resample_poly_f32(const float* x, const float* taps, int n_taps, int up, int down, int64_t n_pre_remove, int channels, int64_t n_in,
                                         int64_t n_out, float* y, void* stream) {
  B2_CHECK_ARG(x && taps && y && n_taps >= 1 && up >= 1 && down >= 1 && n_pre_remove >= 0 && channels >= 1 && n_in >= 1 && n_out >= 1,
               "resample_poly_f32: bad argument");
  dim3 grid((unsigned)std::min<int64_t>(cdiv(n_out, 256), kNumSMs * 8), channels);
  resample_poly_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(x, taps, n_taps, up, down, n_pre_remove, n_in, n_out, y);
  B2_LAUNCHED();
  return B200SEP_OK;
}

extern "C" int b200sep_lstm_bidir_f32(const float* x_proj, const float* w_hh, float* out, int T, int N, int hid, void* stream) {
  B2_CHECK_ARG(x_proj && w_hh && out && T >= 1 && N >= 1 && hid >= 1 && hid <= 96, "lstm_bidir_f32: bad argument (hid must be <= 96)");
  const int smem = (4 * hid * hid + 5 * hid) * (int)sizeof(float);
  static int attr[kMaxDevices] = {};  // the largest limit set so far, per device
  B2_DEVICE_SLOT(dev);
  if (smem > attr[dev]) {
    B2_CUDA(cudaFuncSetAttribute(lstm_bidir_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    attr[dev] = smem;
  }
  lstm_bidir_kernel<<<dim3(N, 2), 4 * hid, smem, (cudaStream_t)stream>>>(x_proj, w_hh, out, T, N, hid);
  B2_LAUNCHED();
  return B200SEP_OK;
}

extern "C" int b200sep_vr_mask_pow(float* mask, int mask_stride, int bins, int frames, int split_bin, float exp_low_left, float exp_high_left, float exp_low_right,
                                   float exp_high_right, void* stream) {
  B2_CHECK_ARG(mask && bins >= 1 && frames >= 1 && mask_stride >= frames && split_bin >= 0, "vr_mask_pow: bad argument");
  const int64_t n = (int64_t)2 * bins * frames;
  vr_mask_pow_kernel<<<ew_grid(n), 256, 0, (cudaStream_t)stream>>>(mask, mask_stride, bins, frames, split_bin, exp_low_left, exp_high_left, exp_low_right, exp_high_right, n);
  B2_LAUNCHED();
  return B200SEP_OK;
}

extern "C" int b200sep_vr_frame_min(const float* mask, int mask_stride, int rows, int frames, float* out, void* stream) {
  B2_CHECK_ARG(mask && out && rows >= 1 && frames >= 1 && mask_stride >= frames, "vr_frame_min: bad argument");
  vr_frame_min_kernel<<<cdiv(frames, 128), 128, 0, (cudaStream_t)stream>>>(mask, mask_stride, rows, frames, out);
  B2_LAUNCHED();
  return B200SEP_OK;
}

extern "C" int b200sep_vr_mask_merge(float* mask, const float* frame_weight, int mask_stride, int rows, int frames, void* stream) {
  B2_CHECK_ARG(mask && frame_weight && rows >= 1 && frames >= 1 && mask_stride >= frames, "vr_mask_merge: bad argument");
  const int64_t n = (int64_t)rows * frames;
  vr_mask_merge_kernel<<<ew_grid(n), 256, 0, (cudaStream_t)stream>>>(mask, frame_weight, mask_stride, frames, n);
  B2_LAUNCHED();
  return B200SEP_OK;
}

extern "C" int b200sep_vr_mirror_high_end(const float* spec_m, int bins, const float* high_end, int high_rows, int high_frames, float* band_spec, int band_bins, int frames,
                                          int h, int max_bin, int pre_filter_start, void* stream) {
  B2_CHECK_ARG(spec_m && high_end && band_spec && bins >= 1 && frames >= 1 && h >= 1 && h <= high_rows && frames <= high_frames && max_bin <= band_bins && max_bin - h >= 0,
               "vr_mirror_high_end: bad argument");
  B2_CHECK_ARG(pre_filter_start - 10 - h >= 0 && pre_filter_start - 11 < bins, "vr_mirror_high_end: the mirrored bins [%d, %d) fall outside the combined spectrogram",
               pre_filter_start - 10 - h, pre_filter_start - 10);
  const int64_t n = (int64_t)2 * h * frames;
  vr_mirror_kernel<<<ew_grid(n), 256, 0, (cudaStream_t)stream>>>(spec_m, bins, high_end, high_rows, high_frames, band_spec, band_bins, frames, h, max_bin, pre_filter_start, n);
  B2_LAUNCHED();
  return B200SEP_OK;
}
