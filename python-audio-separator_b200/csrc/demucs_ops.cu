// The two ends of the time-domain Demucs v3 forward (uvr_lib_v5/demucs/demucs.py:405-442), each one pass over the signal:
//   in:  mono statistics, (x - mean) / (1e-5 + std), the centred zero pad to valid_length, julius.resample_frac(x, 1, 2);
//   out: julius.resample_frac(x, 2, 1), x * std + mean, center_trim to the chunk length.
// julius's ResampleFrac(old, new) replicate-pads its input by (width, width + old) and runs a stride-`old` convolution with `new` phase
// filters of 2 * width + old taps, interleaving the phases.  The tap tables come from the host (b200/demucs_v3.py builds them in float64).
#include <algorithm>

#include "common.cuh"

namespace b200sep {
namespace {

constexpr int kStatBlocks = 128;  // partial sums per sample: the work layout of b200sep_meanstd_work_floats
constexpr int kThreads = 256;
constexpr int kUpTile = 2 * kThreads;  // input positions (x 2 phases) per CTA of the x2 filter
constexpr int kDownTile = kThreads;    // output samples per CTA of the /2 filter

// mix.mean(dim=1) (two channels) summed in double: kStatBlocks CTAs per sample leave (sum, sum of squares), one warp per sample adds them in a
// fixed order -> stats[b] = {mean, unbiased std}.  Deterministic: the partition depends on the length only.
__global__ void __launch_bounds__(kThreads) mono_stats_partial_kernel(const float* __restrict__ x, int64_t n, double2* __restrict__ part) {
  __shared__ double rs[kThreads / 32], rq[kThreads / 32];
  const float* x0 = x + (int64_t)blockIdx.y * 2 * n;
  const float* x1 = x0 + n;
  double s = 0.0, q = 0.0;
  for (int64_t i = (int64_t)blockIdx.x * kThreads + threadIdx.x; i < n; i += (int64_t)kStatBlocks * kThreads) {
    const double v = (double)((__ldg(&x0[i]) + __ldg(&x1[i])) * 0.5f);  // the float channel mean, as torch forms it
    s += v;
    q += v * v;
  }
  for (int o = 16; o > 0; o >>= 1) {
    s += __shfl_xor_sync(0xffffffffu, s, o);
    q += __shfl_xor_sync(0xffffffffu, q, o);
  }
  if ((threadIdx.x & 31) == 0) {
    rs[threadIdx.x >> 5] = s;
    rq[threadIdx.x >> 5] = q;
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    double S = 0.0, Q = 0.0;
    for (int w = 0; w < kThreads / 32; ++w) {
      S += rs[w];
      Q += rq[w];
    }
    part[(int64_t)blockIdx.y * kStatBlocks + blockIdx.x] = make_double2(S, Q);
  }
}

__global__ void mono_stats_final_kernel(const double2* __restrict__ part, int64_t n, float* __restrict__ stats) {
  const double2* ps = part + (int64_t)blockIdx.x * kStatBlocks;
  double s = 0.0, q = 0.0;
  for (int i = threadIdx.x; i < kStatBlocks; i += 32) {
    s += ps[i].x;
    q += ps[i].y;
  }
  for (int o = 16; o > 0; o >>= 1) {
    s += __shfl_xor_sync(0xffffffffu, s, o);
    q += __shfl_xor_sync(0xffffffffu, q, o);
  }
  if (threadIdx.x == 0) {
    const double mean = s / (double)n;
    const double var = (q - s * mean) / (double)(n - 1);
    stats[2 * blockIdx.x] = (float)mean;
    stats[2 * blockIdx.x + 1] = (float)sqrt(var > 0.0 ? var : 0.0);
  }
}

// y[2m + p] = sum_k taps[p][k] * z[clamp(m + k - width, 0, valid - 1)],  z = the normalised input at [pad_l, pad_l + n) of `valid` zeros.
// One CTA: kUpTile consecutive m of one (b, c) row, staged with their 2 * width halo.
__global__ void __launch_bounds__(kThreads) upsample2_kernel(const float* __restrict__ x, int64_t n, int64_t valid, int64_t pad_l,
                                                             const float* __restrict__ taps, int width, const float* __restrict__ stats,
                                                             float* __restrict__ y) {
  extern __shared__ __align__(16) float up_smem[];
  const int K = 2 * width + 1;
  float* tk = up_smem;            // 2 phases x K taps
  float* zs = up_smem + 2 * K;    // kUpTile + 2 * width samples
  const int row = blockIdx.y;     // b * 2 + c
  const float mean = stats[2 * (row >> 1)], den = 1e-5f + stats[2 * (row >> 1) + 1];
  const float* xr = x + (int64_t)row * n;
  const int64_t m0 = (int64_t)blockIdx.x * kUpTile;
  for (int i = threadIdx.x; i < 2 * K; i += kThreads) tk[i] = taps[i];
  for (int i = threadIdx.x; i < kUpTile + 2 * width; i += kThreads) {
    const int64_t j = min(max(m0 + i - width, (int64_t)0), valid - 1) - pad_l;
    zs[i] = (j >= 0 && j < n) ? (__ldg(&xr[j]) - mean) / den : 0.f;
  }
  __syncthreads();
  float2* yr = reinterpret_cast<float2*>(y + (int64_t)row * 2 * valid);
#pragma unroll
  for (int h = 0; h < kUpTile / kThreads; ++h) {
    const int t = threadIdx.x + h * kThreads;
    if (m0 + t >= valid) break;
    float a0 = 0.f, a1 = 0.f;
    for (int k = 0; k < K; ++k) {
      const float v = zs[t + k];
      a0 = fmaf(tk[k], v, a0);
      a1 = fmaf(tk[K + k], v, a1);
    }
    yr[m0 + t] = make_float2(a0, a1);
  }
}

// out[t] = (sum_k taps[k] * x[clamp(2 (t + trim) + k - width, 0, n2 - 1)]) * std + mean for t < n_out: one CTA per kDownTile outputs of a row.
__global__ void __launch_bounds__(kThreads) downsample2_kernel(const float* __restrict__ x, int64_t n2, int64_t trim, int64_t n_out,
                                                               const float* __restrict__ taps, int width, const float* __restrict__ stats,
                                                               int channels, float* __restrict__ y) {
  extern __shared__ __align__(16) float dn_smem[];
  const int K = 2 * width + 2;
  float* tk = dn_smem;
  float* xs = dn_smem + K;  // 2 * kDownTile + K samples
  const int row = blockIdx.y;  // b * channels + c
  const int b = row / channels;
  const float mean = stats[2 * b], sd = stats[2 * b + 1];
  const float* xr = x + (int64_t)row * n2;
  const int64_t t0 = (int64_t)blockIdx.x * kDownTile;
  const int64_t j0 = 2 * (t0 + trim) - width;
  for (int i = threadIdx.x; i < K; i += kThreads) tk[i] = taps[i];
  for (int i = threadIdx.x; i < 2 * kDownTile + K; i += kThreads) xs[i] = __ldg(&xr[min(max(j0 + i, (int64_t)0), n2 - 1)]);
  __syncthreads();
  const int t = threadIdx.x;
  if (t0 + t >= n_out) return;
  float acc = 0.f;
  for (int k = 0; k < K; ++k) acc = fmaf(tk[k], xs[2 * t + k], acc);
  y[(int64_t)row * n_out + t0 + t] = acc * sd + mean;
}

}  // namespace

extern "C" int b200sep_demucs_upsample2_f32(const float* x, int B, int64_t length, int64_t valid, const float* taps, int width, float* stats, float* y,
                                            float* work, void* stream) {
  B2_CHECK_ARG(x && taps && stats && y && work && B >= 1 && B <= 65535 && length >= 2 && valid >= length && width >= 1 && width <= 256,
               "demucs_upsample2_f32: bad argument");
  B2_CHECK_ARG((reinterpret_cast<uintptr_t>(work) & 15) == 0, "demucs_upsample2_f32: work must be 16-byte aligned");
  B2_CHECK_ARG((valid + kUpTile - 1) / kUpTile < (1ll << 31), "demucs_upsample2_f32: %lld samples is too long", (long long)valid);
  cudaStream_t s = (cudaStream_t)stream;
  mono_stats_partial_kernel<<<dim3(kStatBlocks, B), kThreads, 0, s>>>(x, length, reinterpret_cast<double2*>(work));
  B2_LAUNCHED();
  mono_stats_final_kernel<<<B, 32, 0, s>>>(reinterpret_cast<const double2*>(work), length, stats);
  B2_LAUNCHED();
  const size_t smem = (size_t)(2 * (2 * width + 1) + kUpTile + 2 * width) * sizeof(float);
  upsample2_kernel<<<dim3((unsigned)((valid + kUpTile - 1) / kUpTile), 2 * B), kThreads, smem, s>>>(x, length, valid, (valid - length) / 2, taps, width,
                                                                                                   stats, y);
  B2_LAUNCHED();
  return B200SEP_OK;
}

extern "C" int b200sep_demucs_downsample2_f32(const float* x, int B, int channels, int64_t valid, int64_t length, const float* taps, int width,
                                              const float* stats, float* y, void* stream) {
  B2_CHECK_ARG(x && taps && stats && y && B >= 1 && channels >= 1 && (int64_t)B * channels <= 65535 && length >= 1 && valid >= length && width >= 1 &&
                   width <= 256,
               "demucs_downsample2_f32: bad argument");
  const size_t smem = (size_t)((2 * width + 2) + 2 * kDownTile + (2 * width + 2)) * sizeof(float);
  downsample2_kernel<<<dim3((unsigned)((length + kDownTile - 1) / kDownTile), B * channels), kThreads, smem, (cudaStream_t)stream>>>(
      x, 2 * valid, (valid - length) / 2, length, taps, width, stats, channels, y);
  B2_LAUNCHED();
  return B200SEP_OK;
}

}  // namespace b200sep
