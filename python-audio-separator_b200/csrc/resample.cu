// Band-limited resampling at any ratio: the windowed-sinc interpolator behind librosa.resample's soxr / libsamplerate / resampy
// res_types (the filter sets are chosen by b200/resample.py).
//   y[c][n] = g * sum_k x[c][k] * h(g * |n*step - k|),  step = 1 / ratio,  g = min(1, ratio)
// h is a table of per_zero points per zero crossing over [0, n_zeros], linearly interpolated.
//
// Persistent CTAs: each loads the table into shared memory once, then walks tiles of blockDim outputs of one channel.  A tile stages
// the input span its outputs touch (zero outside [0, n_in)).  One thread computes one output: the left wing k = floor(t), floor(t)-1, ...
// and the right wing k = floor(t)+1, ...  The output's position t = n*step is computed in double from n, never accumulated; along a
// wing the table coordinate u = g*per_zero*|t - k| advances by a constant, carried as 32.32 fixed point so it stays exact over the
// 2*16*n_zeros taps of the lowest ratio (a float32 coordinate near 32768 would be off by 1/256 of a table step).
#include <math.h>

#include <algorithm>

#include "common.cuh"

namespace b200sep {

namespace {

constexpr int kSmemLimit = 227 * 1024;  // H100 opt-in dynamic shared memory per block

// frac in [0, 1) from the low word of a 32.32 coordinate (23 mantissa bits; avoids the integer->float conversion pipe)
__device__ __forceinline__ float frac_of(uint32_t lo) { return __uint_as_float(0x3f800000u | (lo >> 9)) - 1.0f; }

__device__ __forceinline__ float wing(const float* __restrict__ tab, const float* __restrict__ xs, int64_t k, int dk, uint64_t u, uint64_t du,
                                      uint64_t u_end) {
  float acc = 0.f;
  for (; u < u_end; u += du, k += dk) {
    const int i = (int)(u >> 32);
    const float t0 = tab[i];
    const float h = fmaf(frac_of((uint32_t)u), tab[i + 1] - t0, t0);
    acc = fmaf(xs[k], h, acc);
  }
  return acc;
}

__global__ void __launch_bounds__(1024) resample_sinc_kernel(const float* __restrict__ x, int64_t n_in, const float* __restrict__ table, int n_tab,
                                                             double step, double g, double half_width, double scale, int64_t n_out, int n_tiles,
                                                             int channels, int span_max, float* __restrict__ y) {
  extern __shared__ __align__(16) float rs_smem[];
  float* tab = rs_smem;                    // n_tab + 1 entries
  float* xs = rs_smem + ((n_tab + 4) & ~3);  // span_max entries
  for (int i = threadIdx.x; i <= n_tab; i += blockDim.x) tab[i] = table[i];
  const uint64_t u_end = (uint64_t)n_tab << 32;
  const uint64_t du = (uint64_t)llrint(scale * 4294967296.0);
  for (int tile = blockIdx.x; tile < n_tiles * channels; tile += gridDim.x) {
    const int c = tile / n_tiles;
    const int64_t n0 = (int64_t)(tile % n_tiles) * blockDim.x;
    const int64_t n1 = min(n0 + (int64_t)blockDim.x, n_out) - 1;
    const int64_t k_lo = (int64_t)floor((double)n0 * step - half_width) - 1;
    const int64_t k_hi = (int64_t)floor((double)n1 * step + half_width) + 2;
    const int span = (int)min(k_hi - k_lo + 1, (int64_t)span_max);
    const float* xc = x + (int64_t)c * n_in;
    __syncthreads();  // the previous tile's readers are done with xs (and the table load is done on the first pass)
    for (int i = threadIdx.x; i < span; i += blockDim.x) {
      const int64_t k = k_lo + i;
      xs[i] = (k >= 0 && k < n_in) ? __ldg(&xc[k]) : 0.f;
    }
    __syncthreads();
    const int64_t n = n0 + threadIdx.x;
    if (n > n1) continue;
    const double t = (double)n * step;
    const double kf = floor(t);
    const double f = t - kf;
    const int64_t k0 = (int64_t)kf - k_lo;  // floor(t) as an index into xs
    const uint64_t ul = (uint64_t)llrint(scale * f * 4294967296.0);
    const uint64_t ur = (uint64_t)llrint(scale * (1.0 - f) * 4294967296.0);
    const float acc = wing(tab, xs, k0, -1, ul, du, u_end) + wing(tab, xs, k0 + 1, 1, ur, du, u_end);
    y[(int64_t)c * n_out + n] = (float)g * acc;
  }
}

}  // namespace

extern "C" int b200sep_resample_sinc_f32(const float* x, int channels, int64_t n_in, const float* table, int n_zeros, int per_zero, double ratio,
                                         int64_t n_out, float* y, void* stream) {
  B2_CHECK_ARG(x && table && y && channels >= 1 && n_in >= 1 && n_out >= 1 && n_zeros >= 1 && per_zero >= 1, "resample_sinc_f32: bad argument");
  B2_CHECK_ARG(ratio >= 1.0 / 16.0 && ratio <= 16.0, "resample_sinc_f32: ratio %.9g is outside [1/16, 16]", ratio);
  const int64_t n_tab = (int64_t)n_zeros * per_zero;
  const double step = 1.0 / ratio, g = std::min(1.0, ratio);
  const double half_width = n_zeros / g;  // input samples on each side of t that the filter reaches
  const int64_t tab_floats = (n_tab + 4) & ~3;
  int threads = 1024;
  int64_t span_max = 0, smem = 0;
  for (; threads >= 128; threads /= 2) {
    span_max = (int64_t)ceil((threads - 1) * step + 2.0 * half_width) + 8;
    smem = (tab_floats + span_max) * (int64_t)sizeof(float);
    if (smem <= kSmemLimit) break;
  }
  B2_CHECK_ARG(threads >= 128, "resample_sinc_f32: a table of %lld entries does not fit in shared memory", (long long)(n_tab + 1));
  const int64_t n_tiles = (n_out + threads - 1) / threads;
  B2_CHECK_ARG(n_tiles * channels < (1ll << 31), "resample_sinc_f32: %lld outputs per channel is too many", (long long)n_out);
  B2_CUDA(cudaFuncSetAttribute(resample_sinc_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  int per_sm = 0;
  B2_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, resample_sinc_kernel, threads, (size_t)smem));
  const int64_t grid = std::min<int64_t>(n_tiles * channels, (int64_t)kNumSMs * std::max(per_sm, 1));
  resample_sinc_kernel<<<(unsigned)grid, threads, smem, (cudaStream_t)stream>>>(x, n_in, table, (int)n_tab, step, g, half_width, g * per_zero, n_out,
                                                                               (int)n_tiles, channels, (int)span_max, y);
  B2_LAUNCHED();
  return B200SEP_OK;
}

}  // namespace b200sep
