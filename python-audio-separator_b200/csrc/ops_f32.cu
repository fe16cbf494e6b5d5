// fp32 operators for the HTDemucs path (hdemucs.py / demucs.py / transformer.py of the reference): GroupNorm(1,C),
// GLU (+LayerScale residual), LayerNorm, batched TN GEMM with bias / activation / scaled residual, row softmax,
// small element-wise helpers, whole-tensor mean/std, and the triangle-window segment overlap-add of apply_model.
#include <math.h>

#include "common.cuh"
#include "tc_f32.cuh"

namespace b200sep {

__device__ __forceinline__ float f32_act(float v, int act) {
  if (act == 1) return fmaxf(v, 0.f);
  if (act == 2) return 0.5f * v * (1.f + erff(v * 0.70710678118654752440f));
  if (act == 3) return v > 0.f ? v : 0.01f * v;
  if (act == 4) return 1.f / (1.f + expf(-v));
  if (act == 5) return tanhf(v);
  return v;
}

__device__ __forceinline__ float2 block_sum2(float a, float b, float* red) {
  for (int o = 16; o > 0; o >>= 1) {
    a += __shfl_xor_sync(0xffffffffu, a, o);
    b += __shfl_xor_sync(0xffffffffu, b, o);
  }
  const int w = threadIdx.x >> 5, l = threadIdx.x & 31, nw = blockDim.x >> 5;
  __syncthreads();
  if (l == 0) {
    red[w] = a;
    red[32 + w] = b;
  }
  __syncthreads();
  float ta = (threadIdx.x < nw) ? red[threadIdx.x] : 0.f, tb = (threadIdx.x < nw) ? red[32 + threadIdx.x] : 0.f;
  if (w == 0) {
    for (int o = 16; o > 0; o >>= 1) {
      ta += __shfl_xor_sync(0xffffffffu, ta, o);
      tb += __shfl_xor_sync(0xffffffffu, tb, o);
    }
    if (l == 0) {
      red[0] = ta;
      red[32] = tb;
    }
  }
  __syncthreads();
  return make_float2(red[0], red[32]);
}

// GroupNorm(num_groups=1, C) over one sample of n = C*L elements, affine per channel, optional activation (hdemucs.py:79-80 norm_fn,
// demucs.py:139-141; eps 1e-5, biased variance).  Two kernels so that a single huge sample (the time branch: 96 x 85995) still fills
// the GPU: (1) `nblk` CTAs per sample reduce shifted sums  sum(x - x0), sum((x - x0)^2)  (x0 = the sample's first element) into double
// partials; (2) every CTA re-reduces the partials of its sample in a fixed order (deterministic) and normalises its slice.
// Every thread accumulates in double: the shift removes the E[x^2] - mean^2 cancellation only when x0 is typical, and with an outlier
// x0 (30 sigma) fp32 per-thread sums of ~256 squares already cost 4e-6 of rstd.  The mean is applied as a float hi + lo pair, so a
// large mean (1e3 at std 1) is not rounded to fp32 before the subtraction.
// Layouts: channel-first (B, C, Fr, L) where sample (b, fr) owns x[((b*C + c)*Fr + fr)*L + l]  (Fr = 1: plain (B, C, L); Fr > 1: DConv
// applied per frequency row of a (B, C, Fr, T) tensor without the permute of hdemucs.py:141-146), or channel-last (samples, L, C)
// (MyGroupNorm on (B, T, C) tokens, transformer.py:184-193).
struct GnGeom {
  int C, Fr, channel_last;
  uint32_t L, n, chunk;
  int groups;  // > 1: nn.GroupNorm(groups, C_total) on channel-first data: sample = b * groups + g owns C consecutive channels, affine index g * C + c
};
__device__ __forceinline__ int64_t gn_index(const GnGeom& g, int sample, uint32_t i) {
  if (g.channel_last || g.Fr == 1) return (int64_t)sample * g.n + i;
  const uint32_t c = i / g.L, l = i - c * g.L;
  const int b = sample / g.Fr, fr = sample - b * g.Fr;
  return (((int64_t)b * g.C + c) * g.Fr + fr) * g.L + l;
}

__global__ void __launch_bounds__(256) gn_partial_kernel(const float* __restrict__ x, GnGeom g, double2* __restrict__ part) {
  __shared__ double rs[8], rq[8];
  const int sample = blockIdx.y;
  const float x0 = __ldg(&x[gn_index(g, sample, 0)]);
  const uint32_t lo = blockIdx.x * g.chunk, hi = min(g.n, lo + g.chunk);
  double ds = 0.0, dq = 0.0;
  for (uint32_t i = lo + threadIdx.x; i < hi; i += 256) {
    const double d = (double)__ldg(&x[gn_index(g, sample, i)]) - (double)x0;
    ds += d;
    dq = fma(d, d, dq);
  }
  for (int o = 16; o > 0; o >>= 1) {
    ds += __shfl_xor_sync(0xffffffffu, ds, o);
    dq += __shfl_xor_sync(0xffffffffu, dq, o);
  }
  if ((threadIdx.x & 31) == 0) {
    rs[threadIdx.x >> 5] = ds;
    rq[threadIdx.x >> 5] = dq;
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    double S = 0.0, Q = 0.0;
    for (int w = 0; w < 8; ++w) {
      S += rs[w];
      Q += rq[w];
    }
    double2* ps = part + (int64_t)sample * (gridDim.x + 1);
    ps[blockIdx.x] = make_double2(S, Q);
    if (blockIdx.x == 0) ps[gridDim.x] = make_double2((double)x0, 0.0);  // the apply pass may run in place: it must not re-read x0 from x
  }
}

__global__ void __launch_bounds__(256) gn_apply_kernel(const float* __restrict__ x, const float* __restrict__ gamma, const float* __restrict__ beta,
                                                      float* __restrict__ y, GnGeom g, const double2* __restrict__ part, int act) {
  __shared__ float stat[3];
  const int sample = blockIdx.y;
  if (threadIdx.x == 0) {
    double S = 0.0, Q = 0.0;
    const double2* ps = part + (int64_t)sample * (gridDim.x + 1);
    for (unsigned k = 0; k < gridDim.x; ++k) {
      S += ps[k].x;
      Q += ps[k].y;
    }
    const double md = S / (double)g.n;  // mean of (x - x0)
    double var = Q / (double)g.n - md * md;
    if (var < 0.0) var = 0.0;
    const double mean = ps[gridDim.x].x + md;
    stat[0] = (float)mean;
    stat[1] = (float)(mean - (double)stat[0]);
    stat[2] = (float)(1.0 / sqrt(var + 1e-5));
  }
  __syncthreads();
  const float mean_hi = stat[0], mean_lo = stat[1], rstd = stat[2];
  const uint32_t lo = blockIdx.x * g.chunk, hi = min(g.n, lo + g.chunk);
  for (uint32_t i = lo + threadIdx.x; i < hi; i += 256) {
    const int c = (g.channel_last ? (int)(i % (uint32_t)g.C) : (int)(i / g.L)) + (sample % g.groups) * g.C;
    const int64_t o = gn_index(g, sample, i);
    y[o] = f32_act(((x[o] - mean_hi) - mean_lo) * rstd * __ldg(&gamma[c]) + __ldg(&beta[c]), act);
  }
}

// CTAs per sample: a function of the sample size ONLY.  (It used to shrink with the number of samples in the launch; the partition of the partial sums then
// depended on the batch size of a forward, and a time-sharded run -- whose ranks batch their segments differently -- differed from the single-GPU run in the
// last bits: 4e-6 after de-normalisation in tests/test_sharded_gpu.py.)
static int gn_blocks_per_sample(int /*samples*/, int64_t n) {
  return (int)std::min<int64_t>(std::max<int64_t>(1, n / 65536), 1024);
}

// out[perm(i)] = in[i] for a 4-D tensor: out dims = in dims permuted by (p0,p1,p2,p3) ("b c fr t -> b t fr c" etc., transformer.py:532,555)
__global__ void permute4_kernel(const float* __restrict__ x, float* __restrict__ y, int d0, int d1, int d2, int d3, int p0, int p1, int p2, int p3, int64_t n) {
  const int din[4] = {d0, d1, d2, d3};
  const int perm[4] = {p0, p1, p2, p3};
  const int64_t sin_[4] = {(int64_t)d1 * d2 * d3, (int64_t)d2 * d3, d3, 1};
  for (int64_t o = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; o < n; o += (int64_t)gridDim.x * blockDim.x) {
    int64_t r = o, src = 0;
    for (int k = 3; k >= 0; --k) {
      const int dk = din[perm[k]];
      src += (r % dk) * sin_[perm[k]];
      r /= dk;
    }
    y[o] = x[src];
  }
}

// y[b][c][l] = (res ? res + scale[c] * g : g),  g = a[b][c][l] * sigmoid(a[b][C + c][l])   (F.glu(dim=1); LayerScale, demucs.py:92-93)
__global__ void glu_kernel(const float* __restrict__ a, const float* __restrict__ res, const float* __restrict__ scale, float* __restrict__ y, int C, int64_t L,
                           int64_t n) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t l = i % L;
    const int64_t bc = i / L;
    const int c = (int)(bc % C);
    const int64_t b = bc / C;
    const float u = a[((b * 2 * C) + c) * L + l], v = a[((b * 2 * C) + C + c) * L + l];
    float g = u / (1.f + expf(-v));
    if (res) g = res[i] + __ldg(&scale[c]) * g;
    y[i] = g;
  }
}

// LayerNorm over the last dimension C of (rows, C); one warp per row.  eps 1e-5.  The sums are taken in double and the mean is applied as a
// float hi + lo pair, as in GroupNorm above: with a row mean of 100 at std 1, fp32 sums of the raw values and an fp32-rounded mean cost 2e-5.
__global__ void layernorm_kernel(const float* __restrict__ x, const float* __restrict__ gamma, const float* __restrict__ beta, float* __restrict__ y, int64_t rows,
                                 int C) {
  const int64_t row = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (row >= rows) return;
  const int lane = threadIdx.x & 31;
  const float* xr = x + row * C;
  double s = 0.0;
  for (int c = lane; c < C; c += 32) s += (double)xr[c];
  for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  const double mean = s / C;
  double q = 0.0;
  for (int c = lane; c < C; c += 32) {
    const double d = (double)xr[c] - mean;
    q = fma(d, d, q);
  }
  for (int o = 16; o > 0; o >>= 1) q += __shfl_xor_sync(0xffffffffu, q, o);
  const float mean_hi = (float)mean, mean_lo = (float)(mean - (double)mean_hi);
  const float rstd = (float)(1.0 / sqrt(q / C + 1e-5));
  float* yr = y + row * C;
  for (int c = lane; c < C; c += 32) yr[c] = ((xr[c] - mean_hi) - mean_lo) * rstd * __ldg(&gamma[c]) + __ldg(&beta[c]);
}

// Batched SGEMM TN: C[z][m][n] = epi( sum_k A[z][m][k] * Bw[z][n][k] ), 128x128x16 tiles, 8x8 per thread.
// epi: v = acc * alpha + (bias_n ? bias[n] : 0) + (bias_m ? bias_row[m] : 0); v = act(v); if res: v = res + (rs ? rs[n] : 1) * v
struct GemmF32 {
  const float* A;
  const float* Bw;
  float* C;
  const float* bias_n;
  const float* bias_m;
  const float* res;
  const float* res_scale;
  int M, N, K, lda, ldb, ldc;
  int64_t sA, sB, sC;  // batch strides (elements)
  float alpha;
  int act;
  int b_kn;  // B given as (K, N) row-major instead of (N, K)
};
constexpr int FBM = 128, FBN = 128, FBK = 16;
__global__ void __launch_bounds__(256) gemm_f32_kernel(GemmF32 p) {
  __shared__ __align__(16) float As[FBK][FBM + 4];
  __shared__ __align__(16) float Bs[FBK][FBN + 4];
  const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4;
  const int m0 = blockIdx.y * FBM, n0 = blockIdx.x * FBN;
  const float* A = p.A + (int64_t)blockIdx.z * p.sA;
  const float* Bw = p.Bw + (int64_t)blockIdx.z * p.sB;
  float* C = p.C + (int64_t)blockIdx.z * p.sC;
  const float* res = p.res ? p.res + (int64_t)blockIdx.z * p.sC : nullptr;
  const bool vec = !p.b_kn && ((p.lda | p.ldb) & 3) == 0 && ((reinterpret_cast<uintptr_t>(A) | reinterpret_cast<uintptr_t>(Bw)) & 15) == 0;
  float acc[8][8];
#pragma unroll
  for (int i = 0; i < 8; ++i)
#pragma unroll
    for (int j = 0; j < 8; ++j) acc[i][j] = 0.f;
  for (int k0 = 0; k0 < p.K; k0 += FBK) {
#pragma unroll
    for (int it = 0; it < 2; ++it) {
      const int idx = tid + it * 256;
      const int row = idx >> 2, kq = idx & 3, k = k0 + kq * 4;
      float av[4] = {0.f, 0.f, 0.f, 0.f}, bv[4] = {0.f, 0.f, 0.f, 0.f};
      if (vec && k + 3 < p.K) {
        if (m0 + row < p.M) {
          const float4 t = __ldg(reinterpret_cast<const float4*>(&A[(int64_t)(m0 + row) * p.lda + k]));
          av[0] = t.x; av[1] = t.y; av[2] = t.z; av[3] = t.w;
        }
        if (n0 + row < p.N) {
          const float4 t = __ldg(reinterpret_cast<const float4*>(&Bw[(int64_t)(n0 + row) * p.ldb + k]));
          bv[0] = t.x; bv[1] = t.y; bv[2] = t.z; bv[3] = t.w;
        }
      } else {
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          if (m0 + row < p.M && k + e < p.K) av[e] = __ldg(&A[(int64_t)(m0 + row) * p.lda + k + e]);
          if (n0 + row < p.N && k + e < p.K) bv[e] = __ldg(p.b_kn ? &Bw[(int64_t)(k + e) * p.ldb + n0 + row] : &Bw[(int64_t)(n0 + row) * p.ldb + k + e]);
        }
      }
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        As[kq * 4 + e][row] = av[e];
        Bs[kq * 4 + e][row] = bv[e];
      }
    }
    __syncthreads();
#pragma unroll
    for (int k = 0; k < FBK; ++k) {
      const float4 a0 = *reinterpret_cast<const float4*>(&As[k][ty * 8]);
      const float4 a1 = *reinterpret_cast<const float4*>(&As[k][ty * 8 + 4]);
      const float4 b0 = *reinterpret_cast<const float4*>(&Bs[k][tx * 8]);
      const float4 b1 = *reinterpret_cast<const float4*>(&Bs[k][tx * 8 + 4]);
      const float av[8] = {a0.x, a0.y, a0.z, a0.w, a1.x, a1.y, a1.z, a1.w};
      const float bv[8] = {b0.x, b0.y, b0.z, b0.w, b1.x, b1.y, b1.z, b1.w};
#pragma unroll
      for (int i = 0; i < 8; ++i)
#pragma unroll
        for (int j = 0; j < 8; ++j) acc[i][j] = fmaf(av[i], bv[j], acc[i][j]);
    }
    __syncthreads();
  }
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const int m = m0 + ty * 8 + i;
    if (m >= p.M) continue;
    const float bm = p.bias_m ? __ldg(&p.bias_m[m]) : 0.f;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const int n = n0 + tx * 8 + j;
      if (n >= p.N) continue;
      float v = fmaf(acc[i][j], p.alpha, bm + (p.bias_n ? __ldg(&p.bias_n[n]) : 0.f));
      v = f32_act(v, p.act);
      const int64_t o = (int64_t)m * p.ldc + n;
      if (res) v = res[o] + (p.res_scale ? __ldg(&p.res_scale[n]) : 1.f) * v;
      C[o] = v;
    }
  }
}

// in-place softmax over the first n columns of rows with stride ld; one CTA per row.  Rows of up to 2048 columns are held in registers
// (one global read + one write per element instead of three reads + two writes): the attention score matrices are HBM-bound.
constexpr int kSmReg = 8;
__global__ void __launch_bounds__(256) softmax_rows_kernel(float* __restrict__ x, int n, int64_t ld) {
  __shared__ float red[64];
  float* r = x + (int64_t)blockIdx.x * ld;
  if (n <= 256 * kSmReg) {
    float v[kSmReg];
    float m = -INFINITY;
#pragma unroll
    for (int j = 0; j < kSmReg; ++j) {
      const int i = threadIdx.x + j * 256;
      v[j] = (i < n) ? r[i] : -INFINITY;
      m = fmaxf(m, v[j]);
    }
    for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = m;
    __syncthreads();
    m = red[0];
#pragma unroll
    for (int w = 1; w < 8; ++w) m = fmaxf(m, red[w]);
    __syncthreads();
    float s = 0.f;
#pragma unroll
    for (int j = 0; j < kSmReg; ++j) {
      v[j] = expf(v[j] - m);  // exp(-inf) = 0 for the padding slots
      s += v[j];
    }
    const float inv = 1.f / block_sum2(s, 0.f, red).x;
#pragma unroll
    for (int j = 0; j < kSmReg; ++j) {
      const int i = threadIdx.x + j * 256;
      if (i < n) r[i] = v[j] * inv;
    }
    return;
  }
  float m = -INFINITY;
  for (int i = threadIdx.x; i < n; i += blockDim.x) m = fmaxf(m, r[i]);
  for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = m;
  __syncthreads();
  m = red[0];
  for (int w = 1; w < (blockDim.x >> 5); ++w) m = fmaxf(m, red[w]);
  __syncthreads();
  float s = 0.f;
  for (int i = threadIdx.x; i < n; i += blockDim.x) {
    const float e = expf(r[i] - m);
    r[i] = e;
    s += e;
  }
  const float tot = block_sum2(s, 0.f, red).x;
  const float inv = 1.f / tot;
  for (int i = threadIdx.x; i < n; i += blockDim.x) r[i] *= inv;
}

// warp-per-row variant for rows of up to 32 * PER columns (attention rows: 62 and 801 in the BS-Roformer): the row lives in registers, no
// block-level synchronisation, 8 rows per CTA.
template <int PER>
__global__ void __launch_bounds__(256) softmax_rows_warp_kernel(float* __restrict__ x, int64_t rows, int n, int64_t ld) {
  const int64_t row = (int64_t)blockIdx.x * 8 + (threadIdx.x >> 5);
  if (row >= rows) return;
  const int lane = threadIdx.x & 31;
  float* r = x + row * ld;
  float v[PER];
  float m = -INFINITY;
#pragma unroll
  for (int j = 0; j < PER; ++j) {
    const int i = lane + j * 32;
    v[j] = (i < n) ? r[i] : -INFINITY;
    m = fmaxf(m, v[j]);
  }
  for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
  float s = 0.f;
#pragma unroll
  for (int j = 0; j < PER; ++j) {
    v[j] = expf(v[j] - m);
    s += v[j];
  }
  for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  const float inv = 1.f / s;
#pragma unroll
  for (int j = 0; j < PER; ++j) {
    const int i = lane + j * 32;
    if (i < n) r[i] = v[j] * inv;
  }
}

// GEMM with a tiny N (the 8 attention gates of the Roformer, bs_roformer.py:78): one warp per row of A, the N weight rows stay in L1.
// C[m][n] = act(alpha * A[m] . Bw[n] + bias_n[n] + bias_m[m]) (+ residual as in gemm_f32_kernel)
constexpr int kSmallN = 16;
template <int NN>
__global__ void __launch_bounds__(256) gemm_small_n_kernel(GemmF32 p) {
  const int64_t row = (int64_t)blockIdx.x * 8 + (threadIdx.x >> 5);
  if (row >= p.M) return;
  const int lane = threadIdx.x & 31;
  const float* A = p.A + (int64_t)blockIdx.z * p.sA + row * p.lda;
  const float* Bw = p.Bw + (int64_t)blockIdx.z * p.sB;
  float acc[NN];
#pragma unroll
  for (int j = 0; j < NN; ++j) acc[j] = 0.f;
  const bool vec = ((p.lda | p.ldb) & 3) == 0 && ((reinterpret_cast<uintptr_t>(A) | reinterpret_cast<uintptr_t>(Bw)) & 15) == 0;
  int k = 0;
  if (vec) {
    for (k = 4 * lane; k + 3 < p.K; k += 128) {
      const float4 a = *reinterpret_cast<const float4*>(A + k);
#pragma unroll
      for (int j = 0; j < NN; ++j) {
        if (j < p.N) {
          const float4 w = __ldg(reinterpret_cast<const float4*>(Bw + (int64_t)j * p.ldb + k));
          acc[j] = fmaf(a.x, w.x, fmaf(a.y, w.y, fmaf(a.z, w.z, fmaf(a.w, w.w, acc[j]))));
        }
      }
    }
    k = (p.K / 4) * 4 + lane;  // the K % 4 tail
  } else {
    k = lane;
  }
  for (; k < p.K; k += 32) {
    const float a = A[k];
#pragma unroll
    for (int j = 0; j < NN; ++j)
      if (j < p.N) acc[j] = fmaf(a, __ldg(&Bw[(int64_t)j * p.ldb + k]), acc[j]);
  }
#pragma unroll
  for (int j = 0; j < NN; ++j)
    for (int o = 16; o > 0; o >>= 1) acc[j] += __shfl_xor_sync(0xffffffffu, acc[j], o);
  if (lane < p.N) {
    float v = 0.f;
#pragma unroll
    for (int j = 0; j < NN; ++j)
      if (j == lane) v = acc[j];
    v = fmaf(v, p.alpha, (p.bias_m ? __ldg(&p.bias_m[row]) : 0.f) + (p.bias_n ? __ldg(&p.bias_n[lane]) : 0.f));
    v = f32_act(v, p.act);
    const int64_t o = (int64_t)blockIdx.z * p.sC + row * p.ldc + lane;
    if (p.res) v = p.res[o] + (p.res_scale ? __ldg(&p.res_scale[lane]) : 1.f) * v;
    p.C[o] = v;
  }
}

// op 0: out = alpha * a + beta * b (b may be null: + beta);  op 1: out = a * b;
// op 2: out = (a - b[0]) / (1e-5 + b[1]);  op 3: out = a * b[1] + b[0]   (b = device {mean, std}; htdemucs.py:501-510, :588-589, :611-612)
__global__ void ew_kernel(const float* __restrict__ a, const float* __restrict__ b, float* __restrict__ out, int64_t n, float alpha, float beta, int op) {
  float m = 0.f, sd = 0.f;
  if (op >= 2) {
    m = __ldg(&b[0]);
    sd = __ldg(&b[1]);
  }
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    float v;
    if (op == 1) v = a[i] * b[i];
    else if (op == 2) v = (a[i] - m) / (1e-5f + sd);
    else if (op == 3) v = a[i] * sd + m;
    else v = alpha * a[i] + (b ? beta * b[i] : beta);
    out[i] = v;
  }
}

// sum and sum of squares (double accumulation) -> out[0] = mean, out[1] = unbiased std  (x.mean(), x.std() of htdemucs.py:501-510).
// Two deterministic passes: kMsBlocks CTAs per sample leave (sum, sum of squares) partials, one CTA per sample adds them in a fixed order.
constexpr int kMsBlocks = 128;
__global__ void __launch_bounds__(256) meanstd_partial_kernel(const float* __restrict__ x, int64_t n, int64_t x_stride, double2* __restrict__ part) {
  __shared__ double rs[8], rq[8];
  const float* xs = x + (int64_t)blockIdx.y * x_stride;
  double s = 0.0, q = 0.0;
  for (int64_t i = (int64_t)blockIdx.x * 256 + threadIdx.x; i < n; i += (int64_t)kMsBlocks * 256) {
    const double v = xs[i];
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
    for (int w = 0; w < 8; ++w) {
      S += rs[w];
      Q += rq[w];
    }
    part[(int64_t)blockIdx.y * kMsBlocks + blockIdx.x] = make_double2(S, Q);
  }
}
__global__ void meanstd_final_kernel(const double2* __restrict__ part, int64_t n, float* __restrict__ out, int out_stride) {
  const double2* ps = part + (int64_t)blockIdx.x * kMsBlocks;
  double s = 0.0, q = 0.0;
  for (int i = threadIdx.x; i < kMsBlocks; i += 32) {
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
    out[(int64_t)blockIdx.x * out_stride] = (float)mean;
    out[(int64_t)blockIdx.x * out_stride + 1] = (float)sqrt(var > 0.0 ? var : 0.0);
  }
}

// apply_model's split branch (demucs/apply.py:215-250) as a gather: out[c][q] = sum_i w[q - o_i] * seg_i[c][q - o_i] / sum_i w[q - o_i],
// segments i start at o_i = i * stride, have `seg_len` samples except the last (clipped at `length`); triangle weight of `seg_len`.
// Output sample n of channel c is position q = q0 + n of the overlap-added signal, times scale * chan_scale[c]; `accumulate` adds to out
// (the shift-trick average, apply.py:197-214, and the per-source bag weights, apply.py:169-195, folded into the same pass).
__global__ void tri_ola_kernel(const float* __restrict__ segs, int first_seg, int n_segs, int channels, int seg_len, int64_t stride, int64_t length, int64_t q0,
                               int64_t n_out, float scale, const float* __restrict__ chan_scale, int accumulate, float* __restrict__ out, int64_t out_ld, int64_t out_off) {
  const int c = blockIdx.y;
  const float wmax = (float)(seg_len - seg_len / 2 > seg_len / 2 ? seg_len - seg_len / 2 : seg_len / 2);
  const float sc = scale * (chan_scale ? __ldg(&chan_scale[c]) : 1.f);
  for (int64_t n_o = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; n_o < n_out; n_o += (int64_t)gridDim.x * blockDim.x) {
    const int64_t q = q0 + n_o;
    int64_t i_hi = q / stride;
    if (i_hi > n_segs - 1) i_hi = n_segs - 1;
    int64_t i_lo = (q - seg_len + 1 <= 0) ? 0 : (q - seg_len + stride) / stride;
    float acc = 0.f, sw = 0.f;
    for (int64_t i = i_lo; i <= i_hi; ++i) {
      const int64_t n = q - i * stride;  // position inside segment i (its valid part is always long enough: clipped only at `length`)
      const float w = ((n < seg_len / 2) ? (float)(n + 1) : (float)(seg_len - n)) / wmax;  // cat(arange(1, s/2+1), arange(s - s/2, 0, -1)) / max
      acc += w * __ldg(&segs[((int64_t)(i - first_seg) * channels + c) * seg_len + n]);  // segs[0] is global segment `first_seg`
      sw += w;
    }
    const int64_t o = (int64_t)c * out_ld + out_off + n_o;
    const float v = sc * (acc / sw);
    out[o] = accumulate ? out[o] + v : v;
  }
}

}  // namespace b200sep

using namespace b200sep;

extern "C" int64_t b200sep_groupnorm1_work_floats(int B, int C, int Fr, int64_t L) {
  if (B < 1 || C < 1 || Fr < 1 || L < 1) return 0;
  return (int64_t)B * Fr * (gn_blocks_per_sample(B * Fr, (int64_t)C * L) + 1) * 4;  // one double2 per CTA + the shift x0
}

extern "C" int b200sep_groupnorm1_f32(const float* x, const float* gamma, const float* beta, float* y, int B, int C, int Fr, int64_t L, int act, int channel_last,
                                      float* work, void* stream) {
  B2_CHECK_ARG(x && gamma && beta && y && work && B >= 1 && C >= 1 && Fr >= 1 && L >= 1, "groupnorm1_f32: bad argument");
  B2_CHECK_ARG(!(channel_last && Fr != 1), "groupnorm1_f32: channel_last layout has no frequency rows");
  B2_CHECK_ARG((int64_t)C * L < (1ll << 31) && (int64_t)B * Fr <= 65535, "groupnorm1_f32: sample of %lld elements / %lld samples too large", (long long)C * L,
               (long long)B * Fr);
  B2_CHECK_ARG((reinterpret_cast<uintptr_t>(work) & 15) == 0, "groupnorm1_f32: work must be 16-byte aligned");
  const int samples = B * Fr;
  const int nblk = gn_blocks_per_sample(samples, (int64_t)C * L);
  GnGeom g;
  g.C = C; g.Fr = Fr; g.channel_last = channel_last; g.L = (uint32_t)L; g.n = (uint32_t)((int64_t)C * L); g.groups = 1;
  g.chunk = (uint32_t)cdiv((int64_t)g.n, nblk);
  dim3 grid(nblk, samples);
  gn_partial_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(x, g, reinterpret_cast<double2*>(work));
  B2_LAUNCHED();
  gn_apply_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(x, gamma, beta, y, g, reinterpret_cast<const double2*>(work), act);
  B2_LAUNCHED();
  return B200SEP_OK;
}

// nn.GroupNorm(groups, C) on a contiguous channel-first (B, C, X) tensor (hdemucs.py:87-88 norm_fn with norm_groups = 4): group (b, g) is the
// contiguous block of (C / groups) * X elements, i.e. one "sample" of the kernels above; gamma / beta are indexed by the absolute channel.
extern "C" int64_t b200sep_groupnorm_work_floats(int B, int C, int groups, int64_t X) {
  if (B < 1 || C < 1 || groups < 1 || X < 1 || C % groups) return 0;
  return (int64_t)B * groups * (gn_blocks_per_sample(B * groups, (int64_t)(C / groups) * X) + 1) * 4;
}

extern "C" int b200sep_groupnorm_f32(const float* x, const float* gamma, const float* beta, float* y, int B, int C, int groups, int64_t X, int act, float* work,
                                     void* stream) {
  B2_CHECK_ARG(x && gamma && beta && y && work && B >= 1 && C >= 1 && groups >= 1 && X >= 1 && C % groups == 0, "groupnorm_f32: bad argument");
  const int Cg = C / groups, samples = B * groups;
  B2_CHECK_ARG((int64_t)Cg * X < (1ll << 31) && samples <= 65535, "groupnorm_f32: group of %lld elements / %d groups too large", (long long)Cg * X, samples);
  B2_CHECK_ARG((reinterpret_cast<uintptr_t>(work) & 15) == 0, "groupnorm_f32: work must be 16-byte aligned");
  const int nblk = gn_blocks_per_sample(samples, (int64_t)Cg * X);
  GnGeom g;
  g.C = Cg; g.Fr = 1; g.channel_last = 0; g.L = (uint32_t)X; g.n = (uint32_t)((int64_t)Cg * X); g.groups = groups;
  g.chunk = (uint32_t)cdiv((int64_t)g.n, nblk);
  dim3 grid(nblk, samples);
  gn_partial_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(x, g, reinterpret_cast<double2*>(work));
  B2_LAUNCHED();
  gn_apply_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(x, gamma, beta, y, g, reinterpret_cast<const double2*>(work), act);
  B2_LAUNCHED();
  return B200SEP_OK;
}

// permutations that keep the innermost dimension in place (the "b t f d <-> b f t d" swaps around the Roformer transformers) move whole
// float4s: same index arithmetic on d3/4 "elements" of 16 bytes
__global__ void permute4_vec_kernel(const float4* __restrict__ x, float4* __restrict__ y, int d0, int d1, int d2, int d3q, int p0, int p1, int p2, int64_t n) {
  const int din[3] = {d0, d1, d2};
  const int perm[3] = {p0, p1, p2};
  const int64_t sin_[3] = {(int64_t)d1 * d2 * d3q, (int64_t)d2 * d3q, d3q};
  for (int64_t o = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; o < n; o += (int64_t)gridDim.x * blockDim.x) {
    int64_t r = o / d3q, src = o - r * d3q;
    for (int k = 2; k >= 0; --k) {
      const int dk = din[perm[k]];
      src += (r % dk) * sin_[perm[k]];
      r /= dk;
    }
    y[o] = x[src];
  }
}

extern "C" int b200sep_permute4_f32(const float* x, float* y, int d0, int d1, int d2, int d3, int p0, int p1, int p2, int p3, void* stream) {
  B2_CHECK_ARG(x && y && d0 >= 1 && d1 >= 1 && d2 >= 1 && d3 >= 1, "permute4_f32: bad argument");
  if (p3 == 3 && d3 % 4 == 0 && ((reinterpret_cast<uintptr_t>(x) | reinterpret_cast<uintptr_t>(y)) & 15) == 0 && p0 >= 0 && p0 < 3 && p1 >= 0 && p1 < 3 && p2 >= 0 && p2 < 3 &&
      ((1 << p0) | (1 << p1) | (1 << p2)) == 7) {
    const int64_t nq = (int64_t)d0 * d1 * d2 * (d3 / 4);
    permute4_vec_kernel<<<(int)std::min<int64_t>(cdiv(nq, 256), kNumSMs * 16), 256, 0, (cudaStream_t)stream>>>(reinterpret_cast<const float4*>(x), reinterpret_cast<float4*>(y), d0,
                                                                                                                 d1, d2, d3 / 4, p0, p1, p2, nq);
    B2_LAUNCHED();
    return B200SEP_OK;
  }
  const int seen = (1 << p0) | (1 << p1) | (1 << p2) | (1 << p3);
  B2_CHECK_ARG(p0 >= 0 && p0 < 4 && p1 >= 0 && p1 < 4 && p2 >= 0 && p2 < 4 && p3 >= 0 && p3 < 4 && seen == 15, "permute4_f32: not a permutation");
  const int64_t n = (int64_t)d0 * d1 * d2 * d3;
  permute4_kernel<<<(int)std::min<int64_t>(cdiv(n, 256), kNumSMs * 16), 256, 0, (cudaStream_t)stream>>>(x, y, d0, d1, d2, d3, p0, p1, p2, p3, n);
  B2_LAUNCHED();
  return B200SEP_OK;
}

extern "C" int b200sep_glu_f32(const float* a, const float* res, const float* scale, float* y, int B, int C, int64_t L, void* stream) {
  B2_CHECK_ARG(a && y && (res == nullptr || scale != nullptr), "glu_f32: bad argument");
  const int64_t n = (int64_t)B * C * L;
  if (n == 0) return B200SEP_OK;
  glu_kernel<<<(int)std::min<int64_t>(cdiv(n, 256), kNumSMs * 16), 256, 0, (cudaStream_t)stream>>>(a, res, scale, y, C, L, n);
  B2_LAUNCHED();
  return B200SEP_OK;
}

extern "C" int b200sep_layernorm_f32(const float* x, const float* gamma, const float* beta, float* y, int64_t rows, int C, void* stream) {
  B2_CHECK_ARG(x && gamma && beta && y && rows >= 0 && C >= 1, "layernorm_f32: bad argument");
  if (rows == 0) return B200SEP_OK;
  layernorm_kernel<<<cdiv(rows, 8), 256, 0, (cudaStream_t)stream>>>(x, gamma, beta, y, rows, C);
  B2_LAUNCHED();
  return B200SEP_OK;
}

// math selects the tensor-core arithmetic (B200SEP_MATH_*); the SIMT kernels below are fp32 in every mode
extern "C" int b200sep_gemm_f32_math(const float* A, const float* Bw, float* C, int M, int N, int K, int lda, int ldb, int ldc, int batch, int64_t strideA,
                                     int64_t strideB, int64_t strideC, float alpha, const float* bias_n, const float* bias_m, int act, const float* res,
                                     const float* res_scale, const void* w_packed, int math, void* stream) {
  B2_CHECK_ARG(A && Bw && C && M >= 1 && N >= 1 && K >= 1 && batch >= 1 && batch <= 65535, "gemm_f32: bad argument");
  B2_CHECK_ARG(math == B200SEP_MATH_BF16X3 || math == B200SEP_MATH_FP16, "gemm_f32: unknown math mode %d", math);
  B2_CHECK_ARG(w_packed == nullptr || tc_packed_matches(w_packed, math), "gemm_f32: w_packed was packed for the other math mode (asked for %d)", math);
  if (tc_gemm_usable(M, N, K, batch))
    return tc_gemm_f32(A, Bw, C, M, N, K, lda, ldb, ldc, batch, strideA, strideB, strideC, alpha, bias_n, bias_m, act, res, res_scale,
                       (batch == 1 || strideB == 0) ? w_packed : nullptr, 0, math, (cudaStream_t)stream);
  GemmF32 p{A, Bw, C, bias_n, bias_m, res, res_scale, M, N, K, lda, ldb, ldc, strideA, strideB, strideC, alpha, act, 0};
  if (N <= kSmallN && M >= 1024) {
    dim3 g(cdiv(M, 8), 1, batch);
    if (N <= 8) gemm_small_n_kernel<8><<<g, 256, 0, (cudaStream_t)stream>>>(p);
    else gemm_small_n_kernel<kSmallN><<<g, 256, 0, (cudaStream_t)stream>>>(p);
    B2_LAUNCHED();
    return B200SEP_OK;
  }
  dim3 grid(cdiv(N, FBN), cdiv(M, FBM), batch);
  B2_CHECK_ARG(grid.y <= 65535, "gemm_f32: M too large");
  gemm_f32_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(p);
  B2_LAUNCHED();
  return B200SEP_OK;
}

extern "C" int b200sep_gemm_f32(const float* A, const float* Bw, float* C, int M, int N, int K, int lda, int ldb, int ldc, int batch, int64_t strideA,
                                int64_t strideB, int64_t strideC, float alpha, const float* bias_n, const float* bias_m, int act, const float* res,
                                const float* res_scale, const void* w_packed, void* stream) {
  return b200sep_gemm_f32_math(A, Bw, C, M, N, K, lda, ldb, ldc, batch, strideA, strideB, strideC, alpha, bias_n, bias_m, act, res, res_scale, w_packed,
                               B200SEP_MATH_BF16X3, stream);
}

extern "C" int b200sep_softmax_rows_f32(float* x, int64_t rows, int n, int64_t ld, void* stream) {
  B2_CHECK_ARG(x && rows >= 0 && n >= 1 && rows <= 0x7fffffff && ld >= n, "softmax_rows_f32: bad argument");
  if (rows == 0) return B200SEP_OK;
  const unsigned wgrid = (unsigned)cdiv(rows, 8);
  if (n <= 64) softmax_rows_warp_kernel<2><<<wgrid, 256, 0, (cudaStream_t)stream>>>(x, rows, n, ld);
  else if (n <= 256) softmax_rows_warp_kernel<8><<<wgrid, 256, 0, (cudaStream_t)stream>>>(x, rows, n, ld);
  else if (n <= 832) softmax_rows_warp_kernel<26><<<wgrid, 256, 0, (cudaStream_t)stream>>>(x, rows, n, ld);
  else softmax_rows_kernel<<<(unsigned)rows, 256, 0, (cudaStream_t)stream>>>(x, n, ld);
  B2_LAUNCHED();
  return B200SEP_OK;
}

extern "C" int b200sep_ew_f32(const float* a, const float* b, float* out, int64_t n, float alpha, float beta, int op, void* stream) {
  B2_CHECK_ARG(a && out && n >= 0 && op >= 0 && op <= 3 && (op == 0 || b), "ew_f32: bad argument");
  if (n == 0) return B200SEP_OK;
  ew_kernel<<<(int)std::min<int64_t>(cdiv(n, 256), kNumSMs * 16), 256, 0, (cudaStream_t)stream>>>(a, b, out, n, alpha, beta, op);
  B2_LAUNCHED();
  return B200SEP_OK;
}

extern "C" int64_t b200sep_meanstd_work_floats(int batch) { return batch >= 1 ? (int64_t)batch * kMsBlocks * 4 : 0; }

extern "C" int b200sep_meanstd_batch_f32(const float* x, int64_t n, int batch, int64_t x_stride, float* out, int out_stride, float* work, void* stream) {
  B2_CHECK_ARG(x && out && work && n >= 2 && batch >= 1 && batch <= 65535 && out_stride >= 2, "meanstd_batch_f32: need at least 2 elements per sample");
  B2_CHECK_ARG((reinterpret_cast<uintptr_t>(work) & 15) == 0, "meanstd_batch_f32: work must be 16-byte aligned");
  meanstd_partial_kernel<<<dim3(kMsBlocks, batch), 256, 0, (cudaStream_t)stream>>>(x, n, x_stride, reinterpret_cast<double2*>(work));
  B2_LAUNCHED();
  meanstd_final_kernel<<<batch, 32, 0, (cudaStream_t)stream>>>(reinterpret_cast<const double2*>(work), n, out, out_stride);
  B2_LAUNCHED();
  return B200SEP_OK;
}

// single-sample form: the partials live in a per-device scratch buffer owned by the library (allocated on first use; calls on different streams
// of one device must not overlap -- the engines issue everything on one stream)
extern "C" int b200sep_meanstd_f32(const float* x, int64_t n, float* out2, void* stream) {
  B2_CHECK_ARG(x && out2 && n >= 2, "meanstd_f32: need at least 2 elements");
  static float* scratch[64] = {nullptr};
  int dev = 0;
  B2_CUDA(cudaGetDevice(&dev));
  B2_CHECK_ARG(dev >= 0 && dev < 64, "meanstd_f32: device index %d", dev);
  if (!scratch[dev]) B2_CUDA(cudaMalloc(&scratch[dev], kMsBlocks * 4 * sizeof(float)));
  return b200sep_meanstd_batch_f32(x, n, 1, 0, out2, 2, scratch[dev], stream);
}

extern "C" int b200sep_triangle_overlap_add_range(const float* segs, int first_seg, int n_local, int n_segs, int channels, int seg_len, int64_t stride, int64_t length,
                                                  int64_t q0, int64_t n_out, float scale, const float* chan_scale, int accumulate, float* out, int64_t out_ld,
                                                  int64_t out_off, void* stream) {
  B2_CHECK_ARG(segs && out && n_segs >= 1 && channels >= 1 && seg_len >= 2 && stride >= 1 && length >= 1, "triangle_overlap_add: bad argument");
  B2_CHECK_ARG(q0 >= 0 && n_out >= 0 && q0 + n_out <= length, "triangle_overlap_add: output range [%lld, %lld) outside the signal of %lld samples",
               (long long)q0, (long long)(q0 + n_out), (long long)length);
  B2_CHECK_ARG((int64_t)(n_segs - 1) * stride < length, "triangle_overlap_add: more segments than the signal holds");
  B2_CHECK_ARG(out_off >= 0 && out_off + n_out <= out_ld, "triangle_overlap_add: output slice [%lld, %lld) outside rows of %lld", (long long)out_off,
               (long long)(out_off + n_out), (long long)out_ld);
  if (n_out == 0) return B200SEP_OK;
  // every segment that covers [q0, q0 + n_out) must be present in the local buffer
  const int64_t need_lo = (q0 - seg_len + 1 <= 0) ? 0 : (q0 - seg_len + stride) / stride;
  const int64_t need_hi = std::min<int64_t>((q0 + n_out - 1) / stride, n_segs - 1);
  B2_CHECK_ARG(need_lo >= first_seg && need_hi < (int64_t)first_seg + n_local, "triangle_overlap_add: outputs [%lld,%lld) need segments [%lld,%lld] but the buffer holds [%d,%d)",
               (long long)q0, (long long)(q0 + n_out), (long long)need_lo, (long long)need_hi, first_seg, first_seg + n_local);
  dim3 grid((unsigned)std::min<int64_t>(cdiv(n_out, 256), kNumSMs * 8), channels);
  tri_ola_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(segs, first_seg, n_segs, channels, seg_len, stride, length, q0, n_out, scale, chan_scale, accumulate, out, out_ld,
                                                         out_off);
  B2_LAUNCHED();
  return B200SEP_OK;
}

extern "C" int b200sep_triangle_overlap_add(const float* segs, int n_segs, int channels, int seg_len, int64_t stride, int64_t length, int64_t q0, int64_t n_out,
                                            float scale, const float* chan_scale, int accumulate, float* out, void* stream) {
  B2_CHECK_ARG(n_out >= 1, "triangle_overlap_add: empty output");
  return b200sep_triangle_overlap_add_range(segs, 0, n_segs, n_segs, channels, seg_len, stride, length, q0, n_out, scale, chan_scale, accumulate, out, n_out, 0, stream);
}

extern "C" int b200sep_gemm_kn_f32(const float* A, const float* B_kn, float* C, int M, int N, int K, int lda, int ldb, int ldc, int batch, int64_t strideA, int64_t strideB,
                                   int64_t strideC, float alpha, void* stream) {
  B2_CHECK_ARG(A && B_kn && C && M >= 1 && N >= 1 && K >= 1 && batch >= 1 && lda >= K && ldb >= N && ldc >= N, "gemm_kn_f32: bad argument");
  if (!tc_gemm_usable(M, N, K, batch)) {  // small shapes: the SIMT kernel reads B transposed
    B2_CHECK_ARG(batch <= 65535, "gemm_kn_f32: batch too large for the SIMT path");
    GemmF32 p{A, B_kn, C, nullptr, nullptr, nullptr, nullptr, M, N, K, lda, ldb, ldc, strideA, strideB, strideC, alpha, 0, 1};
    dim3 grid(cdiv(N, FBN), cdiv(M, FBM), batch);
    gemm_f32_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(p);
    B2_LAUNCHED();
    return B200SEP_OK;
  }
  return tc_gemm_f32(A, B_kn, C, M, N, K, lda, ldb, ldc, batch, strideA, strideB, strideC, alpha, nullptr, nullptr, 0, nullptr, nullptr, nullptr, 1, B200SEP_MATH_BF16X3,
                     (cudaStream_t)stream);
}

extern "C" int64_t b200sep_tc_packed_floats_math(int N, int K, int math) {
  return (N >= 1 && K >= 1 && (math == B200SEP_MATH_BF16X3 || math == B200SEP_MATH_FP16)) ? tc_packed_bytes(N, K, math) / 4 : 0;
}

extern "C" int64_t b200sep_tc_packed_floats(int N, int K) { return b200sep_tc_packed_floats_math(N, K, B200SEP_MATH_BF16X3); }

extern "C" int b200sep_tc_pack_linear_weights_math(const float* W, int N, int K, int ldw, float* packed, int math, void* stream) {
  B2_CHECK_ARG(W && packed && N >= 1 && K >= 1 && ldw >= K, "tc_pack_linear_weights: bad argument");
  B2_CHECK_ARG((reinterpret_cast<uintptr_t>(packed) & 15) == 0, "tc_pack_linear_weights: packed must be 16-byte aligned");
  return tc_pack_linear(W, N, K, ldw, packed, math, (cudaStream_t)stream);
}

extern "C" int b200sep_tc_pack_linear_weights(const float* W, int N, int K, int ldw, float* packed, void* stream) {
  return b200sep_tc_pack_linear_weights_math(W, N, K, ldw, packed, B200SEP_MATH_BF16X3, stream);
}

extern "C" int b200sep_tc_pack_conv_weights_math(const float* w_blocked, int Cin, int taps, int Cout, float* packed, int math, void* stream) {
  B2_CHECK_ARG(w_blocked && packed && Cin >= 1 && taps >= 1 && Cout >= 1, "tc_pack_conv_weights: bad argument");
  B2_CHECK_ARG((reinterpret_cast<uintptr_t>(packed) & 15) == 0, "tc_pack_conv_weights: packed must be 16-byte aligned");
  return tc_pack_conv(w_blocked, Cin, taps, Cout, cdiv(Cout, 48) * 48, packed, math, (cudaStream_t)stream);
}

extern "C" int b200sep_tc_pack_conv_weights(const float* w_blocked, int Cin, int taps, int Cout, float* packed, void* stream) {
  return b200sep_tc_pack_conv_weights_math(w_blocked, Cin, taps, Cout, packed, B200SEP_MATH_BF16X3, stream);
}
