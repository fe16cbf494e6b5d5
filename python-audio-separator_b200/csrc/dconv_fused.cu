// Fused DConv residual branch of Demucs (uvr_lib_v5/demucs/demucs.py:85-168, one `layers[d]` of DConv.forward :166-168):
//
//     x += LayerScale * GLU( GroupNorm(1, 2C)( Conv1d(C/8 -> 2C, 1)( GELU( GroupNorm(1, C/8)( Conv1d(C -> C/8, 3, dilation d)(x) ) ) ) ) )
//
// on (B, C, Fr, L) tensors where every (b, fr) row is one GroupNorm sample (the reference folds the frequency axis of the spectrogram
// branch into the batch, hdemucs.py:141-146).  The operator-by-operator form materialises the 2C-channel tensor and walks it five times
// (1x1 conv write, GroupNorm statistics, GroupNorm apply read + write, GLU read); it is HBM-bound and was 45 % of an HTDemucs forward
// (profiles/r02_htdemucs_launches_b4.txt).  Here the hidden tensor u (C/8 channels, 1/8 of x) is the only intermediate that reaches
// memory; the 2C-channel tensor is recomputed from it on the fly, once for its GroupNorm statistics and once for the output:
//     K1  u = conv3(x) + b0, per-tile partial sums of u, u^2                       reads x, writes u
//     K2  h = GELU(GN(u)); z = W3 h + b3 per position, partial sums of z, z^2      reads u
//     K3  the same z, normalised, GLU, LayerScale, residual                        reads u, x; writes y (in place allowed)
// with a tiny finalise kernel after K1 and K2 turning the partial sums (double) into (mean, rstd) per sample.
// All arithmetic is fp32 FMA (no tensor cores: 2*hid*2C flops per position against 4*(2C + C/4) bytes is below the ridge even for
// fp32 SIMT); thread = P positions, the small weight matrices sit in shared memory and are read as broadcast float4.
#include <algorithm>

#include "common.cuh"

namespace b200sep {
namespace {

constexpr int kDcThreads = 128;

struct DconvParams {
  const float* x;
  float* y;
  const float *w0, *b0, *g1, *be1, *w3, *b3, *g4, *be4, *ls;
  float* u;         // (B, hid, Fr, L)
  double2* part_u;  // [samples][nblk]
  double2* part_z;  // [samples][nblk]
  float2* stat_u;   // [samples] (mean, rstd)
  float2* stat_z;
  int B, C, Fr, L, dil, nblk, tiles;
};

__device__ __forceinline__ float gelu_erf(float v) { return 0.5f * v * (1.f + erff(v * 0.70710678118654752440f)); }

__device__ __forceinline__ void block_sum2(double& s, double& q, double* sm) {
  for (int o = 16; o > 0; o >>= 1) {
    s += __shfl_xor_sync(0xffffffffu, s, o);
    q += __shfl_xor_sync(0xffffffffu, q, o);
  }
  const int w = threadIdx.x >> 5;
  __syncthreads();  // sm may still be read from the previous tile
  if ((threadIdx.x & 31) == 0) {
    sm[2 * w] = s;
    sm[2 * w + 1] = q;
  }
  __syncthreads();
  s = 0.0;
  q = 0.0;
  for (int i = 0; i < kDcThreads / 32; ++i) {
    s += sm[2 * i];
    q += sm[2 * i + 1];
  }
}

// K1: u[b][k][fr][l] = b0[k] + sum_{c,t} w0[k][c][t] * x[b][c][fr][l + (t-1)*dil]      (zero padding at the row ends)
template <int HID, int P>
__global__ void __launch_bounds__(kDcThreads) dconv_k1_kernel(const DconvParams p) {
  extern __shared__ __align__(16) float smem_dc[];
  constexpr int HP = (HID + 3) / 4 * 4;  // rows padded to whole float4s (zeros)
  float* ws = smem_dc;  // [C][3][HP]
  __shared__ double red[2 * kDcThreads / 32];
  for (int i = threadIdx.x; i < HP * p.C * 3; i += kDcThreads) {
    const int k = i / (p.C * 3), r = i - k * (p.C * 3);  // w0 is (HID, C, 3): r = c*3 + t
    ws[r * HP + k] = k < HID ? __ldg(&p.w0[i]) : 0.f;
  }
  __syncthreads();
  constexpr int TP = kDcThreads * P;
  for (int tile = blockIdx.x; tile < p.tiles; tile += gridDim.x) {
    const int sample = tile / p.nblk, tb = tile - sample * p.nblk;
    const int b = sample / p.Fr, fr = sample - b * p.Fr;
    const float* xr = p.x + ((int64_t)b * p.C * p.Fr + fr) * p.L;  // + c * Fr * L
    const int64_t cs = (int64_t)p.Fr * p.L;
    float acc[P][HP];
    int pos[P];
#pragma unroll
    for (int j = 0; j < P; ++j) {
      pos[j] = tb * TP + j * kDcThreads + threadIdx.x;
#pragma unroll
      for (int k = 0; k < HP; ++k) acc[j][k] = k < HID ? __ldg(&p.b0[k]) : 0.f;
    }
    for (int c = 0; c < p.C; ++c) {
      const float* xc = xr + c * cs;
      float xv[P][3];
#pragma unroll
      for (int j = 0; j < P; ++j) {
#pragma unroll
        for (int t = 0; t < 3; ++t) {
          const int l = pos[j] + (t - 1) * p.dil;
          xv[j][t] = (l >= 0 && l < p.L) ? __ldg(&xc[l]) : 0.f;
        }
      }
      const float* wc = ws + c * 3 * HP;
#pragma unroll
      for (int t = 0; t < 3; ++t) {
#pragma unroll
        for (int k4 = 0; k4 < HP; k4 += 4) {
          const float4 w = *reinterpret_cast<const float4*>(&wc[t * HP + k4]);
#pragma unroll
          for (int j = 0; j < P; ++j) {
            acc[j][k4] = fmaf(w.x, xv[j][t], acc[j][k4]);
            acc[j][k4 + 1] = fmaf(w.y, xv[j][t], acc[j][k4 + 1]);
            acc[j][k4 + 2] = fmaf(w.z, xv[j][t], acc[j][k4 + 2]);
            acc[j][k4 + 3] = fmaf(w.w, xv[j][t], acc[j][k4 + 3]);
          }
        }
      }
    }
    double s = 0.0, q = 0.0;
#pragma unroll
    for (int j = 0; j < P; ++j) {
      if (pos[j] < p.L) {
        float fs = 0.f, fq = 0.f;
#pragma unroll
        for (int k = 0; k < HID; ++k) {
          p.u[(((int64_t)b * HID + k) * p.Fr + fr) * p.L + pos[j]] = acc[j][k];
          fs += acc[j][k];
          fq = fmaf(acc[j][k], acc[j][k], fq);
        }
        s += fs;
        q += fq;
      }
    }
    block_sum2(s, q, red);
    if (threadIdx.x == 0) p.part_u[(int64_t)sample * p.nblk + tb] = make_double2(s, q);
  }
}

// statistics of a u that another operator produced (hid = 48: the C -> C/8 convolution runs on the tensor cores)
template <int HID, int P>
__global__ void __launch_bounds__(kDcThreads) dconv_ustats_kernel(const DconvParams p) {
  __shared__ double red[2 * kDcThreads / 32];
  constexpr int TP = kDcThreads * P;
  for (int tile = blockIdx.x; tile < p.tiles; tile += gridDim.x) {
    const int sample = tile / p.nblk, tb = tile - sample * p.nblk;
    const int b = sample / p.Fr, fr = sample - b * p.Fr;
    double s = 0.0, q = 0.0;
#pragma unroll
    for (int j = 0; j < P; ++j) {
      const int pos = tb * TP + j * kDcThreads + threadIdx.x;
      if (pos < p.L) {
        float fs = 0.f, fq = 0.f;
#pragma unroll 8
        for (int k = 0; k < HID; ++k) {
          const float v = p.u[(((int64_t)b * HID + k) * p.Fr + fr) * p.L + pos];
          fs += v;
          fq = fmaf(v, v, fq);
        }
        s += fs;
        q += fq;
      }
    }
    block_sum2(s, q, red);
    if (threadIdx.x == 0) p.part_u[(int64_t)sample * p.nblk + tb] = make_double2(s, q);
  }
}

// partial sums -> (mean, rstd) of GroupNorm(1, channels) per sample (biased variance, eps 1e-5)
__global__ void dconv_finalize_kernel(const double2* __restrict__ part, float2* __restrict__ stat, int samples, int nblk, double n) {
  const int sample = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (sample >= samples) return;
  double s = 0.0, q = 0.0;
  for (int i = threadIdx.x & 31; i < nblk; i += 32) {
    const double2 v = part[(int64_t)sample * nblk + i];
    s += v.x;
    q += v.y;
  }
  for (int o = 16; o > 0; o >>= 1) {
    s += __shfl_xor_sync(0xffffffffu, s, o);
    q += __shfl_xor_sync(0xffffffffu, q, o);
  }
  if ((threadIdx.x & 31) == 0) {
    const double mean = s / n;
    double var = q / n - mean * mean;
    if (var < 0.0) var = 0.0;
    stat[sample] = make_float2((float)mean, (float)(1.0 / sqrt(var + 1e-5)));
  }
}

// K2 (APPLY = false): partial sums of z = W3 h + b3;  K3 (APPLY = true): y = x + ls * GN(z)[:C] * sigmoid(GN(z)[C:])
template <int HID, int P, bool APPLY>
__global__ void __launch_bounds__(kDcThreads) dconv_k23_kernel(const DconvParams p) {
  extern __shared__ __align__(16) float smem_dc[];
  constexpr int HP = (HID + 3) / 4 * 4;      // rows padded to whole float4s (zeros)
  float* ws = smem_dc;                       // [C][2][HP]: rows c (value) and C + c (gate) of w3 side by side
  float* cst = ws + (size_t)p.C * 2 * HP;    // [C][8]: b3[c], b3[C+c], g4[c], be4[c], g4[C+c], be4[C+c], ls[c], -
  __shared__ double red[2 * kDcThreads / 32];
  for (int i = threadIdx.x; i < 2 * p.C * HP; i += kDcThreads) {
    const int row = i / HP, k = i - row * HP;  // w3 is (2C, HID)
    const int c = row < p.C ? row : row - p.C, half = row < p.C ? 0 : 1;
    ws[(c * 2 + half) * HP + k] = k < HID ? __ldg(&p.w3[row * HID + k]) : 0.f;
  }
  for (int c = threadIdx.x; c < p.C; c += kDcThreads) {
    float* o = cst + c * 8;
    o[0] = __ldg(&p.b3[c]); o[1] = __ldg(&p.b3[p.C + c]);
    o[2] = __ldg(&p.g4[c]); o[3] = __ldg(&p.be4[c]); o[4] = __ldg(&p.g4[p.C + c]); o[5] = __ldg(&p.be4[p.C + c]);
    o[6] = __ldg(&p.ls[c]); o[7] = 0.f;
  }
  __syncthreads();
  constexpr int TP = kDcThreads * P;
  const int64_t cs = (int64_t)p.Fr * p.L;
  for (int tile = blockIdx.x; tile < p.tiles; tile += gridDim.x) {
    const int sample = tile / p.nblk, tb = tile - sample * p.nblk;
    const int b = sample / p.Fr, fr = sample - b * p.Fr;
    const float2 su = __ldg(&p.stat_u[sample]);
    float h[P][HP];
    int pos[P];
#pragma unroll
    for (int j = 0; j < P; ++j) {
      pos[j] = tb * TP + j * kDcThreads + threadIdx.x;
      const int l = pos[j] < p.L ? pos[j] : p.L - 1;  // out-of-range lanes compute on a valid address and are masked at the end
#pragma unroll
      for (int k = 0; k < HP; ++k) {
        h[j][k] = 0.f;
        if (k < HID) {
          const float v = p.u[(((int64_t)b * HID + k) * p.Fr + fr) * p.L + l];
          h[j][k] = gelu_erf(fmaf((v - su.x) * su.y, __ldg(&p.g1[k]), __ldg(&p.be1[k])));
        }
      }
    }
    float2 sz = make_float2(0.f, 1.f);
    if (APPLY) sz = __ldg(&p.stat_z[sample]);
    const float* xr = p.x + ((int64_t)b * p.C * p.Fr + fr) * p.L;
    float* yr = p.y + ((int64_t)b * p.C * p.Fr + fr) * p.L;
    float fs[P], fq[P];
#pragma unroll
    for (int j = 0; j < P; ++j) fs[j] = fq[j] = 0.f;
    for (int c = 0; c < p.C; ++c) {
      const float4 k0 = *reinterpret_cast<const float4*>(&cst[c * 8]);
      float a[P], g[P];
#pragma unroll
      for (int j = 0; j < P; ++j) {
        a[j] = k0.x;
        g[j] = k0.y;
      }
      const float* wc = ws + c * 2 * HP;
#pragma unroll
      for (int k = 0; k < HP; k += 4) {
        const float4 wa = *reinterpret_cast<const float4*>(&wc[k]);
        const float4 wg = *reinterpret_cast<const float4*>(&wc[HP + k]);
#pragma unroll
        for (int j = 0; j < P; ++j) {
          a[j] = fmaf(wa.x, h[j][k], a[j]);
          a[j] = fmaf(wa.y, h[j][k + 1], a[j]);
          a[j] = fmaf(wa.z, h[j][k + 2], a[j]);
          a[j] = fmaf(wa.w, h[j][k + 3], a[j]);
          g[j] = fmaf(wg.x, h[j][k], g[j]);
          g[j] = fmaf(wg.y, h[j][k + 1], g[j]);
          g[j] = fmaf(wg.z, h[j][k + 2], g[j]);
          g[j] = fmaf(wg.w, h[j][k + 3], g[j]);
        }
      }
      if (APPLY) {
        const float4 k1 = *reinterpret_cast<const float4*>(&cst[c * 8 + 4]);
#pragma unroll
        for (int j = 0; j < P; ++j) {
          if (pos[j] < p.L) {
            const float an = fmaf((a[j] - sz.x) * sz.y, k0.z, k0.w);
            const float gn = fmaf((g[j] - sz.x) * sz.y, k1.x, k1.y);
            const int64_t o = (int64_t)c * cs + pos[j];
            yr[o] = xr[o] + k1.z * (an / (1.f + expf(-gn)));
          }
        }
      } else {
#pragma unroll
        for (int j = 0; j < P; ++j) {
          fs[j] += a[j] + g[j];
          fq[j] = fmaf(a[j], a[j], fmaf(g[j], g[j], fq[j]));
        }
      }
    }
    if (!APPLY) {
      double s = 0.0, q = 0.0;
#pragma unroll
      for (int j = 0; j < P; ++j) {
        if (pos[j] < p.L) {
          s += fs[j];
          q += fq[j];
        }
      }
      block_sum2(s, q, red);
      if (threadIdx.x == 0) p.part_z[(int64_t)sample * p.nblk + tb] = make_double2(s, q);
    }
  }
}

template <int HID, int P>
int dconv_launch(DconvParams p, bool have_u, cudaStream_t st) {
  const int samples = p.B * p.Fr;
  p.nblk = cdiv(p.L, kDcThreads * P);
  p.tiles = samples * p.nblk;
  constexpr int HP = (HID + 3) / 4 * 4;
  const size_t smem1 = (size_t)HP * p.C * 3 * sizeof(float);
  const size_t smem23 = ((size_t)p.C * 2 * HP + (size_t)p.C * 8) * sizeof(float);
  B2_CHECK_ARG(smem23 <= 200 * 1024 && (have_u || smem1 <= 200 * 1024), "dconv_f32: C=%d hid=%d weights do not fit in shared memory", p.C, HID);
  static bool attr_set[kMaxDevices] = {};
  B2_DEVICE_SLOT(dev);
  if (!attr_set[dev]) {
    B2_CUDA(cudaFuncSetAttribute(dconv_k1_kernel<HID, P>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
    B2_CUDA(cudaFuncSetAttribute(dconv_k23_kernel<HID, P, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
    B2_CUDA(cudaFuncSetAttribute(dconv_k23_kernel<HID, P, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
    attr_set[dev] = true;
  }
  // persistent CTAs (the weights are staged once per CTA); as many per SM as the shared-memory image allows
  auto grid_for = [&](size_t smem) {
    const int per_sm = (int)std::max<size_t>(1, std::min<size_t>(8, (200 * 1024) / std::max<size_t>(smem, 1024)));
    return std::min(p.tiles, kNumSMs * per_sm);
  };
  if (have_u) dconv_ustats_kernel<HID, P><<<std::min(p.tiles, kNumSMs * 8), kDcThreads, 0, st>>>(p);
  else dconv_k1_kernel<HID, P><<<grid_for(smem1), kDcThreads, smem1, st>>>(p);
  B2_LAUNCHED();
  dconv_finalize_kernel<<<cdiv(samples, 4), 128, 0, st>>>(p.part_u, p.stat_u, samples, p.nblk, (double)HID * p.L);
  B2_LAUNCHED();
  dconv_k23_kernel<HID, P, false><<<grid_for(smem23), kDcThreads, smem23, st>>>(p);
  B2_LAUNCHED();
  dconv_finalize_kernel<<<cdiv(samples, 4), 128, 0, st>>>(p.part_z, p.stat_z, samples, p.nblk, 2.0 * p.C * p.L);
  B2_LAUNCHED();
  dconv_k23_kernel<HID, P, true><<<grid_for(smem23), kDcThreads, smem23, st>>>(p);
  B2_LAUNCHED();
  return B200SEP_OK;
}

// ---------------------------------------------------------------------------------------------------------------------------------
// Single-pass form for rows that fit in shared memory (the frequency branch: one GroupNorm sample = one (b, fr) row of C x L values, 64 KB at C = 48,
// L = 336): the row is read ONCE, both GroupNorm reductions happen inside the CTA, and the result is written once -- instead of three passes over x, the
// hidden tensor through HBM and two partial-sum round trips.  Persistent CTAs walk the rows; the weights are staged once per CTA.
constexpr int kRowMaxThreads = 512;

__device__ __forceinline__ void row_sum2(double& s, double& q, double* sm) {
  for (int o = 16; o > 0; o >>= 1) {
    s += __shfl_xor_sync(0xffffffffu, s, o);
    q += __shfl_xor_sync(0xffffffffu, q, o);
  }
  const int w = threadIdx.x >> 5, nw = blockDim.x >> 5;
  __syncthreads();  // sm may still be read from the previous reduction
  if ((threadIdx.x & 31) == 0) {
    sm[2 * w] = s;
    sm[2 * w + 1] = q;
  }
  __syncthreads();
  s = 0.0;
  q = 0.0;
  for (int i = 0; i < nw; ++i) {
    s += sm[2 * i];
    q += sm[2 * i + 1];
  }
}

template <int HID>
__global__ void __launch_bounds__(kRowMaxThreads) dconv_row_kernel(const DconvParams p) {
  constexpr int HP = (HID + 3) / 4 * 4;
  extern __shared__ __align__(16) float smem_dc[];
  const int C = p.C, L = p.L;
  float* xs = smem_dc;                        // [C][L]
  float* us = xs + (size_t)C * L;             // [HP][L]: u, then h = GELU(GN(u)) in place
  float* w0s = us + (size_t)HP * L;           // [C][3][HP]
  float* w3s = w0s + (size_t)C * 3 * HP;      // [C][2][HP]: rows c (value) and C + c (gate) of w3
  float* cst = w3s + (size_t)C * 2 * HP;      // [C][8]: b3[c], b3[C+c], g4[c], be4[c], g4[C+c], be4[C+c], ls[c], -
  float* k1s = cst + (size_t)C * 8;           // [HP][4]: b0, g1, be1, -
  __shared__ double red[2 * kRowMaxThreads / 32];
  const int NT = blockDim.x;
  for (int i = threadIdx.x; i < HP * C * 3; i += NT) {
    const int k = i / (C * 3), r = i - k * (C * 3);  // w0 is (HID, C, 3): r = c*3 + t
    w0s[r * HP + k] = k < HID ? __ldg(&p.w0[i]) : 0.f;
  }
  for (int i = threadIdx.x; i < 2 * C * HP; i += NT) {
    const int row = i / HP, k = i - row * HP;  // w3 is (2C, HID)
    const int c = row < C ? row : row - C, half = row < C ? 0 : 1;
    w3s[(c * 2 + half) * HP + k] = k < HID ? __ldg(&p.w3[row * HID + k]) : 0.f;
  }
  for (int c = threadIdx.x; c < C; c += NT) {
    float* o = cst + c * 8;
    o[0] = __ldg(&p.b3[c]); o[1] = __ldg(&p.b3[C + c]);
    o[2] = __ldg(&p.g4[c]); o[3] = __ldg(&p.be4[c]); o[4] = __ldg(&p.g4[C + c]); o[5] = __ldg(&p.be4[C + c]);
    o[6] = __ldg(&p.ls[c]); o[7] = 0.f;
  }
  for (int k = threadIdx.x; k < HP; k += NT) {
    k1s[k * 4] = k < HID ? __ldg(&p.b0[k]) : 0.f;
    k1s[k * 4 + 1] = k < HID ? __ldg(&p.g1[k]) : 0.f;
    k1s[k * 4 + 2] = k < HID ? __ldg(&p.be1[k]) : 0.f;
    k1s[k * 4 + 3] = 0.f;
  }
  const int samples = p.B * p.Fr;
  const int64_t cs = (int64_t)p.Fr * L;
  for (int sample = blockIdx.x; sample < samples; sample += gridDim.x) {
    const int b = sample / p.Fr, fr = sample - b * p.Fr;
    const float* xr = p.x + ((int64_t)b * C * p.Fr + fr) * L;
    float* yr = p.y + ((int64_t)b * C * p.Fr + fr) * L;
    __syncthreads();  // the previous row's xs / us are dead (and the staged weights are visible)
    for (int i = threadIdx.x; i < C * L; i += NT) {
      const int c = i / L, l = i - c * L;
      xs[i] = __ldg(&xr[(int64_t)c * cs + l]);
    }
    __syncthreads();
    // ---- u = conv3(x) + b0 and its statistics
    double s = 0.0, q = 0.0;
    for (int l = threadIdx.x; l < L; l += NT) {
      float acc[HP];
#pragma unroll
      for (int k = 0; k < HP; ++k) acc[k] = k1s[k * 4];
      for (int c = 0; c < C; ++c) {
        const float* xc = xs + (size_t)c * L;
        const float* wc = w0s + c * 3 * HP;
#pragma unroll
        for (int t = 0; t < 3; ++t) {
          const int ll = l + (t - 1) * p.dil;
          const float xv = (ll >= 0 && ll < L) ? xc[ll] : 0.f;
#pragma unroll
          for (int k4 = 0; k4 < HP; k4 += 4) {
            const float4 w = *reinterpret_cast<const float4*>(&wc[t * HP + k4]);
            acc[k4] = fmaf(w.x, xv, acc[k4]);
            acc[k4 + 1] = fmaf(w.y, xv, acc[k4 + 1]);
            acc[k4 + 2] = fmaf(w.z, xv, acc[k4 + 2]);
            acc[k4 + 3] = fmaf(w.w, xv, acc[k4 + 3]);
          }
        }
      }
      float fs = 0.f, fq = 0.f;
#pragma unroll
      for (int k = 0; k < HID; ++k) {
        us[(size_t)k * L + l] = acc[k];
        fs += acc[k];
        fq = fmaf(acc[k], acc[k], fq);
      }
      s += fs;
      q += fq;
    }
    row_sum2(s, q, red);
    const double nu = (double)HID * L;
    const double mu_d = s / nu;
    double var_u = q / nu - mu_d * mu_d;
    if (var_u < 0.0) var_u = 0.0;
    const float mu = (float)mu_d, ru = (float)(1.0 / sqrt(var_u + 1e-5));
    // ---- h = GELU(GN(u)) kept in registers per position; z = W3 h + b3: statistics first, then the output
    double sz = 0.0, qz = 0.0;
    for (int l = threadIdx.x; l < L; l += NT) {
      float h[HP];
#pragma unroll
      for (int k = 0; k < HP; ++k) h[k] = k < HID ? gelu_erf(fmaf((us[(size_t)k * L + l] - mu) * ru, k1s[k * 4 + 1], k1s[k * 4 + 2])) : 0.f;
#pragma unroll
      for (int k = 0; k < HID; ++k) us[(size_t)k * L + l] = h[k];  // only this thread touches column l
      float fs = 0.f, fq = 0.f;
      for (int c = 0; c < C; ++c) {
        const float* wc = w3s + c * 2 * HP;
        float a = cst[c * 8], g = cst[c * 8 + 1];
#pragma unroll
        for (int k = 0; k < HP; k += 4) {
          const float4 wa = *reinterpret_cast<const float4*>(&wc[k]);
          const float4 wg = *reinterpret_cast<const float4*>(&wc[HP + k]);
          a = fmaf(wa.x, h[k], a); a = fmaf(wa.y, h[k + 1], a); a = fmaf(wa.z, h[k + 2], a); a = fmaf(wa.w, h[k + 3], a);
          g = fmaf(wg.x, h[k], g); g = fmaf(wg.y, h[k + 1], g); g = fmaf(wg.z, h[k + 2], g); g = fmaf(wg.w, h[k + 3], g);
        }
        fs += a + g;
        fq = fmaf(a, a, fmaf(g, g, fq));
      }
      sz += fs;
      qz += fq;
    }
    row_sum2(sz, qz, red);
    const double nz = 2.0 * C * L;
    const double mz_d = sz / nz;
    double var_z = qz / nz - mz_d * mz_d;
    if (var_z < 0.0) var_z = 0.0;
    const float mz = (float)mz_d, rz = (float)(1.0 / sqrt(var_z + 1e-5));
    for (int l = threadIdx.x; l < L; l += NT) {
      float h[HP];
#pragma unroll
      for (int k = 0; k < HP; ++k) h[k] = k < HID ? us[(size_t)k * L + l] : 0.f;
      for (int c = 0; c < C; ++c) {
        const float* wc = w3s + c * 2 * HP;
        const float4 k0 = *reinterpret_cast<const float4*>(&cst[c * 8]);
        const float4 k1 = *reinterpret_cast<const float4*>(&cst[c * 8 + 4]);
        float a = k0.x, g = k0.y;
#pragma unroll
        for (int k = 0; k < HP; k += 4) {
          const float4 wa = *reinterpret_cast<const float4*>(&wc[k]);
          const float4 wg = *reinterpret_cast<const float4*>(&wc[HP + k]);
          a = fmaf(wa.x, h[k], a); a = fmaf(wa.y, h[k + 1], a); a = fmaf(wa.z, h[k + 2], a); a = fmaf(wa.w, h[k + 3], a);
          g = fmaf(wg.x, h[k], g); g = fmaf(wg.y, h[k + 1], g); g = fmaf(wg.z, h[k + 2], g); g = fmaf(wg.w, h[k + 3], g);
        }
        const float an = fmaf((a - mz) * rz, k0.z, k0.w);
        const float gn = fmaf((g - mz) * rz, k1.x, k1.y);
        yr[(int64_t)c * cs + l] = xs[(size_t)c * L + l] + k1.z * (an / (1.f + expf(-gn)));
      }
    }
  }
}

template <int HID>
size_t dconv_row_smem(int C, int L) {
  constexpr int HP = (HID + 3) / 4 * 4;
  return ((size_t)C * L + (size_t)HP * L + (size_t)C * 3 * HP + (size_t)C * 2 * HP + (size_t)C * 8 + (size_t)HP * 4) * sizeof(float);
}

template <int HID>
int dconv_row_launch(const DconvParams& p, cudaStream_t st) {
  const size_t smem = dconv_row_smem<HID>(p.C, p.L);
  static bool attr_set[kMaxDevices] = {};
  B2_DEVICE_SLOT(dev);
  if (!attr_set[dev]) {
    B2_CUDA(cudaFuncSetAttribute(dconv_row_kernel<HID>, cudaFuncAttributeMaxDynamicSharedMemorySize, 220 * 1024));
    attr_set[dev] = true;
  }
  const int threads = std::min(kRowMaxThreads, std::max(128, (p.L + 31) / 32 * 32));
  const int per_sm = (int)std::max<size_t>(1, std::min<size_t>(4, (220 * 1024) / smem));
  dconv_row_kernel<HID><<<std::min(p.B * p.Fr, kNumSMs * per_sm), threads, smem, st>>>(p);
  B2_LAUNCHED();
  return B200SEP_OK;
}

int dconv_positions_per_thread(int L) { return L >= 2048 ? 2 : 1; }

}  // namespace
}  // namespace b200sep

using namespace b200sep;

extern "C" int64_t b200sep_dconv_work_floats(int B, int C, int Fr, int64_t L, int hid) {
  if (B < 1 || C < 1 || Fr < 1 || L < 1 || hid < 1) return 0;
  const int64_t samples = (int64_t)B * Fr;
  const int64_t nblk = cdiv(L, kDcThreads * dconv_positions_per_thread((int)L));
  // u | part_u, part_z (double2 = 4 floats each) | stat_u, stat_z (float2); every section 16-byte aligned
  return ((int64_t)B * hid * Fr * L + 3) / 4 * 4 + 2 * samples * nblk * 4 + 2 * ((samples * 2 + 3) / 4 * 4);
}

extern "C" int b200sep_dconv_f32(const float* x, float* y, const float* w0, const float* b0, const float* g1, const float* be1, const float* w3, const float* b3,
                                 const float* g4, const float* be4, const float* ls, int B, int C, int Fr, int64_t L, int hid, int dilation, const float* u_in,
                                 float* work, void* stream) {
  B2_CHECK_ARG(x && y && b0 && g1 && be1 && w3 && b3 && g4 && be4 && ls && work && (w0 || u_in), "dconv_f32: NULL argument");
  B2_CHECK_ARG(B >= 1 && C >= 1 && Fr >= 1 && L >= 1 && L < (1ll << 30) && dilation >= 1, "dconv_f32: bad sizes");
  B2_CHECK_ARG((reinterpret_cast<uintptr_t>(work) & 15) == 0, "dconv_f32: work must be 16-byte aligned");
  const int64_t samples = (int64_t)B * Fr;
  const int P = dconv_positions_per_thread((int)L);
  const int64_t nblk = cdiv(L, kDcThreads * P);
  DconvParams p{};
  p.x = x; p.y = y; p.w0 = w0; p.b0 = b0; p.g1 = g1; p.be1 = be1; p.w3 = w3; p.b3 = b3; p.g4 = g4; p.be4 = be4; p.ls = ls;
  float* cur = work;
  p.u = u_in ? const_cast<float*>(u_in) : cur;
  cur += ((int64_t)B * hid * Fr * L + 3) / 4 * 4;
  p.part_u = reinterpret_cast<double2*>(cur); cur += samples * nblk * 4;
  p.part_z = reinterpret_cast<double2*>(cur); cur += samples * nblk * 4;
  p.stat_u = reinterpret_cast<float2*>(cur); cur += (samples * 2 + 3) / 4 * 4;
  p.stat_z = reinterpret_cast<float2*>(cur);
  p.B = B; p.C = C; p.Fr = Fr; p.L = (int)L; p.dil = dilation;
  cudaStream_t st = (cudaStream_t)stream;
  const bool have_u = u_in != nullptr;
  // rows that fit in shared memory (the frequency branch) take the single-pass kernel
  if (!have_u && Fr > 1 && L <= 4096) {
#define B2_DCONV_ROW_CASE(h) \
  if (hid == h && dconv_row_smem<h>(C, (int)L) <= 216 * 1024) return dconv_row_launch<h>(p, st);
    B2_DCONV_ROW_CASE(6)
    B2_DCONV_ROW_CASE(12)
    B2_DCONV_ROW_CASE(24)
    B2_DCONV_ROW_CASE(4)
    B2_DCONV_ROW_CASE(8)
    B2_DCONV_ROW_CASE(16)
#undef B2_DCONV_ROW_CASE
  }
#define B2_DCONV_CASE(h)                                                   \
  if (hid == h) return P == 2 ? dconv_launch<h, 2>(p, have_u, st) : dconv_launch<h, 1>(p, have_u, st);
  B2_DCONV_CASE(6)
  B2_DCONV_CASE(12)
  B2_DCONV_CASE(24)
  B2_DCONV_CASE(48)
  B2_DCONV_CASE(4)
  B2_DCONV_CASE(8)
  B2_DCONV_CASE(16)
  B2_DCONV_CASE(32)
#undef B2_DCONV_CASE
  set_error("dconv_f32: hidden width %d has no kernel instance (4, 6, 8, 12, 16, 24, 32, 48)", hid);
  return B200SEP_ERR_ARG;
}
