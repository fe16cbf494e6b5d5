// FP32 SIMT operators (see simt_ops.cuh).  Register-tiled implicit-GEMM convolution and a TN SGEMM.
#include "simt_ops.cuh"

#include <cuda_bf16.h>

namespace b200sep {

using bf16 = __nv_bfloat16;
__device__ __forceinline__ float pair_load(const void* hi, const void* lo, int64_t i) {
  return __bfloat162float(static_cast<const bf16*>(hi)[i]) + __bfloat162float(static_cast<const bf16*>(lo)[i]);
}
__device__ __forceinline__ void pair_store(void* hi, void* lo, int64_t i, float v) {
  const bf16 h = __float2bfloat16_rn(v);
  static_cast<bf16*>(hi)[i] = h;
  static_cast<bf16*>(lo)[i] = __float2bfloat16_rn(v - __bfloat162float(h));
}

// ---------------------------------------------------------------------------------------------------------
// conv2d: block tile = 128 (w) x 2 (h) output pixels x 48 output channels, 256 threads,
// thread tile = 4 consecutive w x 12 channels.  Input channels are staged 8 at a time through shared memory.
constexpr int TW = 128, TH = 2, TCO = 48, CI = 8, CONV_NT = 256;

template <int KH, int KW, int S>
struct ConvGeom {
  static constexpr int PAD = (S == 1) ? (KH - 1) / 2 : 0;
  static constexpr int ROWS = (TH - 1) * S + KH;
  static constexpr int COLS = (TW - 1) * S + KW;
  static constexpr int OFF = (4 - PAD) % 4;  // so that the thread's first non-halo column is 16-byte aligned
  static constexpr int COLS_PAD = ((OFF + COLS + 3) / 4) * 4 + 4;
  static constexpr int TAPS = KH * KW;
  static constexpr int XV = 3 * S + KW;
  static constexpr int SMEM_FLOATS = CI * ROWS * COLS_PAD + CI * TAPS * TCO;
};

template <int KH, int KW, int S>
__global__ void __launch_bounds__(CONV_NT) conv2d_simt_kernel(ConvParams p) {
  using G = ConvGeom<KH, KW, S>;
  extern __shared__ float smem_f[];
  float* in_s = smem_f;                             // [CI][ROWS][COLS_PAD]
  float* w_s = smem_f + CI * G::ROWS * G::COLS_PAD;  // [CI][TAPS][TCO]

  const int tid = threadIdx.x;
  const int tx = tid & 31, ty = (tid >> 5) & 1, tc = tid >> 6;
  const int n_cot = p.CoutPad / TCO;
  const int cot = blockIdx.z % n_cot, b = blockIdx.z / n_cot;
  const int co0 = cot * TCO;
  const int w0 = blockIdx.x * TW, h0 = blockIdx.y * TH;

  float acc[4][12];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 12; ++j) acc[i][j] = 0.f;

  const int64_t xoff = (int64_t)b * p.Cin * p.H * p.W;
  const float* xb = p.x + xoff;
  for (int ci0 = 0; ci0 < p.Cin; ci0 += CI) {
    for (int idx = tid; idx < CI * G::ROWS * G::COLS; idx += CONV_NT) {
      const int c = idx % G::COLS;
      const int r = (idx / G::COLS) % G::ROWS;
      const int ci = idx / (G::COLS * G::ROWS);
      const int hi = h0 * S - G::PAD + r, wi = w0 * S - G::PAD + c;
      float v = 0.f;
      if (ci0 + ci < p.Cin && hi >= 0 && hi < p.H && wi >= 0 && wi < p.W) {
        const int64_t xi = ((int64_t)(ci0 + ci) * p.H + hi) * p.W + wi;
        v = p.x_lo ? pair_load(p.x, p.x_lo, xoff + xi) : __ldg(&xb[xi]);
      }
      in_s[(ci * G::ROWS + r) * G::COLS_PAD + G::OFF + c] = v;
    }
    for (int idx = tid; idx < CI * G::TAPS * (TCO / 4); idx += CONV_NT) {
      const int q = idx % (TCO / 4);
      const int tap = (idx / (TCO / 4)) % G::TAPS;
      const int ci = idx / ((TCO / 4) * G::TAPS);
      float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
      if (ci0 + ci < p.Cin) v = __ldg(reinterpret_cast<const float4*>(&p.w[((int64_t)(ci0 + ci) * G::TAPS + tap) * p.CoutPad + co0 + q * 4]));
      *reinterpret_cast<float4*>(&w_s[(ci * G::TAPS + tap) * TCO + q * 4]) = v;
    }
    __syncthreads();
#pragma unroll 2
    for (int ci = 0; ci < CI; ++ci) {
#pragma unroll
      for (int kh = 0; kh < KH; ++kh) {
        const float* row = &in_s[(ci * G::ROWS + ty * S + kh) * G::COLS_PAD + G::OFF + 4 * S * tx];
        float xv[G::XV];
#pragma unroll
        for (int j = 0; j < G::XV; ++j) xv[j] = row[j];
#pragma unroll
        for (int kw = 0; kw < KW; ++kw) {
          const float4* wp = reinterpret_cast<const float4*>(&w_s[(ci * G::TAPS + kh * KW + kw) * TCO + tc * 12]);
          const float4 wa = wp[0], wb = wp[1], wc = wp[2];
          const float wv[12] = {wa.x, wa.y, wa.z, wa.w, wb.x, wb.y, wb.z, wb.w, wc.x, wc.y, wc.z, wc.w};
#pragma unroll
          for (int i = 0; i < 4; ++i)
#pragma unroll
            for (int j = 0; j < 12; ++j) acc[i][j] = fmaf(xv[i * S + kw], wv[j], acc[i][j]);
        }
      }
    }
    __syncthreads();
  }

  const int h = h0 + ty;
  if (h >= p.Ho) return;
  const int wbase = w0 + 4 * tx;
#pragma unroll
  for (int j = 0; j < 12; ++j) {
    const int co = co0 + tc * 12 + j;
    if (co >= p.Cout) continue;
    const float sc = __ldg(&p.scale[co]), sh = __ldg(&p.shift[co]);
    if (p.epilogue == EPI_NORMAL) {
      const int64_t o = (((int64_t)b * p.Cout + co) * p.Ho + h) * p.Wo + wbase;
      float v[4];
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        v[i] = fmaf(acc[i][j], sc, sh);
        if (p.relu) v[i] = fmaxf(v[i], 0.f);
      }
      if (p.y_lo || p.mul_lo) {
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          if (wbase + i >= p.Wo) continue;
          float r = v[i];
          if (p.mul) r *= p.mul_lo ? pair_load(p.mul, p.mul_lo, o + i) : __ldg(&p.mul[o + i]);
          if (p.y_lo) pair_store(p.y, p.y_lo, o + i, r);
          else p.y[o + i] = r;
        }
      } else if (wbase + 3 < p.Wo && (p.Wo & 3) == 0) {
        if (p.mul) {
          const float4 m = __ldg(reinterpret_cast<const float4*>(&p.mul[o]));
          v[0] *= m.x; v[1] *= m.y; v[2] *= m.z; v[3] *= m.w;
        }
        *reinterpret_cast<float4*>(&p.y[o]) = make_float4(v[0], v[1], v[2], v[3]);
      } else {
#pragma unroll
        for (int i = 0; i < 4; ++i)
          if (wbase + i < p.Wo) p.y[o + i] = p.mul ? v[i] * __ldg(&p.mul[o + i]) : v[i];
      }
    } else {  // EPI_CONVT2X2
      const int cr = p.Cout / 4;
      const int q = co / cr, c = co - q * cr;
      const int dy = q >> 1, dx = q & 1;
      const int H2 = p.Ho * 2, W2 = p.Wo * 2;
      const int64_t orow = (((int64_t)b * cr + c) * H2 + 2 * h + dy) * W2;
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        if (wbase + i >= p.Wo) continue;
        float v = fmaf(acc[i][j], sc, sh);
        if (p.relu) v = fmaxf(v, 0.f);
        const int64_t o = orow + 2 * (wbase + i) + dx;
        if (p.mul) v *= p.mul_lo ? pair_load(p.mul, p.mul_lo, o) : __ldg(&p.mul[o]);
        if (p.y_lo) pair_store(p.y, p.y_lo, o, v);
        else p.y[o] = v;
      }
    }
  }
}

template <int KH, int KW, int S>
static int launch_conv(const ConvParams& p, cudaStream_t stream) {
  using G = ConvGeom<KH, KW, S>;
  const int smem = G::SMEM_FLOATS * (int)sizeof(float);
  static bool attr_set[kMaxDevices] = {};
  B2_DEVICE_SLOT(dev);
  if (!attr_set[dev]) {
    B2_CUDA(cudaFuncSetAttribute(conv2d_simt_kernel<KH, KW, S>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    attr_set[dev] = true;
  }
  dim3 grid(cdiv(p.Wo, TW), cdiv(p.Ho, TH), p.B * (p.CoutPad / TCO));
  B2_CHECK_ARG(grid.y <= 65535 && grid.z <= 65535, "conv2d_simt: grid too large (Ho=%d, B*co_tiles=%d)", p.Ho, (int)grid.z);
  conv2d_simt_kernel<KH, KW, S><<<grid, CONV_NT, smem, stream>>>(p);
  B2_LAUNCHED();
  return B200SEP_OK;
}

int conv2d_simt(const ConvParams& p, int KH, int KW, int S, cudaStream_t stream) {
  B2_CHECK_ARG(p.CoutPad % TCO == 0 && p.Cout <= p.CoutPad, "conv2d_simt: CoutPad=%d must be a multiple of %d", p.CoutPad, TCO);
  if (KH == 3 && KW == 3 && S == 1) return launch_conv<3, 3, 1>(p, stream);
  if (KH == 1 && KW == 1 && S == 1) return launch_conv<1, 1, 1>(p, stream);
  if (KH == 2 && KW == 2 && S == 2) return launch_conv<2, 2, 2>(p, stream);
  set_error("conv2d_simt: unsupported kernel %dx%d stride %d", KH, KW, S);
  return B200SEP_ERR_ARG;
}

// ---------------------------------------------------------------------------------------------------------
// SGEMM TN: C[M][N] = A[M][K] * Bw[N][K]^T, 128x128x16 block tile, 8x8 thread tile
constexpr int BM = 128, BN = 128, BK = 16, GEMM_NT = 256;

__global__ void __launch_bounds__(GEMM_NT) gemm_tn_simt_kernel(GemmParams p) {
  __shared__ __align__(16) float As[BK][BM + 4];
  __shared__ __align__(16) float Bs[BK][BN + 4];
  const int tid = threadIdx.x;
  const int tx = tid & 15, ty = tid >> 4;
  const int m0 = blockIdx.y * BM, n0 = blockIdx.x * BN;
  const bool vec = (p.K & 3) == 0 && p.A_lo == nullptr;  // float4 global loads need 16-byte aligned fp32 rows
  float acc[8][8];
#pragma unroll
  for (int i = 0; i < 8; ++i)
#pragma unroll
    for (int j = 0; j < 8; ++j) acc[i][j] = 0.f;

  for (int k0 = 0; k0 < p.K; k0 += BK) {
#pragma unroll
    for (int it = 0; it < 2; ++it) {
      const int idx = tid + it * GEMM_NT;
      const int row = idx >> 2, kq = idx & 3;
      const int k = k0 + kq * 4;
      float4 a = make_float4(0.f, 0.f, 0.f, 0.f), bb = a;
      if (vec) {
        if (m0 + row < p.M && k < p.K) a = __ldg(reinterpret_cast<const float4*>(&p.A[(int64_t)(m0 + row) * p.K + k]));
        if (n0 + row < p.N && k < p.K) bb = __ldg(reinterpret_cast<const float4*>(&p.Bw[(int64_t)(n0 + row) * p.K + k]));
      } else {
        float av[4] = {0.f, 0.f, 0.f, 0.f}, bv[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          if (m0 + row < p.M && k + e < p.K) {
            const int64_t ai = (int64_t)(m0 + row) * p.K + k + e;
            av[e] = p.A_lo ? pair_load(p.A, p.A_lo, ai) : __ldg(&p.A[ai]);
          }
          if (n0 + row < p.N && k + e < p.K) bv[e] = __ldg(&p.Bw[(int64_t)(n0 + row) * p.K + k + e]);
        }
        a = make_float4(av[0], av[1], av[2], av[3]);
        bb = make_float4(bv[0], bv[1], bv[2], bv[3]);
      }
      As[kq * 4 + 0][row] = a.x; As[kq * 4 + 1][row] = a.y; As[kq * 4 + 2][row] = a.z; As[kq * 4 + 3][row] = a.w;
      Bs[kq * 4 + 0][row] = bb.x; Bs[kq * 4 + 1][row] = bb.y; Bs[kq * 4 + 2][row] = bb.z; Bs[kq * 4 + 3][row] = bb.w;
    }
    __syncthreads();
#pragma unroll
    for (int k = 0; k < BK; ++k) {
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
    const int r = m0 + ty * 8 + i;
    if (r >= p.M) continue;
    const int c = (r / p.rows_per_channel) % p.channels;
    const float sc = p.scale ? __ldg(&p.scale[c]) : 1.f, sh = p.shift ? __ldg(&p.shift[c]) : 0.f;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const int n = n0 + tx * 8 + j;
      if (n >= p.N) continue;
      float v = fmaf(acc[i][j], sc, sh);
      if (p.relu) v = fmaxf(v, 0.f);
      const int64_t o = (int64_t)r * p.N + n;
      if (p.res) v += p.res_lo ? pair_load(p.res, p.res_lo, o) : p.res[o];
      if (p.C_lo) pair_store(p.C, p.C_lo, o, v);
      else p.C[o] = v;
    }
  }
}

int gemm_tn_simt(const GemmParams& p, cudaStream_t stream) {
  B2_CHECK_ARG(p.M > 0 && p.N > 0 && p.rows_per_channel > 0 && p.channels > 0, "gemm_tn_simt: bad sizes");
  dim3 grid(cdiv(p.N, BN), cdiv(p.M, BM));
  B2_CHECK_ARG(grid.y <= 65535, "gemm_tn_simt: M=%d too large", p.M);
  gemm_tn_simt_kernel<<<grid, GEMM_NT, 0, stream>>>(p);
  B2_LAUNCHED();
  return B200SEP_OK;
}

// ---------------------------------------------------------------------------------------------------------
// Bandwidth-bound 1x1 convolutions at the network's ends in pair mode (8 pixels per thread, 16-byte plane accesses).
// first: fp32 (B,Cin<=8,P) -> pair (B,Cout,P) with BN+ReLU;  last: pair (B,Cin,P) -> fp32 (B,Cout<=8,P), bias only.
__global__ void __launch_bounds__(256) pointwise_first_kernel(const float* __restrict__ x, const float* __restrict__ w, int w_stride,
                                                             const float* __restrict__ scale, const float* __restrict__ shift, int relu, bf16* __restrict__ y_hi,
                                                             bf16* __restrict__ y_lo, int Cin, int Cout, int64_t P) {
  const int b = blockIdx.y;
  const int64_t p0 = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) * 8;
  if (p0 >= P) return;
  float xv[8][8];
  for (int ci = 0; ci < Cin; ++ci) {
    const float4* s = reinterpret_cast<const float4*>(x + ((int64_t)b * Cin + ci) * P + p0);
    const float4 a = __ldg(s), c = __ldg(s + 1);
    xv[ci][0] = a.x; xv[ci][1] = a.y; xv[ci][2] = a.z; xv[ci][3] = a.w; xv[ci][4] = c.x; xv[ci][5] = c.y; xv[ci][6] = c.z; xv[ci][7] = c.w;
  }
  for (int co = 0; co < Cout; ++co) {
    float acc[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
    for (int ci = 0; ci < Cin; ++ci) {
      const float wv = __ldg(&w[ci * w_stride + co]);
#pragma unroll
      for (int i = 0; i < 8; ++i) acc[i] = fmaf(xv[ci][i], wv, acc[i]);
    }
    const float sc = __ldg(&scale[co]), sh = __ldg(&shift[co]);
    __align__(16) bf16 h[8];
    __align__(16) bf16 l[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      float v = fmaf(acc[i], sc, sh);
      if (relu) v = fmaxf(v, 0.f);
      h[i] = __float2bfloat16_rn(v);
      l[i] = __float2bfloat16_rn(v - __bfloat162float(h[i]));
    }
    const int64_t o = ((int64_t)b * Cout + co) * P + p0;
    *reinterpret_cast<uint4*>(y_hi + o) = *reinterpret_cast<const uint4*>(h);
    *reinterpret_cast<uint4*>(y_lo + o) = *reinterpret_cast<const uint4*>(l);
  }
}

__global__ void __launch_bounds__(256) pointwise_last_kernel(const bf16* __restrict__ x_hi, const bf16* __restrict__ x_lo, const float* __restrict__ w, int w_stride,
                                                            const float* __restrict__ scale, const float* __restrict__ shift, int relu, float* __restrict__ y, int Cin,
                                                            int Cout, int64_t P) {
  const int b = blockIdx.y;
  const int64_t p0 = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) * 8;
  if (p0 >= P) return;
  float acc[8][8];
#pragma unroll
  for (int co = 0; co < 8; ++co)
#pragma unroll
    for (int i = 0; i < 8; ++i) acc[co][i] = 0.f;
  for (int ci = 0; ci < Cin; ++ci) {
    const int64_t o = ((int64_t)b * Cin + ci) * P + p0;
    const uint4 hv = __ldg(reinterpret_cast<const uint4*>(x_hi + o)), lv = __ldg(reinterpret_cast<const uint4*>(x_lo + o));
    const bf16* h = reinterpret_cast<const bf16*>(&hv);
    const bf16* l = reinterpret_cast<const bf16*>(&lv);
    float v[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) v[i] = __bfloat162float(h[i]) + __bfloat162float(l[i]);
#pragma unroll
    for (int co = 0; co < 8; ++co) {
      if (co < Cout) {
        const float wv = __ldg(&w[ci * w_stride + co]);
#pragma unroll
        for (int i = 0; i < 8; ++i) acc[co][i] = fmaf(v[i], wv, acc[co][i]);
      }
    }
  }
#pragma unroll
  for (int co = 0; co < 8; ++co) {
    if (co < Cout) {
      const float sc = __ldg(&scale[co]), sh = __ldg(&shift[co]);
      float r[8];
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        r[i] = fmaf(acc[co][i], sc, sh);
        if (relu) r[i] = fmaxf(r[i], 0.f);
      }
      float4* d = reinterpret_cast<float4*>(y + ((int64_t)b * Cout + co) * P + p0);
      d[0] = make_float4(r[0], r[1], r[2], r[3]);
      d[1] = make_float4(r[4], r[5], r[6], r[7]);
    }
  }
}

bool pointwise_pair_supported(int Cin, int Cout, int64_t P, int first) { return P % 8 == 0 && (first ? Cin <= 8 : Cout <= 8); }

int pointwise_first_pair(const float* x, const float* w, int w_stride, const float* scale, const float* shift, int relu, void* y_hi, void* y_lo, int B, int Cin,
                         int Cout, int64_t P, cudaStream_t st) {
  dim3 grid(cdiv(P / 8, 256), B);
  pointwise_first_kernel<<<grid, 256, 0, st>>>(x, w, w_stride, scale, shift, relu, (bf16*)y_hi, (bf16*)y_lo, Cin, Cout, P);
  B2_LAUNCHED();
  return B200SEP_OK;
}
int pointwise_last_pair(const void* x_hi, const void* x_lo, const float* w, int w_stride, const float* scale, const float* shift, int relu, float* y, int B, int Cin,
                        int Cout, int64_t P, cudaStream_t st) {
  dim3 grid(cdiv(P / 8, 256), B);
  pointwise_last_kernel<<<grid, 256, 0, st>>>((const bf16*)x_hi, (const bf16*)x_lo, w, w_stride, scale, shift, relu, y, Cin, Cout, P);
  B2_LAUNCHED();
  return B200SEP_OK;
}

// ---------------------------------------------------------------------------------------------------------
__global__ void transpose_hw_kernel(const float* __restrict__ x, float* __restrict__ y, int H, int W) {
  __shared__ float tile[32][33];
  const int64_t plane = (int64_t)blockIdx.z * H * W;
  const int w0 = blockIdx.x * 32, h0 = blockIdx.y * 32;
  for (int i = threadIdx.y; i < 32; i += blockDim.y) {
    const int h = h0 + i, w = w0 + threadIdx.x;
    tile[i][threadIdx.x] = (h < H && w < W) ? x[plane + (int64_t)h * W + w] : 0.f;
  }
  __syncthreads();
  for (int i = threadIdx.y; i < 32; i += blockDim.y) {
    const int w = w0 + i, h = h0 + threadIdx.x;
    if (h < H && w < W) y[plane + (int64_t)w * H + h] = tile[threadIdx.x][i];
  }
}

int transpose_hw(const float* x, float* y, int planes, int H, int W, cudaStream_t stream) {
  dim3 grid(cdiv(W, 32), cdiv(H, 32), planes);
  B2_CHECK_ARG(grid.y <= 65535 && grid.z <= 65535, "transpose_hw: grid too large");
  transpose_hw_kernel<<<grid, dim3(32, 8), 0, stream>>>(x, y, H, W);
  B2_LAUNCHED();
  return B200SEP_OK;
}

}  // namespace b200sep
