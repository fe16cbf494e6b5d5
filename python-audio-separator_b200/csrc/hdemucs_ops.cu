// Operators of the Hybrid Demucs v3 DConv branches (uvr_lib_v5/demucs/demucs.py:19-67 BLSTM, :171-231 LocalState): the recurrence of a
// bidirectional LSTM whose recurrent matrix does not fit one SM (a thread-block cluster splits the hidden units and exchanges h_t through
// distributed shared memory), the overlapping-frame gather / scatter around it, and the LocalState attention as one flash-style kernel.
#include <cooperative_groups.h>

#include <algorithm>

#include "common.cuh"

namespace cg = cooperative_groups;

namespace b200sep {
namespace {

__device__ __forceinline__ float sigmoidf_(float v) { return 1.f / (1.f + expf(-v)); }

// ----------------------------------------------------------------------------------------------------------------------------------
// BLSTM framing (demucs.py:38-45, utils.py:35-50 unfold): x (B, C, T) -> frames (width, B * nf, C); frame k of batch entry b holds
// samples [k * stride, k * stride + width) (zero beyond T).  nf = 1, width = T: the plain "b c t -> t b c" permute of an unframed input.
__global__ void lstm_frames_gather_kernel(const float* __restrict__ x, float* __restrict__ out, int B, int C, int T, int nf, int width, int stride, int64_t total) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int c = (int)(i % C);
    int64_t r = i / C;
    const int n = (int)(r % ((int64_t)B * nf));
    const int t = (int)(r / ((int64_t)B * nf));
    const int b = n / nf, k = n - b * nf;
    const int tt = k * stride + t;
    out[i] = tt < T ? __ldg(&x[((int64_t)b * C + c) * T + tt]) : 0.f;
  }
}

// The inverse (demucs.py:52-64): y[b, c, tt] = skip[b, c, tt] + frames[t, b * nf + k, c] where frame k contributes its samples
// [limit, width - limit) (the first frame from 0, the last frame to its end), limit = stride / 2.
__global__ void lstm_frames_scatter_kernel(const float* __restrict__ fr, const float* __restrict__ skip, float* __restrict__ y, int B, int C, int T, int nf, int width,
                                           int stride, int64_t total) {
  const int limit = stride / 2;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int tt = (int)(i % T);
    const int64_t bc = i / T;
    const int c = (int)(bc % C), b = (int)(bc / C);
    int k = 0;
    if (nf > 1 && tt >= width - limit) k = min((tt - limit) / stride, nf - 1);
    const int t = tt - k * stride;
    const float v = __ldg(&fr[((int64_t)t * B * nf + (int64_t)b * nf + k) * C + c]);
    y[i] = skip ? v + __ldg(&skip[i]) : v;
  }
}

// ----------------------------------------------------------------------------------------------------------------------------------
// Bidirectional LSTM recurrence for any hidden size.  One cluster of CL CTAs per (group of NS sequences, direction); CTA r owns the hidden
// units [r * UH, (r + 1) * UH) and the GL = 4 * UH gate columns that feed them.  Thread = (gate column, k-split kq of KS): NS accumulators over
// its quarter of the hidden dimension -- KS > 1 keeps KS times more weight loads in flight when the CTA's slice of W_hh^T does not fit shared
// memory and is streamed from L2 every step (the loop is latency-bound).  h_t is written into every CTA's shared memory (double-buffered),
// one cluster barrier per step.
template <int NS>
__global__ void __launch_bounds__(768) lstm_bidir_cluster_kernel(const float* __restrict__ xp, const float* __restrict__ whh_t, float* __restrict__ out, int T, int N, int hid, int w_in_smem,
                                          int KS) {
  cg::cluster_group cluster = cg::this_cluster();
  const int CL = (int)cluster.num_blocks();
  const int r = (int)cluster.block_rank();
  const int UH = hid / CL, GL = 4 * UH, G = 4 * hid;
  const int nthreads = GL * KS;
  const int tid = threadIdx.x;
  const int col = tid % GL, kq = tid / GL;
  const int gate = col / UH, ul = col - gate * UH;
  const int j = gate * hid + r * UH + ul;  // this thread's column of the (T, N, 4 * hid) gate pre-activations
  const int kspan = hid / KS, k_lo = kq * kspan, k_hi = k_lo + kspan;
  const int grp = blockIdx.x / CL, dir = blockIdx.y;
  const int n0 = grp * NS;
  extern __shared__ __align__(16) float lsm[];
  float* hs = lsm;                     // [2][hid][NS]
  float* gs = hs + 2 * hid * NS;       // [KS][NS][GL]
  float* cs = gs + KS * NS * GL;       // [UH][NS] cell states
  float* hl = cs + NS * UH;            // [UH][NS] this step's h slice before it is broadcast
  float* ws = hl + NS * UH;            // [hid][GL] when w_in_smem
  const float* w = whh_t + (int64_t)dir * hid * G;
  if (w_in_smem)
    for (int k = k_lo; k < k_hi; ++k) ws[k * GL + col] = __ldg(&w[(int64_t)k * G + j]);
  for (int i = tid; i < 2 * hid * NS; i += nthreads) hs[i] = 0.f;
  for (int i = tid; i < NS * UH; i += nthreads) cs[i] = 0.f;
  cluster.sync();  // every CTA's h buffers are zero before the first remote write can land
  const float* xpd = xp + (int64_t)dir * T * N * G;
  int cur = 0;
  for (int s = 0; s < T; ++s) {
    const int t = dir ? T - 1 - s : s;
    float acc[NS];
#pragma unroll
    for (int n = 0; n < NS; ++n) acc[n] = (kq == 0 && n0 + n < N) ? __ldg(&xpd[((int64_t)t * N + n0 + n) * G + j]) : 0.f;
    const float* hc = hs + cur * hid * NS;
    if (w_in_smem) {
#pragma unroll 4
      for (int k = k_lo; k < k_hi; ++k) {
        const float wv = ws[k * GL + col];
#pragma unroll
        for (int n = 0; n < NS; n += 4) {
          const float4 hv = *reinterpret_cast<const float4*>(&hc[k * NS + n]);
          acc[n] = fmaf(wv, hv.x, acc[n]);
          acc[n + 1] = fmaf(wv, hv.y, acc[n + 1]);
          acc[n + 2] = fmaf(wv, hv.z, acc[n + 2]);
          acc[n + 3] = fmaf(wv, hv.w, acc[n + 3]);
        }
      }
    } else {
#pragma unroll 16
      for (int k = k_lo; k < k_hi; ++k) {
        const float wv = __ldg(&w[(int64_t)k * G + j]);
#pragma unroll
        for (int n = 0; n < NS; n += 4) {
          const float4 hv = *reinterpret_cast<const float4*>(&hc[k * NS + n]);
          acc[n] = fmaf(wv, hv.x, acc[n]);
          acc[n + 1] = fmaf(wv, hv.y, acc[n + 1]);
          acc[n + 2] = fmaf(wv, hv.z, acc[n + 2]);
          acc[n + 3] = fmaf(wv, hv.w, acc[n + 3]);
        }
      }
    }
#pragma unroll
    for (int n = 0; n < NS; ++n) gs[(kq * NS + n) * GL + col] = acc[n];
    __syncthreads();
    float* hn = hs + (cur ^ 1) * hid * NS;
    for (int i = tid; i < NS * UH; i += nthreads) {
      const int u = i / NS, n = i - u * NS;  // n fastest: hl[u][n] below is written as contiguous rows
      float g4[4] = {0.f, 0.f, 0.f, 0.f};
      for (int q = 0; q < KS; ++q) {
        const float* gp = gs + (q * NS + n) * GL + u;
        g4[0] += gp[0];
        g4[1] += gp[UH];
        g4[2] += gp[2 * UH];
        g4[3] += gp[3 * UH];
      }
      const float ig = sigmoidf_(g4[0]), fg = sigmoidf_(g4[1]), gg = tanhf(g4[2]), og = sigmoidf_(g4[3]);
      const float c = fg * cs[i] + ig * gg;
      cs[i] = c;
      const float h = og * tanhf(c);
      if (n0 + n < N) out[((int64_t)t * N + n0 + n) * (2 * hid) + dir * hid + r * UH + u] = h;
      hl[i] = h;  // [UH][NS]: this CTA's slice of h_t
    }
    __syncthreads();
    // broadcast the slice into every CTA's next-step buffer as 16-byte distributed-shared-memory stores (one per thread at 768 threads), not 4-byte ones
    for (int i = tid; i < CL * UH * (NS / 4); i += nthreads) {
      const int q = i / (UH * (NS / 4)), w4 = i - q * (UH * (NS / 4));
      const float4 v = *reinterpret_cast<const float4*>(&hl[w4 * 4]);
      *reinterpret_cast<float4*>(&cluster.map_shared_rank(hn, q)[r * UH * NS + w4 * 4]) = v;
    }
    cluster.sync();  // h_t visible everywhere; gs / the other h buffer are free again
    cur ^= 1;
  }
}

// ----------------------------------------------------------------------------------------------------------------------------------
// LocalState attention (demucs.py:197-231, nfreqs = 0): for every (batch b, head h, query position s)
//   dots[t] = <key[:, t], query[:, s]> / sqrt(CH) - |t - s| * D[s],   D[s] = sum_f (f + 1) * sigmoid(decay[f, s]) / (2 sqrt(ndecay)),
//   dots[s] = -100,  w = softmax_t(dots),  out[:, s] = sum_t w[t] content[:, t].
// One warp per query; the 8 warps of a CTA share shared-memory tiles of 64 key positions; running softmax with a warp-uniform maximum
// so the CH lane-local accumulators are rescaled once per tile.
template <int CH>
__global__ void __launch_bounds__(256) local_state_attn_kernel(const float* __restrict__ q, const float* __restrict__ k, const float* __restrict__ content,
                                                               const float* __restrict__ decay, float* __restrict__ out, int C, int T, int nd) {
  constexpr int R = CH > 48 ? 1 : 2, TT = 32 * R;  // key positions per lane and per tile (two 24 KB tiles at CH = 48 and CH = 96)
  __shared__ float ks[CH][TT];
  __shared__ float cs[CH][TT];
  __shared__ float qs[8][CH];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int h = blockIdx.y, b = blockIdx.z, H = gridDim.y;
  const int s = blockIdx.x * 8 + warp;
  const int sq = min(s, T - 1);  // warps past the end compute a valid column and drop it
  const int64_t base = ((int64_t)b * C + (int64_t)h * CH) * T;
  for (int c = lane; c < CH; c += 32) qs[warp][c] = __ldg(&q[base + (int64_t)c * T + sq]);
  float D = 0.f;
  for (int f = 0; f < nd; ++f) D += (float)(f + 1) * sigmoidf_(__ldg(&decay[((int64_t)b * H * nd + (int64_t)h * nd + f) * T + sq]));
  D *= 0.5f / sqrtf((float)nd);
  const float scale = 1.f / sqrtf((float)CH);
  float m = -INFINITY, l = 0.f;
  float acc[CH];
#pragma unroll
  for (int c = 0; c < CH; ++c) acc[c] = 0.f;
  for (int t0 = 0; t0 < T; t0 += TT) {
    __syncthreads();
    for (int i = threadIdx.x; i < CH * TT; i += 256) {
      const int c = i / TT, tt = i - c * TT;
      const bool ok = t0 + tt < T;
      ks[c][tt] = ok ? __ldg(&k[base + (int64_t)c * T + t0 + tt]) : 0.f;
      cs[c][tt] = ok ? __ldg(&content[base + (int64_t)c * T + t0 + tt]) : 0.f;
    }
    __syncthreads();
    float d[R];
#pragma unroll
    for (int r = 0; r < R; ++r) d[r] = 0.f;
#pragma unroll
    for (int c = 0; c < CH; ++c) {
      const float qv = qs[warp][c];
#pragma unroll
      for (int r = 0; r < R; ++r) d[r] = fmaf(ks[c][lane + 32 * r], qv, d[r]);
    }
    float mx = -INFINITY;
#pragma unroll
    for (int r = 0; r < R; ++r) {
      const int t = t0 + lane + 32 * r;
      d[r] = t < T ? (t == sq ? -100.f : d[r] * scale - fabsf((float)(t - sq)) * D) : -INFINITY;
      mx = fmaxf(mx, d[r]);
    }
    for (int o = 16; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
    const float mn = fmaxf(m, mx);  // finite: lane 0's first position of every tile is < T
    const float corr = expf(m - mn);
    m = mn;
    l *= corr;
#pragma unroll
    for (int r = 0; r < R; ++r) {
      d[r] = expf(d[r] - mn);
      l += d[r];
    }
#pragma unroll
    for (int c = 0; c < CH; ++c) {
      float a = acc[c] * corr;
#pragma unroll
      for (int r = 0; r < R; ++r) a = fmaf(d[r], cs[c][lane + 32 * r], a);
      acc[c] = a;
    }
  }
  for (int o = 16; o > 0; o >>= 1) l += __shfl_xor_sync(0xffffffffu, l, o);
  const float inv = 1.f / l;
#pragma unroll
  for (int c = 0; c < CH; ++c) {
    float v = acc[c];
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    if (lane == (c & 31) && s < T) out[base + (int64_t)c * T + s] = v * inv;
  }
}

// x[b][r][l] += v[r]: the frequency embedding added after the first encoder (hdemucs.py:708-713), r = channel * Fr + fr
__global__ void add_rowvec_kernel(float* __restrict__ x, const float* __restrict__ v, int R, int L, int64_t total) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) x[i] += __ldg(&v[(i / L) % R]);
}

template <int CH>
int launch_local_state(const float* q, const float* k, const float* content, const float* decay, float* out, int B, int C, int T, int heads, int nd, cudaStream_t st) {
  dim3 grid(cdiv(T, 8), heads, B);
  local_state_attn_kernel<CH><<<grid, 256, 0, st>>>(q, k, content, decay, out, C, T, nd);
  B2_LAUNCHED();
  return B200SEP_OK;
}

static inline int ew_grid(int64_t n) { return (int)std::min<int64_t>(cdiv(n, 256), kNumSMs * 16); }

}  // namespace
}  // namespace b200sep

using namespace b200sep;

extern "C" int b200sep_add_rowvec_f32(float* x, const float* v, int B, int R, int64_t L, void* stream) {
  B2_CHECK_ARG(x && v && B >= 1 && R >= 1 && L >= 1 && L <= 0x7fffffff, "add_rowvec_f32: bad argument");
  const int64_t total = (int64_t)B * R * L;
  add_rowvec_kernel<<<ew_grid(total), 256, 0, (cudaStream_t)stream>>>(x, v, R, (int)L, total);
  B2_LAUNCHED();
  return B200SEP_OK;
}

extern "C" int b200sep_lstm_frames_gather_f32(const float* x, float* frames, int B, int C, int T, int n_frames, int width, int stride, void* stream) {
  B2_CHECK_ARG(x && frames && B >= 1 && C >= 1 && T >= 1 && n_frames >= 1 && width >= 1 && stride >= 1, "lstm_frames_gather_f32: bad argument");
  const int64_t total = (int64_t)width * B * n_frames * C;
  lstm_frames_gather_kernel<<<ew_grid(total), 256, 0, (cudaStream_t)stream>>>(x, frames, B, C, T, n_frames, width, stride, total);
  B2_LAUNCHED();
  return B200SEP_OK;
}

extern "C" int b200sep_lstm_frames_scatter_f32(const float* frames, const float* skip, float* y, int B, int C, int T, int n_frames, int width, int stride, void* stream) {
  B2_CHECK_ARG(frames && y && B >= 1 && C >= 1 && T >= 1 && n_frames >= 1 && width >= 1 && stride >= 1, "lstm_frames_scatter_f32: bad argument");
  B2_CHECK_ARG(n_frames == 1 ? width >= T : ((n_frames - 1) * stride + width >= T && stride % 2 == 0 && width == 2 * stride),
               "lstm_frames_scatter_f32: %d frames of %d every %d do not tile %d samples", n_frames, width, stride, T);
  const int64_t total = (int64_t)B * C * T;
  lstm_frames_scatter_kernel<<<ew_grid(total), 256, 0, (cudaStream_t)stream>>>(frames, skip, y, B, C, T, n_frames, width, stride, total);
  B2_LAUNCHED();
  return B200SEP_OK;
}

extern "C" int b200sep_lstm_bidir_wide_f32(const float* x_proj, const float* w_hh_t, float* out, int T, int N, int hid, void* stream) {
  B2_CHECK_ARG(x_proj && w_hh_t && out && T >= 1 && N >= 1 && hid >= 1, "lstm_bidir_wide_f32: bad argument");
  constexpr int NS = 8;
  int CL = 1;
  for (int c : {8, 4, 2})
    if (hid % c == 0 && 4 * (hid / c) >= 32) {
      CL = c;
      break;
    }
  const int UH = hid / CL, GL = 4 * UH;
  B2_CHECK_ARG(GL <= 768, "lstm_bidir_wide_f32: hidden size %d needs %d threads per CTA", hid, GL);
  const size_t wbytes = (size_t)hid * GL * sizeof(float);
  const size_t base1 = ((size_t)2 * hid * NS + (size_t)NS * GL + (size_t)2 * NS * UH) * sizeof(float);
  const int w_in_smem = base1 + wbytes <= 200 * 1024;
  int KS = 1;  // k-splits per gate column: streamed weights want many loads in flight
  if (!w_in_smem)
    for (int c : {4, 2})
      if (hid % c == 0 && GL * c <= 768) {
        KS = c;
        break;
      }
  size_t smem = ((size_t)2 * hid * NS + (size_t)KS * NS * GL + (size_t)2 * NS * UH) * sizeof(float) + (w_in_smem ? wbytes : 0);
  static size_t attr[kMaxDevices] = {};  // the largest limit set so far, per device
  B2_DEVICE_SLOT(dev);
  if (smem > attr[dev]) {
    B2_CUDA(cudaFuncSetAttribute(lstm_bidir_cluster_kernel<NS>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    attr[dev] = smem;
  }
  cudaLaunchConfig_t cfg{};
  cfg.gridDim = dim3((unsigned)(cdiv(N, NS) * CL), 2);
  cfg.blockDim = dim3((unsigned)(GL * KS));
  cfg.dynamicSmemBytes = smem;
  cfg.stream = (cudaStream_t)stream;
  cudaLaunchAttribute at[1];
  at[0].id = cudaLaunchAttributeClusterDimension;
  at[0].val.clusterDim.x = (unsigned)CL;
  at[0].val.clusterDim.y = 1;
  at[0].val.clusterDim.z = 1;
  cfg.attrs = at;
  cfg.numAttrs = 1;
  B2_CUDA(cudaLaunchKernelEx(&cfg, lstm_bidir_cluster_kernel<NS>, x_proj, w_hh_t, out, T, N, hid, w_in_smem, KS));
  count_launch();
  return B200SEP_OK;
}

extern "C" int b200sep_local_state_attn_f32(const float* query, const float* key, const float* content, const float* decay, float* out, int B, int C, int T, int heads,
                                            int ndecay, void* stream) {
  B2_CHECK_ARG(query && key && content && decay && out && B >= 1 && C >= 1 && T >= 1 && heads >= 1 && ndecay >= 1 && C % heads == 0, "local_state_attn_f32: bad argument");
  B2_CHECK_ARG(B <= 65535 && heads <= 65535, "local_state_attn_f32: batch / heads too large");
  cudaStream_t st = (cudaStream_t)stream;
  switch (C / heads) {
#define B2_LS_CASE(ch) \
  case ch:             \
    return launch_local_state<ch>(query, key, content, decay, out, B, C, T, heads, ndecay, st);
    B2_LS_CASE(1) B2_LS_CASE(2) B2_LS_CASE(3) B2_LS_CASE(4) B2_LS_CASE(6) B2_LS_CASE(8) B2_LS_CASE(12) B2_LS_CASE(16) B2_LS_CASE(24) B2_LS_CASE(32) B2_LS_CASE(48)
    B2_LS_CASE(64) B2_LS_CASE(96)
#undef B2_LS_CASE
    default:
      B2_CHECK_ARG(false, "local_state_attn_f32: %d channels per head is not instantiated (1, 2, 3, 4, 6, 8, 12, 16, 24, 32, 48, 64, 96)", C / heads);
  }
  return B200SEP_OK;
}
