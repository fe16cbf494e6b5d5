// fp32-in / fp32-out GEMM and implicit-GEMM convolution on the Hopper tensor cores (wgmma, sm_90a).
//
// The operands stay plain fp32 tensors in HBM (any strides, batched).  Producer warps read them, split every value on the fly into a
// bf16 "hi" and a bf16 "lo" part (x ~= hi + lo, 16 mantissa bits) and write both into shared memory in the canonical K-major
// SWIZZLE_128B layout; two consumer warpgroups (64 rows of the 128-row tile each) then issue, per 64-wide k-block, the three products
// Ah*Bh + Ah*Bl + Al*Bh as wgmma instructions accumulating in fp32 registers (relative error ~1e-5 per contraction, see DESIGN.md) and
// apply bias / activation / residual to their accumulator fragments before storing fp32.
//
//   warps 0..7    : consumers (wgmma issue + epilogue)
//   warps 8..15   : producers: global fp32 -> registers -> split -> swizzled st.shared -> fence.proxy.async -> mbarrier arrive
//
// Persistent CTAs (one per SM) walk the (batch, m-tile, n-tile) list; the shared-memory ring (full/empty mbarriers) runs continuously
// across tiles, so the producers fill the next tile's stages while the consumers run an epilogue.
//
// Used by b200sep_gemm_f32 (nn.Linear / attention of the HTDemucs cross-transformer) and b200sep_conv2d_f32 (Demucs encoders /
// DConv / rewrite convolutions, the VR CascadedASPPNet convolutions) when the shape is large enough; the SIMT kernels in ops_f32.cu /
// conv_gen.cu remain for tiny or oddly aligned shapes and for the transposed (scatter) convolution.
#include <cuda_bf16.h>
#include <stdlib.h>

#include <algorithm>

#include "common.cuh"
#include "tc_f32.cuh"
#include "umma.cuh"

namespace b200sep {

namespace {

constexpr int kTM = 128, kTN = 128, kTK = 64;
constexpr int kProducerWarps = 8;
constexpr int kConsThreads = 256;  // two consumer warpgroups
constexpr int kProdThreads = 32 * kProducerWarps;
constexpr int kThreads = kConsThreads + kProdThreads;  // 512

struct TcParams {
  // A operand (M rows): mode 0 GEMM  a[z*a_sz + m*a_rs + k]  (k contiguous);  mode 1 convolution gather (see below)
  const float* a;
  int64_t a_sz, a_rs;
  // B operand (N rows):  b[z*b_sz + n*b_rs + k*b_ks]   (b_ks == 1: K-major source; b_rs == 1: N-major source, e.g. blocked conv weights)
  const float* b;
  int64_t b_sz, b_rs, b_ks;
  int M, N, K, batch;
  int n_tile, stages;
  int m_tiles, n_tiles, num_tiles, num_iters;
  uint32_t a_bytes, b_bytes, stage_bytes;
  int a_vec, b_vec;  // 16-byte aligned K-major sources: float4 loads
  // convolution geometry (mode 1): x (batch, Cin, H, W), output pixels M = Ho*Wo, K = Cin*KH*KW ordered (ci, kh, kw)
  int mode, Cin, Cin8, H, W, Wo, KH, KW, SH, SW, PH, PW, DH, DW;
  // epilogue: v = acc*alpha + bias_n[n] + bias_m[m]; (+ add before act); act; (+ add after act | res + res_scale[n]*v);
  // out[z*o_sz + m*o_sm + n*o_sn];  res / add indexed  res[z*r_sz + m*r_sm + n*r_sn]
  float* out;
  int64_t o_sz, o_sm, o_sn;
  const float* res;
  int64_t r_sz, r_sm, r_sn;
  const float* res_scale;
  const float* bias_n;
  const float* bias_m;
  float alpha;
  int act, add_before_act;
  // transposed-convolution scatter (mode 1 only; same contract as conv_gen.cu): GEMM column n = r * up_cout + co, output index along the strided axis =
  // q * up + r - trim (kept when 0 <= index < out_len); up_axis 1 = H, 2 = W; bias_n has up_cout entries; up_cout % 16 == 0
  int up_axis, up, trim, out_len, up_cout, Ho;
  // B operand pre-split into the kernel's shared-memory image (tc_pack_*): per (n-tile, k-block) one [hi plane | lo plane] block that a
  // single cp.async.bulk drops into the stage -- static weights cost the producer warps nothing
  const uint8_t* b_packed;
  int sleep_ns;  // > 0: waiting producer / epilogue warps sleep between polls (B200SEP_WAIT_SLEEP_NS)
};

__device__ __forceinline__ float tc_act(float v, int act) {
  if (act == 1) return fmaxf(v, 0.f);
  if (act == 2) return 0.5f * v * (1.f + erff(v * 0.70710678118654752440f));
  if (act == 3) return v > 0.f ? v : 0.01f * v;
  if (act == 4) return 1.f / (1.f + expf(-v));
  if (act == 5) return tanhf(v);
  return v;
}

// x -> (hi, lo) bf16 pair for two values, packed little-endian: element 0 in the low half
__device__ __forceinline__ void split2(float x0, float x1, uint32_t& hi, uint32_t& lo) {
  const __nv_bfloat162 h = __floats2bfloat162_rn(x0, x1);
  const float r0 = x0 - __bfloat162float(h.x), r1 = x1 - __bfloat162float(h.y);
  const __nv_bfloat162 l = __floats2bfloat162_rn(r0, r1);
  hi = *reinterpret_cast<const uint32_t*>(&h);
  lo = *reinterpret_cast<const uint32_t*>(&l);
}

// 8 consecutive k of one row -> one 16-byte chunk in each plane, at the SWIZZLE_128B position of (row, chunk)
__device__ __forceinline__ void store_chunk(uint8_t* plane_hi, uint8_t* plane_lo, int row, int chunk, const float* v) {
  uint4 h, l;
  split2(v[0], v[1], h.x, l.x);
  split2(v[2], v[3], h.y, l.y);
  split2(v[4], v[5], h.z, l.z);
  split2(v[6], v[7], h.w, l.w);
  const uint32_t off = (uint32_t)(row >> 3) * 1024u + (uint32_t)(row & 7) * 128u + (uint32_t)((chunk ^ (row & 7)) << 4);
  *reinterpret_cast<uint4*>(plane_hi + off) = h;
  *reinterpret_cast<uint4*>(plane_lo + off) = l;
}

// The fills below handle their 16-byte chunks ("items") in groups of kG: all global loads of a group are issued before the first
// conversion / shared store, so every producer thread keeps kG*8 loads in flight (the loop is latency-, not issue-bound).
constexpr int kG = 4;

// K-major source: rows x 64 k, element (r, k) at src[r*rs + k].  pt = producer thread index (0..255).
template <int NT = kProdThreads>
__device__ __forceinline__ void fill_kmajor(uint8_t* hi, uint8_t* lo, const float* __restrict__ src, int64_t rs, int rows_tile, int row0, int rows_total, int k0,
                                            int K, int vec, int pt) {
  const int items = rows_tile * 8;
  for (int base = pt; base < items; base += kG * NT) {
    float v[kG][8];
#pragma unroll
    for (int g = 0; g < kG; ++g) {
      const int id = base + g * NT;
      const int r = id >> 3, c = id & 7;
      const int k = k0 + c * 8;
#pragma unroll
      for (int e = 0; e < 8; ++e) v[g][e] = 0.f;
      if (id < items && row0 + r < rows_total && k < K) {
        const float* p = src + (int64_t)(row0 + r) * rs + k;
        if (vec && k + 7 < K) {
          const float4 a = __ldg(reinterpret_cast<const float4*>(p)), b = __ldg(reinterpret_cast<const float4*>(p) + 1);
          v[g][0] = a.x; v[g][1] = a.y; v[g][2] = a.z; v[g][3] = a.w; v[g][4] = b.x; v[g][5] = b.y; v[g][6] = b.z; v[g][7] = b.w;
        } else {
#pragma unroll
          for (int e = 0; e < 8; ++e)
            if (k + e < K) v[g][e] = __ldg(p + e);
        }
      }
    }
#pragma unroll
    for (int g = 0; g < kG; ++g) {
      const int id = base + g * NT;
      if (id < items) store_chunk(hi, lo, id >> 3, id & 7, v[g]);
    }
  }
}

// row-major ("N-major") source: element (r, k) at src[r + k*ks]; lanes walk consecutive rows so the loads coalesce
template <int NT = kProdThreads>
__device__ __forceinline__ void fill_nmajor(uint8_t* hi, uint8_t* lo, const float* __restrict__ src, int64_t ks, int rows_tile, int row0, int rows_total, int k0, int K,
                                            int pt) {
  const int sh = (rows_tile == 256) ? 8 : (rows_tile == 128) ? 7 : 6;  // tiles are 64, 128 or 256 rows
  const int items = rows_tile * 8;
  for (int base = pt; base < items; base += kG * NT) {
    float v[kG][8];
#pragma unroll
    for (int g = 0; g < kG; ++g) {
      const int id = base + g * NT;
      const int r = id & (rows_tile - 1), c = id >> sh;
      const int k = k0 + c * 8;
#pragma unroll
      for (int e = 0; e < 8; ++e) v[g][e] = 0.f;
      if (id < items && row0 + r < rows_total) {
        const float* p = src + (row0 + r) + (int64_t)k * ks;
#pragma unroll
        for (int e = 0; e < 8; ++e)
          if (k + e < K) v[g][e] = __ldg(p + (int64_t)e * ks);
      }
    }
#pragma unroll
    for (int g = 0; g < kG; ++g) {
      const int id = base + g * NT;
      if (id < items) store_chunk(hi, lo, id & (rows_tile - 1), id >> sh, v[g]);
    }
  }
}

// convolution weights blocked [Cin][taps][CoutPad] (output channel contiguous) read in the kernel's (tap, ci) K order
__device__ __forceinline__ void fill_conv_weights(uint8_t* hi, uint8_t* lo, const float* __restrict__ w, int64_t cout_pad, int rows_tile, int n0, int N, int k0, int Cin,
                                                  int Cin8, int taps, int pt) {
  const int sh = (rows_tile == 256) ? 8 : 7;
  const int items = rows_tile * 8;
  for (int base = pt; base < items; base += kG * kProdThreads) {
    float v[kG][8];
#pragma unroll
    for (int g = 0; g < kG; ++g) {
      const int id = base + g * kProdThreads;
      const int r = id & (rows_tile - 1), c = id >> sh;
      const int kg = k0 + c * 8;
      const int tap = kg / Cin8, ci0 = kg - tap * Cin8;
#pragma unroll
      for (int e = 0; e < 8; ++e) v[g][e] = 0.f;
      if (id < items && n0 + r < N && tap < taps) {
        const float* p = w + ((int64_t)ci0 * taps + tap) * cout_pad + n0 + r;
#pragma unroll
        for (int e = 0; e < 8; ++e)
          if (ci0 + e < Cin) v[g][e] = __ldg(p + (int64_t)e * taps * cout_pad);
      }
    }
#pragma unroll
    for (int g = 0; g < kG; ++g) {
      const int id = base + g * kProdThreads;
      if (id < items) store_chunk(hi, lo, id & (rows_tile - 1), id >> sh, v[g]);
    }
  }
}

// one output element of the generic epilogue: v = acc*alpha + bias_m[m] + bias_n[n] (+ add before act); act; (+ add after act | res + res_scale[n]*v)
__device__ __forceinline__ void tc_store(const TcParams& p, int z, int m, int n, float v) {
  if (p.up_axis) {
    // ConvTranspose as a 2-tap convolution over the coarse index: column n is phase r of real channel co
    const int r = n / p.up_cout, co = n - r * p.up_cout;
    const int hq = m / p.Wo, wq = m - hq * p.Wo;
    const int pos = ((p.up_axis == 1) ? hq : wq) * p.up + r - p.trim;
    if (pos < 0 || pos >= p.out_len) return;
    const int64_t cs = (p.up_axis == 1) ? (int64_t)p.out_len * p.Wo : (int64_t)p.Ho * p.out_len;
    float x = v;
    if (p.bias_n) x += __ldg(&p.bias_n[co]);
    p.out[(int64_t)z * p.o_sz + (int64_t)co * cs + ((p.up_axis == 1) ? (int64_t)pos * p.Wo + wq : (int64_t)hq * p.out_len + pos)] = tc_act(x, p.act);
    return;
  }
  float x = fmaf(v, p.alpha, p.bias_m ? __ldg(&p.bias_m[m]) : 0.f);
  if (p.bias_n) x += __ldg(&p.bias_n[n]);
  const float* rrow = p.res ? p.res + (int64_t)z * p.r_sz + (int64_t)m * p.r_sm : nullptr;
  if (rrow && p.add_before_act) x += __ldg(&rrow[(int64_t)n * p.r_sn]);
  x = tc_act(x, p.act);
  if (rrow && !p.add_before_act) {
    if (p.res_scale) x = __ldg(&rrow[(int64_t)n * p.r_sn]) + __ldg(&p.res_scale[n]) * x;
    else x += __ldg(&rrow[(int64_t)n * p.r_sn]);
  }
  p.out[(int64_t)z * p.o_sz + (int64_t)m * p.o_sm + (int64_t)n * p.o_sn] = x;
}

__global__ void __launch_bounds__(kThreads, 1) tc_f32_kernel(const TcParams p) {
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = smem_raw + ((1024u - (ptx::smem_u32(smem_raw) & 1023u)) & 1023u);
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + (size_t)p.stages * p.stage_bytes);
  uint64_t* empty_bar = full_bar + p.stages;

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (threadIdx.x == 0) {
    for (int s = 0; s < p.stages; ++s) {
      ptx::mbar_init(&full_bar[s], kProducerWarps + (p.b_packed ? 1 : 0));
      ptx::mbar_init(&empty_bar[s], kConsThreads);
    }
    ptx::fence_barrier_init();
  }
  __syncthreads();
  const int tiles_per_z = p.m_tiles * p.n_tiles;

  if (warp >= kConsThreads / 32) {
    // ===== producers =====
    const int pt = threadIdx.x - kConsThreads;
    int s = 0;
    uint32_t phase = 0;
    const int taps = p.KH * p.KW;
    const int64_t plane = (int64_t)p.H * p.W;
    for (int tile = blockIdx.x; tile < p.num_tiles; tile += gridDim.x) {
      const int z = tile / tiles_per_z, rem = tile - z * tiles_per_z;
      const int m0 = (rem / p.n_tiles) * kTM, n0 = (rem % p.n_tiles) * p.n_tile;
      const float* bz = p.b + (int64_t)z * p.b_sz;
      // convolution: this thread always fills tile row (pt & 127) -> decode its output pixel once per tile
      const int arow = pt & (kTM - 1);
      int hi0 = 0, wi0 = 0;
      bool arow_ok = false;
      const float* xz = p.a + (int64_t)z * p.a_sz;
      if (p.mode == 1) {
        const int m = m0 + arow;
        arow_ok = m < p.M;
        const int ho = m / p.Wo, wo = m - ho * p.Wo;
        hi0 = ho * p.SH - p.PH;
        wi0 = wo * p.SW - p.PW;
      }
      for (int i = 0; i < p.num_iters; ++i) {
        ptx::mbar_wait_opt(&empty_bar[s], phase ^ 1, p.sleep_ns, 100 + i);
        uint8_t* st = smem + (size_t)s * p.stage_bytes;
        uint8_t* a_hi = st;
        uint8_t* a_lo = st + p.a_bytes;
        uint8_t* b_hi = st + 2 * p.a_bytes;
        uint8_t* b_lo = b_hi + p.b_bytes;
        const int k0 = i * kTK;
        if (p.b_packed && pt == 0) {  // static weights: one bulk copy of the pre-split image, in flight while the A tile is converted
          ptx::mbar_arrive_expect_tx(&full_bar[s], 2 * p.b_bytes);
          ptx::bulk_load_1d(b_hi, p.b_packed + ((size_t)(n0 / p.n_tile) * p.num_iters + i) * (size_t)(2 * p.b_bytes), 2 * p.b_bytes, &full_bar[s]);
        }
        if (p.mode == 0) {
          fill_kmajor(a_hi, a_lo, xz, p.a_rs, kTM, m0, p.M, k0, p.K, p.a_vec, pt);
        } else {
          // implicit-GEMM gather.  K is ordered (tap, ci) with ci padded to a multiple of 8, so one 16-byte chunk = 8 consecutive input
          // channels of ONE tap: a single bounds test and 8 loads at a constant stride.  Two threads per pixel row, 4 chunks each.
          float v[4][8];
#pragma unroll
          for (int g = 0; g < 4; ++g) {
            const int c = (pt >> 7) + 2 * g;
#pragma unroll
            for (int e = 0; e < 8; ++e) v[g][e] = 0.f;
            const int kg = k0 + c * 8;
            const int tap = kg / p.Cin8, ci0 = kg - tap * p.Cin8;
            const int kh = tap / p.KW, kw = tap - kh * p.KW;
            const int hi = hi0 + kh * p.DH, wi = wi0 + kw * p.DW;
            if (arow_ok && tap < taps && hi >= 0 && hi < p.H && wi >= 0 && wi < p.W) {
              const float* px = xz + ((int64_t)ci0 * p.H + hi) * p.W + wi;
              if (ci0 + 8 <= p.Cin) {
#pragma unroll
                for (int e = 0; e < 8; ++e) {
                  v[g][e] = __ldg(px);
                  px += plane;
                }
              } else {
#pragma unroll
                for (int e = 0; e < 8; ++e)
                  if (ci0 + e < p.Cin) v[g][e] = __ldg(px + (int64_t)e * plane);
              }
            }
          }
#pragma unroll
          for (int g = 0; g < 4; ++g) store_chunk(a_hi, a_lo, arow, (pt >> 7) + 2 * g, v[g]);
        }
        if (p.b_packed) {
          // issued above, right after the stage became free
        } else if (p.mode == 1) fill_conv_weights(b_hi, b_lo, bz, p.b_ks, p.n_tile, n0, p.N, k0, p.Cin, p.Cin8, taps, pt);
        else if (p.b_ks == 1) fill_kmajor(b_hi, b_lo, bz, p.b_rs, p.n_tile, n0, p.N, k0, p.K, p.b_vec, pt);
        else fill_nmajor(b_hi, b_lo, bz, p.b_ks, p.n_tile, n0, p.N, k0, p.K, pt);
        ptx::fence_proxy_async();  // generic-proxy smem writes -> visible to the tensor core's async proxy
        __syncwarp();
        if (lane == 0) ptx::mbar_arrive(&full_bar[s]);
        if (++s == p.stages) {
          s = 0;
          phase ^= 1;
        }
      }
    }
    return;
  }
  // ===== consumers: wgmma main loop into registers, then the epilogue from the accumulator fragments =====
  const int wg = warp >> 2, g = lane >> 2, cq = lane & 3;
  const int mrow0 = wg * 64 + (warp & 3) * 16 + g;  // tile rows mrow0 and mrow0 + 8
  int s = 0;
  uint32_t phase = 0;
  float acc[kTN / 2];
  for (int tile = blockIdx.x; tile < p.num_tiles; tile += gridDim.x) {
    const int z = tile / tiles_per_z, rem = tile - z * tiles_per_z;
    const int m0 = (rem / p.n_tiles) * kTM, n0 = (rem % p.n_tiles) * kTN;
    int prev = -1;
    for (int i = 0; i < p.num_iters; ++i) {
      ptx::mbar_wait(&full_bar[s], phase, 200 + i);
      const uint32_t st = ptx::smem_u32(smem + (size_t)s * p.stage_bytes);
      const uint32_t a_hi = st + (uint32_t)wg * 8192u, a_lo = a_hi + p.a_bytes, b_hi = st + 2 * p.a_bytes, b_lo = b_hi + p.b_bytes;
      ptx::wgmma_fence();
#pragma unroll
      for (int j = 0; j < kTK / 16; ++j) {
        const uint64_t dah = ptx::smem_desc(a_hi + j * 32, 16, 1024, ptx::kLayoutSW128);
        const uint64_t dal = ptx::smem_desc(a_lo + j * 32, 16, 1024, ptx::kLayoutSW128);
        const uint64_t dbh = ptx::smem_desc(b_hi + j * 32, 16, 1024, ptx::kLayoutSW128);
        const uint64_t dbl = ptx::smem_desc(b_lo + j * 32, 16, 1024, ptx::kLayoutSW128);
        ptx::wgmma_ss_n128<0>(acc, dah, dbh, (i | j) != 0 ? 1 : 0);
        ptx::wgmma_ss_n128<0>(acc, dah, dbl, 1);
        ptx::wgmma_ss_n128<0>(acc, dal, dbh, 1);
      }
      ptx::wgmma_commit();
      ptx::wgmma_wait<1>();  // the previous stage's group has completed: release it
      if (prev >= 0) ptx::mbar_arrive(&empty_bar[prev]);
      prev = s;
      if (++s == p.stages) {
        s = 0;
        phase ^= 1;
      }
    }
    ptx::wgmma_wait<0>();
    if (prev >= 0) ptx::mbar_arrive(&empty_bar[prev]);
    ptx::fence_regs(acc);
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int m = m0 + mrow0 + 8 * h;
      if (m >= p.M) continue;
#pragma unroll
      for (int i = 0; i < kTN / 8; ++i) {
        const int n = n0 + 8 * i + 2 * cq;
        if (n < p.N) tc_store(p, z, m, n, acc[4 * i + 2 * h]);
        if (n + 1 < p.N) tc_store(p, z, m, n + 1, acc[4 * i + 2 * h + 1]);
      }
    }
  }
}

static int pick_n_tile(int) { return kTN; }

// one thread per 16-byte chunk of the packed image: (n-tile, k-block, row, chunk)
__global__ void tc_pack_kernel(const float* __restrict__ src, int conv, int64_t rs, int64_t ks, int N, int K, int Cin, int Cin8, int taps, int n_tile, int num_iters,
                               uint8_t* __restrict__ packed, int64_t total) {
  for (int64_t id = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; id < total; id += (int64_t)gridDim.x * blockDim.x) {
    const int c = (int)(id & 7);
    const int r = (int)((id >> 3) % n_tile);
    const int64_t blk = (id >> 3) / n_tile;  // tn * num_iters + i
    const int i = (int)(blk % num_iters), tn = (int)(blk / num_iters);
    const int n = tn * n_tile + r, kg = i * kTK + c * 8;
    float v[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
    if (n < N) {
      if (conv) {  // src = blocked conv weights [Cin][taps][cout_pad = ks]; kernel K order (tap, ci padded to 8)
        const int tap = kg / Cin8, ci0 = kg - tap * Cin8;
        if (tap < taps)
          for (int e = 0; e < 8; ++e)
            if (ci0 + e < Cin) v[e] = src[((int64_t)(ci0 + e) * taps + tap) * ks + n];
      } else {
        for (int e = 0; e < 8; ++e)
          if (kg + e < K) v[e] = src[(int64_t)n * rs + kg + e];
      }
    }
    const size_t plane = (size_t)n_tile * 128;
    uint8_t* base = packed + (size_t)blk * 2 * plane;
    store_chunk(base, base + plane, r, c, v);
  }
}

int wait_sleep_ns() {
  static const int ns = [] {
    const char* e = getenv("B200SEP_WAIT_SLEEP_NS");
    return e ? atoi(e) : 0;
  }();
  return ns;
}

int tc_launch(TcParams& p, cudaStream_t st) {
  p.sleep_ns = wait_sleep_ns();
  p.n_tile = pick_n_tile(p.N);
  p.stages = 3;
  p.a_bytes = kTM * 128;
  p.b_bytes = (uint32_t)p.n_tile * 128;
  p.stage_bytes = 2 * p.a_bytes + 2 * p.b_bytes;
  p.m_tiles = cdiv(p.M, kTM);
  p.n_tiles = cdiv(p.N, p.n_tile);
  const int64_t nt = (int64_t)p.batch * p.m_tiles * p.n_tiles;
  B2_CHECK_ARG(nt < (1ll << 31), "tc_f32: too many tiles");
  p.num_tiles = (int)nt;
  p.num_iters = cdiv(p.K, kTK);
  const size_t smem = (size_t)p.stages * p.stage_bytes + 1024 + 256;
  static bool attr_set = false;
  if (!attr_set) {
    B2_CUDA(cudaFuncSetAttribute(tc_f32_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024));
    attr_set = true;
  }
  const int grid = std::min(p.num_tiles, kNumSMs);
  tc_f32_kernel<<<grid, kThreads, smem, st>>>(p);
  B2_LAUNCHED();
  return B200SEP_OK;
}

bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; }

// ===================================================================================================================================
// Fused attention for head dimension 64:  O = softmax(alpha * Q K^T) V  per (batch, head), fp32 in / out, every product as bf16 hi/lo x3 on
// wgmma with fp32 accumulation in registers -- the score matrix never reaches HBM (the unfused form wrote, re-read, normalised and re-read
// B*H*Lq*Lk floats: 0.9 GB per HTDemucs frequency layer at batch 4).  Q / K / V^T arrive as pre-split tile images (att_pack_kernel).
//
//   one CTA per (128-query tile, batch*head);  key tiles of 128:
//   warps 0..7 : two consumer warpgroups, 64 query rows each: S_j = Q K_j^T (64 x 128, K = 64) into registers, online softmax on the
//                fragments (row max / sum over the 4 lanes of a quad), P_j split into bf16 hi/lo in registers and fed as the A operand of
//                O += P_j V_j (64 x 64, K = 128); O lives in registers and is rescaled when the row maximum moves
//   warp 8     : loader: one thread, bulk copies of the 32 KB tile images into a two-slot ring (K and V slots freed independently)
constexpr int kAttConsumers = 256;
constexpr int kAttThreads = kAttConsumers + 32;
constexpr int kAttQ = 128, kAttKeys = 128, kAttD = 64;
constexpr uint32_t kAttQBytes = kAttQ * 128;            // one plane of Q: 128 rows x 64 bf16
constexpr uint32_t kAttKBytes = kAttKeys * 128;         // one plane of K_j
constexpr uint32_t kAttVBlk = kAttD * 128;              // one plane of one 64-key block of V^T_j
constexpr uint32_t kAttStage = 2 * kAttKBytes + 4 * kAttVBlk;  // 64 KB
constexpr uint32_t kAttOffStage = 2 * kAttQBytes;
constexpr uint32_t kAttSmem = kAttOffStage + 2 * kAttStage;  // 160 KB

struct AttParams {
  const float* q;   // q[b * q_bs + m * q_rs + h * 64 + d]
  const float* k;   // k[b * k_bs + n * k_rs + h * 64 + d]
  const float* vt;  // vt[b * vt_bs + (h * 64 + d) * vt_rs + n]   (V transposed: keys contiguous)
  float* out;       // out[b * o_bs + m * o_rs + h * 64 + d]
  int64_t q_bs, q_rs, k_bs, k_rs, vt_bs, vt_rs, o_bs, o_rs;
  int H, Lq, Lk;
  float alpha;
  int o_vec;
  int v_kn;  // 1: V given untransposed, v[b * vt_bs + n * vt_rs + h * 64 + d] (the pack kernel gathers it d-major)
  // Q / K / V^T split into bf16 hi / lo and laid out as the kernel's shared-memory tiles by att_pack_kernel, 32 KB per tile:
  //   qimg[(z * mq_tiles + mt)] = [hi 128 x 128 B | lo],  kimg[(z * nk + j)] = [hi | lo],  vimg[(z * nk + j)] = [hi kb0 | hi kb1 | lo kb0 | lo kb1] (64 rows x 128 B each)
  const uint8_t* qimg;
  const uint8_t* kimg;
  const uint8_t* vimg;
  int mq_tiles;
};

__device__ __forceinline__ float ex2_approx(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}

// one 16-byte chunk (8 values) of a tile image per thread; see AttParams for the image layouts
__global__ void att_pack_kernel(const AttParams p, uint8_t* __restrict__ qimg, uint8_t* __restrict__ kimg, uint8_t* __restrict__ vimg, int nk, int64_t nq_chunks,
                                int64_t nk_chunks) {
  const int64_t total = nq_chunks + 2 * nk_chunks;
  for (int64_t id = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; id < total; id += (int64_t)gridDim.x * blockDim.x) {
    float v[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
    if (id < nq_chunks + nk_chunks) {  // Q or K: rows = tokens, 8 consecutive head-dimension values
      const bool is_q = id < nq_chunks;
      const int64_t cid = is_q ? id : id - nq_chunks;
      const int c = (int)(cid & 7), r = (int)((cid >> 3) & 127);
      const int64_t img = cid >> 10;
      const int tiles = is_q ? p.mq_tiles : nk;
      const int z = (int)(img / tiles), t = (int)(img - (int64_t)z * tiles);
      const int b = z / p.H, h = z - b * p.H;
      const int row = t * 128 + r;
      if (row < (is_q ? p.Lq : p.Lk)) {
        const float* src = is_q ? p.q + (int64_t)b * p.q_bs + (int64_t)row * p.q_rs : p.k + (int64_t)b * p.k_bs + (int64_t)row * p.k_rs;
        src += h * kAttD + c * 8;
#pragma unroll
        for (int e = 0; e < 8; ++e) v[e] = __ldg(src + e);
      }
      uint8_t* base = (is_q ? qimg : kimg) + img * 32768;
      store_chunk(base, base + 16384, r, c, v);
    } else {  // V^T: rows = head dimension, 8 consecutive keys
      const int64_t cid = id - nq_chunks - nk_chunks;
      const int c = (int)(cid & 7), r = (int)((cid >> 3) & 63), kb = (int)((cid >> 9) & 1);
      const int64_t img = cid >> 10;
      const int z = (int)(img / nk), j = (int)(img - (int64_t)z * nk);
      const int b = z / p.H, h = z - b * p.H;
      const int n0 = j * kAttKeys + kb * 64 + c * 8;
      const float* vb = p.vt + (int64_t)b * p.vt_bs;
#pragma unroll
      for (int e = 0; e < 8; ++e)
        if (n0 + e < p.Lk) v[e] = p.v_kn ? __ldg(vb + (int64_t)(n0 + e) * p.vt_rs + h * kAttD + r) : __ldg(vb + (int64_t)(h * kAttD + r) * p.vt_rs + n0 + e);
      uint8_t* base = vimg + img * 32768 + kb * kAttVBlk;
      store_chunk(base, base + 2 * kAttVBlk, r, c, v);
    }
  }
}

__global__ void __launch_bounds__(kAttThreads, 1) tc_attention_kernel(const AttParams p) {
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = smem_raw + ((1024u - (ptx::smem_u32(smem_raw) & 1023u)) & 1023u);
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + kAttSmem);
  uint64_t* q_full = bars;       // [1]
  uint64_t* k_full = bars + 1;   // [2]  K_j landed
  uint64_t* k_empty = bars + 3;  // [2]  S_j done: K slot free
  uint64_t* v_full = bars + 5;   // [2]
  uint64_t* v_empty = bars + 7;  // [2]  O += P_j V_j done: V slot free

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (threadIdx.x == 0) {
    ptx::mbar_init(q_full, 1);
    for (int a = 0; a < 2; ++a) {
      ptx::mbar_init(&k_full[a], 1);
      ptx::mbar_init(&k_empty[a], kAttConsumers);
      ptx::mbar_init(&v_full[a], 1);
      ptx::mbar_init(&v_empty[a], kAttConsumers);
    }
    ptx::fence_barrier_init();
  }
  __syncthreads();

  const int z = blockIdx.y, b = z / p.H, h = z - b * p.H;
  const int m0 = blockIdx.x * kAttQ;
  const int nk = (p.Lk + kAttKeys - 1) / kAttKeys;

  if (warp == kAttConsumers / 32) {
    // ===== loader: K and V streams polled independently =====
    if (lane == 0) {
      const int64_t zq = (int64_t)z * p.mq_tiles + blockIdx.x, zk = (int64_t)z * nk;
      ptx::mbar_arrive_expect_tx(q_full, 32768);
      ptx::bulk_load_1d(smem, p.qimg + zq * 32768, 32768, q_full);
      int jk = 0, jv = 0;
      uint32_t idle = 0;
      while (jk < nk || jv < nk) {
        bool did = false;
        if (jk < nk) {
          const int st = jk & 1;
          if (ptx::mbar_try_wait(&k_empty[st], ((uint32_t)(jk >> 1) & 1u) ^ 1u)) {
            ptx::mbar_arrive_expect_tx(&k_full[st], 32768);
            ptx::bulk_load_1d(smem + kAttOffStage + (size_t)st * kAttStage, p.kimg + (zk + jk) * 32768, 32768, &k_full[st]);
            ++jk;
            did = true;
          }
        }
        if (jv < nk) {
          const int st = jv & 1;
          if (ptx::mbar_try_wait(&v_empty[st], ((uint32_t)(jv >> 1) & 1u) ^ 1u)) {
            ptx::mbar_arrive_expect_tx(&v_full[st], 32768);
            ptx::bulk_load_1d(smem + kAttOffStage + (size_t)st * kAttStage + 2 * kAttKBytes, p.vimg + (zk + jv) * 32768, 32768, &v_full[st]);
            ++jv;
            did = true;
          }
        }
        if (did) {
          idle = 0;
        } else if (__nanosleep(100), ++idle > (1u << 22)) {
          __trap();  // stalled pipeline
        }
      }
    }
    return;
  }

  // ===== consumers: thread = rows r0 and r0 + 8 of the query tile, columns 8i + 2*cq + {0, 1} of every fragment =====
  const int wg = warp >> 2, g = lane >> 2, cq = lane & 3;
  const int r0 = wg * 64 + (warp & 3) * 16 + g;
  // base-2 domain: p = 2^(s * a2 - m2) with a2 = alpha * log2(e): one FFMA + one MUFU.EX2 per score
  const float a2 = p.alpha * 1.4426950408889634f;
  float mrun[2] = {-INFINITY, -INFINITY}, l[2] = {0.f, 0.f};
  float O[kAttD / 2];
#pragma unroll
  for (int e = 0; e < kAttD / 2; ++e) O[e] = 0.f;
  const uint32_t qh = ptx::smem_u32(smem) + (uint32_t)wg * 8192u, ql = qh + kAttQBytes;
  ptx::mbar_wait(q_full, 0, 500);
  for (int j = 0; j < nk; ++j) {
    const int st = j & 1;
    const uint32_t ph = (uint32_t)(j >> 1) & 1u;
    const uint32_t kh = ptx::smem_u32(smem + kAttOffStage + (size_t)st * kAttStage), kl = kh + kAttKBytes;
    ptx::mbar_wait(&k_full[st], ph, 560 + st);
    float S[kAttKeys / 2];
    ptx::wgmma_fence();
#pragma unroll
    for (int jj = 0; jj < kAttD / 16; ++jj) {
      const uint64_t dqh = ptx::smem_desc(qh + jj * 32, 16, 1024, ptx::kLayoutSW128), dql = ptx::smem_desc(ql + jj * 32, 16, 1024, ptx::kLayoutSW128);
      const uint64_t dkh = ptx::smem_desc(kh + jj * 32, 16, 1024, ptx::kLayoutSW128), dkl = ptx::smem_desc(kl + jj * 32, 16, 1024, ptx::kLayoutSW128);
      ptx::wgmma_ss_n128<0>(S, dqh, dkh, jj != 0 ? 1 : 0);
      ptx::wgmma_ss_n128<0>(S, dqh, dkl, 1);
      ptx::wgmma_ss_n128<0>(S, dql, dkh, 1);
    }
    ptx::wgmma_commit();
    ptx::wgmma_wait<0>();
    ptx::fence_regs(S);
    ptx::mbar_arrive(&k_empty[st]);

    const int nvalid = min(kAttKeys, p.Lk - j * kAttKeys);
    float mx[2] = {-INFINITY, -INFINITY};
#pragma unroll
    for (int i = 0; i < kAttKeys / 8; ++i)
#pragma unroll
      for (int e = 0; e < 2; ++e)
        if (8 * i + 2 * cq + e < nvalid) {
          mx[0] = fmaxf(mx[0], S[4 * i + e]);
          mx[1] = fmaxf(mx[1], S[4 * i + 2 + e]);
        }
    float mnew[2], corr[2];
#pragma unroll
    for (int hh = 0; hh < 2; ++hh) {
      mx[hh] = fmaxf(mx[hh], __shfl_xor_sync(0xffffffffu, mx[hh], 1));
      mx[hh] = fmaxf(mx[hh], __shfl_xor_sync(0xffffffffu, mx[hh], 2));
      mnew[hh] = fmaxf(mrun[hh], mx[hh] * a2);
      corr[hh] = ex2_approx(mrun[hh] - mnew[hh]);  // first tile: 2^(-inf) = 0
      mrun[hh] = mnew[hh];
    }
    // P_j as the register A operand of the second product: k-step kk covers keys 16kk..16kk+15; A register q holds row r0 + 8*(q & 1),
    // keys 16kk + 8*(q >> 1) + 2*cq + {0, 1} -- exactly S[8kk + 2q], S[8kk + 2q + 1]
    uint32_t ah[kAttKeys / 16][4], al[kAttKeys / 16][4];
    float lsum[2] = {0.f, 0.f};
#pragma unroll
    for (int kk = 0; kk < kAttKeys / 16; ++kk)
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        const int hh = q & 1, col = 16 * kk + 8 * (q >> 1) + 2 * cq;
        float x0 = ex2_approx(fmaf(S[8 * kk + 2 * q], a2, -mnew[hh])), x1 = ex2_approx(fmaf(S[8 * kk + 2 * q + 1], a2, -mnew[hh]));
        if (col >= nvalid) x0 = 0.f;
        if (col + 1 >= nvalid) x1 = 0.f;
        lsum[hh] += x0 + x1;
        split2(x0, x1, ah[kk][q], al[kk][q]);
      }
#pragma unroll
    for (int hh = 0; hh < 2; ++hh) l[hh] = l[hh] * corr[hh] + lsum[hh];
#pragma unroll
    for (int i = 0; i < kAttD / 8; ++i) {
      O[4 * i] *= corr[0];
      O[4 * i + 1] *= corr[0];
      O[4 * i + 2] *= corr[1];
      O[4 * i + 3] *= corr[1];
    }
    ptx::mbar_wait(&v_full[st], ph, 580 + st);
    const uint32_t vh = kh + 2 * kAttKBytes, vl = vh + 2 * kAttVBlk;
    ptx::wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < kAttKeys / 16; ++kk) {
      const uint32_t off = (uint32_t)(kk >> 2) * kAttVBlk + (uint32_t)(kk & 3) * 32u;
      const uint64_t dvh = ptx::smem_desc(vh + off, 16, 1024, ptx::kLayoutSW128), dvl = ptx::smem_desc(vl + off, 16, 1024, ptx::kLayoutSW128);
      ptx::wgmma_rs_n64(O, ah[kk], dvh);
      ptx::wgmma_rs_n64(O, ah[kk], dvl);
      ptx::wgmma_rs_n64(O, al[kk], dvh);
    }
    ptx::wgmma_commit();
    ptx::wgmma_wait<0>();
    ptx::fence_regs(O);
#pragma unroll
    for (int kk = 0; kk < kAttKeys / 16; ++kk) {
      ptx::fence_regs(ah[kk]);
      ptx::fence_regs(al[kk]);
    }
    ptx::mbar_arrive(&v_empty[st]);
  }
#pragma unroll
  for (int hh = 0; hh < 2; ++hh) {
    l[hh] += __shfl_xor_sync(0xffffffffu, l[hh], 1);
    l[hh] += __shfl_xor_sync(0xffffffffu, l[hh], 2);
    const int m = m0 + r0 + 8 * hh;
    if (m >= p.Lq) continue;
    const float inv = 1.f / l[hh];
    float* o = p.out + (int64_t)b * p.o_bs + (int64_t)m * p.o_rs + (int64_t)h * kAttD;
#pragma unroll
    for (int i = 0; i < kAttD / 8; ++i) {
      const int col = 8 * i + 2 * cq;
      if (p.o_vec) {
        *reinterpret_cast<float2*>(o + col) = make_float2(O[4 * i + 2 * hh] * inv, O[4 * i + 2 * hh + 1] * inv);
      } else {
        o[col] = O[4 * i + 2 * hh] * inv;
        o[col + 1] = O[4 * i + 2 * hh + 1] * inv;
      }
    }
  }
}

}  // namespace

bool tc_attention_usable(int hd, int Lq, int Lk) { return tc_enabled() && hd == kAttD && Lq >= 1 && Lk >= 1; }

// bytes of scratch for the pre-split Q / K / V^T tile images (one 32 KB image per 128-row tile and (batch, head))
int64_t tc_attention_work_bytes(int B, int H, int Lq, int Lk) {
  return (int64_t)B * H * ((int64_t)cdiv(Lq, kAttQ) + 2 * (int64_t)cdiv(Lk, kAttKeys)) * 32768;
}

int tc_attention_f32(const float* q, const float* k, const float* vt, float* out, int B, int H, int Lq, int Lk, int64_t q_bs, int64_t q_rs, int64_t k_bs, int64_t k_rs,
                     int64_t vt_bs, int64_t vt_rs, int64_t o_bs, int64_t o_rs, float alpha, int v_kn, void* work, cudaStream_t st) {
  AttParams p{};
  p.v_kn = v_kn;
  p.q = q; p.k = k; p.vt = vt; p.out = out;
  p.q_bs = q_bs; p.q_rs = q_rs; p.k_bs = k_bs; p.k_rs = k_rs; p.vt_bs = vt_bs; p.vt_rs = vt_rs; p.o_bs = o_bs; p.o_rs = o_rs;
  p.H = H; p.Lq = Lq; p.Lk = Lk; p.alpha = alpha;
  p.o_vec = (o_rs % 4 == 0) && (o_bs % 4 == 0) && aligned16(out);
  const size_t smem = (size_t)kAttSmem + 1024 + 256;
  B2_CHECK_ARG((int64_t)B * H <= 65535, "attention_f32: batch * heads too large");
  dim3 grid((unsigned)cdiv(Lq, kAttQ), (unsigned)(B * H));
  // Every K / V tile is consumed by all query tiles of its (batch, head): it is split into bf16 hi / lo ONCE, here, not once per consumer inside the
  // attention kernel.  Without caller scratch the images live in a stream-ordered allocation for the duration of the call.
  void* scratch = nullptr;
  if (!work) {
    B2_CUDA(cudaMallocAsync(&scratch, (size_t)tc_attention_work_bytes(B, H, Lq, Lk), st));
    work = scratch;
  }
  B2_CHECK_ARG(aligned16(work), "attention_f32: work must be 16-byte aligned");
  static bool attr_set = false;
  if (!attr_set) {
    B2_CUDA(cudaFuncSetAttribute(tc_attention_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    attr_set = true;
  }
  const int nk = cdiv(Lk, kAttKeys);
  p.mq_tiles = cdiv(Lq, kAttQ);
  uint8_t* qimg = (uint8_t*)work;
  uint8_t* kimg = qimg + (int64_t)B * H * p.mq_tiles * 32768;
  uint8_t* vimg = kimg + (int64_t)B * H * nk * 32768;
  p.qimg = qimg; p.kimg = kimg; p.vimg = vimg;
  const int64_t nq_chunks = (int64_t)B * H * p.mq_tiles * 1024, nk_chunks = (int64_t)B * H * nk * 1024;
  att_pack_kernel<<<(int)std::min<int64_t>(cdiv(nq_chunks + 2 * nk_chunks, 256), kNumSMs * 32), 256, 0, st>>>(p, qimg, kimg, vimg, nk, nq_chunks, nk_chunks);
  B2_LAUNCHED();
  tc_attention_kernel<<<grid, kAttThreads, smem, st>>>(p);
  B2_LAUNCHED();
  if (scratch) B2_CUDA(cudaFreeAsync(scratch, st));
  return B200SEP_OK;
}


bool tc_enabled() {
  static const bool on = [] {
    const char* e = getenv("B200SEP_TC");
    return !(e && e[0] == '0');
  }();
  return on;
}

int64_t tc_packed_bytes(int N, int K) {
  const int nt = pick_n_tile(N);
  return (int64_t)cdiv(N, nt) * cdiv(K, kTK) * 2 * nt * 128;
}

int tc_pack_linear(const float* W, int N, int K, int ldw, void* packed, cudaStream_t st) {
  const int nt = pick_n_tile(N), iters = cdiv(K, kTK);
  const int64_t total = (int64_t)cdiv(N, nt) * iters * nt * 8;
  tc_pack_kernel<<<(int)std::min<int64_t>(cdiv(total, 256), kNumSMs * 16), 256, 0, st>>>(W, 0, ldw, 1, N, K, 0, 8, 1, nt, iters, (uint8_t*)packed, total);
  B2_LAUNCHED();
  return B200SEP_OK;
}

int tc_pack_conv(const float* w_blocked, int Cin, int taps, int Cout, int CoutPad, void* packed, cudaStream_t st) {
  const int cin8 = (Cin + 7) / 8 * 8, K = cin8 * taps;
  const int nt = pick_n_tile(Cout), iters = cdiv(K, kTK);
  const int64_t total = (int64_t)cdiv(Cout, nt) * iters * nt * 8;
  tc_pack_kernel<<<(int)std::min<int64_t>(cdiv(total, 256), kNumSMs * 16), 256, 0, st>>>(w_blocked, 1, 0, CoutPad, Cout, K, Cin, cin8, taps, nt, iters, (uint8_t*)packed,
                                                                                          total);
  B2_LAUNCHED();
  return B200SEP_OK;
}

bool tc_gemm_usable(int M, int N, int K, int batch) {
  // tiny problems do not fill a 128 x 128 x 64 tile pipeline; the SIMT kernel is faster there
  return K >= 32 && N >= 32 && (int64_t)M * N * batch >= 128 * 128;
}

int tc_gemm_f32(const float* A, const float* Bw, float* C, int M, int N, int K, int lda, int ldb, int ldc, int batch, int64_t sA, int64_t sB, int64_t sC, float alpha,
                const float* bias_n, const float* bias_m, int act, const float* res, const float* res_scale, const void* w_packed, int b_is_kn,
                cudaStream_t st) {
  TcParams p{};
  p.mode = 0;
  p.b_packed = (const uint8_t*)w_packed;
  p.a = A; p.a_sz = sA; p.a_rs = lda;
  p.b = Bw; p.b_sz = sB;
  if (b_is_kn) {  // B given as (K, N) row-major (e.g. V in P @ V): the producers gather it n-major, no transposed copy needed
    p.b_rs = 1; p.b_ks = ldb;
  } else {
    p.b_rs = ldb; p.b_ks = 1;
  }
  p.M = M; p.N = N; p.K = K; p.batch = batch;
  p.a_vec = (lda % 4 == 0) && (sA % 4 == 0) && aligned16(A);
  p.b_vec = (ldb % 4 == 0) && (sB % 4 == 0) && aligned16(Bw);
  p.KH = p.KW = 1; p.Cin8 = 8; p.DH = p.DW = 1;
  p.out = C; p.o_sz = sC; p.o_sm = ldc; p.o_sn = 1;
  p.res = res; p.r_sz = sC; p.r_sm = ldc; p.r_sn = 1;
  p.res_scale = res_scale; p.bias_n = bias_n; p.bias_m = bias_m; p.alpha = alpha; p.act = act; p.add_before_act = 0;
  return tc_launch(p, st);
}

bool tc_conv_usable(int Cin, int Cout, int KH, int KW, int Ho, int Wo, int B) {
  return Cin * KH * KW >= 32 && Cout >= 16 && (int64_t)Ho * Wo * B >= 512;
}

int tc_conv2d_f32(const float* x, const float* w_blocked, const float* bias, const float* add, float* y, int B, int Cin, int H, int W, int Cout, int CoutPad, int Ho,
                  int Wo, int KH, int KW, int SH, int SW, int PH, int PW, int DH, int DW, int act, int add_before_act, int out_c_total, int out_c_off, const void* w_packed,
                  cudaStream_t st, int up_axis, int up, int trim, int out_len) {
  TcParams p{};
  p.mode = 1;
  p.b_packed = (const uint8_t*)w_packed;
  p.a = x; p.a_sz = (int64_t)Cin * H * W; p.a_rs = 0;
  p.b = w_blocked; p.b_sz = 0; p.b_rs = 1; p.b_ks = CoutPad;  // [Cin][KH*KW][CoutPad]: k = (ci, tap) rows, output channel contiguous
  p.Cin8 = (Cin + 7) / 8 * 8;
  p.M = Ho * Wo; p.N = Cout; p.K = p.Cin8 * KH * KW; p.batch = B;  // K in the kernel's (tap, ci padded to 8) order
  p.Cin = Cin; p.H = H; p.W = W; p.Wo = Wo; p.KH = KH; p.KW = KW; p.SH = SH; p.SW = SW; p.PH = PH; p.PW = PW; p.DH = DH; p.DW = DW;
  const int64_t P = (int64_t)Ho * Wo;
  const int ct = out_c_total ? out_c_total : Cout;
  p.out = y + (int64_t)(out_c_total ? out_c_off : 0) * P; p.o_sz = ct * P; p.o_sm = 1; p.o_sn = P;
  p.res = add; p.r_sz = (int64_t)Cout * P; p.r_sm = 1; p.r_sn = P;
  p.res_scale = nullptr; p.bias_n = bias; p.bias_m = nullptr; p.alpha = 1.f; p.act = act; p.add_before_act = add_before_act;
  if (up_axis) {
    B2_CHECK_ARG(up >= 1 && Cout % up == 0 && (Cout / up) % 16 == 0 && add == nullptr && out_c_total == 0, "tc_conv2d_f32: transposed mode needs Cout/up a multiple of 16 and no residual");
    p.up_axis = up_axis; p.up = up; p.trim = trim; p.out_len = out_len; p.up_cout = Cout / up; p.Ho = Ho;
    p.o_sz = (int64_t)(Cout / up) * (up_axis == 1 ? (int64_t)out_len * Wo : (int64_t)Ho * out_len);
  }
  return tc_launch(p, st);
}

}  // namespace b200sep

// softmax(alpha Q K^T) V per (batch, head) for head dimension 64 without materialising the scores (nn.MultiheadAttention of the HTDemucs
// cross-transformer, transformer.py:196-409; Attend of the Roformers).  Layouts in the header.
extern "C" int b200sep_attention_f32(const float* q, const float* k, const float* vt, float* out, int B, int H, int Lq, int Lk, int head_dim, int64_t q_batch_stride,
                                     int64_t q_row_stride, int64_t k_batch_stride, int64_t k_row_stride, int64_t vt_batch_stride, int64_t vt_row_stride,
                                     int64_t out_batch_stride, int64_t out_row_stride, float alpha, int v_is_kn, float* work, void* stream) {
  using namespace b200sep;
  B2_CHECK_ARG(q && k && vt && out && B >= 1 && H >= 1 && Lq >= 1 && Lk >= 1 && alpha > 0.f, "attention_f32: bad argument");
  B2_CHECK_ARG(head_dim == 64, "attention_f32: head dimension %d is not supported (64 only)", head_dim);
  B2_CHECK_ARG(v_is_kn ? vt_row_stride >= 64 : vt_row_stride >= Lk, "attention_f32: V row stride %lld too short", (long long)vt_row_stride);
  return tc_attention_f32(q, k, vt, out, B, H, Lq, Lk, q_batch_stride, q_row_stride, k_batch_stride, k_row_stride, vt_batch_stride, vt_row_stride, out_batch_stride,
                          out_row_stride, alpha, v_is_kn, work, (cudaStream_t)stream);
}

extern "C" int64_t b200sep_attention_work_floats(int B, int H, int Lq, int Lk) {
  if (B < 1 || H < 1 || Lq < 1 || Lk < 1) return 0;
  return b200sep::tc_attention_work_bytes(B, H, Lq, Lk) / 4;
}
