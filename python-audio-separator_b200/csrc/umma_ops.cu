// Hopper (sm_90a) tensor-core operators on "pair" tensors (fp32 values stored as two bf16 planes, hi + lo).
//
// Why pairs: the reference computes the networks in fp32 and parity is gated at 1e-4 on PCM samples; a single
// TF32/BF16 pass misses that (measured 5e-4 / 3e-3 relative on the ConvTDFNet), so every contraction is evaluated as
//      A*B ~= Ah*Bh + Ah*Bl + Al*Bh          (Ah = bf16(A), Al = bf16(A - Ah); dropped terms <= 2^-16 |A||B|)
// with fp32 accumulation: three bf16 wgmma products per k-step at the bf16 rate (measured error 7e-6 relative,
// DESIGN.md).  Producers write activations already split, so a pair tensor costs the same 4 bytes/element as fp32
// and its planes are fed to the tensor cores straight from TMA-written shared memory, no register staging.
//
// One kernel, two addressing modes:
//   GEMM : D[M][N] = A[M][K] * W[N][K]^T     (TDF linears; A, W K-major, TMA SWIZZLE_128B tiles of 64 k)
//   CONV : implicit GEMM for the 3x3 stride-1 convolution on (B,C,T,F) pairs.  The A tile of one filter ROW dy is a
//          TMA box [kc channels][128 pixels along F] at row t+dy-1 (out-of-bounds rows zero-filled = the padding); it
//          lands MN-major (pixels contiguous), which wgmma consumes directly (transposed A).  TMA cannot shift a box
//          by one bf16 along the innermost axis (box starts must be 16-byte aligned), so the horizontal taps are moved
//          to the OUTPUT side: B holds the three dx filter columns side by side (N = 3*n_c accumulator columns,
//          P_dx[m] = W[dy][dx] . x[f0+m]) and the epilogue forms out[f0+j] = P_0[j-1] + P_1[j] + P_2[j+1] with warp
//          shuffles (+ a small smem exchange at warp edges).
// Warp roles per CTA (288 threads): warps 0-7 = two consumer warpgroups (wgmma issue + epilogue), warp 8 = TMA producer.
#include <cuda_bf16.h>
#include <stdlib.h>
#include <string.h>

#include <map>
#include <mutex>
#include <tuple>
#include <vector>

#include "common.cuh"
#include "umma.cuh"
#include "umma_ops.cuh"

namespace b200sep {

using bf16 = __nv_bfloat16;
constexpr int kConsumerThreads = 256;                 // two consumer warpgroups: rows 0-63 and 64-127 of a 128-row tile
constexpr int kUmmaThreads = kConsumerThreads + 32;   // + the TMA producer warp (warp 8)
constexpr int kMaxChannels = 1024;  // per-channel scale/shift staged in shared memory (conv modes)
constexpr int kTileM = 128;
constexpr int kMaxNTile = 128;      // accumulator columns of umma_pair_kernel: n_tile / 2 fp32 registers per consumer thread
constexpr int kConvStride = 112;    // output pixels per 3x3 tile: rows 8..119 of the 128 loaded pixels [f0 - 8, f0 + 120), so that loads AND stores start 16-byte aligned
constexpr int kEpiBar = 1;          // named barrier of the 256 consumer threads

struct UmmaParams {
  int mode;  // 0 GEMM, 1 CONV3x3, 2 UP (ConvTranspose2d k2 s2), 3 DOWN (Conv2d k2 s2), 4 PW (Conv2d 1x1)
  int f_stride, t_mul, t_off;  // implicit-GEMM addressing: tile f0 = blockIdx.x*f_stride, input row = t*t_mul + r + t_off
  int f_off;                   // first input pixel of a tile = f0 + f_off (CONV3x3: -8, so that the 112 outputs of a tile start 16-byte aligned)
  int b_resident;              // CONV3x3 with one weight tile that fits (Cin = Cout = 48: 83 KB): the whole B operand is loaded ONCE per CTA and the ring carries only A
  uint32_t b_res_off;          //   byte offset of the resident image [num_iters][hi | lo] from the start of dynamic shared memory (after alignment)
  int n_tile, n_total;
  int num_iters, ksteps, stages;
  int sleep_ns;  // > 0: the waiting producer sleeps between polls (B200SEP_WAIT_SLEEP_NS)
  int num_tiles, n_ftiles, t_tiles;  // persistent tile walk (n_tiles below = tiles along N / output channels)
  uint32_t a_bytes, b_bytes, stage_bytes;
  // CONV
  int n_chunks, kc, T, F, Cin, Cout, n_tiles, n_c;  // n_c = output channels per CTA
  const bf16* wb_hi;
  const bf16* wb_lo;
  // GEMM
  int M, K, rows_per_channel, channels;
  // epilogue
  const float* scale;
  const float* shift;
  int act;  // 0 none, 1 ReLU, 2 GELU (erf)
  bf16* out_hi;
  bf16* out_lo;
  float* out_f32;      // PW only: write plain fp32 instead of a pair
  const bf16* res_hi;  // GEMM / CONV3x3 / PW: residual (output-shaped, own channel count) ADDED after the activation.  UP: skip tensor MULTIPLIED.
  const bf16* res_lo;
  const bf16* mul_hi;  // CONV3x3 / PW: output-shaped tensor multiplied last
  const bf16* mul_lo;
  int out_c_total, out_c_off;  // conv modes: the output occupies channels [out_c_off, out_c_off + Cout) of a (B, out_c_total, T', F') tensor
};

__device__ __forceinline__ float act1(float x, int act) {
  if (act == 1) return fmaxf(x, 0.f);
  if (act == 2) return 0.5f * x * (1.f + erff(x * 0.70710678118654752440f));
  return x;
}

__device__ __forceinline__ void split_store2(float v, bf16& hi, bf16& lo) {
  hi = __float2bfloat16_rn(v);
  lo = __float2bfloat16_rn(v - __bfloat162float(hi));
}
__device__ __forceinline__ float pair_at(const bf16* hi, const bf16* lo, size_t o) { return __bfloat162float(hi[o]) + __bfloat162float(lo[o]); }

struct TileCoord {
  int m0, n_idx, f0, t, b;
};
// Tile order keeps concurrently running CTAs on neighbouring tiles (same A rows / same weights stay hot in L2).
__device__ __forceinline__ TileCoord decode_tile(const UmmaParams& p, int tile) {
  TileCoord c{0, 0, 0, 0, 0};
  if (p.mode == 0) {
    c.n_idx = tile % p.n_tiles;
    c.m0 = (tile / p.n_tiles) * kTileM;
  } else {
    const int fx = tile % p.n_ftiles;
    int r = tile / p.n_ftiles;
    c.t = r % p.t_tiles;
    r /= p.t_tiles;
    c.n_idx = r % p.n_tiles;
    c.b = r / p.n_tiles;
    c.f0 = fx * p.f_stride;
  }
  return c;
}

// ===== TMA producer (one thread): fills the shared-memory ring, continuous across the tiles of this CTA =====
__device__ __forceinline__ void umma_producer_loop(const CUtensorMap& tmA_hi, const CUtensorMap& tmA_lo, const CUtensorMap& tmB_hi, const CUtensorMap& tmB_lo,
                                                   const UmmaParams& p, uint8_t* smem, uint64_t* full_bar, uint64_t* empty_bar, uint64_t* wres_bar = nullptr) {
  int s = 0;
  uint32_t phase = 0;
  if (p.b_resident) {  // the layer's whole weight operand, once: [iteration][hi | lo] blocks of b_bytes
    ptx::mbar_arrive_expect_tx(wres_bar, 2u * p.b_bytes * (uint32_t)p.num_iters);
    for (int i = 0; i < p.num_iters; ++i) {
      uint8_t* dst = smem + p.b_res_off + (size_t)i * 2 * p.b_bytes;
      ptx::bulk_load_1d(dst, p.wb_hi + (size_t)i * (p.b_bytes / 2), p.b_bytes, wres_bar);
      ptx::bulk_load_1d(dst + p.b_bytes, p.wb_lo + (size_t)i * (p.b_bytes / 2), p.b_bytes, wres_bar);
    }
  }
  for (int tile = blockIdx.x; tile < p.num_tiles; tile += gridDim.x) {
    const TileCoord tc = decode_tile(p, tile);
    const int n0 = tc.n_idx * p.n_tile;
    for (int i = 0; i < p.num_iters; ++i) {
      ptx::mbar_wait_opt(&empty_bar[s], phase ^ 1, p.sleep_ns, 100 + i);
      uint8_t* st = smem + (size_t)s * p.stage_bytes;
      uint8_t* a_hi = st;
      uint8_t* a_lo = st + p.a_bytes;
      uint8_t* b_hi = st + 2 * p.a_bytes;
      uint8_t* b_lo = b_hi + p.b_bytes;
      ptx::mbar_arrive_expect_tx(&full_bar[s], 2 * p.a_bytes + (p.b_resident ? 0 : 2 * p.b_bytes));
      if (p.mode == 0) {
        const int k0 = i * 64;
        ptx::tma_load_2d(a_hi, &tmA_hi, &full_bar[s], k0, tc.m0);
        ptx::tma_load_2d(a_lo, &tmA_lo, &full_bar[s], k0, tc.m0);
        ptx::tma_load_2d(b_hi, &tmB_hi, &full_bar[s], k0, n0);
        ptx::tma_load_2d(b_lo, &tmB_lo, &full_bar[s], k0, n0);
      } else {
        const int r = i / p.n_chunks, chunk = i - r * p.n_chunks;
        const int cf = tc.f0 + p.f_off, ct = tc.t * p.t_mul + r + p.t_off, cc = tc.b * p.Cin + chunk * p.kc;
        const uint32_t box = (uint32_t)p.kc * 128u;
        ptx::tma_load_3d(a_hi, &tmA_hi, &full_bar[s], cf, ct, cc);
        ptx::tma_load_3d(a_hi + box, &tmA_hi, &full_bar[s], cf + 64, ct, cc);
        ptx::tma_load_3d(a_lo, &tmA_lo, &full_bar[s], cf, ct, cc);
        ptx::tma_load_3d(a_lo + box, &tmA_lo, &full_bar[s], cf + 64, ct, cc);
        if (!p.b_resident) {
          const size_t woff = ((size_t)tc.n_idx * p.num_iters + i) * (size_t)(p.b_bytes / 2);
          ptx::bulk_load_1d(b_hi, p.wb_hi + woff, p.b_bytes, &full_bar[s]);
          ptx::bulk_load_1d(b_lo, p.wb_lo + woff, p.b_bytes, &full_bar[s]);
        }
      }
      if (++s == p.stages) {
        s = 0;
        phase ^= 1;
      }
    }
  }
}

// ===== one tile's main loop of a consumer warpgroup =====
// Per ring stage and 16-deep k-step, mma() issues the three products Ah*Bh + Ah*Bl + Al*Bh into the register accumulator.  A stage is released
// (one arrive per consumer thread) when the wgmma group that read it has completed, one stage late, so the tensor core always has the next group queued.
template <class Mma>
__device__ __forceinline__ void consumer_mainloop(const UmmaParams& p, uint8_t* smem, uint64_t* full_bar, uint64_t* empty_bar, int& s, uint32_t& phase, Mma mma) {
  int prev = -1;
  for (int i = 0; i < p.num_iters; ++i) {
    ptx::mbar_wait(&full_bar[s], phase, 200 + i);
    const uint32_t st = ptx::smem_u32(smem + (size_t)s * p.stage_bytes);
    const uint32_t a_hi = st, a_lo = st + p.a_bytes;
    const uint32_t b_hi = p.b_resident ? ptx::smem_u32(smem + p.b_res_off + (size_t)i * 2 * p.b_bytes) : st + 2 * p.a_bytes, b_lo = b_hi + p.b_bytes;
    ptx::wgmma_fence();
    for (int j = 0; j < p.ksteps; ++j) mma(a_hi, a_lo, b_hi, b_lo, j, (i | j) != 0 ? 1 : 0);
    ptx::wgmma_commit();
    ptx::wgmma_wait<1>();
    if (prev >= 0) ptx::mbar_arrive(&empty_bar[prev]);
    prev = s;
    if (++s == p.stages) {
      s = 0;
      phase ^= 1;
    }
  }
  ptx::wgmma_wait<0>();
  if (prev >= 0) ptx::mbar_arrive(&empty_bar[prev]);
}

// A operand descriptors of consumer warpgroup wg (rows 64*wg..): GEMM = K-major 128-byte-swizzled rows of 64 k; conv modes = the two TMA boxes of
// 64 pixels (MN-major, pixels contiguous), box wg; k-step j
__device__ __forceinline__ uint64_t a_desc(const UmmaParams& p, uint32_t a, int wg, int j) {
  if (p.mode == 0) return ptx::smem_desc(a + (uint32_t)wg * 8192u + (uint32_t)j * 32u, 16, 1024, ptx::kLayoutSW128);
  const uint32_t lbo = (uint32_t)p.kc * 128u;
  return ptx::smem_desc(a + (uint32_t)wg * lbo + (uint32_t)j * 2048u, lbo, 1024, ptx::kLayoutSW128);
}
// B operand: GEMM = K-major swizzled rows of 64 k; conv modes = one [n_tile][16] block of 8x8 core matrices per k-step
__device__ __forceinline__ uint64_t b_desc(const UmmaParams& p, uint32_t b, int j) {
  if (p.mode == 0) return ptx::smem_desc(b + (uint32_t)j * 32u, 16, 1024, ptx::kLayoutSW128);
  return ptx::smem_desc(b + (uint32_t)j * (uint32_t)p.n_tile * 32u, 128, 256, ptx::kLayoutNone);
}

// Persistent kernel: grid = min(#tiles, #SMs); every CTA walks tiles blockIdx.x, +gridDim.x, ...  The producer warp keeps the shared-memory ring
// (full/empty mbarriers) filled across tiles while the two consumer warpgroups multiply (wgmma, fp32 accumulators in registers) and run the
// epilogue straight from their accumulator fragments.
// Accumulator column layouts (the weight blocking below produces them): GEMM n; UP co*4 + (dy*2 + dx); DOWN co*2 + dx; PW co -- so the
// columns a thread holds in one register pair (2c, 2c + 1) always belong together.
__global__ void __launch_bounds__(kUmmaThreads, 1) umma_pair_kernel(const __grid_constant__ CUtensorMap tmA_hi, const __grid_constant__ CUtensorMap tmA_lo,
                                                                    const __grid_constant__ CUtensorMap tmB_hi, const __grid_constant__ CUtensorMap tmB_lo,
                                                                    const UmmaParams p) {
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  // 1024-byte alignment for SWIZZLE_128B tiles.  The offset is applied to the __shared__ array itself (not through an integer
  // round trip) so every derived pointer keeps the shared address space.
  uint8_t* smem = smem_raw + ((1024u - (ptx::smem_u32(smem_raw) & 1023u)) & 1023u);
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + (size_t)p.stages * p.stage_bytes);
  uint64_t* empty_bar = full_bar + p.stages;
  float* sc_s = reinterpret_cast<float*>(empty_bar + p.stages + 2);  // conv modes: folded BatchNorm scale / shift per output channel
  float* sh_s = sc_s + kMaxChannels;

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;

  if (threadIdx.x == 0) {
    for (int s = 0; s < p.stages; ++s) {
      ptx::mbar_init(&full_bar[s], 1);
      ptx::mbar_init(&empty_bar[s], kConsumerThreads);
    }
    ptx::fence_barrier_init();
    ptx::prefetch_tensormap(&tmA_hi);
    ptx::prefetch_tensormap(&tmA_lo);
    if (p.mode == 0) {
      ptx::prefetch_tensormap(&tmB_hi);
      ptx::prefetch_tensormap(&tmB_lo);
    }
  }
  if (p.mode != 0) {
    for (int i = threadIdx.x; i < p.Cout; i += blockDim.x) {
      sc_s[i] = p.scale ? __ldg(&p.scale[i]) : 1.f;
      sh_s[i] = p.shift ? __ldg(&p.shift[i]) : 0.f;
    }
  }
  __syncthreads();

  if (warp == kConsumerThreads / 32) {
    if (lane == 0) umma_producer_loop(tmA_hi, tmA_lo, tmB_hi, tmB_lo, p, smem, full_bar, empty_bar);
    return;
  }
  const int wg = warp >> 2, g = lane >> 2, cq = lane & 3;
  const int mrow0 = wg * 64 + (warp & 3) * 16 + g;  // tile rows of this thread: mrow0 and mrow0 + 8
  int s = 0;
  uint32_t phase = 0;
  float acc[kMaxNTile / 2];
  for (int tile = blockIdx.x; tile < p.num_tiles; tile += gridDim.x) {
    const TileCoord tc = decode_tile(p, tile);
    if (p.mode == 0) {
      consumer_mainloop(p, smem, full_bar, empty_bar, s, phase, [&](uint32_t ah, uint32_t al, uint32_t bh, uint32_t bl, int j, int accum) {
        const uint64_t dah = a_desc(p, ah, wg, j), dal = a_desc(p, al, wg, j), dbh = b_desc(p, bh, j), dbl = b_desc(p, bl, j);
        ptx::wgmma_ss<0>(p.n_tile, acc, dah, dbh, accum);
        ptx::wgmma_ss<0>(p.n_tile, acc, dah, dbl, 1);
        ptx::wgmma_ss<0>(p.n_tile, acc, dal, dbh, 1);
      });
    } else {
      consumer_mainloop(p, smem, full_bar, empty_bar, s, phase, [&](uint32_t ah, uint32_t al, uint32_t bh, uint32_t bl, int j, int accum) {
        const uint64_t dah = a_desc(p, ah, wg, j), dal = a_desc(p, al, wg, j), dbh = b_desc(p, bh, j), dbl = b_desc(p, bl, j);
        ptx::wgmma_ss<1>(p.n_tile, acc, dah, dbh, accum);
        ptx::wgmma_ss<1>(p.n_tile, acc, dah, dbl, 1);
        ptx::wgmma_ss<1>(p.n_tile, acc, dal, dbh, 1);
      });
    }
    ptx::fence_regs(acc);

    // ===== epilogue: accumulator fragments -> BN/act(/+res, *skip) -> split into bf16 hi/lo -> global =====
    if (p.mode == 0) {
      const int n0 = tc.n_idx * p.n_tile;
      float sc[2], sh[2];
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int r = tc.m0 + mrow0 + 8 * h;
        sc[h] = 1.f;
        sh[h] = 0.f;
        if (r < p.M) {
          const int c = (r / p.rows_per_channel) % p.channels;
          sc[h] = p.scale ? __ldg(&p.scale[c]) : 1.f;
          sh[h] = p.shift ? __ldg(&p.shift[c]) : 0.f;
        }
      }
#pragma unroll
      for (int i = 0; i < kMaxNTile / 8; ++i) {
        if (8 * i >= p.n_tile) break;
        const int n = n0 + 8 * i + 2 * cq;
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const int r = tc.m0 + mrow0 + 8 * h;
          if (r >= p.M) continue;
          const size_t o = (size_t)r * p.n_total + n;
          float y0 = act1(fmaf(acc[4 * i + 2 * h], sc[h], sh[h]), p.act), y1 = act1(fmaf(acc[4 * i + 2 * h + 1], sc[h], sh[h]), p.act);
          if (p.res_hi) {
            y0 += pair_at(p.res_hi, p.res_lo, o);
            y1 += pair_at(p.res_hi, p.res_lo, o + 1);
          }
          __nv_bfloat162 oh, ol;
          split_store2(y0, oh.x, ol.x);
          split_store2(y1, oh.y, ol.y);
          *reinterpret_cast<__nv_bfloat162*>(p.out_hi + o) = oh;
          *reinterpret_cast<__nv_bfloat162*>(p.out_lo + o) = ol;
        }
      }
    } else if (p.mode == 2) {
      // ConvTranspose2d k2 s2: the register pair (col, col + 1), col = co*4 + dy*2, holds output pixels (2t+dy, 2f) and (2t+dy, 2f+1) of channel co,
      // f = f0 + row; then BN + ReLU, times the skip tensor (uvr_lib_v5/mdxnet.py:111-112), stored as one 4-byte pair per plane.
      const int c0 = tc.n_idx * p.n_c;
      const int T2 = 2 * p.T, F2 = 2 * p.F;
      const size_t plane = (size_t)T2 * F2;
#pragma unroll
      for (int i = 0; i < kMaxNTile / 8; ++i) {
        if (8 * i >= p.n_tile) break;
        const int col = 8 * i + 2 * cq, co = c0 + (col >> 2), dy = (col >> 1) & 1;
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const int f = tc.f0 + mrow0 + 8 * h;
          if (f >= p.F) continue;
          const size_t pix = (size_t)(2 * tc.t + dy) * F2 + 2 * f;
          const size_t o = ((size_t)tc.b * p.out_c_total + p.out_c_off + co) * plane + pix;
          float x0 = act1(fmaf(acc[4 * i + 2 * h], sc_s[co], sh_s[co]), p.act), x1 = act1(fmaf(acc[4 * i + 2 * h + 1], sc_s[co], sh_s[co]), p.act);
          if (p.res_hi) {  // skip tensor: own channel count; bf16 -> fp32 is a 16-bit shift: low half = dx 0, high half = dx 1
            const size_t so = ((size_t)tc.b * p.Cout + co) * plane + pix;
            const uint32_t sk_h = __ldg(reinterpret_cast<const unsigned int*>(p.res_hi + so)), sk_l = __ldg(reinterpret_cast<const unsigned int*>(p.res_lo + so));
            x0 *= __uint_as_float(sk_h << 16) + __uint_as_float(sk_l << 16);
            x1 *= __uint_as_float(sk_h & 0xffff0000u) + __uint_as_float(sk_l & 0xffff0000u);
          }
          __nv_bfloat162 oh, ol;
          split_store2(x0, oh.x, ol.x);
          split_store2(x1, oh.y, ol.y);
          *reinterpret_cast<__nv_bfloat162*>(p.out_hi + o) = oh;
          *reinterpret_cast<__nv_bfloat162*>(p.out_lo + o) = ol;
        }
      }
    } else if (p.mode == 3) {
      // Conv2d k2 s2: the register pair (col, col + 1), col = co*2, holds P_0 and P_1 of channel co, the partial sums over (ci, dy) at INPUT pixel
      // f0 + row; out[(f0+row)/2] = P_0[row] + P_1[row+1] for even rows (row + 1 is lane + 4: same register, same warp).
      const int c0 = tc.n_idx * p.n_c;
      const int Fo = p.F >> 1, To = p.T >> 1;
      const size_t plane = (size_t)To * Fo;
#pragma unroll
      for (int i = 0; i < kMaxNTile / 8; ++i) {
        if (8 * i >= p.n_tile) break;
        const int co = c0 + 4 * i + cq;
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const float p1 = __shfl_down_sync(0xffffffffu, acc[4 * i + 2 * h + 1], 4);
          const int fo = (tc.f0 + mrow0 + 8 * h) >> 1;
          if ((g & 1) == 0 && fo < Fo) {
            const float y = act1(fmaf(acc[4 * i + 2 * h] + p1, sc_s[co], sh_s[co]), p.act);
            const size_t o = ((size_t)tc.b * p.out_c_total + p.out_c_off + co) * plane + (size_t)tc.t * Fo + fo;
            split_store2(y, p.out_hi[o], p.out_lo[o]);
          }
        }
      }
    } else if (p.mode == 4) {
      // 1x1 convolution: column co is channel c0 + co at output pixel f0 + row
      const int c0 = tc.n_idx * p.n_c;
      const size_t plane = (size_t)p.T * p.F;
#pragma unroll
      for (int i = 0; i < kMaxNTile / 8; ++i) {
        if (8 * i >= p.n_tile) break;
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const int f = tc.f0 + mrow0 + 8 * h;
          if (f >= p.F) continue;
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            const int co = c0 + 8 * i + 2 * cq + e;
            float y = act1(fmaf(acc[4 * i + 2 * h + e], sc_s[co], sh_s[co]), p.act);
            const size_t ro = ((size_t)tc.b * p.Cout + co) * plane + (size_t)tc.t * p.F + f;
            if (p.res_hi) y += pair_at(p.res_hi, p.res_lo, ro);
            if (p.mul_hi) y *= pair_at(p.mul_hi, p.mul_lo, ro);
            const size_t o = ((size_t)tc.b * p.out_c_total + p.out_c_off + co) * plane + (size_t)tc.t * p.F + f;
            if (p.out_f32) p.out_f32[o] = y;
            else split_store2(y, p.out_hi[o], p.out_lo[o]);
          }
        }
      }
    }  // (CONV3x3 has its own kernel, umma_conv3_kernel)
  }
}

// ---------------------------------------------------------------------------------------------------------
// CONV3x3 kernel (NC = output channels per CTA).  Same producer / ring as umma_pair_kernel; accumulator column dx*NC + co holds
// P_dx[row] = W[dy][dx] . x[f0 - 8 + row] summed over (ci, dy), and the epilogue forms out[j] = P_0[j-1] + P_1[j] + P_2[j+1]:
//   * a tile loads the 128 pixels [f0 - 8, f0 + 120) (TMA zero-fills the left / right padding) and produces the 112 outputs
//     [f0, f0 + 112) = rows 8..119, so both the loads and the STORES start 16-byte aligned (TMA faults on any other innermost coordinate);
//   * row +-1 of a fragment row is lane +-4 (warp shuffles); the rows across a warp boundary go through a small shared-memory exchange;
//   * folded BatchNorm + activation (+ residual, * multiplier), bf16 hi/lo split, staged in shared memory as [channel][pixel] planes
//     and written with one cp.async.bulk.tensor store per plane: full 224-byte rows per channel.
template <int NC>
__device__ __forceinline__ void conv3_mma(float (&acc)[3 * NC / 2], uint64_t da, uint64_t db, int accum) {
  if constexpr (NC == 16) ptx::wgmma_ss_n48<1>(acc, da, db, accum);
  else if constexpr (NC == 32) ptx::wgmma_ss_n96<1>(acc, da, db, accum);
  else if constexpr (NC == 48) ptx::wgmma_ss_n144<1>(acc, da, db, accum);
  else if constexpr (NC == 64) ptx::wgmma_ss_n192<1>(acc, da, db, accum);
  else ptx::wgmma_ss_n240<1>(acc, da, db, accum);
}

template <int NC>
__global__ void __launch_bounds__(kUmmaThreads, 1) umma_conv3_kernel(const __grid_constant__ CUtensorMap tmA_hi, const __grid_constant__ CUtensorMap tmA_lo,
                                                                     const __grid_constant__ CUtensorMap tmO_hi, const __grid_constant__ CUtensorMap tmO_lo,
                                                                     const UmmaParams p) {
  constexpr int kPlane = NC * kConvStride;  // bf16 elements of one staged plane [NC][112]
  constexpr int G = NC / 8;                 // 8-column groups per dx
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = smem_raw + ((1024u - (ptx::smem_u32(smem_raw) & 1023u)) & 1023u);
  // [ring: stages x stage_bytes][resident weights, when b_resident][output staging hi | lo][barriers][BN coefficients][edge rows]
  bf16* s_hi = reinterpret_cast<bf16*>(smem + (size_t)p.stages * p.stage_bytes + (p.b_resident ? (size_t)2 * p.b_bytes * p.num_iters : 0));
  bf16* s_lo = s_hi + kPlane;
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(s_lo + kPlane);
  uint64_t* empty_bar = full_bar + p.stages;
  uint64_t* wres_bar = empty_bar + p.stages;
  float* sc_s = reinterpret_cast<float*>(wres_bar + 2);
  float* sh_s = sc_s + kMaxChannels;
  float* edge0 = sh_s + kMaxChannels;  // [8 warps][NC]: P_0 of the warp's last row (row 16w + 15)
  float* edge2 = edge0 + 8 * NC;       // [8 warps][NC]: P_2 of the warp's first row (row 16w)

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (threadIdx.x == 0) {
    for (int s = 0; s < p.stages; ++s) {
      ptx::mbar_init(&full_bar[s], 1);
      ptx::mbar_init(&empty_bar[s], kConsumerThreads);
    }
    ptx::mbar_init(wres_bar, 1);
    ptx::fence_barrier_init();
    ptx::prefetch_tensormap(&tmA_hi);
    ptx::prefetch_tensormap(&tmA_lo);
    ptx::prefetch_tensormap(&tmO_hi);
    ptx::prefetch_tensormap(&tmO_lo);
  }
  for (int i = threadIdx.x; i < p.Cout; i += blockDim.x) {
    sc_s[i] = p.scale ? __ldg(&p.scale[i]) : 1.f;
    sh_s[i] = p.shift ? __ldg(&p.shift[i]) : 0.f;
  }
  __syncthreads();

  if (warp == kConsumerThreads / 32) {
    if (lane == 0) umma_producer_loop(tmA_hi, tmA_lo, tmA_hi, tmA_lo, p, smem, full_bar, empty_bar, wres_bar);
    return;
  }
  const int wg = warp >> 2, g = lane >> 2, cq = lane & 3;
  const int mrow0 = wg * 64 + (warp & 3) * 16 + g;  // tile rows mrow0 and mrow0 + 8
  const bool issuer = threadIdx.x == 0;             // owns the bulk store groups
  if (p.b_resident) ptx::mbar_wait(wres_bar, 0, 500);  // the resident weight image has landed
  int s = 0;
  uint32_t phase = 0;
  float acc[3 * NC / 2];
  for (int tile = blockIdx.x; tile < p.num_tiles; tile += gridDim.x) {
    const TileCoord tc = decode_tile(p, tile);
    consumer_mainloop(p, smem, full_bar, empty_bar, s, phase, [&](uint32_t ah, uint32_t al, uint32_t bh, uint32_t bl, int j, int accum) {
      const uint64_t dah = a_desc(p, ah, wg, j), dal = a_desc(p, al, wg, j), dbh = b_desc(p, bh, j), dbl = b_desc(p, bl, j);
      conv3_mma<NC>(acc, dah, dbh, accum);
      conv3_mma<NC>(acc, dah, dbl, 1);
      conv3_mma<NC>(acc, dal, dbh, 1);
    });
    ptx::fence_regs(acc);
    // boundary rows for the neighbouring warps
#pragma unroll
    for (int i = 0; i < G; ++i) {
      const int col = 8 * i + 2 * cq;
      if (g == 7) *reinterpret_cast<float2*>(&edge0[warp * NC + col]) = make_float2(acc[4 * i + 2], acc[4 * i + 3]);
      if (g == 0) *reinterpret_cast<float2*>(&edge2[warp * NC + col]) = make_float2(acc[4 * (2 * G + i)], acc[4 * (2 * G + i) + 1]);
    }
    // the staging planes must have been read out by the previous tile's store
    if (issuer) ptx::bulk_wait_read<0>();
    asm volatile("bar.sync %0, %1;" ::"n"(kEpiBar), "n"(kConsumerThreads) : "memory");
    const int n0 = tc.n_idx * NC;
#pragma unroll
    for (int i = 0; i < G; ++i) {
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        const int col = 8 * i + 2 * cq + e;
        const float p0a = acc[4 * i + e], p0b = acc[4 * i + 2 + e];
        const float p1a = acc[4 * (G + i) + e], p1b = acc[4 * (G + i) + 2 + e];
        const float p2a = acc[4 * (2 * G + i) + e], p2b = acc[4 * (2 * G + i) + 2 + e];
        const float up_a = __shfl_sync(0xffffffffu, p0a, (lane + 28) & 31), up_b = __shfl_sync(0xffffffffu, p0b, (lane + 28) & 31);
        const float dn_a = __shfl_sync(0xffffffffu, p2a, (lane + 4) & 31), dn_b = __shfl_sync(0xffffffffu, p2b, (lane + 4) & 31);
        const float prev = (g == 0 && warp > 0) ? edge0[(warp - 1) * NC + col] : 0.f;
        const float next = (g == 7 && warp < 7) ? edge2[(warp + 1) * NC + col] : 0.f;
        float x[2];
        x[0] = p1a + ((g > 0) ? up_a : prev) + ((g < 7) ? dn_a : dn_b);
        x[1] = p1b + ((g > 0) ? up_b : up_a) + ((g < 7) ? dn_b : next);
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const int m = mrow0 + 8 * h;
          if (m < 8 || m >= 8 + kConvStride) continue;
          float y = act1(fmaf(x[h], sc_s[n0 + col], sh_s[n0 + col]), p.act);
          const int f = tc.f0 + m - 8;
          if ((p.res_hi || p.mul_hi) && f < p.F) {
            const size_t plane = (size_t)p.T * p.F;
            const size_t ro = ((size_t)tc.b * p.Cout + n0 + col) * plane + (size_t)tc.t * p.F + f;  // residual / multiplier: (B, Cout, T, F)
            if (p.res_hi) y += pair_at(p.res_hi, p.res_lo, ro);
            if (p.mul_hi) y *= pair_at(p.mul_hi, p.mul_lo, ro);
          }
          split_store2(y, s_hi[col * kConvStride + (m - 8)], s_lo[col * kConvStride + (m - 8)]);
        }
      }
    }
    ptx::fence_proxy_async();
    asm volatile("bar.sync %0, %1;" ::"n"(kEpiBar), "n"(kConsumerThreads) : "memory");
    if (issuer) {
      const int cc = tc.b * p.out_c_total + p.out_c_off + n0;
      ptx::tma_store_3d(&tmO_hi, s_hi, tc.f0, tc.t, cc);
      ptx::tma_store_3d(&tmO_lo, s_lo, tc.f0, tc.t, cc);
      ptx::bulk_commit();
    }
  }
  if (issuer) ptx::bulk_wait_all();
}

// ---------------------------------------------------------------------------------------------------------
// host side
typedef CUresult (*PFN_encodeTiled)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*, const cuuint32_t*,
                                    const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static PFN_encodeTiled get_encode() {
  static PFN_encodeTiled fn = nullptr;
  if (!fn) {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult qres;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qres) == cudaSuccess && qres == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<PFN_encodeTiled>(p);
  }
  return fn;
}

// bf16 tensor map, SWIZZLE_128B, zero OOB fill.  dims/box innermost first; strides in BYTES for dims 1..rank-1.
static int make_map(CUtensorMap* map, const void* base, int rank, const uint64_t* dims, const uint64_t* strides_bytes, const uint32_t* box,
                    CUtensorMapSwizzle swizzle = CU_TENSOR_MAP_SWIZZLE_128B) {
  PFN_encodeTiled enc = get_encode();
  if (!enc) {
    set_error("cuTensorMapEncodeTiled is not available from the driver");
    return B200SEP_ERR_CUDA;
  }
  cuuint64_t gd[5], gs[4];
  cuuint32_t bx[5], es[5];
  for (int i = 0; i < rank; ++i) {
    gd[i] = dims[i];
    bx[i] = box[i];
    es[i] = 1;
    if (i > 0) gs[i - 1] = strides_bytes[i - 1];
  }
  CUresult r = enc(map, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, (cuuint32_t)rank, const_cast<void*>(base), gd, gs, bx, es, CU_TENSOR_MAP_INTERLEAVE_NONE,
                   swizzle, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    set_error("cuTensorMapEncodeTiled failed (CUresult %d) rank=%d dims=[%llu,%llu,%llu] box=[%u,%u,%u]", (int)r, rank, (unsigned long long)dims[0],
              (unsigned long long)(rank > 1 ? dims[1] : 0), (unsigned long long)(rank > 2 ? dims[2] : 0), box[0], rank > 1 ? box[1] : 0, rank > 2 ? box[2] : 0);
    return B200SEP_ERR_CUDA;
  }
  return B200SEP_OK;
}

static int num_sms() {
  static int n = 0;
  if (n == 0) {
    int dev = 0;
    cudaGetDevice(&dev);
    if (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || n <= 0) n = kNumSMs;
  }
  return n;
}

static int umma_wait_sleep_ns() {
  static const int ns = [] {
    const char* e = getenv("B200SEP_WAIT_SLEEP_NS");
    return e ? atoi(e) : 0;
  }();
  return ns;
}

// Persistent launch: one CTA per SM.
template <class Kernel, class... Args>
static int launch_persistent(Kernel kernel, int num_tiles, size_t smem, cudaStream_t st, Args... args) {
  const int grid = std::min(num_tiles, num_sms());
  kernel<<<grid, kUmmaThreads, smem, st>>>(args...);
  B2_LAUNCHED();
  return B200SEP_OK;
}

// `tiles` is the logical tile grid: GEMM (n tiles, m tiles, 1); conv modes (f tiles, output rows, batch * channel tiles).
static int launch(const CUtensorMap& a_hi, const CUtensorMap& a_lo, const CUtensorMap& b_hi, const CUtensorMap& b_lo, UmmaParams& p, dim3 tiles,
                  cudaStream_t st) {
  p.sleep_ns = umma_wait_sleep_ns();
  B2_CHECK_ARG(p.n_tile % 16 == 0 && p.n_tile >= 16 && p.n_tile <= kMaxNTile, "umma: n_tile=%d is not a multiple of 16 in [16, %d]", p.n_tile, kMaxNTile);
  p.stage_bytes = ((2 * p.a_bytes + 2 * p.b_bytes + 1023) / 1024) * 1024;
  if (p.mode == 0) p.n_tiles = (int)tiles.x;
  p.n_ftiles = (int)tiles.x;
  p.t_tiles = (int)tiles.y;
  p.num_tiles = (int)(tiles.x * tiles.y * tiles.z);
  const size_t fixed = 1024 /*alignment slack*/ + 64 * sizeof(uint64_t) + 64 + 2 * kMaxChannels * sizeof(float);
  B2_CHECK_ARG(p.mode == 0 || p.Cout <= kMaxChannels, "umma: more than %d output channels", kMaxChannels);
  const size_t budget = 227 * 1024 - fixed;  // one persistent CTA per SM
  int stages = (int)(budget / p.stage_bytes);
  if (stages > 8) stages = 8;
  B2_CHECK_ARG(stages >= 2, "umma: a pipeline stage of %u bytes does not fit twice in shared memory", p.stage_bytes);
  p.stages = stages;
  const size_t smem = (size_t)stages * p.stage_bytes + fixed;
  static bool attr_set = false;
  if (!attr_set) {
    B2_CUDA(cudaFuncSetAttribute(umma_pair_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024));
    attr_set = true;
  }
  return launch_persistent(umma_pair_kernel, p.num_tiles, smem, st, a_hi, a_lo, b_hi, b_lo, p);
}

bool umma_gemm_supported(int M, int N, int K) { return M >= 1 && N % 16 == 0 && K % 8 == 0 && N >= 16 && K >= 16; }

int umma_gemm_plan_create(UmmaGemmPlan* pl, const void* a_hi, const void* a_lo, const void* w_hi, const void* w_lo, int M, int N, int K) {
  pl->M = M; pl->N = N; pl->K = K;
  int n_tile = N <= 128 ? N : 128;
  if (N > 128 && N % 128 != 0) {
    for (n_tile = 128; n_tile >= 16; n_tile -= 16)
      if (N % n_tile == 0) break;
  }
  pl->n_tile = n_tile;
  const uint64_t da[2] = {(uint64_t)K, (uint64_t)M}, sa[1] = {(uint64_t)K * 2};
  const uint32_t ba[2] = {64, 128};
  const uint64_t db[2] = {(uint64_t)K, (uint64_t)N};
  const uint32_t bb[2] = {64, (uint32_t)n_tile};
  int rc = make_map(&pl->a_hi, a_hi, 2, da, sa, ba);
  if (!rc) rc = make_map(&pl->a_lo, a_lo, 2, da, sa, ba);
  if (!rc) rc = make_map(&pl->b_hi, w_hi, 2, db, sa, bb);
  if (!rc) rc = make_map(&pl->b_lo, w_lo, 2, db, sa, bb);
  return rc;
}

static void fill_epilogue(UmmaParams& p, const UmmaEpilogue& e, int Cout) {
  p.scale = e.scale; p.shift = e.shift; p.act = e.act;
  p.out_hi = (bf16*)e.out_hi; p.out_lo = (bf16*)e.out_lo; p.out_f32 = e.out_f32;
  p.res_hi = (const bf16*)e.res_hi; p.res_lo = (const bf16*)e.res_lo;
  p.mul_hi = (const bf16*)e.mul_hi; p.mul_lo = (const bf16*)e.mul_lo;
  p.out_c_total = e.out_c_total > 0 ? e.out_c_total : Cout;
  p.out_c_off = e.out_c_off;
}

int umma_gemm_run(const UmmaGemmPlan& pl, const float* scale, const float* shift, int rows_per_channel, int channels, int relu, void* out_hi,
                  void* out_lo, const void* res_hi, const void* res_lo, int M_active, cudaStream_t st) {
  UmmaEpilogue e;
  e.scale = scale; e.shift = shift; e.act = relu ? 1 : 0; e.out_hi = out_hi; e.out_lo = out_lo; e.res_hi = res_hi; e.res_lo = res_lo;
  return umma_gemm_run_ex(pl, rows_per_channel, channels, M_active, e, st);
}

int umma_gemm_run_ex(const UmmaGemmPlan& pl, int rows_per_channel, int channels, int M_active, const UmmaEpilogue& e, cudaStream_t st) {
  const float* scale = e.scale; const float* shift = e.shift; const int relu = e.act;
  void* out_hi = e.out_hi; void* out_lo = e.out_lo; const void* res_hi = e.res_hi; const void* res_lo = e.res_lo;
  UmmaParams p{};
  p.mode = 0;
  p.n_tile = pl.n_tile; p.n_total = pl.N;
  p.num_iters = (pl.K + 63) / 64; p.ksteps = 4;
  p.a_bytes = 128 * 128; p.b_bytes = (uint32_t)pl.n_tile * 128;
  p.M = M_active; p.K = pl.K; p.rows_per_channel = rows_per_channel; p.channels = channels;
  p.scale = scale; p.shift = shift; p.act = relu;
  p.out_hi = (bf16*)out_hi; p.out_lo = (bf16*)out_lo; p.res_hi = (const bf16*)res_hi; p.res_lo = (const bf16*)res_lo;
  dim3 grid(pl.N / pl.n_tile, cdiv(M_active, kTileM));
  return launch(pl.a_hi, pl.a_lo, pl.b_hi, pl.b_lo, p, grid, st);
}

bool umma_conv_supported(int Cin, int Cout, int F, int kh, int kw) {
  return Cin % 16 == 0 && Cout % 16 == 0 && F % 8 == 0 && kh == 3 && kw == 3;
}

// kc = input channels per pipeline stage, n_c = output channels per CTA (3*n_c accumulator columns <= 256)
int umma_conv_choose(int Cin, int Cout, int* kc, int* n_c) {
  int k = 64;
  while (k > 16 && Cin % k != 0) k -= 16;
  if (Cin % 48 == 0) k = 48;
  int nc = 16;
  const int cand[5] = {48, 80, 64, 32, 16};
  for (int i = 0; i < 5; ++i)
    if (Cout % cand[i] == 0) {
      nc = cand[i];
      break;
    }
  // the ring needs at least two stages next to the output staging tile of the TMA-store epilogue: shrink the channel step of wide tiles
  // (n_c = 80 with 64 channels per stage is a 92 KB stage: MDX23C's 640-channel scale)
  auto fits = [&](int kk) {
    const size_t stage = ((size_t)2 * kk * 256 + (size_t)2 * (kk / 16) * (3 * nc) * 32 + 1023) / 1024 * 1024;
    const size_t staging = (size_t)2 * nc * kConvStride * 2;  // hi + lo output planes
    return 2 * stage + staging + 16 * 1024 <= 227 * 1024;
  };
  while (!fits(k) && k > 16) {
    int kk = k - 16;
    while (kk > 16 && Cin % kk != 0) kk -= 16;
    if (Cin % kk != 0) break;
    k = kk;
  }
  *kc = k;
  *n_c = nc;
  return 0;
}

int umma_conv_plan_create(UmmaConvPlan* pl, const void* x_hi, const void* x_lo, int Bmax, int Cin, int T, int F, int kc) {
  pl->Cin = Cin; pl->T = T; pl->F = F; pl->kc = kc;
  const uint64_t d[3] = {(uint64_t)F, (uint64_t)T, (uint64_t)Bmax * Cin};
  const uint64_t s[2] = {(uint64_t)F * 2, (uint64_t)T * F * 2};
  const uint32_t bx[3] = {64, 1, (uint32_t)kc};
  int rc = make_map(&pl->a_hi, x_hi, 3, d, s, bx);
  if (!rc) rc = make_map(&pl->a_lo, x_lo, 3, d, s, bx);
  return rc;
}

int umma_conv_run(const UmmaConvPlan& pl, const void* wb_hi, const void* wb_lo, int B, int Cout, int n_c, int ksize, const float* scale,
                  const float* shift, int relu, void* out_hi, void* out_lo, cudaStream_t st) {
  B2_CHECK_ARG(ksize == 3, "umma_conv: only 3x3 kernels");
  UmmaEpilogue e;
  e.scale = scale; e.shift = shift; e.act = relu ? 1 : 0; e.out_hi = out_hi; e.out_lo = out_lo;
  return umma_conv_run_ex(pl, wb_hi, wb_lo, B, Cout, n_c, e, st);
}

// TMA store maps of a conv3x3 output: the (F, T, B * C_total) bf16 planes with a [112 px][1 row][NC channels] box, no swizzle.  Encoding a map costs a few
// microseconds on the host and the same activation buffers are written forward after forward, so the maps are cached by (plane address, geometry).
struct StoreMapKey {
  const void* base; int F, T, C, box_c;
  bool operator<(const StoreMapKey& o) const { return std::tie(base, F, T, C, box_c) < std::tie(o.base, o.F, o.T, o.C, o.box_c); }
};
static int store_map(const void* base, int F, int T, int C, int box_c, CUtensorMap* out) {
  static std::map<StoreMapKey, CUtensorMap> cache;
  static std::mutex mu;
  std::lock_guard<std::mutex> lock(mu);
  const StoreMapKey key{base, F, T, C, box_c};
  auto it = cache.find(key);
  if (it == cache.end()) {
    CUtensorMap m;
    const uint64_t d[3] = {(uint64_t)F, (uint64_t)T, (uint64_t)C};
    const uint64_t st[2] = {(uint64_t)F * 2, (uint64_t)T * F * 2};
    const uint32_t bx[3] = {(uint32_t)kConvStride, 1, (uint32_t)box_c};
    int rc = make_map(&m, base, 3, d, st, bx, CU_TENSOR_MAP_SWIZZLE_NONE);
    if (rc) return rc;
    if (cache.size() > 4096) cache.clear();
    it = cache.emplace(key, m).first;
  }
  *out = it->second;
  return B200SEP_OK;
}

template <int NC>
static int launch_conv3(const CUtensorMap& a_hi, const CUtensorMap& a_lo, const CUtensorMap& o_hi, const CUtensorMap& o_lo, UmmaParams& p, size_t smem, cudaStream_t st) {
  static bool attr_set = false;
  if (!attr_set) {
    B2_CUDA(cudaFuncSetAttribute(umma_conv3_kernel<NC>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024));
    attr_set = true;
  }
  p.sleep_ns = umma_wait_sleep_ns();
  return launch_persistent(umma_conv3_kernel<NC>, p.num_tiles, smem, st, a_hi, a_lo, o_hi, o_lo, p);
}

int umma_conv_run_ex(const UmmaConvPlan& pl, const void* wb_hi, const void* wb_lo, int B, int Cout, int n_c, const UmmaEpilogue& e, cudaStream_t st) {
  UmmaParams p{};
  p.mode = 1; p.f_stride = kConvStride; p.f_off = -8; p.t_mul = 1; p.t_off = -1;
  p.n_c = n_c; p.n_tile = 3 * n_c; p.n_total = Cout;
  p.kc = pl.kc; p.n_chunks = pl.Cin / pl.kc;
  p.num_iters = 3 * p.n_chunks; p.ksteps = pl.kc / 16;
  p.a_bytes = (uint32_t)pl.kc * 256; p.b_bytes = (uint32_t)p.ksteps * p.n_tile * 32;
  p.T = pl.T; p.F = pl.F; p.Cin = pl.Cin; p.Cout = Cout; p.n_tiles = Cout / n_c;
  p.wb_hi = (const bf16*)wb_hi; p.wb_lo = (const bf16*)wb_lo;
  fill_epilogue(p, e, Cout);
  B2_CHECK_ARG(Cout <= kMaxChannels, "umma_conv: more than %d output channels", kMaxChannels);
  B2_CHECK_ARG(e.out_f32 == nullptr, "umma_conv: 3x3 convolutions write pair tensors only");
  // one weight tile whose whole B operand fits next to the ring (Cin = Cout = 48: 83 KB): keep it resident; the shared-memory data pipe is the kernel's
  // limiter (TC operand fetch + TMA fill + epilogue stores, profiles/README.md round 2) and the per-tile weight refill was 30 % of the TMA fill
  const size_t b_all = (size_t)2 * p.b_bytes * p.num_iters;
  static const bool allow_res = !(getenv("B200SEP_WRES") && atoi(getenv("B200SEP_WRES")) == 0);
  p.b_resident = (allow_res && p.n_tiles == 1 && b_all <= 96 * 1024) ? 1 : 0;
  p.stage_bytes = ((2 * p.a_bytes + (p.b_resident ? 0 : 2 * p.b_bytes) + 1023) / 1024) * 1024;
  p.n_ftiles = cdiv(pl.F, kConvStride);
  p.t_tiles = pl.T;
  p.num_tiles = p.n_ftiles * pl.T * B * p.n_tiles;
  B2_CHECK_ARG(n_c % 16 == 0 && n_c <= 80, "umma_conv: n_c=%d is not a multiple of 16 up to 80", n_c);
  const size_t sbuf_bytes = (size_t)2 * n_c * kConvStride * 2;  // staged output: hi + lo planes [n_c][112] bf16
  const size_t fixed = 1024 /*alignment slack*/ + 64 * sizeof(uint64_t) + 64 + 2 * kMaxChannels * sizeof(float) + (size_t)16 * n_c * sizeof(float) +
                       (p.b_resident ? b_all : 0);
  const size_t budget = 227 * 1024 - fixed;
  int stages = (int)((budget - sbuf_bytes) / p.stage_bytes);
  if (stages > 8) stages = 8;
  B2_CHECK_ARG(stages >= 2, "umma_conv: a pipeline stage of %u bytes does not fit twice in shared memory", p.stage_bytes);
  p.stages = stages;
  p.b_res_off = (uint32_t)((size_t)stages * p.stage_bytes);
  const size_t smem = (size_t)stages * p.stage_bytes + sbuf_bytes + fixed;
  CUtensorMap o_hi, o_lo;
  int rc = store_map(p.out_hi, pl.F, pl.T, B * p.out_c_total, n_c, &o_hi);
  if (!rc) rc = store_map(p.out_lo, pl.F, pl.T, B * p.out_c_total, n_c, &o_lo);
  if (rc) return rc;
  switch (n_c) {
    case 16: return launch_conv3<16>(pl.a_hi, pl.a_lo, o_hi, o_lo, p, smem, st);
    case 32: return launch_conv3<32>(pl.a_hi, pl.a_lo, o_hi, o_lo, p, smem, st);
    case 48: return launch_conv3<48>(pl.a_hi, pl.a_lo, o_hi, o_lo, p, smem, st);
    case 64: return launch_conv3<64>(pl.a_hi, pl.a_lo, o_hi, o_lo, p, smem, st);
    case 80: return launch_conv3<80>(pl.a_hi, pl.a_lo, o_hi, o_lo, p, smem, st);
  }
  set_error("umma_conv: n_c=%d has no kernel instance", n_c);
  return B200SEP_ERR_ARG;
}

static int pick_nc(int Cout, int mult, int limit) {  // largest n_c | Cout with mult*n_c <= limit and mult*n_c % 16 == 0
  for (int nc = Cout; nc >= 4; --nc)
    if (Cout % nc == 0 && mult * nc <= limit && (mult * nc) % 16 == 0 && nc % 16 == 0) return nc;
  return 0;
}
bool umma_updown_supported(int Cin, int Cout, int F_in, int up) {
  return Cin % 16 == 0 && F_in % 8 == 0 && pick_nc(Cout, up ? 4 : 2, kMaxNTile) > 0 && (up || F_in % 2 == 0);
}
int umma_updown_choose(int Cin, int Cout, int up, int* kc, int* n_c) {
  int k = 64;
  while (k > 16 && Cin % k != 0) k -= 16;
  if (Cin % 48 == 0) k = 48;
  *kc = k;
  *n_c = pick_nc(Cout, up ? 4 : 2, kMaxNTile);
  return 0;
}

// x: pair (B, Cin, T, F) -> ConvTranspose2d(k2,s2)+BN+ReLU (* skip) -> pair (B, Cout, 2T, 2F)
int umma_up_run(const UmmaConvPlan& pl, const void* wb_hi, const void* wb_lo, int B, int Cout, int n_c, const float* scale, const float* shift, int relu,
                const void* skip_hi, const void* skip_lo, void* out_hi, void* out_lo, cudaStream_t st) {
  UmmaEpilogue e;
  e.scale = scale; e.shift = shift; e.act = relu ? 1 : 0; e.out_hi = out_hi; e.out_lo = out_lo; e.res_hi = skip_hi; e.res_lo = skip_lo;
  return umma_up_run_ex(pl, wb_hi, wb_lo, B, Cout, n_c, e, st);
}

int umma_up_run_ex(const UmmaConvPlan& pl, const void* wb_hi, const void* wb_lo, int B, int Cout, int n_c, const UmmaEpilogue& e, cudaStream_t st) {
  UmmaParams p{};
  p.mode = 2; p.f_stride = kTileM; p.t_mul = 1; p.t_off = 0;
  p.n_c = n_c; p.n_tile = 4 * n_c; p.n_total = Cout;
  p.kc = pl.kc; p.n_chunks = pl.Cin / pl.kc; p.num_iters = p.n_chunks; p.ksteps = pl.kc / 16;
  p.a_bytes = (uint32_t)pl.kc * 256; p.b_bytes = (uint32_t)p.ksteps * p.n_tile * 32;
  p.T = pl.T; p.F = pl.F; p.Cin = pl.Cin; p.Cout = Cout; p.n_tiles = Cout / n_c;
  p.wb_hi = (const bf16*)wb_hi; p.wb_lo = (const bf16*)wb_lo;
  fill_epilogue(p, e, Cout);
  dim3 grid(cdiv(pl.F, kTileM), pl.T, B * p.n_tiles);
  return launch(pl.a_hi, pl.a_lo, pl.a_hi, pl.a_lo, p, grid, st);
}

// x: pair (B, Cin, T, F) -> Conv2d(k2,s2)+BN+ReLU -> pair (B, Cout, T/2, F/2)
int umma_down_run(const UmmaConvPlan& pl, const void* wb_hi, const void* wb_lo, int B, int Cout, int n_c, const float* scale, const float* shift, int relu,
                  void* out_hi, void* out_lo, cudaStream_t st) {
  UmmaEpilogue e;
  e.scale = scale; e.shift = shift; e.act = relu ? 1 : 0; e.out_hi = out_hi; e.out_lo = out_lo;
  return umma_down_run_ex(pl, wb_hi, wb_lo, B, Cout, n_c, e, st);
}

int umma_down_run_ex(const UmmaConvPlan& pl, const void* wb_hi, const void* wb_lo, int B, int Cout, int n_c, const UmmaEpilogue& e, cudaStream_t st) {
  UmmaParams p{};
  p.mode = 3; p.f_stride = kTileM; p.t_mul = 2; p.t_off = 0;
  p.n_c = n_c; p.n_tile = 2 * n_c; p.n_total = Cout;
  p.kc = pl.kc; p.n_chunks = pl.Cin / pl.kc; p.num_iters = 2 * p.n_chunks; p.ksteps = pl.kc / 16;
  p.a_bytes = (uint32_t)pl.kc * 256; p.b_bytes = (uint32_t)p.ksteps * p.n_tile * 32;
  p.T = pl.T; p.F = pl.F; p.Cin = pl.Cin; p.Cout = Cout; p.n_tiles = Cout / n_c;
  p.wb_hi = (const bf16*)wb_hi; p.wb_lo = (const bf16*)wb_lo;
  fill_epilogue(p, e, Cout);
  dim3 grid(cdiv(pl.F, kTileM), pl.T / 2, B * p.n_tiles);
  return launch(pl.a_hi, pl.a_lo, pl.a_hi, pl.a_lo, p, grid, st);
}

// Generic blocking: value(row, r, ci) for B rows [rows], row taps [n_r], -> [Cout/n_c][r][Cin/kc][kc/16][rows x 16 core-matrix tiled]
template <class F>
static void block_weights(int n_tiles, int n_r, int Cin, int kc, int rows, F value, std::vector<uint16_t>& hi, std::vector<uint16_t>& lo) {
  auto f2bf = [](float f) {
    uint32_t u;
    memcpy(&u, &f, 4);
    u += 0x7fffu + ((u >> 16) & 1u);
    return (uint16_t)(u >> 16);
  };
  auto bf2f = [](uint16_t h) {
    uint32_t u = (uint32_t)h << 16;
    float f;
    memcpy(&f, &u, 4);
    return f;
  };
  const int n_chunks = Cin / kc, ksteps = kc / 16;
  hi.assign((size_t)n_tiles * n_r * Cin * rows, 0);
  lo.assign(hi.size(), 0);
  size_t pos = 0;
  for (int nt = 0; nt < n_tiles; ++nt)
    for (int r = 0; r < n_r; ++r)
      for (int ch = 0; ch < n_chunks; ++ch)
        for (int j = 0; j < ksteps; ++j) {
          for (int row = 0; row < rows; ++row)
            for (int kk = 0; kk < 16; ++kk) {
              const float v = value(nt, row, r, ch * kc + j * 16 + kk);
              const size_t o = pos + (size_t)((row / 8) * 2 + kk / 8) * 64 + (row % 8) * 8 + (kk % 8);
              hi[o] = f2bf(v);
              lo[o] = f2bf(v - bf2f(hi[o]));
            }
          pos += (size_t)rows * 16;
        }
}
// ConvTranspose2d weight (Cin, Cout, 2, 2): B rows = (co_local, q = dy*2+dx)
void umma_up_block_weights(const float* w, int Cin, int Cout, int kc, int n_c, std::vector<uint16_t>& hi, std::vector<uint16_t>& lo) {
  block_weights(Cout / n_c, 1, Cin, kc, 4 * n_c, [&](int nt, int row, int, int ci) {
    const int q = row & 3, co = nt * n_c + (row >> 2);
    return w[((size_t)ci * Cout + co) * 4 + q];
  }, hi, lo);
}
// Conv2d weight (Cout, Cin, 2, 2) stride 2: row taps r = dy, B rows = (co_local, dx)
void umma_down_block_weights(const float* w, int Cout, int Cin, int kc, int n_c, std::vector<uint16_t>& hi, std::vector<uint16_t>& lo) {
  block_weights(Cout / n_c, 2, Cin, kc, 2 * n_c, [&](int nt, int row, int dy, int ci) {
    const int dx = row & 1, co = nt * n_c + (row >> 1);
    return w[(((size_t)co * Cin + ci) * 2 + dy) * 2 + dx];
  }, hi, lo);
}

// Conv2d weight (Cout, Cin, 1, 1): one tap, B rows = co_local
void umma_pw_block_weights(const float* w, int Cout, int Cin, int kc, int n_c, std::vector<uint16_t>& hi, std::vector<uint16_t>& lo) {
  block_weights(Cout / n_c, 1, Cin, kc, n_c, [&](int nt, int row, int, int ci) { return w[(size_t)(nt * n_c + row) * Cin + ci]; }, hi, lo);
}
bool umma_pw_supported(int Cin, int Cout, int F) { return Cin % 16 == 0 && Cout % 16 == 0 && F % 8 == 0; }
int umma_pw_choose(int Cin, int Cout, int* kc, int* n_c) {
  int k = 64;
  while (k > 16 && Cin % k != 0) k -= 16;
  if (Cin % 48 == 0) k = 48;
  *kc = k;
  *n_c = pick_nc(Cout, 1, kMaxNTile);
  return 0;
}
// x: pair (B, Cin, T, F) -> Conv2d 1x1 (+affine, act, +res, *mul) -> pair or fp32 (B, Cout, T, F)
int umma_pw_run_ex(const UmmaConvPlan& pl, const void* wb_hi, const void* wb_lo, int B, int Cout, int n_c, const UmmaEpilogue& e, cudaStream_t st) {
  UmmaParams p{};
  p.mode = 4; p.f_stride = kTileM; p.t_mul = 1; p.t_off = 0;
  p.n_c = n_c; p.n_tile = n_c; p.n_total = Cout;
  p.kc = pl.kc; p.n_chunks = pl.Cin / pl.kc; p.num_iters = p.n_chunks; p.ksteps = pl.kc / 16;
  p.a_bytes = (uint32_t)pl.kc * 256; p.b_bytes = (uint32_t)p.ksteps * p.n_tile * 32;
  p.T = pl.T; p.F = pl.F; p.Cin = pl.Cin; p.Cout = Cout; p.n_tiles = Cout / n_c;
  p.wb_hi = (const bf16*)wb_hi; p.wb_lo = (const bf16*)wb_lo;
  fill_epilogue(p, e, Cout);
  dim3 grid(cdiv(pl.F, kTileM), pl.T, B * p.n_tiles);
  return launch(pl.a_hi, pl.a_lo, pl.a_hi, pl.a_lo, p, grid, st);
}

// Host-side blocking of a (Cout, Cin, 3, 3) fp32 filter into the B operand stream of umma_conv_run:
// [Cout/n_c][dy][Cin/kc][kc/16] blocks of [3*n_c rows = (dx, co)][16 k] stored as 8x8 core matrices (K-major, no swizzle).
void umma_conv_block_weights(const float* w, int Cout, int Cin, int kc, int n_c, std::vector<uint16_t>& hi, std::vector<uint16_t>& lo) {
  auto f2bf = [](float f) {
    uint32_t u;
    memcpy(&u, &f, 4);
    u += 0x7fffu + ((u >> 16) & 1u);
    return (uint16_t)(u >> 16);
  };
  auto bf2f = [](uint16_t h) {
    uint32_t u = (uint32_t)h << 16;
    float f;
    memcpy(&f, &u, 4);
    return f;
  };
  const int n_tiles = Cout / n_c, n_chunks = Cin / kc, ksteps = kc / 16, rows = 3 * n_c;
  hi.assign((size_t)Cout * Cin * 9, 0);
  lo.assign(hi.size(), 0);
  size_t pos = 0;
  for (int nt = 0; nt < n_tiles; ++nt)
    for (int dy = 0; dy < 3; ++dy)
      for (int ch = 0; ch < n_chunks; ++ch)
        for (int j = 0; j < ksteps; ++j) {
          for (int r = 0; r < rows; ++r)
            for (int kk = 0; kk < 16; ++kk) {
              const int dx = r / n_c, co = nt * n_c + r % n_c, ci = ch * kc + j * 16 + kk;
              const float v = w[(((size_t)co * Cin + ci) * 3 + dy) * 3 + dx];
              const size_t o = pos + (size_t)((r / 8) * 2 + kk / 8) * 64 + (r % 8) * 8 + (kk % 8);
              hi[o] = f2bf(v);
              lo[o] = f2bf(v - bf2f(hi[o]));
            }
          pos += (size_t)rows * 16;
        }
}

// ---------------------------------------------------------------------------------------------------------
// pair <-> fp32 helpers
__global__ void split_pair_kernel(const float* __restrict__ x, bf16* __restrict__ hi, bf16* __restrict__ lo, int64_t n) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) split_store2(x[i], hi[i], lo[i]);
}
__global__ void join_pair_kernel(const bf16* __restrict__ hi, const bf16* __restrict__ lo, float* __restrict__ y, int64_t n) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x)
    y[i] = __bfloat162float(hi[i]) + __bfloat162float(lo[i]);
}
int split_pair(const float* x, void* hi, void* lo, int64_t n, cudaStream_t st) {
  if (n == 0) return B200SEP_OK;
  split_pair_kernel<<<(int)std::min<int64_t>(cdiv(n, 1024), kNumSMs * 8), 256, 0, st>>>(x, (bf16*)hi, (bf16*)lo, n);
  B2_LAUNCHED();
  return B200SEP_OK;
}
int join_pair(const void* hi, const void* lo, float* y, int64_t n, cudaStream_t st) {
  if (n == 0) return B200SEP_OK;
  join_pair_kernel<<<(int)std::min<int64_t>(cdiv(n, 1024), kNumSMs * 8), 256, 0, st>>>((const bf16*)hi, (const bf16*)lo, y, n);
  B2_LAUNCHED();
  return B200SEP_OK;
}

}  // namespace b200sep

// ---------------------------------------------------------------------------------------------------------
// self-test entry points (exported through the C ABI so the GPU test-suite can check each tensor-core operator in
// isolation against a plain fp32 reference): fp32 in -> split -> wgmma op -> join -> fp32 out.
using namespace b200sep;

extern "C" int b200sep_selftest_umma_gemm(const float* a, const float* w, const float* res, float* out, int M, int N, int K, int rows_per_channel,
                                          int channels, const float* scale, const float* shift, int relu, void* stream) {
  B2_CHECK_ARG(a && w && out && scale && shift, "selftest_umma_gemm: NULL argument");
  B2_CHECK_ARG(umma_gemm_supported(M, N, K), "selftest_umma_gemm: shape M=%d N=%d K=%d not supported by the tensor-core path", M, N, K);
  cudaStream_t st = (cudaStream_t)stream;
  uint16_t *a_p = nullptr, *w_p = nullptr, *o_p = nullptr, *r_p = nullptr;
  const int64_t na = (int64_t)M * K, nw = (int64_t)N * K, no = (int64_t)M * N;
  B2_CUDA(cudaMalloc(&a_p, na * 4));
  B2_CUDA(cudaMalloc(&w_p, nw * 4));
  B2_CUDA(cudaMalloc(&o_p, no * 4));
  if (res) B2_CUDA(cudaMalloc(&r_p, no * 4));
  int rc = split_pair(a, a_p, a_p + na, na, st);
  if (!rc) rc = split_pair(w, w_p, w_p + nw, nw, st);
  if (!rc && res) rc = split_pair(res, r_p, r_p + no, no, st);
  UmmaGemmPlan pl;
  if (!rc) rc = umma_gemm_plan_create(&pl, a_p, a_p + na, w_p, w_p + nw, M, N, K);
  if (!rc) rc = umma_gemm_run(pl, scale, shift, rows_per_channel, channels, relu, o_p, o_p + no, r_p, r_p ? r_p + no : nullptr, M, st);
  if (!rc) rc = join_pair(o_p, o_p + no, out, no, st);
  cudaStreamSynchronize(st);
  cudaFree(a_p); cudaFree(w_p); cudaFree(o_p);
  if (r_p) cudaFree(r_p);
  return rc;
}

extern "C" int b200sep_selftest_umma_conv3x3(const float* x, const float* w_host, float* out, int B, int Cin, int Cout, int T, int F, const float* scale,
                                             const float* shift, int relu, void* stream) {
  B2_CHECK_ARG(x && w_host && out && scale && shift, "selftest_umma_conv3x3: NULL argument");
  B2_CHECK_ARG(umma_conv_supported(Cin, Cout, F, 3, 3), "selftest_umma_conv3x3: Cin=%d Cout=%d F=%d not supported by the tensor-core path", Cin, Cout, F);
  cudaStream_t st = (cudaStream_t)stream;
  int kc, n_c;
  umma_conv_choose(Cin, Cout, &kc, &n_c);
  std::vector<uint16_t> hi, lo;
  umma_conv_block_weights(w_host, Cout, Cin, kc, n_c, hi, lo);
  uint16_t *x_p = nullptr, *o_p = nullptr, *w_p = nullptr;
  const int64_t nx = (int64_t)B * Cin * T * F, no = (int64_t)B * Cout * T * F, nw = (int64_t)hi.size();
  B2_CUDA(cudaMalloc(&x_p, nx * 4));
  B2_CUDA(cudaMalloc(&o_p, no * 4));
  B2_CUDA(cudaMalloc(&w_p, nw * 4));
  B2_CUDA(cudaMemcpy(w_p, hi.data(), nw * 2, cudaMemcpyHostToDevice));
  B2_CUDA(cudaMemcpy(w_p + nw, lo.data(), nw * 2, cudaMemcpyHostToDevice));
  int rc = split_pair(x, x_p, x_p + nx, nx, st);
  UmmaConvPlan pl;
  if (!rc) rc = umma_conv_plan_create(&pl, x_p, x_p + nx, B, Cin, T, F, kc);
  if (!rc) rc = umma_conv_run(pl, w_p, w_p + nw, B, Cout, n_c, 3, scale, shift, relu, o_p, o_p + no, st);
  if (!rc) rc = join_pair(o_p, o_p + no, out, no, st);
  cudaStreamSynchronize(st);
  cudaFree(x_p); cudaFree(o_p); cudaFree(w_p);
  return rc;
}

extern "C" int b200sep_selftest_umma_updown(const float* x, const float* w_host, const float* skip, float* out, int B, int Cin, int Cout, int T, int F,
                                            const float* scale, const float* shift, int relu, int up, void* stream) {
  B2_CHECK_ARG(x && w_host && out && scale && shift, "selftest_umma_updown: NULL argument");
  B2_CHECK_ARG(umma_updown_supported(Cin, Cout, F, up), "selftest_umma_updown: Cin=%d Cout=%d F=%d not supported by the tensor-core path", Cin, Cout, F);
  cudaStream_t st = (cudaStream_t)stream;
  int kc, n_c;
  umma_updown_choose(Cin, Cout, up, &kc, &n_c);
  std::vector<uint16_t> hi, lo;
  if (up) umma_up_block_weights(w_host, Cin, Cout, kc, n_c, hi, lo);
  else umma_down_block_weights(w_host, Cout, Cin, kc, n_c, hi, lo);
  uint16_t *x_p = nullptr, *o_p = nullptr, *w_p = nullptr, *s_p = nullptr;
  const int64_t nx = (int64_t)B * Cin * T * F, no = up ? (int64_t)B * Cout * 4 * T * F : (int64_t)B * Cout * (T / 2) * (F / 2), nw = (int64_t)hi.size();
  B2_CUDA(cudaMalloc(&x_p, nx * 4));
  B2_CUDA(cudaMalloc(&o_p, no * 4));
  B2_CUDA(cudaMalloc(&w_p, nw * 4));
  if (skip) B2_CUDA(cudaMalloc(&s_p, no * 4));
  B2_CUDA(cudaMemcpy(w_p, hi.data(), nw * 2, cudaMemcpyHostToDevice));
  B2_CUDA(cudaMemcpy(w_p + nw, lo.data(), nw * 2, cudaMemcpyHostToDevice));
  int rc = split_pair(x, x_p, x_p + nx, nx, st);
  if (!rc && skip) rc = split_pair(skip, s_p, s_p + no, no, st);
  UmmaConvPlan pl;
  if (!rc) rc = umma_conv_plan_create(&pl, x_p, x_p + nx, B, Cin, T, F, kc);
  if (!rc) {
    if (up) rc = umma_up_run(pl, w_p, w_p + nw, B, Cout, n_c, scale, shift, relu, s_p, s_p ? s_p + no : nullptr, o_p, o_p + no, st);
    else rc = umma_down_run(pl, w_p, w_p + nw, B, Cout, n_c, scale, shift, relu, o_p, o_p + no, st);
  }
  if (!rc) rc = join_pair(o_p, o_p + no, out, no, st);
  cudaStreamSynchronize(st);
  cudaFree(x_p); cudaFree(o_p); cudaFree(w_p);
  if (s_p) cudaFree(s_p);
  return rc;
}
