// FLAC encoder (RFC 9639) for normalised stereo stems, sm_90a.  Fixed block size 4096; three launches:
//   flac_analyze_kernel  one CTA per frame: quantise the frame exactly like the WAV writer (pcm_quantize), then for each channel candidate
//                        (left, right, mid, side) find wasted bits and CONSTANT, try FIXED orders 0-4 and LPC orders 1-12 (Tukey(0.5)-windowed
//                        autocorrelation in fp64, Levinson-Durbin in one warp, 15-bit quantised coefficients, exact integer residual) with the
//                        cheapest partitioned Rice code (partition orders 0-8, RICE / RICE2, escape partitions), keep the smallest subframe
//                        (VERBATIM when nothing beats it) and pick the channel assignment with the fewest bits.  Every size is an exact bit
//                        count: it becomes the frame's byte length and write offset.
//   flac_offsets_kernel  one CTA: exclusive scan of the frame lengths, total / min / max frame size.
//   flac_pack_kernel     one CTA per frame: recompute the chosen residuals, a block scan of the per-sample code lengths gives each code's bit
//                        offset, codes are OR-ed into a shared-memory frame image, CRC-8 of the header and CRC-16 of the frame (per-thread
//                        partial CRCs combined in GF(2)), then the bytes are stored at the frame's offset.
// Every reduction has a fixed order, so the stream is the same byte for byte from run to run.
#include <limits.h>
#include <math.h>

#include "common.cuh"
#include "flac_common.cuh"
#include "pcm.cuh"

namespace b200sep {
namespace {

using flac::crc8;
using flac::gf2_mulmod16;
using flac::x8_pow_mod16;

constexpr int kBlock = 4096;
constexpr int kThreads = 256;
constexpr int kWarps = kThreads / 32;
constexpr int kMaxLpc = 12;
constexpr int kLpcPrec = 15;              // quantised coefficient precision, sign included
constexpr int kMaxPo = 8;                 // partition orders 0..8
constexpr int kMaxParts = 1 << kMaxPo;    // == kThreads: one finest partition per thread
constexpr int kKs = 32;                   // Rice parameters 0..30 are evaluated (RICE: 0..14)
constexpr int kHeaderMax = 16;            // frame header incl. CRC-8: 4 + 6 (frame number) + 2 (block size) + 2 (rate) + 1 = 15
constexpr uint8_t kEscape = 255;
// A frame never exceeds its independent-channel VERBATIM coding: header + 2 x (8 + bs * bps) bits + CRC-16.
constexpr int frame_bound_bytes(int bps) { return kHeaderMax + 2 + 2 * kBlock * bps / 8 + 2; }
constexpr int kFrameWords = (frame_bound_bytes(24) + 3) / 4;

enum { SF_CONSTANT = 0, SF_VERBATIM = 1, SF_FIXED = 2, SF_LPC = 3 };

struct Sub {
  int type, order, wasted, bps, shift, method, po;  // bps = the channel's sample size before wasted bits are removed
  int coef[kMaxLpc];
  uint8_t k[kMaxParts];  // Rice parameter per partition, kEscape = escape partition of width w[p]
  uint8_t w[kMaxParts];
};
struct FramePlan {
  int assign;  // channel assignment code: 1 independent, 8 left/side, 9 right/side, 10 mid/side
  int bytes;
  Sub sub[2];
};

struct AnalysisSmem {
  int L[kBlock], R[kBlock], sig[kBlock], res[kBlock];
  unsigned long long S[kMaxParts * kKs];  // S[j][k] = sum over partition j of (zigzag residual >> k); doubles as the windowed signal
  Sub best[4];
  unsigned long long bits[4];
  double ac[kMaxLpc + 1];
  double lpc[kMaxLpc][kMaxLpc];
  int qc[kMaxLpc][kMaxLpc], qshift[kMaxLpc], qok[kMaxLpc];
  int nlpc;
  unsigned long long red_u[kWarps];
  double red_d[kWarps];
  int red_i[kWarps];
  uint8_t W[kMaxParts], tk[kMaxParts], tw[kMaxParts];
};

struct PackSmem {
  int sig[2][kBlock];
  unsigned buf[kFrameWords];  // the frame image, big-endian bit order: byte b is bits [24 - 8 (b & 3), +8) of buf[b >> 2]
  Sub sub[2];
  unsigned scan[kWarps];
  unsigned crc_part[kWarps];
  uint16_t crc_tab[256];
};

__device__ __forceinline__ unsigned zigzag(int r) { return ((unsigned)r << 1) ^ (unsigned)(r >> 31); }
__device__ __forceinline__ unsigned low_bits(int v, int n) { return n >= 32 ? (unsigned)v : ((unsigned)v & ((1u << n) - 1u)); }
// bits of the smallest two's-complement field holding r (0 for r == 0: an all-zero escape partition stores nothing)
__device__ __forceinline__ int signed_width(int r) { return r == 0 ? 0 : 33 - __clz(r ^ (r >> 31)); }
__device__ __forceinline__ int bitrev(int j, int nbits) { return nbits ? (int)(__brev((unsigned)j) >> (32 - nbits)) : 0; }

__device__ unsigned long long block_sum(unsigned long long v, unsigned long long* red) {
  for (int o = 16; o; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
  __syncthreads();
  unsigned long long t = 0;
  for (int w = 0; w < kWarps; ++w) t += red[w];
  __syncthreads();
  return t;
}
__device__ double block_sum(double v, double* red) {
  for (int o = 16; o; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
  __syncthreads();
  double t = 0.0;
  for (int w = 0; w < kWarps; ++w) t += red[w];
  __syncthreads();
  return t;
}
template <class Op>
__device__ int block_reduce(int v, int* red, Op op) {
  for (int o = 16; o; o >>= 1) v = op(v, __shfl_xor_sync(0xffffffffu, v, o));
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
  __syncthreads();
  int t = red[0];
  for (int w = 1; w < kWarps; ++w) t = op(t, red[w]);
  __syncthreads();
  return t;
}

// Prediction residual of sample i (i >= order) of a FIXED or LPC subframe; int64 so that an overflowing LPC residual can be detected.
__device__ __forceinline__ long long residual_at(const int* s, int i, int type, int order, const int* coef, int shift) {
  if (type == SF_FIXED) {
    switch (order) {
      case 0: return s[i];
      case 1: return (long long)s[i] - s[i - 1];
      case 2: return (long long)s[i] - 2ll * s[i - 1] + s[i - 2];
      case 3: return (long long)s[i] - 3ll * s[i - 1] + 3ll * s[i - 2] - s[i - 3];
      default: return (long long)s[i] - 4ll * s[i - 1] + 6ll * s[i - 2] - 4ll * s[i - 3] + s[i - 4];
    }
  }
  long long p = 0;
  for (int j = 0; j < order; ++j) p += (long long)coef[j] * s[i - 1 - j];
  return (long long)s[i] - (p >> shift);
}

// Frame header with its CRC-8 -> h (kHeaderMax bytes); returns its length.
__device__ int frame_header(uint8_t* h, unsigned frame, int bs, int sr_code, int sr_extra_bits, int sr_extra, int bps_code, int assign) {
  int n = 0;
  h[n++] = 0xFF;
  h[n++] = 0xF8;  // sync code, reserved bit, fixed-blocksize stream
  const int bs_code = bs == kBlock ? 12 : (bs <= 256 ? 6 : 7);
  h[n++] = (uint8_t)((bs_code << 4) | sr_code);
  h[n++] = (uint8_t)((assign << 4) | (bps_code << 1));
  if (frame < 0x80) {  // frame number, UTF-8 style
    h[n++] = (uint8_t)frame;
  } else {
    int nb = 2;
    while (frame >= (1u << (5 * nb + 1))) ++nb;
    h[n++] = (uint8_t)(((0xFF00 >> nb) & 0xFF) | (frame >> (6 * (nb - 1))));
    for (int j = nb - 2; j >= 0; --j) h[n++] = (uint8_t)(0x80 | ((frame >> (6 * j)) & 0x3F));
  }
  if (bs_code == 6) {
    h[n++] = (uint8_t)(bs - 1);
  } else if (bs_code == 7) {
    h[n++] = (uint8_t)((bs - 1) >> 8);
    h[n++] = (uint8_t)(bs - 1);
  }
  if (sr_extra_bits == 8) {
    h[n++] = (uint8_t)sr_extra;
  } else if (sr_extra_bits == 16) {
    h[n++] = (uint8_t)(sr_extra >> 8);
    h[n++] = (uint8_t)sr_extra;
  }
  h[n] = crc8(h, n);
  return n + 1;
}

__device__ __forceinline__ int candidate(int ch, int l, int r) { return ch == 0 ? l : ch == 1 ? r : ch == 2 ? ((l + r) >> 1) : l - r; }
__device__ __forceinline__ int assign_code(int a) { return a == 0 ? 1 : 7 + a; }
// channel candidates (0 left, 1 right, 2 mid, 3 side) of the two subframes of each assignment (0 independent, 1 left/side, 2 right/side, 3 mid/side)
__device__ __forceinline__ int sub_channel(int a, int c) {
  const int t[4][2] = {{0, 1}, {0, 3}, {3, 1}, {2, 3}};
  return t[a][c];
}

// Bits of the residual section of res[order, bs) (coding method, partition order, partitions) for the cheapest partition order / method;
// their per-partition parameters are left in sm.tk / sm.tw.
__device__ unsigned long long rice_plan(AnalysisSmem& sm, int bs, int order, int& method, int& po_best) {
  const int t = threadIdx.x;
  int pmax = 0;
  while (pmax < kMaxPo && bs % (2 << pmax) == 0 && (bs >> (pmax + 1)) > order) ++pmax;
  const int n0 = bs >> pmax;
  if (t < (1 << pmax)) {
    const int lo = max(t * n0, order), hi = (t + 1) * n0;
    unsigned umax = 0;
    int wmax = 0;
    for (int i = lo; i < hi; ++i) {
      umax = max(umax, zigzag(sm.res[i]));
      wmax = max(wmax, signed_width(sm.res[i]));
    }
    const int j = bitrev(t, pmax);  // bit-reversed storage: the two halves of partition j at the next coarser level are j and j + n/2
    const int kend = 32 - __clz(umax);
    for (int k = 0; k < kKs; ++k) {
      unsigned long long s = 0;
      if (k < kend)
        for (int i = lo; i < hi; ++i) s += zigzag(sm.res[i]) >> k;
      sm.S[j * kKs + k] = s;
    }
    sm.W[j] = (uint8_t)wmax;
  }
  __syncthreads();
  unsigned long long best = ~0ull;
  for (int po = pmax; po >= 0; --po) {
    const int n = 1 << po, psz = bs >> po;
    unsigned long long c1 = 0, c2 = 0;
    int k1 = 0, k2 = 0;
    if (t < n) {
      const unsigned long long cnt = (unsigned long long)(psz - (bitrev(t, po) == 0 ? order : 0));
      const unsigned long long* S = sm.S + t * kKs;
      unsigned long long b1 = ~0ull, b2 = ~0ull;
      for (int k = 0; k <= 30; ++k) {
        const unsigned long long c = cnt * (unsigned long long)(1 + k) + S[k];
        if (c < b2) b2 = c, k2 = k;
        if (k <= 14 && c < b1) b1 = c, k1 = k;
      }
      if (sm.W[t] <= 31) {
        const unsigned long long e = 5 + cnt * sm.W[t];
        if (e < b1) b1 = e, k1 = kEscape;
        if (e < b2) b2 = e, k2 = kEscape;
      }
      c1 = 4 + b1;
      c2 = 5 + b2;
    }
    const unsigned long long s1 = block_sum(c1, sm.red_u), s2 = block_sum(c2, sm.red_u);
    const int m = s2 < s1 ? 1 : 0;
    const unsigned long long cost = 6 + (m ? s2 : s1);
    if (cost < best) {  // every thread sees the same sums
      best = cost;
      method = m;
      po_best = po;
      if (t < n) {
        const int q = bitrev(t, po);
        sm.tk[q] = (uint8_t)(m ? k2 : k1);
        sm.tw[q] = sm.W[t];
      }
    }
    if (po > 0) {
      const int h = n >> 1;
      for (int e = t; e < h * kKs; e += kThreads) sm.S[e] += sm.S[e + h * kKs];
      for (int j = t; j < h; j += kThreads) sm.W[j] = max(sm.W[j], sm.W[j + h]);
      __syncthreads();
    }
  }
  __syncthreads();
  return best;
}

__device__ void commit(AnalysisSmem& sm, Sub& b, int type, int order, int wasted, int bps, int shift, const int* coef, int method, int po) {
  for (int q = threadIdx.x; q < (1 << po); q += kThreads) {
    b.k[q] = sm.tk[q];
    b.w[q] = sm.tw[q];
  }
  if (threadIdx.x == 0) {
    b.type = type, b.order = order, b.wasted = wasted, b.bps = bps, b.shift = shift, b.method = method, b.po = po;
    for (int j = 0; j < order; ++j) b.coef[j] = coef ? coef[j] : 0;
  }
  __syncthreads();
}

// Smallest subframe of channel candidate ch -> sm.best[ch], its exact size in bits -> sm.bits[ch].
__device__ void analyze_channel(AnalysisSmem& sm, int ch, int bs, int bps) {
  const int t = threadIdx.x;
  int orv = 0, mn = INT_MAX, mx = INT_MIN;
  for (int i = t; i < bs; i += kThreads) {
    const int v = candidate(ch, sm.L[i], sm.R[i]);
    sm.sig[i] = v;
    orv |= v;
    mn = min(mn, v);
    mx = max(mx, v);
  }
  orv = block_reduce(orv, sm.red_i, [](int a, int b) { return a | b; });
  mn = block_reduce(mn, sm.red_i, [](int a, int b) { return min(a, b); });
  mx = block_reduce(mx, sm.red_i, [](int a, int b) { return max(a, b); });
  Sub& b = sm.best[ch];
  if (mn == mx) {
    commit(sm, b, SF_CONSTANT, 0, 0, bps, 0, nullptr, 0, 0);
    if (t == 0) sm.bits[ch] = 8 + bps;
    __syncthreads();
    return;
  }
  const int wasted = __ffs(orv) - 1;
  const int bps_e = bps - wasted;
  const unsigned long long hdr = 8 + wasted;  // type byte + unary wasted-bits count
  if (wasted)
    for (int i = t; i < bs; i += kThreads) sm.sig[i] >>= wasted;
  commit(sm, b, SF_VERBATIM, 0, wasted, bps, 0, nullptr, 0, 0);  // also orders the shift before the reads below
  unsigned long long best = hdr + (unsigned long long)bs * bps_e;
  int method, po;
  for (int o = 0; o <= 4 && o < bs; ++o) {
    for (int i = t + o; i < bs; i += kThreads) sm.res[i] = (int)residual_at(sm.sig, i, SF_FIXED, o, nullptr, 0);  // |res| < 2^30
    __syncthreads();
    const unsigned long long c = hdr + (unsigned long long)o * bps_e + rice_plan(sm, bs, o, method, po);
    if (c < best) {
      best = c;
      commit(sm, b, SF_FIXED, o, wasted, bps, 0, nullptr, method, po);
    }
  }
  // LPC: Tukey(0.5) window (cosine tapers over a quarter of the block at each end), autocorrelation in fp64
  const int maxo = min(kMaxLpc, bs - 1);
  if (maxo >= 1) {
    double* xw = reinterpret_cast<double*>(sm.S);
    const int np = bs >> 2;
    for (int i = t; i < bs; i += kThreads) {
      double w = 1.0;
      if (i < np) w = 0.5 - 0.5 * cospi((double)i / np);
      else if (i >= bs - np) w = 0.5 - 0.5 * cospi((double)(bs - 1 - i) / np);
      xw[i] = w * (double)sm.sig[i];
    }
    __syncthreads();
    for (int l = 0; l <= maxo; ++l) {
      double a = 0.0;
      for (int i = t + l; i < bs; i += kThreads) a += xw[i] * xw[i - l];
      a = block_sum(a, sm.red_d);
      if (t == 0) sm.ac[l] = a;
    }
    __syncthreads();
    if (t < 32) {  // Levinson-Durbin: lane j holds coefficient j; the butterfly sums leave the same value in every lane
      double err = sm.ac[0], a = 0.0;
      int valid = 0;
      if (err > 0.0) {
        for (int i = 0; i < maxo; ++i) {
          double p = t < i ? a * sm.ac[i - t] : 0.0;
          for (int o = 16; o; o >>= 1) p += __shfl_xor_sync(0xffffffffu, p, o);
          const double k = (sm.ac[i + 1] - p) / err;
          const double mirror = __shfl_sync(0xffffffffu, a, (i - 1 - t) & 31);
          if (t < i) a -= k * mirror;
          else if (t == i) a = k;
          if (t <= i) sm.lpc[i][t] = a;
          valid = i + 1;
          err *= 1.0 - k * k;
          if (!(err > 0.0)) break;
        }
      }
      if (t == 0) sm.nlpc = valid;
    }
    __syncthreads();
    if (t < sm.nlpc) {  // quantise order t+1 with error feedback
      const int o = t + 1;
      double cmax = 0.0;
      for (int j = 0; j < o; ++j) cmax = fmax(cmax, fabs(sm.lpc[t][j]));
      int e = 0;
      frexp(cmax, &e);
      int shift = min(kLpcPrec - 1 - e, 15);
      const int qmax = (1 << (kLpcPrec - 1)) - 1;
      sm.qok[t] = cmax > 0.0 && shift >= 0 && isfinite(cmax);
      shift = max(shift, 0);
      double acc = 0.0;
      for (int j = 0; j < o; ++j) {
        acc += ldexp(sm.lpc[t][j], shift);
        const double q = fmin(fmax(rint(acc), (double)(-qmax - 1)), (double)qmax);
        sm.qc[t][j] = sm.qok[t] ? (int)q : 0;
        acc -= q;
      }
      sm.qshift[t] = shift;
    }
    __syncthreads();
    for (int o = 1; o <= sm.nlpc; ++o) {
      if (!sm.qok[o - 1]) continue;
      int ovf = 0;
      for (int i = t + o; i < bs; i += kThreads) {
        const long long r = residual_at(sm.sig, i, SF_LPC, o, sm.qc[o - 1], sm.qshift[o - 1]);
        ovf |= r < INT_MIN || r > INT_MAX;
        sm.res[i] = (int)r;
      }
      if (block_reduce(ovf, sm.red_i, [](int a, int b) { return a | b; })) continue;  // a residual must fit in 32 signed bits
      const unsigned long long c = hdr + (unsigned long long)o * bps_e + 4 + 5 + (unsigned long long)o * kLpcPrec + rice_plan(sm, bs, o, method, po);
      if (c < best) {
        best = c;
        commit(sm, b, SF_LPC, o, wasted, bps, sm.qshift[o - 1], sm.qc[o - 1], method, po);
      }
    }
  }
  if (t == 0) sm.bits[ch] = best;
  __syncthreads();
}

__global__ void __launch_bounds__(kThreads, 1) flac_analyze_kernel(const float* __restrict__ x, int64_t n, int bits, int via_int16, int sbps,
                                                                   int sr_code, int sr_extra_bits, int sr_extra, FramePlan* __restrict__ plans) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  AnalysisSmem& sm = *reinterpret_cast<AnalysisSmem*>(smem_raw);
  const int f = blockIdx.x, t = threadIdx.x;
  const int64_t start = (int64_t)f * kBlock;
  const int bs = (int)min((int64_t)kBlock, n - start);
  for (int i = t; i < bs; i += kThreads) {
    const float2 v = reinterpret_cast<const float2*>(x)[start + i];
    sm.L[i] = pcm_quantize(v.x, bits, via_int16) >> (bits - sbps);
    sm.R[i] = pcm_quantize(v.y, bits, via_int16) >> (bits - sbps);
  }
  __syncthreads();
  for (int ch = 0; ch < 4; ++ch) analyze_channel(sm, ch, bs, ch == 3 ? sbps + 1 : sbps);
  int a_best = 0;
  unsigned long long b_best = ~0ull;
  for (int a = 0; a < 4; ++a) {
    const unsigned long long s = sm.bits[sub_channel(a, 0)] + sm.bits[sub_channel(a, 1)];
    if (s < b_best) b_best = s, a_best = a;
  }
  uint8_t h[kHeaderMax];
  const int hb = frame_header(h, (unsigned)f, bs, sr_code, sr_extra_bits, sr_extra, sbps == 16 ? 4 : 6, assign_code(a_best));
  FramePlan& P = plans[f];
  for (int c = 0; c < 2; ++c) {
    const int* src = reinterpret_cast<const int*>(&sm.best[sub_channel(a_best, c)]);
    int* dst = reinterpret_cast<int*>(&P.sub[c]);
    for (int i = t; i < (int)(sizeof(Sub) / 4); i += kThreads) dst[i] = src[i];
  }
  if (t == 0) {
    P.assign = assign_code(a_best);
    P.bytes = hb + (int)((b_best + 7) / 8) + 2;
  }
}

__global__ void __launch_bounds__(1024) flac_offsets_kernel(const FramePlan* __restrict__ plans, int nf, int64_t* __restrict__ offsets,
                                                            int64_t* __restrict__ result) {
  __shared__ long long warp_tot[32];
  __shared__ int warp_min[32], warp_max[32];
  const int t = threadIdx.x, per = (nf + 1023) / 1024;
  const int lo = min(nf, t * per), hi = min(nf, lo + per);
  long long s = 0;
  int mn = INT_MAX, mx = 0;
  for (int f = lo; f < hi; ++f) {
    const int b = plans[f].bytes;
    s += b;
    mn = min(mn, b);
    mx = max(mx, b);
  }
  long long inc = s;  // inclusive scan over the threads
  for (int o = 1; o < 32; o <<= 1) {
    const long long v = __shfl_up_sync(0xffffffffu, inc, o);
    if ((t & 31) >= o) inc += v;
  }
  for (int o = 16; o; o >>= 1) {
    mn = min(mn, __shfl_xor_sync(0xffffffffu, mn, o));
    mx = max(mx, __shfl_xor_sync(0xffffffffu, mx, o));
  }
  if ((t & 31) == 31) warp_tot[t >> 5] = inc;
  if ((t & 31) == 0) warp_min[t >> 5] = mn, warp_max[t >> 5] = mx;
  __syncthreads();
  long long base = 0, total = 0;
  for (int w = 0; w < 32; ++w) {
    if (w < (t >> 5)) base += warp_tot[w];
    total += warp_tot[w];
    mn = min(mn, warp_min[w]);
    mx = max(mx, warp_max[w]);
  }
  long long off = base + inc - s;
  for (int f = lo; f < hi; ++f) {
    offsets[f] = off;
    off += plans[f].bytes;
  }
  if (t == 0) {
    result[0] = total;
    result[1] = nf ? mn : 0;
    result[2] = mx;
    result[3] = 0;
  }
}

__device__ __forceinline__ void put_bits(unsigned* buf, unsigned pos, unsigned v, int n) {
  if (n == 0 || pos + (unsigned)n > (unsigned)kFrameWords * 32u) return;  // cannot happen for a consistent plan (checked after packing)
  const unsigned word = pos >> 5, off = pos & 31;
  if (off + n <= 32) {
    atomicOr(&buf[word], v << (32 - off - n));
  } else {
    atomicOr(&buf[word], v >> (off + n - 32));
    atomicOr(&buf[word + 1], v << (64 - off - n));
  }
}

// Bits of item i (sample i of subframe c plus whatever precedes its code: the subframe header before sample 0, the LPC coefficients and the
// residual header before the first residual, a partition's parameter before its first sample); kWrite also stores them at bit `pos`.
template <bool kWrite>
__device__ unsigned item_bits(PackSmem& sm, int c, int i, int bs, unsigned pos) {
  const Sub& s = sm.sub[c];
  const int* sig = sm.sig[c];
  unsigned len = 0;
  auto put = [&](unsigned v, int nb) {
    if (kWrite) put_bits(sm.buf, pos + len, v, nb);
    len += nb;
  };
  if (i == 0) {
    const int code = s.type == SF_CONSTANT ? 0 : s.type == SF_VERBATIM ? 1 : s.type == SF_FIXED ? 8 + s.order : 31 + s.order;
    put((unsigned)(code << 1) | (s.wasted ? 1u : 0u), 8);
    if (s.wasted) {
      len += s.wasted - 1;
      put(1, 1);
    }
  }
  const int bps_e = s.bps - s.wasted;
  if (s.type == SF_CONSTANT) {
    if (i == 0) put(low_bits(sig[0], s.bps), s.bps);
    return len;
  }
  if (s.type == SF_VERBATIM || i < s.order) {
    put(low_bits(sig[i], bps_e), bps_e);
    return len;
  }
  const int psz = bs >> s.po, p = i / psz;
  if (i == s.order) {
    if (s.type == SF_LPC) {
      put(kLpcPrec - 1, 4);
      put(low_bits(s.shift, 5), 5);
      for (int j = 0; j < s.order; ++j) put(low_bits(s.coef[j], kLpcPrec), kLpcPrec);
    }
    put((unsigned)s.method, 2);
    put((unsigned)s.po, 4);
  }
  const int k = s.k[p];
  if (i == s.order || i == p * psz) {
    const int pb = s.method ? 5 : 4;
    if (k == kEscape) {
      put((1u << pb) - 1, pb);
      put(s.w[p], 5);
    } else {
      put((unsigned)k, pb);
    }
  }
  const int r = (int)residual_at(sig, i, s.type, s.order, s.coef, s.shift);
  if (k == kEscape) {
    put(low_bits(r, s.w[p]), s.w[p]);
  } else {
    const unsigned u = zigzag(r);
    len += u >> k;  // unary quotient: zeros
    put((1u << k) | (u & ((1u << k) - 1u)), k + 1);
  }
  return len;
}

__device__ __forceinline__ unsigned frame_byte(const unsigned* buf, int b) { return (buf[b >> 2] >> (24 - 8 * (b & 3))) & 0xFFu; }

__global__ void __launch_bounds__(kThreads) flac_pack_kernel(const float* __restrict__ x, int64_t n, int bits, int via_int16, int sbps, int sr_code,
                                                             int sr_extra_bits, int sr_extra, const FramePlan* __restrict__ plans,
                                                             const int64_t* __restrict__ offsets, uint8_t* __restrict__ out,
                                                             unsigned long long* __restrict__ bad_frames) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  PackSmem& sm = *reinterpret_cast<PackSmem*>(smem_raw);
  const int f = blockIdx.x, t = threadIdx.x, lane = t & 31, warp = t >> 5;
  const int64_t start = (int64_t)f * kBlock;
  const int bs = (int)min((int64_t)kBlock, n - start);
  const FramePlan& P = plans[f];
  for (int i = t; i < kFrameWords; i += kThreads) sm.buf[i] = 0;
  for (int c = 0; c < 2; ++c) {
    const int* src = reinterpret_cast<const int*>(&P.sub[c]);
    int* dst = reinterpret_cast<int*>(&sm.sub[c]);
    for (int i = t; i < (int)(sizeof(Sub) / 4); i += kThreads) dst[i] = src[i];
  }
  sm.crc_tab[t] = flac::crc16_table_entry((unsigned)t);
  const int a = P.assign == 1 ? 0 : P.assign - 7;
  const int ch0 = sub_channel(a, 0), ch1 = sub_channel(a, 1);
  __syncthreads();
  for (int i = t; i < bs; i += kThreads) {
    const float2 v = reinterpret_cast<const float2*>(x)[start + i];
    const int l = pcm_quantize(v.x, bits, via_int16) >> (bits - sbps), r = pcm_quantize(v.y, bits, via_int16) >> (bits - sbps);
    sm.sig[0][i] = candidate(ch0, l, r) >> sm.sub[0].wasted;
    sm.sig[1][i] = candidate(ch1, l, r) >> sm.sub[1].wasted;
  }
  uint8_t h[kHeaderMax];
  const int hb = frame_header(h, (unsigned)f, bs, sr_code, sr_extra_bits, sr_extra, sbps == 16 ? 4 : 6, P.assign);
  __syncthreads();
  if (t == 0)
    for (int j = 0; j < hb; ++j) put_bits(sm.buf, 8 * j, h[j], 8);
  // items [0, bs) = subframe 0, [bs, 2 bs) = subframe 1, a contiguous run per thread
  const int items = 2 * bs, per = (items + kThreads - 1) / kThreads;
  const int lo = min(items, t * per), hi = min(items, lo + per);
  unsigned len = 0;
  for (int it = lo; it < hi; ++it) len += item_bits<false>(sm, it >= bs, it >= bs ? it - bs : it, bs, 0);
  unsigned inc = len;
  for (int o = 1; o < 32; o <<= 1) {
    const unsigned v = __shfl_up_sync(0xffffffffu, inc, o);
    if (lane >= o) inc += v;
  }
  if (lane == 31) sm.scan[warp] = inc;
  __syncthreads();
  unsigned base = 8u * hb, total = 8u * hb;
  for (int w = 0; w < kWarps; ++w) {
    if (w < warp) base += sm.scan[w];
    total += sm.scan[w];
  }
  unsigned pos = base + inc - len;
  for (int it = lo; it < hi; ++it) pos += item_bits<true>(sm, it >= bs, it >= bs ? it - bs : it, bs, pos);
  const int nb = (int)((total + 7) / 8) + 2;
  if (nb != P.bytes) {  // the analysis and the packer disagree: report it and store only the planned length
    if (t == 0) atomicAdd(bad_frames, 1ull);
    return;
  }
  __syncthreads();
  // CRC-16 of bytes [0, nb - 2): each thread's run with init 0, moved to its place by x^(8 * bytes after it), XOR-combined
  const int nc = nb - 2, cper = (nc + kThreads - 1) / kThreads;
  const int clo = min(nc, t * cper), chi = min(nc, clo + cper);
  unsigned crc = 0;
  for (int b = clo; b < chi; ++b) crc = ((crc << 8) ^ sm.crc_tab[((crc >> 8) ^ frame_byte(sm.buf, b)) & 0xFFu]) & 0xFFFFu;
  crc = gf2_mulmod16(crc, x8_pow_mod16((unsigned)(nc - chi)));
  for (int o = 16; o; o >>= 1) crc ^= __shfl_xor_sync(0xffffffffu, crc, o);
  if (lane == 0) sm.crc_part[warp] = crc;
  __syncthreads();
  unsigned crc16 = 0;
  for (int w = 0; w < kWarps; ++w) crc16 ^= sm.crc_part[w];
  uint8_t* o = out + offsets[f];
  for (int b = t; b < nc; b += kThreads) o[b] = (uint8_t)frame_byte(sm.buf, b);
  if (t == 0) {
    o[nc] = (uint8_t)(crc16 >> 8);
    o[nc + 1] = (uint8_t)crc16;
  }
}

int64_t n_frames(int64_t n_samples) { return (n_samples + kBlock - 1) / kBlock; }

// Sample-rate code of the frame header and the bits / value that follow the header for codes 12-14 (RFC 9639 section 9.1.2).
void sample_rate_code(int rate, int* code, int* extra_bits, int* extra) {
  const int table[11][2] = {{88200, 1}, {176400, 2}, {192000, 3}, {8000, 4}, {16000, 5}, {22050, 6}, {24000, 7}, {32000, 8}, {44100, 9}, {48000, 10}, {96000, 11}};
  *extra_bits = 0, *extra = 0;
  for (const auto& e : table)
    if (e[0] == rate) {
      *code = e[1];
      return;
    }
  if (rate % 1000 == 0 && rate / 1000 <= 255) *code = 12, *extra_bits = 8, *extra = rate / 1000;
  else if (rate <= 65535) *code = 13, *extra_bits = 16, *extra = rate;
  else if (rate % 10 == 0 && rate / 10 <= 65535) *code = 14, *extra_bits = 16, *extra = rate / 10;
  else *code = 0;  // only in STREAMINFO
}

}  // namespace
}  // namespace b200sep

using namespace b200sep;

extern "C" int64_t b200sep_flac_work_bytes(int64_t n_samples) {
  if (n_samples < 0) return -1;
  return n_frames(n_samples) * (int64_t)(sizeof(FramePlan) + sizeof(int64_t));
}

extern "C" int64_t b200sep_flac_max_bytes(int64_t n_samples, int stream_bps) {
  if (n_samples < 0 || (stream_bps != 16 && stream_bps != 24)) return -1;
  return n_frames(n_samples) * (int64_t)frame_bound_bytes(stream_bps);
}

extern "C" int b200sep_flac_encode(const float* x, int64_t n_samples, int bits, int via_int16, int stream_bps, int sample_rate, void* work, uint8_t* out,
                                   int64_t* result, void* stream) {
  B2_CHECK_ARG(x && work && out && result && n_samples >= 0, "flac_encode: bad argument");
  B2_CHECK_ARG(bits == 16 || bits == 24 || bits == 32, "flac_encode: bits must be 16, 24 or 32");
  B2_CHECK_ARG((stream_bps == 16 || stream_bps == 24) && stream_bps <= bits, "flac_encode: stream bps must be 16 or 24 and at most bits (got %d, %d)",
               stream_bps, bits);
  B2_CHECK_ARG(sample_rate > 0 && sample_rate < (1 << 20), "flac_encode: sample rate %d does not fit STREAMINFO", sample_rate);
  B2_CHECK_ARG(((uintptr_t)x & 7) == 0 && ((uintptr_t)work & 7) == 0 && ((uintptr_t)result & 7) == 0, "flac_encode: x, work and result must be 8-byte aligned");
  const int64_t nf = n_frames(n_samples);
  B2_CHECK_ARG(nf < (1ll << 31), "flac_encode: too many frames");
  cudaStream_t st = (cudaStream_t)stream;
  B2_CUDA(cudaMemsetAsync(result, 0, 4 * sizeof(int64_t), st));
  if (nf == 0) return B200SEP_OK;
  int sr_code, sr_extra_bits, sr_extra;
  sample_rate_code(sample_rate, &sr_code, &sr_extra_bits, &sr_extra);
  FramePlan* plans = reinterpret_cast<FramePlan*>(work);
  int64_t* offsets = reinterpret_cast<int64_t*>(plans + nf);
  B2_CUDA(cudaFuncSetAttribute(flac_analyze_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(AnalysisSmem)));
  B2_CUDA(cudaFuncSetAttribute(flac_pack_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(PackSmem)));
  flac_analyze_kernel<<<(unsigned)nf, kThreads, sizeof(AnalysisSmem), st>>>(x, n_samples, bits, via_int16, stream_bps, sr_code, sr_extra_bits, sr_extra, plans);
  B2_LAUNCHED();
  flac_offsets_kernel<<<1, 1024, 0, st>>>(plans, (int)nf, offsets, result);
  B2_LAUNCHED();
  flac_pack_kernel<<<(unsigned)nf, kThreads, sizeof(PackSmem), st>>>(x, n_samples, bits, via_int16, stream_bps, sr_code, sr_extra_bits, sr_extra, plans,
                                                                     offsets, out, reinterpret_cast<unsigned long long*>(result + 3));
  B2_LAUNCHED();
  return B200SEP_OK;
}
