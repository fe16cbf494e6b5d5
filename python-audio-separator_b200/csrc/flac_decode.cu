// FLAC decoder (RFC 9639), sm_90a: the compressed frames in HBM -> the planar float mix prepare_mix returns.  Two host calls, one host read
// between them (the output size is known only once the frames are found):
//   locate  flac_find_kernel<false>  one CTA per 4 KiB tile: count the byte positions whose frame header parses, agrees with STREAMINFO and
//                                    carries a matching CRC-8 (the candidates);
//           flac_scan_kernel         one CTA: exclusive scan of the tile counts;
//           flac_find_kernel<true>   the same search again, storing each candidate (offset, block size, channel assignment, coded number) in
//                                    byte order;
//           flac_span_crc_kernel     one warp per candidate: CRC-16 of the bytes up to the next candidate (per-lane runs combined in GF(2));
//           flac_successor_kernel    one thread per candidate: the nearest later candidate (or the end of the data) whose number follows and for
//                                    which the CRC-16 residue of the span, the stored CRC included, is zero.  Span CRCs combine, so a longer span
//                                    costs one GF(2) product per skipped candidate;
//           flac_chain_kernel        one CTA: follow the successors from the candidate at offset 0 through windows staged in shared memory,
//                                    giving each frame its sample offset (the running sum of the block sizes) and checking the coded numbers
//                                    against it.
//   decode  flac_decode_kernel       one CTA per frame: stage the frame's bytes in shared memory, one thread walks the subframes (residuals and
//                                    prediction are one sequential chain), writing integers into the output rows, then the CTA undoes the stereo
//                                    decorrelation and converts to float in place.
// A damaged stream is an input error in the result array: every read is bounded by the buffer, nothing traps.
#include "common.cuh"
#include "flac_common.cuh"

namespace b200sep {
namespace {

using flac::crc8;
using flac::gf2_mulmod16;
using flac::x8_pow_mod16;

constexpr int kTile = 4096;  // bytes per CTA of the candidate search: 16 per thread
constexpr int kFindThreads = kTile / 16;
constexpr int kScanThreads = 1024;
constexpr int kChainWindow = 2048;             // candidates staged per window of the chain walk
constexpr int kDecodeThreads = 32;  // one warp per frame: the walk is serial, so more frames per SM beat more threads per frame
constexpr int kMaxStagedBytes = 96 * 1024;     // larger frames are read from global memory
constexpr int kMaxOrder = 32;

struct Params {
  int sample_rate, bps, channels, variable;
};
struct WorkHeader {
  Params p;
  int m;                         // candidates
  int pad;
  unsigned long long err_key;    // decode: min over failing frames of (frame << 8 | code)
};
struct FrameRec {
  long long sample_off;
  unsigned pos;
  int bs, assign, hdr_len;
};
struct Layout {
  WorkHeader* hdr;
  int* tile_off;                 // tiles + 1
  unsigned* pos;                 // cap + 1 (pos[m] = n_bytes: the end of the data counts as a candidate)
  unsigned* info;                // block size | header length << 16 | channel assignment << 24
  unsigned long long* num;       // coded frame number (fixed blocking) or sample number (variable blocking)
  unsigned* span_crc;            // CRC-16 of [pos[i], pos[i + 1])
  int* succ;
  FrameRec* frames;
  int64_t bytes;
};

// Two candidates are at least 5 bytes apart: a sync byte 0xFF cannot sit at offsets 2-4 of a valid header (rate code 15 is invalid, the
// reserved bit is zero, 0xFF never starts a coded number).
__host__ __device__ inline int64_t capacity(int64_t n) { return n / 5 + 2; }
__host__ __device__ inline int64_t tiles_of(int64_t n) { return n / kTile + 1; }
__host__ __device__ inline int64_t align8(int64_t x) { return (x + 7) & ~7ll; }

__host__ __device__ inline Layout layout(void* work, int64_t n) {
  const int64_t cap = capacity(n), tiles = tiles_of(n);
  char* base = static_cast<char*>(work);
  int64_t o = 0;
  auto take = [&](int64_t bytes) {
    char* p = base + o;
    o += align8(bytes);
    return p;
  };
  Layout L;
  L.hdr = reinterpret_cast<WorkHeader*>(take(sizeof(WorkHeader)));
  L.tile_off = reinterpret_cast<int*>(take(4 * (tiles + 1)));
  L.pos = reinterpret_cast<unsigned*>(take(4 * (cap + 1)));
  L.info = reinterpret_cast<unsigned*>(take(4 * cap));
  L.num = reinterpret_cast<unsigned long long*>(take(8 * cap));
  L.span_crc = reinterpret_cast<unsigned*>(take(4 * cap));
  L.succ = reinterpret_cast<int*>(take(4 * cap));
  L.frames = reinterpret_cast<FrameRec*>(take((int64_t)sizeof(FrameRec) * cap));
  L.bytes = o;
  return L;
}

struct Hdr {
  int len, bs, assign;
  unsigned long long number;
};

// Frame header at byte p of d[0, n): sync with the stream's blocking bit, no reserved codes, rate / sample size / channels agreeing with
// STREAMINFO or deferring to it, block size 1-65535, coded number of at most 6 (fixed) or 7 (variable) bytes, CRC-8.
__device__ bool parse_header(const uint8_t* __restrict__ d, int64_t n, int64_t p, const Params& sp, Hdr& h) {
  if (p + 6 > n || d[p] != 0xFF || d[p + 1] != (0xF8 | sp.variable)) return false;
  const unsigned b2 = d[p + 2], b3 = d[p + 3];
  const int bs_code = b2 >> 4, sr_code = b2 & 15, ca = b3 >> 4, ss = (b3 >> 1) & 7;
  if (bs_code == 0 || sr_code == 15 || ca > 10 || ss == 3 || (b3 & 1)) return false;
  if (ca < 8 ? ca + 1 != sp.channels : sp.channels != 2) return false;
  if (ss && flac::header_bps(ss) != sp.bps) return false;
  int64_t q = p + 4;
  const unsigned first = d[q++];
  const int more = __clz(~(first << 24));  // leading ones of the first byte
  unsigned long long num = first;
  if (more) {
    if (more == 1 || more > (sp.variable ? 7 : 6)) return false;
    num = first & (0x7Fu >> more);
    for (int k = 1; k < more; ++k) {
      if (q >= n) return false;
      const unsigned c = d[q++];
      if ((c >> 6) != 2) return false;
      num = (num << 6) | (c & 0x3F);
    }
  }
  int bs;
  if (bs_code == 1) {
    bs = 192;
  } else if (bs_code <= 5) {
    bs = 576 << (bs_code - 2);
  } else if (bs_code == 6) {
    if (q >= n) return false;
    bs = d[q++] + 1;
  } else if (bs_code == 7) {
    if (q + 1 >= n) return false;
    bs = ((int)d[q] << 8 | d[q + 1]) + 1;
    q += 2;
  } else {
    bs = 256 << (bs_code - 8);
  }
  if (bs > 65535) return false;
  int rate = sr_code < 12 ? flac::header_rate(sr_code) : 0;
  if (sr_code == 12) {
    if (q >= n) return false;
    rate = d[q++] * 1000;
  } else if (sr_code == 13 || sr_code == 14) {
    if (q + 1 >= n) return false;
    rate = ((int)d[q] << 8 | d[q + 1]) * (sr_code == 14 ? 10 : 1);
    q += 2;
  }
  if (sr_code && rate != sp.sample_rate) return false;
  if (q >= n || crc8(d + p, (int)(q - p)) != d[q]) return false;
  h.len = (int)(q + 1 - p);
  h.bs = bs;
  h.assign = ca;
  h.number = num;
  return true;
}

template <bool kWrite>
__global__ void __launch_bounds__(kFindThreads) flac_find_kernel(const uint8_t* __restrict__ d, int64_t n, Params sp, Layout L) {
  __shared__ int warp_sum[kFindThreads / 32];
  const int t = threadIdx.x, lane = t & 31, warp = t >> 5;
  const int64_t base = (int64_t)blockIdx.x * kTile + 16 * t;
  if (!kWrite && blockIdx.x == 0 && t == 0) L.hdr->p = sp;
  unsigned mask = 0;
  if (base < n) {
    const uint4 v = reinterpret_cast<const uint4*>(d)[base >> 4];  // the buffer is readable up to n rounded up to 16
    const unsigned w[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
    for (int k = 0; k < 16; ++k) {
      Hdr h;
      if (((w[k >> 2] >> (8 * (k & 3))) & 0xFFu) == 0xFFu && parse_header(d, n, base + k, sp, h)) mask |= 1u << k;
    }
  }
  const int cnt = __popc(mask);
  int inc = cnt;
  for (int o = 1; o < 32; o <<= 1) {
    const int x = __shfl_up_sync(0xffffffffu, inc, o);
    if (lane >= o) inc += x;
  }
  if (lane == 31) warp_sum[warp] = inc;
  __syncthreads();
  int before = 0, total = 0;
  for (int w = 0; w < kFindThreads / 32; ++w) {
    if (w < warp) before += warp_sum[w];
    total += warp_sum[w];
  }
  if (!kWrite) {
    if (t == 0) L.tile_off[blockIdx.x] = total;
    return;
  }
  int idx = L.tile_off[blockIdx.x] + before + inc - cnt;
  for (; mask; mask &= mask - 1, ++idx) {
    const int64_t p = base + __ffs(mask) - 1;
    Hdr h;
    parse_header(d, n, p, sp, h);
    L.pos[idx] = (unsigned)p;
    L.info[idx] = (unsigned)h.bs | (unsigned)h.len << 16 | (unsigned)h.assign << 24;
    L.num[idx] = h.number;
  }
}

__global__ void __launch_bounds__(kScanThreads) flac_scan_kernel(Layout L, int tiles, int64_t n) {
  __shared__ int warp_sum[kScanThreads / 32];
  const int t = threadIdx.x, lane = t & 31, warp = t >> 5, per = (tiles + kScanThreads - 1) / kScanThreads;
  const int lo = min(tiles, t * per), hi = min(tiles, lo + per);
  int s = 0;
  for (int i = lo; i < hi; ++i) s += L.tile_off[i];
  int inc = s;
  for (int o = 1; o < 32; o <<= 1) {
    const int x = __shfl_up_sync(0xffffffffu, inc, o);
    if (lane >= o) inc += x;
  }
  if (lane == 31) warp_sum[warp] = inc;
  __syncthreads();
  int off = inc - s, total = 0;
  for (int w = 0; w < kScanThreads / 32; ++w) {
    if (w < warp) off += warp_sum[w];
    total += warp_sum[w];
  }
  for (int i = lo; i < hi; ++i) {
    const int c = L.tile_off[i];
    L.tile_off[i] = off;
    off += c;
  }
  if (t == 0) {
    L.hdr->m = total;
    L.pos[total] = (unsigned)n;
  }
}

__global__ void __launch_bounds__(256) flac_span_crc_kernel(const uint8_t* __restrict__ d, Layout L) {
  __shared__ uint16_t tab[256];
  const int t = threadIdx.x, lane = t & 31;
  tab[t] = flac::crc16_table_entry((unsigned)t);
  __syncthreads();
  const int m = L.hdr->m;
  for (int64_t i = ((int64_t)blockIdx.x * blockDim.x + t) >> 5; i < m; i += ((int64_t)gridDim.x * blockDim.x) >> 5) {
    const unsigned a = L.pos[i], len = L.pos[i + 1] - a, per = (len + 31) / 32;
    const unsigned lo = min(len, lane * per), hi = min(len, lo + per);
    unsigned crc = 0;
    for (unsigned b = lo; b < hi; ++b) crc = ((crc << 8) ^ tab[((crc >> 8) ^ d[a + b]) & 0xFFu]) & 0xFFFFu;
    if (crc) crc = gf2_mulmod16(crc, x8_pow_mod16(len - hi));
    for (int o = 16; o; o >>= 1) crc ^= __shfl_xor_sync(0xffffffffu, crc, o);
    if (lane == 0) L.span_crc[i] = crc;
  }
}

// Longest span searched for a frame's end: 32 bits per sample and channel (more than VERBATIM at 25 bits) plus headers.
__device__ __forceinline__ unsigned long long max_frame_span(int bs, int channels) { return 64ull + (unsigned long long)channels * (4ull * bs + 256); }

__global__ void __launch_bounds__(256) flac_successor_kernel(Layout L) {
  const Params sp = L.hdr->p;
  const int m = L.hdr->m;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < m; i += (int64_t)gridDim.x * blockDim.x) {
    const unsigned pi = L.pos[i];
    const int bs = (int)(L.info[i] & 0xFFFFu);
    const unsigned long long want = sp.variable ? L.num[i] + bs : L.num[i] + 1;
    const unsigned long long limit = max_frame_span(bs, sp.channels);
    unsigned crc = 0;
    int s = -1;
    for (int64_t j = i + 1; j <= m; ++j) {
      const unsigned pj = L.pos[j];
      if (pj - pi > limit) break;
      if (crc) crc = gf2_mulmod16(crc, x8_pow_mod16(pj - L.pos[j - 1]));
      crc ^= L.span_crc[j - 1];
      if (crc == 0 && (j == m || L.num[j] == want)) {
        s = (int)j;
        break;
      }
    }
    L.succ[i] = s;
  }
}

__global__ void __launch_bounds__(kScanThreads) flac_chain_kernel(Layout L, int64_t n, int64_t* __restrict__ result) {
  __shared__ int s_succ[kChainWindow];
  __shared__ unsigned s_pos[kChainWindow], s_info[kChainWindow];
  __shared__ unsigned long long s_num[kChainWindow];
  __shared__ int s_cur, s_done;
  __shared__ long long s_k, s_sum, s_maxlen;
  const int t = threadIdx.x;
  const int m = L.hdr->m;
  const bool variable = L.hdr->p.variable;
  if (t == 0) {
    for (int i = 0; i < 8; ++i) result[i] = 0;
    s_cur = 0, s_k = 0, s_sum = 0, s_maxlen = 0;
    s_done = 0;
    if (n == 0) {
      s_done = 1;
    } else if (m == 0 || L.pos[0] != 0) {
      result[2] = B200SEP_FLAC_ERR_SYNC;
      s_done = 1;
    } else {
      result[6] = (int64_t)L.num[0];
    }
  }
  __syncthreads();
  const unsigned long long first = m ? L.num[0] : 0;
  while (!s_done) {
    const int base = s_cur, cnt = min(kChainWindow, m - base);
    for (int i = t; i < cnt; i += kScanThreads) {
      s_succ[i] = L.succ[base + i];
      s_pos[i] = L.pos[base + i];
      s_info[i] = L.info[base + i];
      s_num[i] = L.num[base + i];
    }
    __syncthreads();
    if (t == 0) {
      int cur = base, done = 0;
      long long k = s_k, sum = s_sum, maxlen = s_maxlen;
      while (cur < base + cnt) {
        const int c = cur - base, s = s_succ[c];
        const unsigned long long want = variable ? first + (unsigned long long)sum : first + (unsigned long long)k;
        int code = s < 0 ? B200SEP_FLAC_ERR_CRC : (s_num[c] != want ? B200SEP_FLAC_ERR_NUMBER : B200SEP_FLAC_OK);
        if (code) {
          result[2] = code, result[3] = k, result[4] = s_pos[c];
          done = 1;
          break;
        }
        const int bs = (int)(s_info[c] & 0xFFFFu);
        L.frames[k] = FrameRec{sum, s_pos[c], bs, (int)(s_info[c] >> 24), (int)((s_info[c] >> 16) & 0xFFu)};
        const unsigned end = s < base + cnt ? s_pos[s - base] : L.pos[s];
        maxlen = max(maxlen, (long long)(end - s_pos[c]));
        sum += bs;
        ++k;
        cur = s;
        if (s == m) {
          done = 1;
          break;
        }
      }
      s_cur = cur, s_k = k, s_sum = sum, s_maxlen = maxlen, s_done = done;
      if (done && result[2] == 0) result[0] = k, result[1] = sum, result[5] = maxlen;
    }
    __syncthreads();
  }
}

// ---- decode ------------------------------------------------------------------------------------------------------------------------

// Big-endian bit reader over 32-bit words (shared or global memory through a generic pointer); words past nw read as zero.
struct BitReader {
  const uint32_t* w;
  unsigned long long nw, next, buf, pos;
  int nb;
  __device__ void init(const uint32_t* words, unsigned long long nwords, unsigned long long bitpos) {
    w = words, nw = nwords, next = bitpos >> 5, buf = 0, nb = 0, pos = bitpos & ~31ull;
    skip((int)(bitpos & 31));
  }
  __device__ __forceinline__ void refill() {  // one word always leaves more than 32 bits
    if (nb <= 32) {
      const uint32_t v = next < nw ? __byte_perm(w[next], 0, 0x0123) : 0u;
      ++next;
      buf |= (unsigned long long)v << (32 - nb);
      nb += 32;
    }
  }
  __device__ __forceinline__ void skip(int n) {  // n <= 32
    refill();
    buf <<= n;
    nb -= n;
    pos += n;
  }
  __device__ __forceinline__ unsigned get(int n) {  // n <= 32
    refill();
    const unsigned v = n ? (unsigned)(buf >> (64 - n)) : 0u;
    buf <<= n;
    nb -= n;
    pos += n;
    return v;
  }
  __device__ __forceinline__ int sget(int n) { return n ? (int)(get(n) << (32 - n)) >> (32 - n) : 0; }
  // zeros before the next one bit; false once the reader passes `limit` without finding one
  __device__ __forceinline__ bool unary(unsigned& q, unsigned long long limit) {
    unsigned z = 0;
    for (;;) {
      refill();
      if (buf) break;
      z += nb, pos += nb, nb = 0;
      if (pos > limit) return false;
    }
    const int c = __clzll(buf);
    buf = (buf << c) << 1;
    nb -= c + 1;
    pos += c + 1;
    q = z + c;
    return true;
  }
};

struct FixedPred {
  int order, h1, h2, h3, h4;
  __device__ __forceinline__ int operator()(int r) {
    unsigned p = 0;
    switch (order) {
      case 1: p = h1; break;
      case 2: p = 2u * h1 - h2; break;
      case 3: p = 3u * h1 - 3u * h2 + h3; break;
      case 4: p = 4u * h1 - 6u * h2 + 4u * h3 - h4; break;
      default: break;
    }
    const int x = (int)(p + (unsigned)r);
    h4 = h3, h3 = h2, h2 = h1, h1 = x;
    return x;
  }
};
// LPC with the last kMaxOrder samples in a shared-memory ring; Acc = int when bps + precision + log2(order) fits 32 bits.
template <class Acc>
struct LpcPred {
  int order, shift, i;
  const int* coef;
  int* hist;
  __device__ __forceinline__ int operator()(int r) {
    Acc s = 0;
    for (int j = 0; j < order; ++j) s += (Acc)coef[j] * (Acc)hist[(i - 1 - j) & (kMaxOrder - 1)];
    const int x = (int)((unsigned)r + (unsigned)(int)(s >> shift));
    hist[i & (kMaxOrder - 1)] = x;
    ++i;
    return x;
  }
};

// Residual of a FIXED / LPC subframe after its warm-up samples, fed through the predictor into dst[order, bs) (dst may be null: a channel that
// is not kept).  Returns a B200SEP_FLAC_* code.
template <class Pred>
__device__ __forceinline__ int residual(BitReader& br, unsigned long long limit, int bs, int order, int wasted, Pred& pred, int* dst) {
  const unsigned method = br.get(2);
  if (method > 1) return B200SEP_FLAC_ERR_SUBFRAME;
  const int pbits = method ? 5 : 4, esc = (1 << pbits) - 1;
  const int po = (int)br.get(4), psz = bs >> po;
  if ((bs & ((1 << po) - 1)) || psz < order) return B200SEP_FLAC_ERR_SUBFRAME;
  int i = order;
  for (int p = 0; p < (1 << po); ++p) {
    const int end = (p + 1) * psz;
    const int k = (int)br.get(pbits);
    if (k == esc) {
      const int w = (int)br.get(5);
      for (; i < end; ++i) {
        const int x = pred(br.sget(w));
        if (dst) dst[i] = (int)((unsigned)x << wasted);
      }
    } else {
      for (; i < end; ++i) {
        unsigned q;
        if (!br.unary(q, limit)) return B200SEP_FLAC_ERR_LENGTH;
        const unsigned v = (q << k) | br.get(k);
        const int x = pred((int)(v >> 1) ^ -(int)(v & 1));
        if (dst) dst[i] = (int)((unsigned)x << wasted);
      }
    }
    if (br.pos > limit) return B200SEP_FLAC_ERR_LENGTH;
  }
  return B200SEP_FLAC_OK;
}

struct SubScratch {
  int coef[kMaxOrder];
  int hist[kMaxOrder];
};

__device__ __forceinline__ int subframe(BitReader& br, unsigned long long limit, int bs, int bps, int* dst, SubScratch& sc) {
  if (br.get(1)) return B200SEP_FLAC_ERR_SUBFRAME;
  const int type = (int)br.get(6);
  int wasted = 0;
  if (br.get(1)) {
    unsigned q;
    if (!br.unary(q, limit)) return B200SEP_FLAC_ERR_LENGTH;
    if (q + 1 >= (unsigned)bps) return B200SEP_FLAC_ERR_SUBFRAME;
    wasted = (int)q + 1;
  }
  const int b = bps - wasted;
  if (type == 0) {
    const int v = (int)((unsigned)br.sget(b) << wasted);
    if (dst)
      for (int i = 0; i < bs; ++i) dst[i] = v;
    return br.pos > limit ? B200SEP_FLAC_ERR_LENGTH : B200SEP_FLAC_OK;
  }
  if (type == 1) {
    for (int i = 0; i < bs; ++i) {
      const int v = (int)((unsigned)br.sget(b) << wasted);
      if (dst) dst[i] = v;
      if ((i & 255) == 0 && br.pos > limit) return B200SEP_FLAC_ERR_LENGTH;
    }
    return br.pos > limit ? B200SEP_FLAC_ERR_LENGTH : B200SEP_FLAC_OK;
  }
  const bool fixed = type >= 8 && type <= 12;
  if (!fixed && type < 32) return B200SEP_FLAC_ERR_SUBFRAME;
  const int order = fixed ? type - 8 : type - 31;
  if (order > bs) return B200SEP_FLAC_ERR_SUBFRAME;
  FixedPred fp{order, 0, 0, 0, 0};
  for (int i = 0; i < order; ++i) {
    const int x = br.sget(b);
    if (dst) dst[i] = (int)((unsigned)x << wasted);
    if (fixed) fp.h4 = fp.h3, fp.h3 = fp.h2, fp.h2 = fp.h1, fp.h1 = x;
    else sc.hist[i] = x;
  }
  if (fixed) {
    FixedPred& pred = fp;
    return residual(br, limit, bs, order, wasted, pred, dst);
  }
  const int prec = (int)br.get(4) + 1;
  const int shift = br.sget(5);
  if (prec == 16 || shift < 0) return B200SEP_FLAC_ERR_SUBFRAME;
  for (int j = 0; j < order; ++j) sc.coef[j] = br.sget(prec);
  if (br.pos > limit) return B200SEP_FLAC_ERR_LENGTH;
  if (b + prec + (32 - __clz(order)) <= 32) {
    LpcPred<int> pred{order, shift, order, sc.coef, sc.hist};
    return residual(br, limit, bs, order, wasted, pred, dst);
  }
  LpcPred<long long> pred{order, shift, order, sc.coef, sc.hist};
  return residual(br, limit, bs, order, wasted, pred, dst);
}

__global__ void __launch_bounds__(kDecodeThreads, 1) flac_decode_kernel(const uint8_t* __restrict__ d, int64_t n, Layout L, int nf, int staged,
                                                                     float* __restrict__ out, int64_t ld) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  __shared__ SubScratch sc;
  __shared__ int s_err;
  const int f = blockIdx.x, t = threadIdx.x;
  const FrameRec fr = L.frames[f];
  const Params sp = L.hdr->p;
  const unsigned start = fr.pos, end = f + 1 < nf ? L.frames[f + 1].pos : (unsigned)n;
  const int bs = fr.bs, assign = fr.assign;
  const int nch = assign < 8 ? assign + 1 : 2, rows = min(sp.channels, 2);
  if (end < start + 2 + 6 || end > n || fr.sample_off + bs > ld) {  // only a caller passing another stream's work gets here
    if (t == 0) atomicMin(&L.hdr->err_key, (unsigned long long)f << 8 | B200SEP_FLAC_ERR_LENGTH);
    return;
  }
  const uint32_t* words;
  unsigned long long nwords, bit0;
  if (staged) {
    const unsigned a0 = start & ~15u, a1 = (end + 15) & ~15u;
    const uint4* src = reinterpret_cast<const uint4*>(d + a0);
    uint4* dst = reinterpret_cast<uint4*>(smem_raw);
    for (unsigned i = t; i < (a1 - a0) / 16; i += kDecodeThreads) dst[i] = src[i];
    words = reinterpret_cast<const uint32_t*>(smem_raw);
    nwords = (a1 - a0) / 4;
    bit0 = 8ull * (start - a0);
  } else {
    words = reinterpret_cast<const uint32_t*>(d);
    nwords = (((unsigned long long)n + 15) & ~15ull) / 4;
    bit0 = 8ull * start;
  }
  __syncthreads();
  int* row0 = reinterpret_cast<int*>(out + fr.sample_off);
  int* row1 = reinterpret_cast<int*>(out + ld + fr.sample_off);
  if (t == 0) {
    // the subframes end, byte-aligned, where the frame's CRC-16 begins
    const unsigned long long limit = bit0 + 8ull * (end - start - 2);
    BitReader br;
    br.init(words, nwords, bit0 + 8ull * fr.hdr_len);
    int err = B200SEP_FLAC_OK;
    for (int c = 0; c < nch && !err; ++c) {
      const int side = (assign == 8 && c == 1) || (assign == 9 && c == 0) || (assign == 10 && c == 1);
      err = subframe(br, limit, bs, sp.bps + side, c == 0 ? row0 : (c == 1 && rows == 2 ? row1 : nullptr), sc);
    }
    if (!err && ((br.pos + 7) & ~7ull) != limit) err = B200SEP_FLAC_ERR_LENGTH;
    if (err) atomicMin(&L.hdr->err_key, (unsigned long long)f << 8 | (unsigned)err);
    s_err = err;
  }
  __syncthreads();
  if (s_err) return;
  // stereo decorrelation, then x * 2^-(bps-1): exact for |x| < 2^24
  const float scale = ldexpf(1.f, 1 - sp.bps);
  for (int i = t; i < bs; i += kDecodeThreads) {
    const int a = row0[i];
    if (rows == 1) {
      out[fr.sample_off + i] = (float)a * scale;
      continue;
    }
    const int b = row1[i];
    int l = a, r = b;
    if (assign == 8) {
      r = (int)((unsigned)a - (unsigned)b);
    } else if (assign == 9) {
      l = (int)((unsigned)a + (unsigned)b);
    } else if (assign == 10) {
      const int mid = (int)(((unsigned)a << 1) | ((unsigned)b & 1u));
      l = (int)((unsigned)mid + (unsigned)b) >> 1;
      r = (int)((unsigned)mid - (unsigned)b) >> 1;
    }
    out[fr.sample_off + i] = (float)l * scale;
    out[ld + fr.sample_off + i] = (float)r * scale;
  }
}

__global__ void flac_decode_status_kernel(Layout L, int64_t* __restrict__ result) {
  const unsigned long long key = L.hdr->err_key;
  if (key != ~0ull && result[2] == 0) {
    result[2] = (int64_t)(key & 0xFF);
    result[3] = (int64_t)(key >> 8);
    result[4] = L.frames[key >> 8].pos;
  }
}

}  // namespace
}  // namespace b200sep

using namespace b200sep;

extern "C" int64_t b200sep_flac_decode_work_bytes(int64_t n_bytes) {
  if (n_bytes < 0 || n_bytes >= (1ll << 31)) return -1;
  return layout(nullptr, n_bytes).bytes;
}

extern "C" int b200sep_flac_locate(const uint8_t* frames, int64_t n_bytes, int sample_rate, int bps, int channels, int variable_blocking, void* work,
                                   int64_t* result, void* stream) {
  B2_CHECK_ARG(frames && work && result && n_bytes >= 0 && n_bytes < (1ll << 31), "flac_locate: bad argument");
  B2_CHECK_ARG(sample_rate > 0 && sample_rate < (1 << 20) && bps >= 4 && bps <= 24 && channels >= 1 && channels <= 8 &&
                   (variable_blocking == 0 || variable_blocking == 1),
               "flac_locate: unsupported stream (rate %d, %d bits, %d channels, blocking %d)", sample_rate, bps, channels, variable_blocking);
  B2_CHECK_ARG(((uintptr_t)frames & 15) == 0 && ((uintptr_t)work & 7) == 0 && ((uintptr_t)result & 7) == 0,
               "flac_locate: frames must be 16-byte aligned, work and result 8-byte aligned");
  cudaStream_t st = (cudaStream_t)stream;
  const Layout L = layout(work, n_bytes);
  const Params sp{sample_rate, bps, channels, variable_blocking};
  const int tiles = (int)tiles_of(n_bytes);
  const int grid = kNumSMs * 8;
  flac_find_kernel<false><<<tiles, kFindThreads, 0, st>>>(frames, n_bytes, sp, L);
  B2_LAUNCHED();
  flac_scan_kernel<<<1, kScanThreads, 0, st>>>(L, tiles, n_bytes);
  B2_LAUNCHED();
  flac_find_kernel<true><<<tiles, kFindThreads, 0, st>>>(frames, n_bytes, sp, L);
  B2_LAUNCHED();
  flac_span_crc_kernel<<<grid, 256, 0, st>>>(frames, L);
  B2_LAUNCHED();
  flac_successor_kernel<<<grid, 256, 0, st>>>(L);
  B2_LAUNCHED();
  flac_chain_kernel<<<1, kScanThreads, 0, st>>>(L, n_bytes, result);
  B2_LAUNCHED();
  return B200SEP_OK;
}

extern "C" int b200sep_flac_decode(const uint8_t* frames, int64_t n_bytes, void* work, int64_t n_frames, int64_t max_frame_bytes, float* out,
                                   int64_t out_ld, int64_t* result, void* stream) {
  B2_CHECK_ARG(frames && work && out && result && n_bytes >= 0 && n_bytes < (1ll << 31), "flac_decode: bad argument");
  B2_CHECK_ARG(n_frames >= 0 && n_frames <= capacity(n_bytes) && max_frame_bytes >= 0 && max_frame_bytes <= n_bytes && out_ld >= 0,
               "flac_decode: frame count / size do not belong to this stream");
  B2_CHECK_ARG(((uintptr_t)frames & 15) == 0 && ((uintptr_t)work & 7) == 0 && ((uintptr_t)out & 3) == 0, "flac_decode: misaligned argument");
  if (n_frames == 0) return B200SEP_OK;
  cudaStream_t st = (cudaStream_t)stream;
  const Layout L = layout(work, n_bytes);
  B2_CUDA(cudaMemsetAsync(&L.hdr->err_key, 0xFF, sizeof(unsigned long long), st));
  const int64_t span = ((max_frame_bytes + 15) & ~15ll) + 16;  // a frame's 16-byte aligned enclosing span
  const int staged = span <= kMaxStagedBytes;
  const int smem = staged ? (int)span : 0;
  B2_CUDA(cudaFuncSetAttribute(flac_decode_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
  flac_decode_kernel<<<(unsigned)n_frames, kDecodeThreads, smem, st>>>(frames, n_bytes, L, (int)n_frames, staged, out, out_ld);
  B2_LAUNCHED();
  flac_decode_status_kernel<<<1, 1, 0, st>>>(L, result);
  B2_LAUNCHED();
  return B200SEP_OK;
}
