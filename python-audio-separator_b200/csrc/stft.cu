// STFT / iSTFT / overlap-add kernels (sm_90a).  Not cuFFT: one CTA transforms one stereo frame as a single
// complex FFT (z = L + iR) with shared-memory Stockham autosort stages of radix 8/4/2/3/5, the two real
// spectra are separated in the epilogue, which also applies the dim_f crop, the low-bin zeroing and the
// complex-as-channels plane split of the reference (uvr_lib_v5/stft.py:20-56).  These kernels are HBM/latency
// bound (~0.1 GFLOP vs 14.7 MB per MDX chunk, SURVEY.md section 8d); all chunks of a track go in one launch.
#include <math.h>

#include <vector>

#include "common.cuh"
#include "internal.h"
#include "pcm.cuh"

namespace b200sep {

constexpr int kFftThreads = 256;
}  // namespace b200sep

namespace b200sep {

__device__ __forceinline__ float2 cmul(float2 a, float2 b) { return make_float2(a.x * b.x - a.y * b.y, a.x * b.y + a.y * b.x); }
__device__ __forceinline__ float2 cadd(float2 a, float2 b) { return make_float2(a.x + b.x, a.y + b.y); }
__device__ __forceinline__ float2 csub(float2 a, float2 b) { return make_float2(a.x - b.x, a.y - b.y); }
// multiply by -i (DIR=-1, forward) or +i (DIR=+1, inverse)
template <int DIR>
__device__ __forceinline__ float2 mul_dir_i(float2 a) {
  return DIR < 0 ? make_float2(a.y, -a.x) : make_float2(-a.y, a.x);
}

template <int DIR>
__device__ __forceinline__ void bfly2(float2* v) {
  float2 a = v[0], b = v[1];
  v[0] = cadd(a, b);
  v[1] = csub(a, b);
}
template <int DIR>
__device__ __forceinline__ void bfly4(float2* v) {
  float2 a = cadd(v[0], v[2]), b = csub(v[0], v[2]);
  float2 c = cadd(v[1], v[3]), d = mul_dir_i<DIR>(csub(v[1], v[3]));
  v[0] = cadd(a, c);
  v[1] = cadd(b, d);
  v[2] = csub(a, c);
  v[3] = csub(b, d);
}
template <int DIR>
__device__ __forceinline__ void bfly8(float2* v) {
  // two radix-4 on even / odd, then twiddle by w8^k
  float2 e[4] = {v[0], v[2], v[4], v[6]};
  float2 o[4] = {v[1], v[3], v[5], v[7]};
  bfly4<DIR>(e);
  bfly4<DIR>(o);
  const float h = 0.70710678118654752440f;
  // w8^1 = (h, DIR*h), w8^2 = DIR*i, w8^3 = (-h, DIR*h)
  float2 t1 = make_float2(h * (o[1].x - DIR * o[1].y), h * (o[1].y + DIR * o[1].x));
  float2 t2 = mul_dir_i<DIR>(o[2]);
  float2 t3 = make_float2(h * (-o[3].x - DIR * o[3].y), h * (-o[3].y + DIR * o[3].x));
  v[0] = cadd(e[0], o[0]);
  v[4] = csub(e[0], o[0]);
  v[1] = cadd(e[1], t1);
  v[5] = csub(e[1], t1);
  v[2] = cadd(e[2], t2);
  v[6] = csub(e[2], t2);
  v[3] = cadd(e[3], t3);
  v[7] = csub(e[3], t3);
}
template <int DIR>
__device__ __forceinline__ void bfly3(float2* v) {
  const float s = 0.86602540378443864676f * DIR;  // sin(2pi/3) with direction sign
  float2 t = cadd(v[1], v[2]);
  float2 d = csub(v[1], v[2]);
  float2 m = make_float2(v[0].x - 0.5f * t.x, v[0].y - 0.5f * t.y);
  float2 r = make_float2(-s * d.y, s * d.x);  // i*s*d
  v[0] = cadd(v[0], t);
  v[1] = cadd(m, r);
  v[2] = csub(m, r);
}
template <int DIR>
__device__ __forceinline__ void bfly5(float2* v) {
  const float c1 = 0.30901699437494742410f, c2 = -0.80901699437494742410f;
  const float s1 = 0.95105651629515357212f * DIR, s2 = 0.58778525229247312917f * DIR;
  float2 a1 = cadd(v[1], v[4]), b1 = csub(v[1], v[4]);
  float2 a2 = cadd(v[2], v[3]), b2 = csub(v[2], v[3]);
  float2 x0 = v[0];
  v[0] = make_float2(x0.x + a1.x + a2.x, x0.y + a1.y + a2.y);
  float2 m1 = make_float2(x0.x + c1 * a1.x + c2 * a2.x, x0.y + c1 * a1.y + c2 * a2.y);
  float2 m2 = make_float2(x0.x + c2 * a1.x + c1 * a2.x, x0.y + c2 * a1.y + c1 * a2.y);
  // i*(s1*b1 + s2*b2), i*(s2*b1 - s1*b2)
  float2 r1 = make_float2(-(s1 * b1.y + s2 * b2.y), s1 * b1.x + s2 * b2.x);
  float2 r2 = make_float2(-(s2 * b1.y - s1 * b2.y), s2 * b1.x - s1 * b2.x);
  v[1] = cadd(m1, r1);
  v[4] = csub(m1, r1);
  v[2] = cadd(m2, r2);
  v[3] = csub(m2, r2);
}

// One Stockham autosort stage of radix R.  ns = product of the radices already applied.  The power-of-two stages come first (factor_fft), so while
// R is 8 / 4 / 2 the index arithmetic is shifts and masks (`lg` = log2(ns), -1 otherwise).
template <int DIR, int R>
__device__ __forceinline__ void stockham_stage(const float2* __restrict__ in, float2* __restrict__ out, int n, int ns, int lg,
                                               const float2* __restrict__ tw) {
  const int nr = n / R;
  const int tw_step = n / (ns * R);
  for (int j = threadIdx.x; j < nr; j += blockDim.x) {
    const int k = lg >= 0 ? (j & (ns - 1)) : (j % ns);
    float2 v[R];
#pragma unroll
    for (int r = 0; r < R; ++r) v[r] = in[j + r * nr];
    if (ns > 1) {
      // exact table twiddles w^r = tw[r k tw_step] (powers built by complex multiplication were measured: no faster, and 3e-7 of extra relative error)
#pragma unroll
      for (int r = 1; r < R; ++r) {
        float2 w = __ldg(&tw[r * k * tw_step]);
        if (DIR > 0) w.y = -w.y;
        v[r] = cmul(v[r], w);
      }
    }
    if (R == 2) bfly2<DIR>(v);
    if (R == 3) bfly3<DIR>(v);
    if (R == 4) bfly4<DIR>(v);
    if (R == 5) bfly5<DIR>(v);
    if (R == 8) bfly8<DIR>(v);
    const int j0 = (lg >= 0 ? ((j >> lg) << lg) : (j / ns) * ns) * R + k;
#pragma unroll
    for (int r = 0; r < R; ++r) out[j0 + r * ns] = v[r];
  }
}

// In-CTA complex FFT of st.n points living in buf0; returns the buffer holding the natural-order result.
template <int DIR>
__device__ float2* fft_smem(float2* buf0, float2* buf1, const FftStages& st, const float2* __restrict__ tw) {
  int ns = 1;
  float2* a = buf0;
  float2* b = buf1;
  for (int s = 0; s < st.n_stages; ++s) {
    const int R = st.radix[s];
    const int lg = (ns & (ns - 1)) == 0 ? 31 - __clz(ns) : -1;
    switch (R) {
      case 8: stockham_stage<DIR, 8>(a, b, st.n, ns, lg, tw); break;
      case 4: stockham_stage<DIR, 4>(a, b, st.n, ns, lg, tw); break;
      case 2: stockham_stage<DIR, 2>(a, b, st.n, ns, lg, tw); break;
      case 3: stockham_stage<DIR, 3>(a, b, st.n, ns, lg, tw); break;
      default: stockham_stage<DIR, 5>(a, b, st.n, ns, lg, tw); break;
    }
    __syncthreads();
    ns *= R;
    float2* t = a;
    a = b;
    b = t;
  }
  return a;
}

// ---------------------------------------------------------------------------------------------------------
// forward: grid (frames, batch)
__global__ void __launch_bounds__(kFftThreads) stft_forward_kernel(FftStages st, const float2* __restrict__ tw,
                                                                   const float* __restrict__ window, const float* __restrict__ wave,
                                                                   int64_t batch_stride, int64_t chan_stride, int64_t valid_len,
                                                                   int hop, int chunk_len, int frames, int dim_f, int zero_bins,
                                                                   int layout, float* __restrict__ spec, int frame_offset, float scale, int zero_pad) {
  extern __shared__ float2 smem[];
  const int N = st.n;
  float2* buf0 = smem;
  float2* buf1 = smem + N;
  const int t = blockIdx.x, b = blockIdx.y;
  const int64_t base = (int64_t)b * batch_stride;
  for (int n = threadIdx.x; n < N; n += blockDim.x) {
    int s = t * hop + n - frame_offset;
    const bool outside = s < 0 || s >= chunk_len;
    if (s < 0) s = -s;                                // reflect (torch.stft center=True, pad_mode="reflect")
    if (s >= chunk_len) s = 2 * (chunk_len - 1) - s;
    float xl = 0.f, xr = 0.f;
    if (!(zero_pad && outside) && (valid_len <= 0 || base + s < valid_len)) {  // zero_pad: librosa.stft's pad_mode="constant"
      xl = __ldg(&wave[base + s]);
      xr = __ldg(&wave[base + chan_stride + s]);
    }
    const float w = __ldg(&window[n]) * scale;
    buf0[n] = make_float2(xl * w, xr * w);
  }
  __syncthreads();
  const float2* Z = fft_smem<-1>(buf0, buf1, st, tw);
  const int64_t plane = (int64_t)frames * dim_f;
  float* out = spec + (int64_t)b * 4 * plane;
  for (int k = threadIdx.x; k < dim_f; k += blockDim.x) {
    float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
    if (k >= zero_bins) {
      const float2 z = Z[k];
      const float2 zc = Z[k == 0 ? 0 : N - k];
      v.x = 0.5f * (z.x + zc.x);  // L re
      v.y = 0.5f * (z.y - zc.y);  // L im
      v.z = 0.5f * (z.y + zc.y);  // R re
      v.w = 0.5f * (zc.x - z.x);  // R im
    }
    if (layout == B200SEP_LAYOUT_CTF) {
      const int64_t o = (int64_t)t * dim_f + k;
      out[o] = v.x;
      out[plane + o] = v.y;
      out[2 * plane + o] = v.z;
      out[3 * plane + o] = v.w;
    } else {
      const int64_t o = (int64_t)k * frames + t;
      out[o] = v.x;
      out[plane + o] = v.y;
      out[2 * plane + o] = v.z;
      out[3 * plane + o] = v.w;
    }
  }
}

// inverse per-frame transform: grid (frames, batch); writes windowed time frames (B,2,frames,N)
__global__ void __launch_bounds__(kFftThreads) istft_frames_kernel(FftStages st, const float2* __restrict__ tw,
                                                                   const float* __restrict__ window, const float* __restrict__ spec,
                                                                   int frames, int dim_f, int layout, float* __restrict__ fr, float scale) {
  extern __shared__ float2 smem[];
  const int N = st.n;
  float2* buf0 = smem;
  float2* buf1 = smem + N;
  const int t = blockIdx.x, b = blockIdx.y;
  const int64_t plane = (int64_t)frames * dim_f;
  const float* in = spec + (int64_t)b * 4 * plane;
  for (int k = threadIdx.x; k < N; k += blockDim.x) {
    const int kk = (k <= N / 2) ? k : N - k;
    float2 z = make_float2(0.f, 0.f);
    if (kk < dim_f) {
      const int64_t o = (layout == B200SEP_LAYOUT_CTF) ? ((int64_t)t * dim_f + kk) : ((int64_t)kk * frames + t);
      const float lre = __ldg(&in[o]), lim = __ldg(&in[plane + o]), rre = __ldg(&in[2 * plane + o]), rim = __ldg(&in[3 * plane + o]);
      if (kk == 0 || 2 * kk == N) {
        z = make_float2(lre, rre);  // c2r ignores the imaginary part of DC / Nyquist
      } else if (k <= N / 2) {
        z = make_float2(lre - rim, lim + rre);
      } else {
        z = make_float2(lre + rim, rre - lim);
      }
    }
    buf0[k] = z;
  }
  __syncthreads();
  const float2* y = fft_smem<+1>(buf0, buf1, st, tw);
  const float inv_n = scale / (float)N;
  float* o_l = fr + (((int64_t)b * 2 + 0) * frames + t) * N;
  float* o_r = fr + (((int64_t)b * 2 + 1) * frames + t) * N;
  for (int n = threadIdx.x; n < N; n += blockDim.x) {
    const float w = __ldg(&window[n]) * inv_n;
    const float2 v = y[n];
    o_l[n] = v.x * w;
    o_r[n] = v.y * w;
  }
}

// overlap-add of the windowed frames / window envelope, trimmed by N/2: (B,2,frames,N) -> (B,2,hop*(frames-1))
// frame t sits at OLA position t*hop; output sample n is OLA position n + ola_offset.  The squared-window envelope also counts
// `env_extra` virtual all-zero frames before frame 0 and after the last one (HTDemucs._ispec pads two such frames, htdemucs.py:405-413).
__global__ void istft_ola_kernel(const float* __restrict__ fr, const float* __restrict__ window, int N, int hop, int frames,
                                 int out_len, float* __restrict__ wave, int ola_offset, int env_extra) {
  const int bc = blockIdx.y;
  const float* f = fr + (int64_t)bc * frames * N;
  for (int n = blockIdx.x * blockDim.x + threadIdx.x; n < out_len; n += gridDim.x * blockDim.x) {
    const int m = n + ola_offset;
    // floor/ceil with negative numerators: shift by a multiple of hop
    const int sh = (env_extra + 1) * hop;
    int t_hi = (m + sh) / hop - (env_extra + 1);
    int t_lo = (m - N + 1 + sh + hop - 1) / hop - (env_extra + 1);  // smallest t with t*hop + N > m
    if (t_hi > frames - 1 + env_extra) t_hi = frames - 1 + env_extra;
    if (t_lo < -env_extra) t_lo = -env_extra;
    float acc = 0.f, env = 0.f;
    for (int t = t_lo; t <= t_hi; ++t) {
      const int i = m - t * hop;
      const float w = __ldg(&window[i]);
      if (t >= 0 && t < frames) acc += __ldg(&f[(int64_t)t * N + i]);
      env += w * w;
    }
    wave[(int64_t)bc * out_len + n] = acc / env;
  }
}

// demix accumulate/divide/trim as a gather over covering chunks (mdx_separator.py:348-401)
__global__ void demix_ola_kernel(const float* __restrict__ chunks, int first_chunk, int n_chunks, int chunk_len, int64_t step, int64_t total_len,
                                 int64_t trim, int64_t n_out, int64_t q_begin, int64_t q_end, int use_window, float out_scale,
                                 const float* __restrict__ mix, int64_t mix_ld, int64_t mix_base, float compensate, int interleave,
                                 float* __restrict__ primary, float* __restrict__ secondary, int64_t out_base, int64_t out_ld) {
  for (int64_t q = q_begin + (int64_t)blockIdx.x * blockDim.x + threadIdx.x; q < q_end; q += (int64_t)gridDim.x * blockDim.x) {
    const int64_t p = q + trim;
    int64_t i_hi = p / step;
    if (i_hi > n_chunks - 1) i_hi = n_chunks - 1;
    int64_t i_lo = (p - chunk_len + step) / step;
    if (p - chunk_len + 1 <= 0) i_lo = 0;
    float res[2] = {0.f, 0.f};
    float div = 0.f;
    for (int64_t i = i_lo; i <= i_hi; ++i) {
      const int64_t s = i * step;
      int64_t e = s + chunk_len;
      if (e > total_len) e = total_len;
      if (p >= e) continue;
      const int64_t actual = e - s;
      const int64_t n = p - s;
      float w = 1.f;
      if (use_window) {
        // np.hanning(M)[n] = 0.5 - 0.5*cos(2*pi*n/(M-1)); np.hanning(1) = [1.]
        w = (actual > 1) ? (float)(0.5 - 0.5 * cospi(2.0 * (double)n / (double)(actual - 1))) : 1.f;
      }
      const float* y = chunks + (int64_t)(i - first_chunk) * 2 * chunk_len;  // chunks[0] is global chunk `first_chunk`
      res[0] += __ldg(&y[n]) * w;
      res[1] += __ldg(&y[chunk_len + n]) * w;
      div += w;
    }
#pragma unroll
    for (int c = 0; c < 2; ++c) {
      const float v = __fmul_rn(res[c] / div, out_scale);
      const int64_t o = interleave ? ((q - out_base) * 2 + c) : ((int64_t)c * out_ld + (q - out_base));
      primary[o] = v;
      if (mix != nullptr) secondary[o] = __fadd_rn(__fmul_rn(-v, compensate), __ldg(&mix[(int64_t)c * mix_ld + (q - mix_base)]));
    }
  }
}

// MDX23C accumulation (mdxc_separator.py:395-402): rectangular overlap-add of full-length chunks placed every `hop`,
// slice [front, front + n_out), divide by the constant `overlap`.  chunks: (n_chunks, C, chunk); out: (C, n_out).
__global__ void rect_ola_kernel(const float* __restrict__ chunks, int first_chunk, int n_chunks, int C, int chunk_len, int64_t hop, int64_t front, int64_t n_out,
                                int64_t q_begin, int64_t q_end, float divisor, float* __restrict__ out, int64_t out_ld, int64_t out_base) {
  const int c = blockIdx.y;
  for (int64_t q = q_begin + (int64_t)blockIdx.x * blockDim.x + threadIdx.x; q < q_end; q += (int64_t)gridDim.x * blockDim.x) {
    const int64_t p = q + front;
    int64_t i_hi = p / hop;
    if (i_hi > n_chunks - 1) i_hi = n_chunks - 1;
    int64_t i_lo = (p - chunk_len + 1 <= 0) ? 0 : (p - chunk_len + hop) / hop;
    float acc = 0.f;
    for (int64_t i = i_lo; i <= i_hi; ++i) acc += __ldg(&chunks[((int64_t)(i - first_chunk) * C + c) * chunk_len + (p - i * hop)]);  // chunks[0] is global chunk `first_chunk`
    out[(int64_t)c * out_ld + (q - out_base)] = acc / divisor;
  }
}

__global__ void absmax_kernel(const float* __restrict__ x, int64_t n, unsigned int* result_bits) {
  float m = 0.f;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) m = fmaxf(m, fabsf(x[i]));
  for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
  if ((threadIdx.x & 31) == 0) atomicMax(result_bits, __float_as_uint(m));  // non-negative floats order like uints
}

__global__ void normalize_kernel(const float* __restrict__ x, int64_t n, const float* __restrict__ absmax, float max_peak, float min_peak,
                                 float* __restrict__ y) {
  const float mv = *absmax;
  float s = 1.f;
  if (mv > max_peak) s = max_peak / mv;
  else if (min_peak >= 0.f && mv < min_peak) s = min_peak / mv;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) y[i] = x[i] * s;
}

__global__ void pcm16_kernel(const float* __restrict__ x, int64_t n, int16_t* __restrict__ y) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    float v = __fmul_rn(x[i], 32767.f);
    y[i] = (int16_t)(int)v;  // truncation toward zero, like ndarray.astype(np.int16) for in-range values
  }
}

// PCM bytes (little endian) at the input file's bit depth; the quantisation rules are pcm_quantize's (pcm.cuh).
__global__ void pcm_bytes_kernel(const float* __restrict__ x, int64_t n, int bits, int via_int16, uint8_t* __restrict__ y) {
  const int width = bits >> 3;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const int v = pcm_quantize(x[i], bits, via_int16);
    uint8_t* o = y + i * width;
    for (int b = 0; b < width; ++b) o[b] = (uint8_t)((unsigned)v >> (8 * b));
  }
}

static int factor_fft(int n, FftStages* st) {
  st->n = n;
  st->n_stages = 0;
  int m = n;
  const int radices[5] = {8, 4, 2, 3, 5};
  for (int ri = 0; ri < 5; ++ri) {
    const int r = radices[ri];
    while (m % r == 0 && m > 1) {
      if (st->n_stages >= kMaxStages) return -1;
      st->radix[st->n_stages++] = r;
      m /= r;
    }
  }
  return m == 1 ? 0 : -1;
}

static int fft_smem_bytes(int n) { return 2 * n * (int)sizeof(float2); }

}  // namespace b200sep

using namespace b200sep;

extern "C" int b200sep_stft_plan_create(b200sep_stft_plan** plan, int n_fft, int hop) {
  B2_CHECK_ARG(plan != nullptr, "stft_plan_create: plan is NULL");
  B2_CHECK_ARG(n_fft >= 8 && hop >= 1 && hop <= n_fft, "stft_plan_create: bad n_fft=%d hop=%d", n_fft, hop);
  FftStages st;
  B2_CHECK_ARG(factor_fft(n_fft, &st) == 0, "stft_plan_create: n_fft=%d does not factor into {2,3,5}", n_fft);
  B2_CHECK_ARG(fft_smem_bytes(n_fft) <= 227 * 1024, "stft_plan_create: n_fft=%d needs more than 227 KB of shared memory", n_fft);
  std::vector<float2> tw(n_fft);
  std::vector<float> win(n_fft);
  for (int m = 0; m < n_fft; ++m) {
    const double a = -2.0 * M_PI * (double)m / (double)n_fft;
    tw[m] = make_float2((float)cos(a), (float)sin(a));
    win[m] = (float)(0.5 - 0.5 * cos(2.0 * M_PI * (double)m / (double)n_fft));  // torch.hann_window(periodic=True)
  }
  b200sep_stft_plan* p = new b200sep_stft_plan();
  p->n_fft = n_fft;
  p->hop = hop;
  p->st = st;
  p->twiddle = nullptr;
  p->window = nullptr;
  cudaError_t e = cudaMalloc(&p->twiddle, sizeof(float2) * n_fft);
  if (e == cudaSuccess) e = cudaMalloc(&p->window, sizeof(float) * n_fft);
  if (e == cudaSuccess) e = cudaMemcpy(p->twiddle, tw.data(), sizeof(float2) * n_fft, cudaMemcpyHostToDevice);
  if (e == cudaSuccess) e = cudaMemcpy(p->window, win.data(), sizeof(float) * n_fft, cudaMemcpyHostToDevice);
  if (e == cudaSuccess) e = cudaFuncSetAttribute(stft_forward_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024);
  if (e == cudaSuccess) e = cudaFuncSetAttribute(istft_frames_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024);
  if (e != cudaSuccess) {
    set_error("stft_plan_create: %s", cudaGetErrorString(e));
    b200sep_stft_plan_destroy(p);
    return B200SEP_ERR_CUDA;
  }
  *plan = p;
  return B200SEP_OK;
}

extern "C" void b200sep_stft_plan_destroy(b200sep_stft_plan* p) {
  if (!p) return;
  if (p->twiddle) cudaFree(p->twiddle);
  if (p->window) cudaFree(p->window);
  delete p;
}

extern "C" int b200sep_stft_forward(const b200sep_stft_plan* plan, const float* wave, int64_t batch_stride, int64_t chan_stride,
                                    int64_t valid_len, int batch, int chunk_len, int dim_f, int zero_bins, int layout, float* spec,
                                    void* stream) {
  B2_CHECK_ARG(plan && wave && spec, "stft_forward: NULL argument");
  B2_CHECK_ARG(batch >= 0 && chunk_len > 0, "stft_forward: chunk_len=%d must be positive", chunk_len);
  B2_CHECK_ARG(chunk_len > plan->n_fft / 2, "stft_forward: reflect padding needs chunk_len=%d > n_fft/2=%d", chunk_len, plan->n_fft / 2);
  B2_CHECK_ARG(dim_f >= 1 && dim_f <= plan->n_fft / 2 + 1, "stft_forward: dim_f=%d out of range", dim_f);
  B2_CHECK_ARG(layout == B200SEP_LAYOUT_CFT || layout == B200SEP_LAYOUT_CTF, "stft_forward: bad layout %d", layout);
  if (batch == 0) return B200SEP_OK;
  const int frames = chunk_len / plan->hop + 1;
  dim3 grid(frames, batch);
  stft_forward_kernel<<<grid, kFftThreads, fft_smem_bytes(plan->n_fft), (cudaStream_t)stream>>>(
      plan->st, plan->twiddle, plan->window, wave, batch_stride, chan_stride, valid_len, plan->hop, chunk_len, frames, dim_f, zero_bins,
      layout, spec, plan->n_fft / 2, 1.0f, 0);
  B2_LAUNCHED();
  return B200SEP_OK;
}

// Generalised framing: frame t covers samples [t*hop - frame_offset, +n_fft) of the chunk (reflected at its ends), `frames` is given
// explicitly and every bin is multiplied by `scale`.  HTDemucs._spec (demucs/htdemucs.py:383-403, spec.py:11-22: normalized=True,
// reflect pad 3*hop/2, frames 2..2+le kept, last bin dropped) is frame_offset = 3*hop/2, frames = ceil(T/hop), scale = n_fft^-1/2, dim_f = n_fft/2.
extern "C" int b200sep_stft_forward_ex(const b200sep_stft_plan* plan, const float* wave, int64_t batch_stride, int64_t chan_stride, int64_t valid_len,
                                       int batch, int chunk_len, int frames, int frame_offset, float scale, int dim_f, int zero_bins, int layout,
                                       int pad_mode, float* spec, void* stream) {
  B2_CHECK_ARG(plan && wave && spec, "stft_forward_ex: NULL argument");
  B2_CHECK_ARG(batch >= 0 && chunk_len > 0 && frames >= 1 && (pad_mode == 0 || pad_mode == 1), "stft_forward_ex: bad sizes");
  B2_CHECK_ARG(pad_mode == 1 || (frame_offset >= 0 && frame_offset < chunk_len && (frames - 1) * plan->hop - frame_offset + plan->n_fft - 1 <= 2 * (chunk_len - 1)),
               "stft_forward_ex: frames reach beyond a single reflection of the chunk");
  B2_CHECK_ARG(pad_mode == 0 || (frame_offset >= 0 && frame_offset <= plan->n_fft && (int64_t)(frames - 1) * plan->hop - frame_offset < chunk_len + plan->n_fft),
               "stft_forward_ex: zero-padded frames lie entirely outside the signal");
  B2_CHECK_ARG(dim_f >= 1 && dim_f <= plan->n_fft / 2 + 1, "stft_forward_ex: dim_f=%d out of range", dim_f);
  B2_CHECK_ARG(layout == B200SEP_LAYOUT_CFT || layout == B200SEP_LAYOUT_CTF, "stft_forward_ex: bad layout %d", layout);
  if (batch == 0) return B200SEP_OK;
  dim3 grid(frames, batch);
  stft_forward_kernel<<<grid, kFftThreads, fft_smem_bytes(plan->n_fft), (cudaStream_t)stream>>>(
      plan->st, plan->twiddle, plan->window, wave, batch_stride, chan_stride, valid_len, plan->hop, chunk_len, frames, dim_f, zero_bins, layout, spec,
      frame_offset, scale, pad_mode);
  B2_LAUNCHED();
  return B200SEP_OK;
}

extern "C" int64_t b200sep_stft_inverse_work_floats(const b200sep_stft_plan* plan, int batch, int frames, int dim_f, int layout) {
  (void)dim_f;
  (void)layout;
  if (!plan) return 0;
  return (int64_t)batch * 2 * frames * plan->n_fft;
}

extern "C" int b200sep_stft_inverse(const b200sep_stft_plan* plan, const float* spec, int batch, int frames, int dim_f, int layout,
                                    float* wave, float* work, void* stream) {
  B2_CHECK_ARG(plan && spec && wave && work, "stft_inverse: NULL argument");
  B2_CHECK_ARG(frames >= 2, "stft_inverse: frames=%d must be >= 2", frames);
  B2_CHECK_ARG(dim_f >= 1 && dim_f <= plan->n_fft / 2 + 1, "stft_inverse: dim_f=%d out of range", dim_f);
  B2_CHECK_ARG(layout == B200SEP_LAYOUT_CFT || layout == B200SEP_LAYOUT_CTF, "stft_inverse: bad layout %d", layout);
  if (batch == 0) return B200SEP_OK;
  dim3 grid(frames, batch);
  istft_frames_kernel<<<grid, kFftThreads, fft_smem_bytes(plan->n_fft), (cudaStream_t)stream>>>(plan->st, plan->twiddle, plan->window, spec,
                                                                                               frames, dim_f, layout, work, 1.0f);
  B2_LAUNCHED();
  const int out_len = plan->hop * (frames - 1);
  dim3 g2(cdiv(out_len, 256), batch * 2);
  istft_ola_kernel<<<g2, 256, 0, (cudaStream_t)stream>>>(work, plan->window, plan->n_fft, plan->hop, frames, out_len, wave, plan->n_fft / 2, 0);
  B2_LAUNCHED();
  return B200SEP_OK;
}

// Generalised inverse: out_len samples, sample n = overlap-add position n + ola_offset, `env_extra` virtual zero frames on each side in
// the window envelope, spectrum multiplied by `scale` first.  HTDemucs._ispec + ispectro (htdemucs.py:405-413, spec.py:25-38) is
// ola_offset = 3*hop/2, env_extra = 2, scale = sqrt(n_fft), out_len = segment length, dim_f = n_fft/2 (Nyquist bin zero).
extern "C" int b200sep_stft_inverse_ex(const b200sep_stft_plan* plan, const float* spec, int batch, int frames, int dim_f, int layout, int out_len,
                                       int ola_offset, int env_extra, float scale, float* wave, float* work, void* stream) {
  B2_CHECK_ARG(plan && spec && wave && work, "stft_inverse_ex: NULL argument");
  B2_CHECK_ARG(frames >= 1 && out_len >= 1 && ola_offset >= 0 && env_extra >= 0, "stft_inverse_ex: bad sizes");
  B2_CHECK_ARG(dim_f >= 1 && dim_f <= plan->n_fft / 2 + 1, "stft_inverse_ex: dim_f=%d out of range", dim_f);
  B2_CHECK_ARG(layout == B200SEP_LAYOUT_CFT || layout == B200SEP_LAYOUT_CTF, "stft_inverse_ex: bad layout %d", layout);
  if (batch == 0) return B200SEP_OK;
  dim3 grid(frames, batch);
  istft_frames_kernel<<<grid, kFftThreads, fft_smem_bytes(plan->n_fft), (cudaStream_t)stream>>>(plan->st, plan->twiddle, plan->window, spec, frames, dim_f,
                                                                                               layout, work, scale);
  B2_LAUNCHED();
  dim3 g2(cdiv(out_len, 256), batch * 2);
  istft_ola_kernel<<<g2, 256, 0, (cudaStream_t)stream>>>(work, plan->window, plan->n_fft, plan->hop, frames, out_len, wave, ola_offset, env_extra);
  B2_LAUNCHED();
  return B200SEP_OK;
}

extern "C" int b200sep_demix_overlap_add_range_ex(const float* chunks, int first_chunk, int n_local_chunks, int n_chunks, int chunk_len, int64_t step,
                                                  int64_t total_len, int64_t trim, int64_t n_out, int64_t q_begin, int64_t q_end, int use_window,
                                                  float out_scale, const float* mix, int64_t mix_ld, int64_t mix_base, float compensate, int interleave,
                                                  float* primary, float* secondary, int64_t out_base, void* stream) {
  B2_CHECK_ARG(chunks && primary, "demix_overlap_add_range: NULL argument");
  B2_CHECK_ARG(mix == nullptr || secondary != nullptr, "demix_overlap_add_range: mix given without a secondary buffer");
  B2_CHECK_ARG(n_chunks >= 1 && chunk_len >= 1 && step >= 1 && total_len >= 1 && trim >= 0 && n_out >= 0, "demix_overlap_add_range: bad sizes");
  B2_CHECK_ARG(trim + n_out <= total_len && 0 <= q_begin && q_begin <= q_end && q_end <= n_out, "demix_overlap_add_range: bad output range");
  B2_CHECK_ARG(out_base >= 0 && out_base <= q_begin && (mix == nullptr || (mix_base >= 0 && mix_base <= q_begin && q_end - mix_base <= mix_ld)),
               "demix_overlap_add_range: output / mix slices do not cover [%lld, %lld)", (long long)q_begin, (long long)q_end);
  B2_CHECK_ARG(interleave || out_base == 0, "demix_overlap_add_range: planar output slices are not supported");
  if (q_end == q_begin) return B200SEP_OK;
  // every chunk that covers [q_begin, q_end) must be present in the local buffer
  const int64_t p0 = q_begin + trim, p1 = q_end - 1 + trim;
  int64_t need_lo = (p0 - chunk_len + 1 <= 0) ? 0 : (p0 - chunk_len + step) / step;
  int64_t need_hi = std::min<int64_t>(p1 / step, n_chunks - 1);
  B2_CHECK_ARG(need_lo >= first_chunk && need_hi < (int64_t)first_chunk + n_local_chunks,
               "demix_overlap_add_range: outputs [%lld,%lld) need chunks [%lld,%lld] but the buffer holds [%d,%d)", (long long)q_begin, (long long)q_end,
               (long long)need_lo, (long long)need_hi, first_chunk, first_chunk + n_local_chunks);
  const int blocks = (int)std::min<int64_t>(cdiv(q_end - q_begin, 256), kNumSMs * 16);
  demix_ola_kernel<<<blocks, 256, 0, (cudaStream_t)stream>>>(chunks, first_chunk, n_chunks, chunk_len, step, total_len, trim, n_out, q_begin, q_end, use_window,
                                                             out_scale, mix, mix_ld, mix_base, compensate, interleave, primary, secondary, out_base, n_out);
  B2_LAUNCHED();
  return B200SEP_OK;
}

extern "C" int b200sep_demix_overlap_add_range(const float* chunks, int first_chunk, int n_local_chunks, int n_chunks, int chunk_len, int64_t step,
                                               int64_t total_len, int64_t trim, int64_t n_out, int64_t q_begin, int64_t q_end, int use_window,
                                               float out_scale, const float* mix, float compensate, int interleave, float* primary,
                                               float* secondary, void* stream) {
  return b200sep_demix_overlap_add_range_ex(chunks, first_chunk, n_local_chunks, n_chunks, chunk_len, step, total_len, trim, n_out, q_begin, q_end, use_window, out_scale,
                                            mix, n_out, 0, compensate, interleave, primary, secondary, 0, stream);
}

extern "C" int b200sep_demix_overlap_add(const float* chunks, int n_chunks, int chunk_len, int64_t step, int64_t total_len, int64_t trim,
                                         int64_t n_out, int use_window, float out_scale, const float* mix, float compensate,
                                         int interleave, float* primary, float* secondary, void* stream) {
  return b200sep_demix_overlap_add_range_ex(chunks, 0, n_chunks, n_chunks, chunk_len, step, total_len, trim, n_out, 0, n_out, use_window, out_scale, mix, n_out, 0,
                                            compensate, interleave, primary, secondary, 0, stream);
}

extern "C" int b200sep_rect_overlap_add_range(const float* chunks, int first_chunk, int n_local, int n_chunks, int channels, int chunk_len, int64_t hop, int64_t front,
                                              int64_t n_out, int64_t q_begin, int64_t q_end, float divisor, float* out, int64_t out_ld, int64_t out_base, void* stream) {
  B2_CHECK_ARG(chunks && out && n_chunks >= 1 && channels >= 1 && chunk_len >= 1 && hop >= 1 && front >= 0 && n_out >= 0 && divisor != 0.f,
               "rect_overlap_add: bad argument");
  B2_CHECK_ARG(front + n_out <= (int64_t)(n_chunks - 1) * hop + chunk_len, "rect_overlap_add: output range exceeds the chunk grid");
  B2_CHECK_ARG(0 <= q_begin && q_begin <= q_end && q_end <= n_out, "rect_overlap_add: bad output range");
  B2_CHECK_ARG(out_base >= 0 && out_base <= q_begin && q_end - out_base <= out_ld, "rect_overlap_add: output slice does not cover [%lld, %lld)", (long long)q_begin, (long long)q_end);
  if (q_end == q_begin) return B200SEP_OK;
  const int64_t p0 = q_begin + front, p1 = q_end - 1 + front;
  const int64_t need_lo = (p0 - chunk_len + 1 <= 0) ? 0 : (p0 - chunk_len + hop) / hop;
  const int64_t need_hi = std::min<int64_t>(p1 / hop, n_chunks - 1);
  B2_CHECK_ARG(need_lo >= first_chunk && need_hi < (int64_t)first_chunk + n_local, "rect_overlap_add: outputs [%lld,%lld) need chunks [%lld,%lld] but the buffer holds [%d,%d)",
               (long long)q_begin, (long long)q_end, (long long)need_lo, (long long)need_hi, first_chunk, first_chunk + n_local);
  dim3 grid((unsigned)std::min<int64_t>(cdiv(q_end - q_begin, 256), kNumSMs * 8), channels);
  rect_ola_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(chunks, first_chunk, n_chunks, channels, chunk_len, hop, front, n_out, q_begin, q_end, divisor, out, out_ld, out_base);
  B2_LAUNCHED();
  return B200SEP_OK;
}

extern "C" int b200sep_rect_overlap_add(const float* chunks, int n_chunks, int channels, int chunk_len, int64_t hop, int64_t front, int64_t n_out,
                                        float divisor, float* out, void* stream) {
  return b200sep_rect_overlap_add_range(chunks, 0, n_chunks, n_chunks, channels, chunk_len, hop, front, n_out, 0, n_out, divisor, out, n_out, 0, stream);
}

extern "C" int b200sep_absmax(const float* x, int64_t n, float* result, void* stream) {
  B2_CHECK_ARG(x && result && n >= 0, "absmax: bad argument");
  B2_CUDA(cudaMemsetAsync(result, 0, sizeof(float), (cudaStream_t)stream));
  if (n == 0) return B200SEP_OK;
  const int blocks = (int)std::min<int64_t>(cdiv(n, 1024), kNumSMs * 8);
  absmax_kernel<<<blocks, 256, 0, (cudaStream_t)stream>>>(x, n, reinterpret_cast<unsigned int*>(result));
  B2_LAUNCHED();
  return B200SEP_OK;
}

extern "C" int b200sep_normalize(const float* x, int64_t n, const float* absmax, float max_peak, float min_peak, float* y, void* stream) {
  B2_CHECK_ARG(x && y && absmax && n >= 0, "normalize: bad argument");
  if (n == 0) return B200SEP_OK;
  const int blocks = (int)std::min<int64_t>(cdiv(n, 1024), kNumSMs * 8);
  normalize_kernel<<<blocks, 256, 0, (cudaStream_t)stream>>>(x, n, absmax, max_peak, min_peak, y);
  B2_LAUNCHED();
  return B200SEP_OK;
}

extern "C" int b200sep_to_pcm_bytes(const float* x, int64_t n, int bits, int via_int16, uint8_t* y, void* stream) {
  B2_CHECK_ARG(x && y && n >= 0 && (bits == 16 || bits == 24 || bits == 32), "to_pcm_bytes: bits must be 16, 24 or 32");
  if (n == 0) return B200SEP_OK;
  const int blocks = (int)std::min<int64_t>(cdiv(n, 1024), kNumSMs * 8);
  pcm_bytes_kernel<<<blocks, 256, 0, (cudaStream_t)stream>>>(x, n, bits, via_int16, y);
  B2_LAUNCHED();
  return B200SEP_OK;
}

extern "C" int b200sep_to_pcm16(const float* x, int64_t n, int16_t* y, void* stream) {
  B2_CHECK_ARG(x && y && n >= 0, "to_pcm16: bad argument");
  if (n == 0) return B200SEP_OK;
  const int blocks = (int)std::min<int64_t>(cdiv(n, 1024), kNumSMs * 8);
  pcm16_kernel<<<blocks, 256, 0, (cudaStream_t)stream>>>(x, n, y);
  B2_LAUNCHED();
  return B200SEP_OK;
}
