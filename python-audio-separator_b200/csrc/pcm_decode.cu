// Uncompressed PCM decoder (WAV, RF64, AIFF / AIFF-C payloads), sm_90a: the interleaved sample bytes of a data / SSND chunk in HBM -> the planar
// float mix prepare_mix returns, converted as libsndfile's sf_read_float with normalisation on (what librosa.load returns).
//   pcm_decode_kernel<F>  one CTA per tile of frames: the tile's bytes (16-byte aligned around it) are staged in shared memory with 16-byte loads,
//                         then each thread assembles whole samples from the staged bytes and writes rows.  Reads stay coalesced whatever the sample
//                         width (3-byte samples) or frame size (6 channels, padded block aligns); writes are coalesced per output row.
// One launch, no host synchronisation; the empty-file check and the mono duplication are the caller's (b200sep_absmax, CommonSeparator._device_mix).
#include "common.cuh"

namespace b200sep {
namespace {

constexpr int kThreads = 256;
constexpr int kMaxTileFrames = 1024;
constexpr int kTileBytes = 32 * 1024;  // staged bytes per CTA: several CTAs per SM keep enough loads in flight
constexpr int kMaxFrameBytes = 65535;  // WAV's nBlockAlign is 16 bits wide

__host__ __device__ constexpr int sample_bytes(int f) { return f <= B200SEP_PCM_S8 ? 1 : f <= B200SEP_PCM_S16BE ? 2 : f <= B200SEP_PCM_S24BE ? 3 : f <= B200SEP_PCM_F32BE ? 4 : 8; }
__host__ __device__ constexpr bool big_endian(int f) { return f >= B200SEP_PCM_S16LE && (f & 1); }

int tile_frames(int frame_bytes) {
  const int t = kTileBytes / frame_bytes;
  return t < 1 ? 1 : t > kMaxTileFrames ? kMaxTileFrames : t;
}

int64_t staged_bytes(int frame_bytes) { return (((int64_t)tile_frames(frame_bytes) * frame_bytes + 15) & ~15ll) + 16; }

template <int F>
__device__ __forceinline__ float to_float(const uint8_t* p) {
  constexpr int B = sample_bytes(F);
  if constexpr (B == 8) {
    unsigned lo = 0, hi = 0;
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      lo |= (unsigned)p[big_endian(F) ? 7 - i : i] << (8 * i);
      hi |= (unsigned)p[big_endian(F) ? 3 - i : 4 + i] << (8 * i);
    }
    const double d = __hiloint2double((int)hi, (int)lo);
    if (d != d)  // a NaN keeps its sign and the top of its payload, quiet bit set (the host's cvtsd2ss / fcvt)
      return __uint_as_float((hi & 0x80000000u) | 0x7FC00000u | (__funnelshift_r(lo, hi, 29) & 0x7FFFFFu));
    return __double2float_rn(d);
  } else {
    unsigned u = 0;
#pragma unroll
    for (int i = 0; i < B; ++i) u |= (unsigned)p[i] << (8 * (big_endian(F) ? B - 1 - i : i));
    if constexpr (F == B200SEP_PCM_U8) {
      return (float)((int)u - 128) * 0x1p-7f;
    } else if constexpr (F == B200SEP_PCM_F32LE || F == B200SEP_PCM_F32BE) {
      return __uint_as_float(u);
    } else {
      constexpr int kShift = 32 - 8 * B;
      constexpr float kScale = 1.0f / (float)(1u << (8 * B - 1));
      return __int2float_rn((int)(u << kShift) >> kShift) * kScale;  // one rounding (32 bits), then an exact power-of-two scale
    }
  }
}

template <int F>
__global__ void __launch_bounds__(kThreads) pcm_decode_kernel(const uint8_t* __restrict__ data, int64_t n_frames, int frame_bytes, int tile,
                                                              int out_channels, float* __restrict__ out, int64_t out_ld) {
  extern __shared__ uint4 staged[];
  const int64_t f0 = (int64_t)blockIdx.x * tile;
  const int n = (int)min((int64_t)tile, n_frames - f0);
  const int64_t begin = f0 * frame_bytes, a0 = begin & ~15ll;
  const int64_t a1 = (begin + (int64_t)n * frame_bytes + 15) & ~15ll;  // within the buffer: it is readable up to the payload rounded up to 16
  const uint4* src = reinterpret_cast<const uint4*>(data + a0);
  const int words = (int)((a1 - a0) >> 4);
  for (int i = threadIdx.x; i < words; i += kThreads) staged[i] = __ldcs(src + i);
  __syncthreads();
  const uint8_t* s = reinterpret_cast<const uint8_t*>(staged) + (begin - a0);
  for (int c = 0; c < out_channels; ++c) {
    float* row = out + c * out_ld + f0;
#pragma unroll 2
    for (int i = threadIdx.x; i < n; i += kThreads) row[i] = to_float<F>(s + i * frame_bytes + c * sample_bytes(F));
  }
}

template <int F>
int launch(const uint8_t* data, int64_t n_frames, int frame_bytes, int out_channels, float* out, int64_t out_ld, cudaStream_t st) {
  const int tile = tile_frames(frame_bytes);
  const int smem = (int)staged_bytes(frame_bytes);
  B2_CUDA(cudaFuncSetAttribute(pcm_decode_kernel<F>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
  pcm_decode_kernel<F><<<(unsigned)((n_frames + tile - 1) / tile), kThreads, smem, st>>>(data, n_frames, frame_bytes, tile, out_channels, out, out_ld);
  B2_LAUNCHED();
  return B200SEP_OK;
}

}  // namespace
}  // namespace b200sep

using namespace b200sep;

extern "C" int b200sep_pcm_decode_f32(const uint8_t* data, int64_t n_frames, int frame_bytes, int channels, int format, int out_channels, float* out,
                                      int64_t out_ld, void* stream) {
  B2_CHECK_ARG(format >= B200SEP_PCM_U8 && format <= B200SEP_PCM_F64BE, "pcm_decode: unknown sample format %d", format);
  B2_CHECK_ARG(n_frames >= 0 && (n_frames == 0 || (data && out)) && channels >= 1 && out_channels >= 1 && out_channels <= channels,
               "pcm_decode: bad argument");
  B2_CHECK_ARG((int64_t)channels * sample_bytes(format) <= frame_bytes && frame_bytes <= kMaxFrameBytes,
               "pcm_decode: %d-byte frames cannot hold %d channels of %d bytes (or exceed %d bytes)", frame_bytes, channels, sample_bytes(format),
               kMaxFrameBytes);
  B2_CHECK_ARG(out_channels == 1 || out_ld >= n_frames, "pcm_decode: out_ld %lld below the %lld frames", (long long)out_ld, (long long)n_frames);
  B2_CHECK_ARG(((uintptr_t)data & 15) == 0 && ((uintptr_t)out & 3) == 0, "pcm_decode: data must be 16-byte aligned, out 4-byte aligned");
  B2_CHECK_ARG((n_frames + tile_frames(frame_bytes) - 1) / tile_frames(frame_bytes) < (1ll << 31), "pcm_decode: %lld frames are too many",
               (long long)n_frames);
  if (n_frames == 0) return B200SEP_OK;
  cudaStream_t st = (cudaStream_t)stream;
  switch (format) {
    case B200SEP_PCM_U8: return launch<B200SEP_PCM_U8>(data, n_frames, frame_bytes, out_channels, out, out_ld, st);
    case B200SEP_PCM_S8: return launch<B200SEP_PCM_S8>(data, n_frames, frame_bytes, out_channels, out, out_ld, st);
    case B200SEP_PCM_S16LE: return launch<B200SEP_PCM_S16LE>(data, n_frames, frame_bytes, out_channels, out, out_ld, st);
    case B200SEP_PCM_S16BE: return launch<B200SEP_PCM_S16BE>(data, n_frames, frame_bytes, out_channels, out, out_ld, st);
    case B200SEP_PCM_S24LE: return launch<B200SEP_PCM_S24LE>(data, n_frames, frame_bytes, out_channels, out, out_ld, st);
    case B200SEP_PCM_S24BE: return launch<B200SEP_PCM_S24BE>(data, n_frames, frame_bytes, out_channels, out, out_ld, st);
    case B200SEP_PCM_S32LE: return launch<B200SEP_PCM_S32LE>(data, n_frames, frame_bytes, out_channels, out, out_ld, st);
    case B200SEP_PCM_S32BE: return launch<B200SEP_PCM_S32BE>(data, n_frames, frame_bytes, out_channels, out, out_ld, st);
    case B200SEP_PCM_F32LE: return launch<B200SEP_PCM_F32LE>(data, n_frames, frame_bytes, out_channels, out, out_ld, st);
    case B200SEP_PCM_F32BE: return launch<B200SEP_PCM_F32BE>(data, n_frames, frame_bytes, out_channels, out, out_ld, st);
    case B200SEP_PCM_F64LE: return launch<B200SEP_PCM_F64LE>(data, n_frames, frame_bytes, out_channels, out, out_ld, st);
    default: return launch<B200SEP_PCM_F64BE>(data, n_frames, frame_bytes, out_channels, out, out_ld, st);
  }
}
