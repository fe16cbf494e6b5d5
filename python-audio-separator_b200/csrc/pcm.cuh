// Float -> integer PCM quantisation of the output writers, shared by the WAV byte packer (stft.cu) and the FLAC encoder (flac.cu)
// so both formats store the same samples.
#pragma once
#include <stdint.h>

namespace b200sep {

// One normalised float sample at the input file's bit depth (common_separator.py:322-383).  via_int16 = the pydub writer: the sample is
// quantised to int16 first ((x * 32767).astype(int16)) and ffmpeg widens it (s16 -> s32 = << 16; pcm_s24le keeps the top three bytes).
// Otherwise the libsndfile writer: lrint(x * (2^(bits-1) - 1)) (PCM_32 scales by 2^31 and saturates).  The result holds `bits` significant
// bits (the low bits of a widened pydub sample are zero).
__device__ __forceinline__ int pcm_quantize(float x, int bits, int via_int16) {
  if (via_int16) {
    const int v = (int)(int16_t)(int)__fmul_rn(x, 32767.f);
    return (int)((unsigned)v << (bits - 16));
  }
  if (bits == 32) {
    const double d = rint((double)x * 2147483648.0);
    return d >= 2147483647.0 ? 2147483647 : (d <= -2147483648.0 ? (int)0x80000000 : (int)d);
  }
  return (int)rintf(__fmul_rn(x, (float)((1 << (bits - 1)) - 1)));
}

}  // namespace b200sep
