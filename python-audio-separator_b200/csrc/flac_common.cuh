// Pieces of FLAC (RFC 9639) shared by the encoder (flac.cu) and the decoder (flac_decode.cu): the header CRC-8, the CRC-16 table entry and the
// GF(2) arithmetic that moves a partial CRC-16 past later bytes, so that the CRC of a long span is a combination of the CRCs of its pieces.
#pragma once
#include <stdint.h>

namespace b200sep {
namespace flac {

__device__ __forceinline__ uint8_t crc8(const uint8_t* p, int n) {
  unsigned c = 0;
  for (int i = 0; i < n; ++i) {
    c ^= p[i];
    for (int b = 0; b < 8; ++b) c = (c & 0x80) ? ((c << 1) ^ 0x07) : (c << 1);
    c &= 0xFF;
  }
  return (uint8_t)c;
}

// Entry i of the byte-wise CRC-16 table (polynomial x^16 + x^15 + x^2 + 1, initial value 0, no reflection).
__device__ __forceinline__ uint16_t crc16_table_entry(unsigned i) {
  unsigned c = i << 8;
  for (int b = 0; b < 8; ++b) c = (c & 0x8000u) ? ((c << 1) ^ 0x8005u) : (c << 1);
  return (uint16_t)c;
}

__device__ __forceinline__ unsigned gf2_mulmod16(unsigned a, unsigned b) {  // a * b mod x^16 + x^15 + x^2 + 1
  unsigned r = 0;
  for (int i = 15; i >= 0; --i) {
    r <<= 1;
    if (r & 0x10000u) r ^= 0x18005u;
    if ((b >> i) & 1u) r ^= a;
  }
  return r;
}

// x^(8n) mod the CRC-16 polynomial: CRC16(A || B) = gf2_mulmod16(CRC16(A), x8_pow_mod16(|B|)) ^ CRC16(B).
__device__ __forceinline__ unsigned x8_pow_mod16(unsigned long long n) {
  unsigned r = 1, b = 0x100;
  for (; n; n >>= 1) {
    if (n & 1u) r = gf2_mulmod16(r, b);
    b = gf2_mulmod16(b, b);
  }
  return r;
}

// Sample rates of the frame-header codes 1-11 (0 = from STREAMINFO, 12-14 = explicit, 15 = invalid).
__device__ __forceinline__ int header_rate(int code) {
  constexpr int kRates[12] = {0, 88200, 176400, 192000, 8000, 16000, 22050, 24000, 32000, 44100, 48000, 96000};
  return code < 12 ? kRates[code] : -1;
}
// Sample sizes of the frame-header codes (0 = from STREAMINFO, 3 = reserved).
__device__ __forceinline__ int header_bps(int code) {
  constexpr int kBps[8] = {0, 8, 12, -1, 16, 20, 24, 32};
  return kBps[code & 7];
}

}  // namespace flac
}  // namespace b200sep
