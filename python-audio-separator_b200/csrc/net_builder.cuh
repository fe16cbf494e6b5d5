// Host helpers of the network builders (mdx_net.cu, tfc_net.cu): reading the flat parameter blob, owning the device allocations and
// preparing a layer's weights for the pair pipeline (umma_ops.cuh).
#pragma once
#include <stdint.h>

#include <vector>

#include "common.cuh"
#include "umma_ops.cuh"

namespace b200sep {

struct ParamReader {
  const float* p;
  int64_t n, pos = 0;
  bool ok = true;
  const float* take(int64_t count) {
    if (pos + count > n) {
      ok = false;
      return p;  // caller checks ok
    }
    const float* r = p + pos;
    pos += count;
    return r;
  }
};

struct DeviceAllocs {  // every allocation of one network handle; freed together by free_all()
  std::vector<void*> ptrs;
  int64_t bytes = 0;
  int alloc(void** ptr, int64_t n_bytes) {
    B2_CUDA(cudaMalloc(ptr, (size_t)n_bytes));
    ptrs.push_back(*ptr);
    bytes += n_bytes;
    return B200SEP_OK;
  }
  int upload_f32(float** dst, const float* src, int64_t n) {
    int rc = alloc((void**)dst, n * 4);
    if (rc) return rc;
    B2_CUDA(cudaMemcpy(*dst, src, n * 4, cudaMemcpyHostToDevice));
    return B200SEP_OK;
  }
  int upload_u16(void** dst, const std::vector<uint16_t>& src) {
    int rc = alloc(dst, (int64_t)src.size() * 2);
    if (rc) return rc;
    B2_CUDA(cudaMemcpy(*dst, src.data(), src.size() * 2, cudaMemcpyHostToDevice));
    return B200SEP_OK;
  }
  void free_all() {
    for (void* p : ptrs) cudaFree(p);
    ptrs.clear();
  }
};

struct PairWeights {  // a layer's weights on the pair pipeline: hi / lo planes
  void* hi = nullptr;
  void* lo = nullptr;
  int n_c = 0;  // convolutions: output channels per CTA
};

// convolution weights (layouts at umma_block_weights); the caller has checked the umma_*_supported predicate of the layer
inline int upload_pair_conv(DeviceAllocs& mem, UmmaConvKind kind, const float* w, int cin, int cout, PairWeights& pw) {
  std::vector<uint16_t> hi, lo;
  pw.n_c = umma_block_weights(kind, w, cin, cout, hi, lo);
  int rc = mem.upload_u16(&pw.hi, hi);
  if (!rc) rc = mem.upload_u16(&pw.lo, lo);
  return rc;
}

// linear weight [n][k]
inline int upload_pair_linear(DeviceAllocs& mem, const float* w, int n, int k, PairWeights& pw) {
  std::vector<uint16_t> hi, lo;
  umma_gemm_split_weights(w, n, k, hi, lo);
  int rc = mem.upload_u16(&pw.hi, hi);
  if (!rc) rc = mem.upload_u16(&pw.lo, lo);
  return rc;
}

}  // namespace b200sep
