// Host interface of the wgmma "pair" operators (umma_ops.cu).
#pragma once
#include <cuda.h>
#include <stdint.h>

#include <vector>

#include "common.cuh"

namespace b200sep {

struct UmmaGemmPlan {
  CUtensorMap a_hi, a_lo, b_hi, b_lo;
  int M, N, K, n_tile;
};
struct UmmaConvPlan {
  CUtensorMap a_hi, a_lo;
  int Cin, T, F, kc;
};

// Epilogue of every mode: y = act(acc * scale[c] + shift[c]); then y += res (GEMM, CONV3x3, PW) or y *= res (UP: skip tensor);
// then y *= mul (CONV3x3, PW); stored as a pair (or plain fp32 when out_f32 is set, PW only) into channels
// [out_c_off, out_c_off + Cout) of a tensor with out_c_total channels (0 = exactly Cout).
struct UmmaEpilogue {
  const float* scale = nullptr;  // nullptr = 1
  const float* shift = nullptr;  // nullptr = 0
  int act = 0;                   // 0 none, 1 ReLU, 2 GELU (erf form)
  const void* res_hi = nullptr;
  const void* res_lo = nullptr;
  const void* mul_hi = nullptr;
  const void* mul_lo = nullptr;
  void* out_hi = nullptr;
  void* out_lo = nullptr;
  float* out_f32 = nullptr;
  int out_c_total = 0, out_c_off = 0;
};

bool umma_gemm_supported(int M, int N, int K);
// A: pair [M][K] (K contiguous), W: pair [N][K].  Tensor maps are bound to these addresses.
int umma_gemm_plan_create(UmmaGemmPlan* pl, const void* a_hi, const void* a_lo, const void* w_hi, const void* w_lo, int M, int N, int K);
// hi / lo planes of a GEMM weight [N][K] (the W operand of umma_gemm_plan_create)
void umma_gemm_split_weights(const float* w, int N, int K, std::vector<uint16_t>& hi, std::vector<uint16_t>& lo);
// out[r][n] = act(acc*scale[c]+shift[c]) (+ res[r][n]),  c = (r / rows_per_channel) % channels;  rows >= M_active are not written
int umma_gemm_run(const UmmaGemmPlan& pl, int rows_per_channel, int channels, int M_active, const UmmaEpilogue& e, cudaStream_t st);

// Convolutions on the same pipeline: 3x3 stride 1; ConvTranspose2d / Conv2d with 2x2 kernels and stride 2 (the U-Nets' up / down sampling); 1x1.
enum UmmaConvKind { UMMA_CONV3, UMMA_UP, UMMA_DOWN, UMMA_PW };
// input checks: shapes that fail them run on the SIMT pair kernels (or are rejected by the caller)
bool umma_conv_supported(int Cin, int Cout, int F, int kh, int kw);
bool umma_updown_supported(int Cin, int Cout, int F_in, int up);
bool umma_pw_supported(int Cin, int Cout, int F);
// output channels per CTA: a property of the blocked weights
int umma_n_c(UmmaConvKind kind, int Cout);
// input channels per pipeline stage: a property of the plan
int umma_kc(UmmaConvKind kind, int Cin, int Cout);
// Blocks fp32 weights -- (Cout, Cin, kh, kw); UP: ConvTranspose2d (Cin, Cout, 2, 2) -- into the hi / lo weight planes of the run functions.
// Returns n_c = umma_n_c(kind, Cout).
int umma_block_weights(UmmaConvKind kind, const float* w, int Cin, int Cout, std::vector<uint16_t>& hi, std::vector<uint16_t>& lo);
// x: pair (Bmax, Cin, T, F); the plan's kc is umma_kc(kind, Cin, Cout)
int umma_conv_plan_create(UmmaConvPlan* pl, UmmaConvKind kind, const void* x_hi, const void* x_lo, int Bmax, int Cin, int Cout, int T, int F);
// x: the plan's input, B <= Bmax; wb_hi / wb_lo: the planes of umma_block_weights
int umma_conv_run(const UmmaConvPlan& pl, const void* wb_hi, const void* wb_lo, int B, int Cout, int n_c, const UmmaEpilogue& e, cudaStream_t st);
int umma_up_run(const UmmaConvPlan& pl, const void* wb_hi, const void* wb_lo, int B, int Cout, int n_c, const UmmaEpilogue& e, cudaStream_t st);
int umma_down_run(const UmmaConvPlan& pl, const void* wb_hi, const void* wb_lo, int B, int Cout, int n_c, const UmmaEpilogue& e, cudaStream_t st);
int umma_pw_run(const UmmaConvPlan& pl, const void* wb_hi, const void* wb_lo, int B, int Cout, int n_c, const UmmaEpilogue& e, cudaStream_t st);

int split_pair(const float* x, void* hi, void* lo, int64_t n, cudaStream_t st);
int join_pair(const void* hi, const void* lo, float* y, int64_t n, cudaStream_t st);

}  // namespace b200sep
