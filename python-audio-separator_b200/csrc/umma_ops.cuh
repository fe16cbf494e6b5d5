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
// out[r][n] = act(acc*scale[c]+shift[c]) (+ res[r][n]),  c = (r / rows_per_channel) % channels;  rows >= M_active are not written
int umma_gemm_run(const UmmaGemmPlan& pl, const float* scale, const float* shift, int rows_per_channel, int channels, int relu, void* out_hi,
                  void* out_lo, const void* res_hi, const void* res_lo, int M_active, cudaStream_t st);

int umma_gemm_run_ex(const UmmaGemmPlan& pl, int rows_per_channel, int channels, int M_active, const UmmaEpilogue& e, cudaStream_t st);

bool umma_conv_supported(int Cin, int Cout, int F, int kh, int kw);
int umma_conv_choose(int Cin, int Cout, int* kc, int* n_c);
void umma_conv_block_weights(const float* w, int Cout, int Cin, int kc, int n_c, std::vector<uint16_t>& hi, std::vector<uint16_t>& lo);
// x: pair (Bmax, Cin, T, F)
int umma_conv_plan_create(UmmaConvPlan* pl, const void* x_hi, const void* x_lo, int Bmax, int Cin, int T, int F, int kc);
// weights pre-blocked by umma_conv_block_weights (hi plane, lo plane)
int umma_conv_run(const UmmaConvPlan& pl, const void* wb_hi, const void* wb_lo, int B, int Cout, int n_c, int ksize, const float* scale,
                  const float* shift, int relu, void* out_hi, void* out_lo, cudaStream_t st);

// ConvTranspose2d / Conv2d with 2x2 kernels and stride 2 (the U-Net's up / down sampling) on the same pipeline
bool umma_updown_supported(int Cin, int Cout, int F_in, int up);
int umma_updown_choose(int Cin, int Cout, int up, int* kc, int* n_c);
void umma_up_block_weights(const float* w /*(Cin,Cout,2,2)*/, int Cin, int Cout, int kc, int n_c, std::vector<uint16_t>& hi, std::vector<uint16_t>& lo);
void umma_down_block_weights(const float* w /*(Cout,Cin,2,2)*/, int Cout, int Cin, int kc, int n_c, std::vector<uint16_t>& hi, std::vector<uint16_t>& lo);
int umma_up_run(const UmmaConvPlan& pl, const void* wb_hi, const void* wb_lo, int B, int Cout, int n_c, const float* scale, const float* shift, int relu,
                const void* skip_hi, const void* skip_lo, void* out_hi, void* out_lo, cudaStream_t st);
int umma_down_run(const UmmaConvPlan& pl, const void* wb_hi, const void* wb_lo, int B, int Cout, int n_c, const float* scale, const float* shift, int relu,
                  void* out_hi, void* out_lo, cudaStream_t st);

int umma_conv_run_ex(const UmmaConvPlan& pl, const void* wb_hi, const void* wb_lo, int B, int Cout, int n_c, const UmmaEpilogue& e, cudaStream_t st);
int umma_up_run_ex(const UmmaConvPlan& pl, const void* wb_hi, const void* wb_lo, int B, int Cout, int n_c, const UmmaEpilogue& e, cudaStream_t st);
int umma_down_run_ex(const UmmaConvPlan& pl, const void* wb_hi, const void* wb_lo, int B, int Cout, int n_c, const UmmaEpilogue& e, cudaStream_t st);
// 1x1 convolution on the same pipeline
bool umma_pw_supported(int Cin, int Cout, int F);
int umma_pw_choose(int Cin, int Cout, int* kc, int* n_c);
void umma_pw_block_weights(const float* w /*(Cout,Cin)*/, int Cout, int Cin, int kc, int n_c, std::vector<uint16_t>& hi, std::vector<uint16_t>& lo);
int umma_pw_run_ex(const UmmaConvPlan& pl, const void* wb_hi, const void* wb_lo, int B, int Cout, int n_c, const UmmaEpilogue& e, cudaStream_t st);

int split_pair(const float* x, void* hi, void* lo, int64_t n, cudaStream_t st);
int join_pair(const void* hi, const void* lo, float* y, int64_t n, cudaStream_t st);

}  // namespace b200sep
