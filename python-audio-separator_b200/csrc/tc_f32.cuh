// Host interface of the fp32-in / fp32-out tensor-core GEMM + implicit-GEMM convolution (tc_f32.cu).  `math` is B200SEP_MATH_BF16X3 (the
// three-product bf16 hi / lo split) or B200SEP_MATH_FP16 (operands rounded once to fp16, one product).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace b200sep {

// the *_usable predicates pick the tensor-core kernels by shape; smaller or unsupported shapes run on the SIMT kernels
bool tc_gemm_usable(int M, int N, int K, int batch);
int tc_gemm_f32(const float* A, const float* Bw, float* C, int M, int N, int K, int lda, int ldb, int ldc, int batch, int64_t sA, int64_t sB, int64_t sC, float alpha,
                const float* bias_n, const float* bias_m, int act, const float* res, const float* res_scale, const void* w_packed, int b_is_kn, int math,
                cudaStream_t st);
bool tc_conv_usable(int Cin, int Cout, int KH, int KW, int Ho, int Wo, int B);
int tc_conv2d_f32(const float* x, const float* w_blocked, const float* bias, const float* add, float* y, int B, int Cin, int H, int W, int Cout, int CoutPad, int Ho,
                  int Wo, int KH, int KW, int SH, int SW, int PH, int PW, int DH, int DW, int act, int add_before_act, int out_c_total, int out_c_off, const void* w_packed,
                  int math, cudaStream_t st, int up_axis = 0, int up = 1, int trim = 0, int out_len = 0);
// fused attention, head dimension 64: out = softmax(alpha q k^T) v with vt = v transposed (keys contiguous); strides in floats (see tc_f32.cu)
int tc_attention_f32(const float* q, const float* k, const float* vt, float* out, int B, int H, int Lq, int Lk, int64_t q_bs, int64_t q_rs, int64_t k_bs, int64_t k_rs,
                     int64_t vt_bs, int64_t vt_rs, int64_t o_bs, int64_t o_rs, float alpha, int v_kn, void* work, int math, cudaStream_t st);
int64_t tc_attention_work_bytes(int B, int H, int Lq, int Lk, int math);
// static B operands (weights) pre-split into the kernel's shared-memory image; K = the kernel's K (convolution: ceil8(Cin) * taps)
int64_t tc_packed_bytes(int N, int K, int math);
int tc_pack_linear(const float* W, int N, int K, int ldw, void* packed, int math, cudaStream_t st);
int tc_pack_conv(const float* w_blocked, int Cin, int taps, int Cout, int CoutPad, void* packed, int math, cudaStream_t st);
// false when `packed` was last written by tc_pack_* for the other math mode (unknown addresses pass)
bool tc_packed_matches(const void* packed, int math);

}  // namespace b200sep
