// Generic fp32 convolution operator (NCHW, W innermost) for the Demucs / VR style networks: arbitrary small kernels,
// strides, dilation along W, zero padding, fused bias + activation + residual add, and a "transposed" scatter epilogue.
// Register-tiled implicit GEMM on CUDA cores (block = 128 w x 2 h x 48 output channels, thread = 4 w x 12 channels,
// input channels staged 8 at a time through shared memory) -- the same scheme as conv2d_simt_kernel, generalised.
// Exact fp32 semantics; the tensor-core ("pair") path covers the shapes in umma_ops.cu.
#include <algorithm>

#include "common.cuh"
#include "tc_f32.cuh"

namespace b200sep {

constexpr int GTW = 128, GTH = 2, GTCO = 48, GCI = 8, GNT = 256;

struct ConvGenParams {
  const float* x;     // (B, Cin, H, W)
  const float* w;     // [Cin][KH*KW][CoutPad]  (CoutPad multiple of 48)
  const float* bias;  // [Cout] or nullptr
  const float* add;   // output-shaped tensor added before / after the activation, or nullptr
  float* y;
  int B, Cin, H, W, Cout, CoutPad, Ho, Wo;
  int PH, PW;         // zero padding (top / left); bottom / right are implied by Ho, Wo
  int act;            // 0 none, 1 ReLU, 2 GELU(erf), 3 LeakyReLU(0.01), 4 sigmoid -- applied after bias (+ add when add_before_act)
  int add_before_act;
  // transposed-convolution scatter: GEMM column co' = r * CoutReal + co; output index along the strided axis = q * up + r - trim,
  // kept when 0 <= index < out_len.  up_axis: 0 = none, 1 = H, 2 = W.
  int up_axis, up, trim, out_len, CoutReal;
  int OutCT, OutCOff;  // the output tensor has OutCT channels and this convolution fills [OutCOff, OutCOff + Cout) (torch.cat fused away)
};

__device__ __forceinline__ float gen_act(float v, int act) {
  if (act == 1) return fmaxf(v, 0.f);
  if (act == 2) return 0.5f * v * (1.f + erff(v * 0.70710678118654752440f));
  if (act == 3) return v > 0.f ? v : 0.01f * v;
  if (act == 4) return 1.f / (1.f + expf(-v));
  if (act == 5) return tanhf(v);
  return v;
}

template <int KH, int KW, int SH, int SW, int DW>
struct GenGeom {
  static constexpr int ROWS = (GTH - 1) * SH + KH;
  static constexpr int COLS = (GTW - 1) * SW + (KW - 1) * DW + 1;
  static constexpr int COLS_PAD = ((COLS + 3) / 4) * 4 + 4;
  static constexpr int TAPS = KH * KW;
  static constexpr int XV = 3 * SW + (KW - 1) * DW + 1;
  static constexpr int OPERAND_FLOATS = GCI * ROWS * COLS_PAD + GCI * TAPS * GTCO;
  static constexpr int STAGE_FLOATS = GTH * GTCO * (GTW + 1);  // output staging of the W-transposed mode
  static constexpr int SMEM_FLOATS = OPERAND_FLOATS > STAGE_FLOATS ? OPERAND_FLOATS : STAGE_FLOATS;
};

template <int KH, int KW, int SH, int SW, int DW>
__global__ void __launch_bounds__(GNT) conv_gen_kernel(ConvGenParams p) {
  using G = GenGeom<KH, KW, SH, SW, DW>;
  extern __shared__ float gsm[];
  float* in_s = gsm;
  float* w_s = gsm + GCI * G::ROWS * G::COLS_PAD;
  const int tid = threadIdx.x;
  const int tx = tid & 31, ty = (tid >> 5) & 1, tc = tid >> 6;
  const int n_cot = p.CoutPad / GTCO;
  const int cot = blockIdx.z % n_cot, b = blockIdx.z / n_cot;
  const int co0 = cot * GTCO;
  const int w0 = blockIdx.x * GTW, h0 = blockIdx.y * GTH;
  float acc[4][12];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 12; ++j) acc[i][j] = 0.f;
  const float* xb = p.x + (int64_t)b * p.Cin * p.H * p.W;
  for (int ci0 = 0; ci0 < p.Cin; ci0 += GCI) {
    for (int idx = tid; idx < GCI * G::ROWS * G::COLS; idx += GNT) {
      const int c = idx % G::COLS;
      const int r = (idx / G::COLS) % G::ROWS;
      const int ci = idx / (G::COLS * G::ROWS);
      const int hi = h0 * SH - p.PH + r, wi = w0 * SW - p.PW + c;
      float v = 0.f;
      if (ci0 + ci < p.Cin && hi >= 0 && hi < p.H && wi >= 0 && wi < p.W) v = __ldg(&xb[((int64_t)(ci0 + ci) * p.H + hi) * p.W + wi]);
      in_s[(ci * G::ROWS + r) * G::COLS_PAD + c] = v;
    }
    for (int idx = tid; idx < GCI * G::TAPS * (GTCO / 4); idx += GNT) {
      const int q = idx % (GTCO / 4);
      const int tap = (idx / (GTCO / 4)) % G::TAPS;
      const int ci = idx / ((GTCO / 4) * G::TAPS);
      float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
      if (ci0 + ci < p.Cin) v = __ldg(reinterpret_cast<const float4*>(&p.w[((int64_t)(ci0 + ci) * G::TAPS + tap) * p.CoutPad + co0 + q * 4]));
      *reinterpret_cast<float4*>(&w_s[(ci * G::TAPS + tap) * GTCO + q * 4]) = v;
    }
    __syncthreads();
#pragma unroll 2
    for (int ci = 0; ci < GCI; ++ci) {
      if (ci0 + ci >= p.Cin) break;  // the 2-channel waveform convolution of the first time encoder: no arithmetic on the zero-filled channels
#pragma unroll
      for (int kh = 0; kh < KH; ++kh) {
        const float* row = &in_s[(ci * G::ROWS + ty * SH + kh) * G::COLS_PAD + 4 * SW * tx];
        float xv[G::XV];
#pragma unroll
        for (int j = 0; j < G::XV; ++j) xv[j] = row[j];
#pragma unroll
        for (int kw = 0; kw < KW; ++kw) {
          const float4* wp = reinterpret_cast<const float4*>(&w_s[(ci * G::TAPS + kh * KW + kw) * GTCO + tc * 12]);
          const float4 wa = wp[0], wb = wp[1], wc = wp[2];
          const float wv[12] = {wa.x, wa.y, wa.z, wa.w, wb.x, wb.y, wb.z, wb.w, wc.x, wc.y, wc.z, wc.w};
#pragma unroll
          for (int i = 0; i < 4; ++i)
#pragma unroll
            for (int j = 0; j < 12; ++j) acc[i][j] = fmaf(xv[i * SW + kw * DW], wv[j], acc[i][j]);
        }
      }
    }
    __syncthreads();
  }
  if (p.up_axis == 2) {
    // Transposed convolution along W: thread (wq, column r * CoutReal + c) owns output sample wq * up + r - trim, i.e. a warp's stores would be `up` floats
    // apart.  Stage the tile in shared memory and write whole rows: for every real channel the block holds the 128 * up CONSECUTIVE samples of each row.
    float* out_s = gsm;  // [GTH][GTCO][GTW + 1]   (the main loop ended with a barrier: the operand tiles are dead)
#pragma unroll
    for (int j = 0; j < 12; ++j)
#pragma unroll
      for (int i = 0; i < 4; ++i) out_s[(ty * GTCO + tc * 12 + j) * (GTW + 1) + 4 * tx + i] = acc[i][j];
    __syncthreads();
    const int span = GTW * p.up;
    for (int idx = tid; idx < GTH * p.CoutReal * span; idx += GNT) {
      const int wl = idx % span;
      const int c_real = (idx / span) % p.CoutReal;
      const int hy = idx / (span * p.CoutReal);
      const int wq_l = wl / p.up, r_up = wl - wq_l * p.up;
      const int col = r_up * p.CoutReal + c_real - co0;
      const int h = h0 + hy, wq = w0 + wq_l;
      if (col < 0 || col >= GTCO || co0 + col >= p.Cout || h >= p.Ho || wq >= p.Wo) continue;
      const int wo = wq * p.up + r_up - p.trim;
      if (wo < 0 || wo >= p.out_len) continue;
      const int64_t o = (((int64_t)b * p.CoutReal + c_real) * p.Ho + h) * p.out_len + wo;
      float v = out_s[(hy * GTCO + col) * (GTW + 1) + wq_l] + (p.bias ? __ldg(&p.bias[c_real]) : 0.f);
      if (p.add && p.add_before_act) v += __ldg(&p.add[o]);
      v = gen_act(v, p.act);
      if (p.add && !p.add_before_act) v += __ldg(&p.add[o]);
      p.y[o] = v;
    }
    return;
  }
  const int h = h0 + ty;
  if (h >= p.Ho) return;
  const int wbase = w0 + 4 * tx;
#pragma unroll
  for (int j = 0; j < 12; ++j) {
    const int co = co0 + tc * 12 + j;
    if (co >= p.Cout) continue;
    int c_real = co, r_up = 0;
    if (p.up_axis) {
      r_up = co / p.CoutReal;
      c_real = co - r_up * p.CoutReal;
    }
    const float bias = p.bias ? __ldg(&p.bias[c_real]) : 0.f;
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const int wq = wbase + i;
      if (wq >= p.Wo) continue;
      int64_t o, o_add;
      if (p.up_axis == 0) {
        o = (((int64_t)b * p.OutCT + p.OutCOff + co) * p.Ho + h) * p.Wo + wq;
        o_add = (((int64_t)b * p.Cout + co) * p.Ho + h) * p.Wo + wq;
      } else if (p.up_axis == 1) {  // scatter along H
        const int ho = h * p.up + r_up - p.trim;
        if (ho < 0 || ho >= p.out_len) continue;
        o = o_add = (((int64_t)b * p.CoutReal + c_real) * p.out_len + ho) * p.Wo + wq;
      } else {  // scatter along W
        const int wo = wq * p.up + r_up - p.trim;
        if (wo < 0 || wo >= p.out_len) continue;
        o = o_add = (((int64_t)b * p.CoutReal + c_real) * p.Ho + h) * p.out_len + wo;
      }
      float v = acc[i][j] + bias;
      if (p.add && p.add_before_act) v += __ldg(&p.add[o_add]);
      v = gen_act(v, p.act);
      if (p.add && !p.add_before_act) v += __ldg(&p.add[o_add]);
      p.y[o] = v;
    }
  }
}

// Any geometry (arbitrary kernel, strides, dilations along H and W): one thread per output element.  Only reached for shapes the tiled
// kernels do not cover AND that are too small for the tensor-core route (e.g. the dilated ASPP convolutions of VR 5.1 on a tiny feature map).
__global__ void conv_direct_kernel(ConvGenParams p, int KH, int KW, int SH, int SW, int DH, int DW, int64_t total) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int wo = (int)(i % p.Wo);
    const int ho = (int)((i / p.Wo) % p.Ho);
    const int co = (int)((i / ((int64_t)p.Wo * p.Ho)) % p.Cout);
    const int b = (int)(i / ((int64_t)p.Wo * p.Ho * p.Cout));
    float acc = 0.f;
    for (int ci = 0; ci < p.Cin; ++ci)
      for (int kh = 0; kh < KH; ++kh) {
        const int hi = ho * SH - p.PH + kh * DH;
        if (hi < 0 || hi >= p.H) continue;
        for (int kw = 0; kw < KW; ++kw) {
          const int wi = wo * SW - p.PW + kw * DW;
          if (wi < 0 || wi >= p.W) continue;
          acc = fmaf(__ldg(&p.x[(((int64_t)b * p.Cin + ci) * p.H + hi) * p.W + wi]), __ldg(&p.w[((int64_t)ci * KH * KW + kh * KW + kw) * p.CoutPad + co]), acc);
        }
      }
    float v = acc + (p.bias ? __ldg(&p.bias[co]) : 0.f);
    if (p.add && p.add_before_act) v += __ldg(&p.add[i]);
    v = gen_act(v, p.act);
    if (p.add && !p.add_before_act) v += __ldg(&p.add[i]);
    p.y[(((int64_t)b * p.OutCT + p.OutCOff + co) * p.Ho + ho) * p.Wo + wo] = v;
  }
}

template <int KH, int KW, int SH, int SW, int DW>
static int launch_gen(const ConvGenParams& p, cudaStream_t st) {
  using G = GenGeom<KH, KW, SH, SW, DW>;
  // the W-transposed mode stages its output tile in shared memory; everything else only needs the operand tiles (keeps the occupancy of the small geometries)
  const int smem = (p.up_axis == 2 ? G::SMEM_FLOATS : G::OPERAND_FLOATS) * (int)sizeof(float);
  static bool attr_set[kMaxDevices] = {};
  B2_DEVICE_SLOT(dev);
  if (!attr_set[dev]) {
    B2_CUDA(cudaFuncSetAttribute(conv_gen_kernel<KH, KW, SH, SW, DW>, cudaFuncAttributeMaxDynamicSharedMemorySize, G::SMEM_FLOATS * (int)sizeof(float)));
    attr_set[dev] = true;
  }
  dim3 grid(cdiv(p.Wo, GTW), cdiv(p.Ho, GTH), p.B * (p.CoutPad / GTCO));
  B2_CHECK_ARG(grid.y <= 65535 && grid.z <= 65535, "conv2d_f32: grid too large (Ho=%d, B*co_tiles=%d)", p.Ho, (int)grid.z);
  conv_gen_kernel<KH, KW, SH, SW, DW><<<grid, GNT, smem, st>>>(p);
  B2_LAUNCHED();
  return B200SEP_OK;
}

}  // namespace b200sep

using namespace b200sep;

// math selects the tensor-core arithmetic (B200SEP_MATH_*); the SIMT kernels below are fp32 in every mode
extern "C" int b200sep_conv2d_f32_math(const float* x, const float* w_blocked, const float* bias, const float* add, float* y, int B, int Cin, int H, int W, int Cout,
                                       int Ho, int Wo, int KH, int KW, int SH, int SW, int PH, int PW, int DH, int DW, int act, int add_before_act, int up_axis, int up,
                                       int trim, int out_len, int out_c_total, int out_c_off, const void* w_packed, int math, void* stream) {
  B2_CHECK_ARG(x && w_blocked && y && B >= 1 && Cin >= 1 && Cout >= 1 && Ho >= 1 && Wo >= 1, "conv2d_f32: bad argument");
  B2_CHECK_ARG(math == B200SEP_MATH_BF16X3 || math == B200SEP_MATH_FP16, "conv2d_f32: unknown math mode %d", math);
  B2_CHECK_ARG(w_packed == nullptr || tc_packed_matches(w_packed, math), "conv2d_f32: w_packed was packed for the other math mode (asked for %d)", math);
  B2_CHECK_ARG(out_c_total == 0 || (up_axis == 0 && out_c_off >= 0 && out_c_off + Cout <= out_c_total), "conv2d_f32: bad output channel slice [%d, %d) of %d",
               out_c_off, out_c_off + Cout, out_c_total);
  ConvGenParams p;
  p.x = x; p.w = w_blocked; p.bias = bias; p.add = add; p.y = y;
  p.B = B; p.Cin = Cin; p.H = H; p.W = W; p.Cout = Cout; p.CoutPad = cdiv(Cout, GTCO) * GTCO; p.Ho = Ho; p.Wo = Wo;
  p.PH = PH; p.PW = PW; p.act = act; p.add_before_act = add_before_act;
  p.OutCT = out_c_total ? out_c_total : Cout; p.OutCOff = out_c_total ? out_c_off : 0;
  p.up_axis = up_axis; p.up = up; p.trim = trim; p.out_len = out_len; p.CoutReal = up_axis ? Cout / up : Cout;
  B2_CHECK_ARG(up_axis == 0 || (up >= 1 && Cout % up == 0), "conv2d_f32: transposed mode needs Cout divisible by the up factor");
  cudaStream_t st = (cudaStream_t)stream;
  if (tc_conv_usable(Cin, Cout, KH, KW, Ho, Wo, B) && (up_axis == 0 || (p.CoutReal % 16 == 0 && add == nullptr)))
    return tc_conv2d_f32(x, w_blocked, bias, add, y, B, Cin, H, W, Cout, p.CoutPad, Ho, Wo, KH, KW, SH, SW, PH, PW, DH, DW, act, add_before_act, out_c_total, out_c_off, w_packed,
                         math, st, up_axis, up, trim, out_len);
#define B2_CONV_CASE(kh, kw, sh, sw, dw) \
  if (DH == 1 && KH == kh && KW == kw && SH == sh && SW == sw && DW == dw) return launch_gen<kh, kw, sh, sw, dw>(p, st);
  B2_CONV_CASE(1, 1, 1, 1, 1)
  B2_CONV_CASE(3, 3, 1, 1, 1)
  B2_CONV_CASE(3, 3, 2, 2, 1)
  B2_CONV_CASE(1, 3, 1, 1, 1)
  B2_CONV_CASE(1, 3, 1, 1, 2)
  B2_CONV_CASE(8, 1, 4, 1, 1)
  B2_CONV_CASE(1, 8, 1, 4, 1)
  B2_CONV_CASE(2, 1, 1, 1, 1)
  B2_CONV_CASE(1, 2, 1, 1, 1)
#undef B2_CONV_CASE
  B2_CHECK_ARG(up_axis == 0 && KH >= 1 && KW >= 1 && SH >= 1 && SW >= 1 && DH >= 1 && DW >= 1, "conv2d_f32: unsupported geometry kernel %dx%d stride %dx%d dilation %dx%d%s", KH, KW,
               SH, SW, DH, DW, up_axis ? " (transposed)" : "");
  const int64_t total = (int64_t)B * Cout * Ho * Wo;
  conv_direct_kernel<<<(int)std::min<int64_t>(cdiv(total, 256), kNumSMs * 16), 256, 0, st>>>(p, KH, KW, SH, SW, DH, DW, total);
  B2_LAUNCHED();
  return B200SEP_OK;
}

extern "C" int b200sep_conv2d_f32(const float* x, const float* w_blocked, const float* bias, const float* add, float* y, int B, int Cin, int H, int W, int Cout,
                                  int Ho, int Wo, int KH, int KW, int SH, int SW, int PH, int PW, int DH, int DW, int act, int add_before_act, int up_axis, int up,
                                  int trim, int out_len, int out_c_total, int out_c_off, const void* w_packed, void* stream) {
  return b200sep_conv2d_f32_math(x, w_blocked, bias, add, y, B, Cin, H, W, Cout, Ho, Wo, KH, KW, SH, SW, PH, PW, DH, DW, act, add_before_act, up_axis, up, trim, out_len,
                                 out_c_total, out_c_off, w_packed, B200SEP_MATH_BF16X3, stream);
}
