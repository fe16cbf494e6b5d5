// ConvTDFNet forward plan (the graph inside UVR-MDX-NET-*.onnx; topology uvr_lib_v5/mdxnet.py:30-120,
// modules.py:1-74 of the reference).  The handle owns the folded / re-laid-out weights and the activation
// arena; forward() is a fixed sequence of kernel launches on the caller's stream (CUDA-graph capturable).
//
// Activation layout: (B, C, T, F) float32, F innermost -- the layout the reference network computes on
// after its transpose(-1,-2) (mdxnet.py:101), which is also what the STFT kernel emits (layout CTF).
#include <math.h>
#include <string.h>

#include <vector>

#include "common.cuh"
#include "simt_ops.cuh"
#include "umma_ops.cuh"

namespace b200sep {

struct ConvW {       // one convolution (+ folded BatchNorm) on the device
  float* w = nullptr;      // [Cin][taps][CoutPad]
  float* scale = nullptr;  // [N]
  float* shift = nullptr;  // [N]
  int cin = 0, n = 0, n_pad = 0, kh = 1, kw = 1, stride = 1;
  // tensor-core path (precision 1): weights split into bf16 hi/lo planes, pre-blocked for umma_conv_run
  bool umma = false;
  void* wb_hi = nullptr;
  void* wb_lo = nullptr;
  int kc = 0, n_tile = 0;  // n_tile = output channels per CTA (n_c)
};
struct LinW {        // TDF linear (+ folded BatchNorm over the channel axis)
  float* w = nullptr;  // [N][K]
  float* scale = nullptr;
  float* shift = nullptr;
  int n = 0, k = 0, channels = 0;
  bool umma = false;
  void* w_hi = nullptr;  // bf16 [N][K]
  void* w_lo = nullptr;
  UmmaGemmPlan plan;
};
struct BlockW {
  std::vector<ConvW> tfc;
  LinW tdf1, tdf2;
};

}  // namespace b200sep

using namespace b200sep;

struct b200sep_mdxnet {
  b200sep_mdxnet_config cfg;
  int n_scales = 0;  // num_blocks / 2
  ConvW first, final;
  std::vector<BlockW> enc, dec;
  BlockW bottleneck;
  std::vector<ConvW> ds, us;
  std::vector<float*> bufA, bufB;  // per scale (0..n_scales), each max_batch * C_i * T_i * F_i floats
  float* tdf_tmp = nullptr;        // max over scales of max_batch * C_i * T_i * (F_i / bn)
  int64_t tdf_tmp_elems = 0;
  float* io_tmp = nullptr;         // CFT<->CTF staging, max_batch * 4 * T * F
  std::vector<int64_t> buf_elems;  // elements of bufA[i] / bufB[i] (= offset of the lo plane in pair mode)
  std::vector<UmmaConvPlan> planA, planB;  // per scale: TMA maps over bufA[i] / bufB[i] as conv inputs
  std::vector<char> plan_ok;
  bool pair = false;               // precision 1: activations are bf16 hi/lo pairs
  std::vector<void*> allocs;
  int64_t device_bytes = 0;
  // optional per-category device timing (bench.py roofline): CUDA events recorded around every launch
  bool profiling = false;
  struct ProfRec { int cat; cudaEvent_t a, b; double flops, bytes; };
  std::vector<ProfRec> prof;
};

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

static int dev_alloc(b200sep_mdxnet* net, void** ptr, int64_t bytes) {
  B2_CUDA(cudaMalloc(ptr, (size_t)bytes));
  net->allocs.push_back(*ptr);
  net->device_bytes += bytes;
  return B200SEP_OK;
}

static int upload(b200sep_mdxnet* net, float** dst, const std::vector<float>& src) {
  int rc = dev_alloc(net, (void**)dst, (int64_t)src.size() * sizeof(float));
  if (rc) return rc;
  B2_CUDA(cudaMemcpy(*dst, src.data(), src.size() * sizeof(float), cudaMemcpyHostToDevice));
  return B200SEP_OK;
}

// BatchNorm(eval) after y = conv(x) + bias:  gamma*(y - mean)/sqrt(var+eps) + beta = y_nobias*s + (bias - mean)*s + beta
static void fold_bn(int c, const float* bias, const float* gamma, const float* beta, const float* mean, const float* var, std::vector<float>& scale,
                    std::vector<float>& shift) {
  scale.resize(c);
  shift.resize(c);
  for (int i = 0; i < c; ++i) {
    const double s = gamma ? (double)gamma[i] / sqrt((double)var[i] + 1e-5) : 1.0;
    const double b = bias ? (double)bias[i] : 0.0;
    const double sh = gamma ? (b - (double)mean[i]) * s + (double)beta[i] : b;
    scale[i] = (float)s;
    shift[i] = (float)sh;
  }
}

static inline uint16_t f2bf(float f) {  // round-to-nearest-even float -> bf16 bits
  uint32_t u;
  memcpy(&u, &f, 4);
  if ((u & 0x7fffffffu) > 0x7f800000u) return (uint16_t)((u >> 16) | 0x40);
  u += 0x7fffu + ((u >> 16) & 1u);
  return (uint16_t)(u >> 16);
}
static inline float bf2f(uint16_t h) {
  uint32_t u = (uint32_t)h << 16;
  float f;
  memcpy(&f, &u, 4);
  return f;
}
static int upload_u16(b200sep_mdxnet* net, void** dst, const std::vector<uint16_t>& src) {
  int rc = dev_alloc(net, dst, (int64_t)src.size() * 2);
  if (rc) return rc;
  B2_CUDA(cudaMemcpy(*dst, src.data(), src.size() * 2, cudaMemcpyHostToDevice));
  return B200SEP_OK;
}

// wgmma B operand of a 3x3 conv (see umma_conv_block_weights)
static int make_conv_umma(b200sep_mdxnet* net, ConvW& cw, const float* w /*(Cout,Cin,3,3)*/) {
  umma_conv_choose(cw.cin, cw.n, &cw.kc, &cw.n_tile);
  std::vector<uint16_t> hi, lo;
  umma_conv_block_weights(w, cw.n, cw.cin, cw.kc, cw.n_tile, hi, lo);
  int rc = upload_u16(net, &cw.wb_hi, hi);
  if (!rc) rc = upload_u16(net, &cw.wb_lo, lo);
  cw.umma = rc == 0;
  return rc;
}

// Conv2d weight (Cout, Cin, kh, kw) -> [Cin][kh*kw][CoutPad]
static int make_conv(b200sep_mdxnet* net, ParamReader& rd, ConvW& cw, int cin, int cout, int k, int stride, bool has_bn) {
  const int taps = k * k;
  const float* w = rd.take((int64_t)cout * cin * taps);
  const float* bias = rd.take(cout);
  const float *g = nullptr, *be = nullptr, *mu = nullptr, *va = nullptr;
  if (has_bn) {
    g = rd.take(cout); be = rd.take(cout); mu = rd.take(cout); va = rd.take(cout);
  }
  if (!rd.ok) return B200SEP_ERR_ARG;
  cw.cin = cin; cw.n = cout; cw.n_pad = cdiv(cout, 48) * 48; cw.kh = cw.kw = k; cw.stride = stride;
  std::vector<float> wr((size_t)cin * taps * cw.n_pad, 0.f);
  for (int co = 0; co < cout; ++co)
    for (int ci = 0; ci < cin; ++ci)
      for (int t = 0; t < taps; ++t) wr[((size_t)ci * taps + t) * cw.n_pad + co] = w[((size_t)co * cin + ci) * taps + t];
  std::vector<float> sc, sh;
  fold_bn(cout, bias, g, be, mu, va, sc, sh);
  int rc = upload(net, &cw.w, wr);
  if (!rc) rc = upload(net, &cw.scale, sc);
  if (!rc) rc = upload(net, &cw.shift, sh);
  if (!rc && net->pair && stride == 1 && k == 3 && umma_conv_supported(cin, cout, 8, k, k)) rc = make_conv_umma(net, cw, w);
  if (!rc && net->pair && stride == 2 && k == 2 && umma_updown_supported(cin, cout, 8, 0)) {
    umma_updown_choose(cin, cout, 0, &cw.kc, &cw.n_tile);
    std::vector<uint16_t> hi, lo;
    umma_down_block_weights(w, cout, cin, cw.kc, cw.n_tile, hi, lo);
    rc = upload_u16(net, &cw.wb_hi, hi);
    if (!rc) rc = upload_u16(net, &cw.wb_lo, lo);
    cw.umma = rc == 0;
  }
  return rc;
}

// ConvTranspose2d weight (Cin, Cout, 2, 2) -> 1x1 implicit GEMM with N = 4*Cout ordered (dy, dx, co): [Cin][1][NPad]
static int make_convt(b200sep_mdxnet* net, ParamReader& rd, ConvW& cw, int cin, int cout) {
  const float* w = rd.take((int64_t)cin * cout * 4);
  const float* bias = rd.take(cout);
  const float* g = rd.take(cout); const float* be = rd.take(cout); const float* mu = rd.take(cout); const float* va = rd.take(cout);
  if (!rd.ok) return B200SEP_ERR_ARG;
  cw.cin = cin; cw.n = 4 * cout; cw.n_pad = cdiv(4 * cout, 48) * 48; cw.kh = cw.kw = 1; cw.stride = 1;
  std::vector<float> wr((size_t)cin * cw.n_pad, 0.f);
  for (int ci = 0; ci < cin; ++ci)
    for (int co = 0; co < cout; ++co)
      for (int q = 0; q < 4; ++q) wr[(size_t)ci * cw.n_pad + q * cout + co] = w[((size_t)ci * cout + co) * 4 + q];
  std::vector<float> sc1, sh1, sc(4 * cout), sh(4 * cout);
  fold_bn(cout, bias, g, be, mu, va, sc1, sh1);
  for (int q = 0; q < 4; ++q)
    for (int co = 0; co < cout; ++co) { sc[q * cout + co] = sc1[co]; sh[q * cout + co] = sh1[co]; }
  int rc = upload(net, &cw.w, wr);
  if (!rc) rc = upload(net, &cw.scale, sc);
  if (!rc) rc = upload(net, &cw.shift, sh);
  if (!rc && net->pair && umma_updown_supported(cin, cout, 8, 1)) {
    umma_updown_choose(cin, cout, 1, &cw.kc, &cw.n_tile);
    std::vector<uint16_t> hi, lo;
    umma_up_block_weights(w, cin, cout, cw.kc, cw.n_tile, hi, lo);
    rc = upload_u16(net, &cw.wb_hi, hi);
    if (!rc) rc = upload_u16(net, &cw.wb_lo, lo);
    cw.umma = rc == 0;
  }
  return rc;
}

static int make_lin(b200sep_mdxnet* net, ParamReader& rd, LinW& lw, int n, int k, int channels) {
  const float* w = rd.take((int64_t)n * k);
  const float* g = rd.take(channels); const float* be = rd.take(channels); const float* mu = rd.take(channels); const float* va = rd.take(channels);
  if (!rd.ok) return B200SEP_ERR_ARG;
  lw.n = n; lw.k = k; lw.channels = channels;
  std::vector<float> wv(w, w + (size_t)n * k), sc, sh;
  fold_bn(channels, nullptr, g, be, mu, va, sc, sh);
  int rc = upload(net, &lw.w, wv);
  if (!rc) rc = upload(net, &lw.scale, sc);
  if (!rc) rc = upload(net, &lw.shift, sh);
  if (!rc && net->pair && umma_gemm_supported(1, n, k)) {
    std::vector<uint16_t> hi((size_t)n * k), lo(hi.size());
    for (size_t i = 0; i < hi.size(); ++i) {
      hi[i] = f2bf(w[i]);
      lo[i] = f2bf(w[i] - bf2f(hi[i]));
    }
    rc = upload_u16(net, &lw.w_hi, hi);
    if (!rc) rc = upload_u16(net, &lw.w_lo, lo);
    lw.umma = rc == 0;  // the TMA plan is bound once the activation arena exists
  }
  return rc;
}

static int make_block(b200sep_mdxnet* net, ParamReader& rd, BlockW& bw, int c, int f) {
  const b200sep_mdxnet_config& cfg = net->cfg;
  bw.tfc.resize(cfg.l);
  for (int i = 0; i < cfg.l; ++i) {
    int rc = make_conv(net, rd, bw.tfc[i], c, c, cfg.k, 1, true);
    if (rc) return rc;
  }
  int rc = make_lin(net, rd, bw.tdf1, f / cfg.bn, f, c);
  if (!rc) rc = make_lin(net, rd, bw.tdf2, f, f / cfg.bn, c);
  return rc;
}

static int64_t block_params(const b200sep_mdxnet_config& c, int64_t ch, int64_t f) {
  return c.l * (ch * ch * c.k * c.k + ch + 4 * ch) + 2 * (f / c.bn) * f + 8 * ch;
}

enum ProfCat { CAT_CONV3X3 = 0, CAT_TDF = 1, CAT_DOWN = 2, CAT_UP = 3, CAT_POINTWISE = 4, CAT_TRANSPOSE = 5, CAT_CONV3X3_S0 = 6, CAT_COUNT = 7 };
// "conv3x3_scale0" = the TFC convolutions at the outermost U-Net scale (the single heaviest launch shape); "conv3x3" = all other scales
static const char* kCatNames[CAT_COUNT] = {"conv3x3", "tdf_linear", "downsample2x2", "upsample2x2", "pointwise1x1", "transpose", "conv3x3_scale0"};

struct ProfScope {  // records an event pair around the launches issued during its lifetime
  b200sep_mdxnet* net; cudaStream_t st; b200sep_mdxnet::ProfRec rec; bool on;
  ProfScope(b200sep_mdxnet* n, cudaStream_t s, int cat, double flops, double bytes) : net(n), st(s), on(n->profiling) {
    if (!on) return;
    rec.cat = cat; rec.flops = flops; rec.bytes = bytes;
    cudaEventCreate(&rec.a); cudaEventCreate(&rec.b);
    cudaEventRecord(rec.a, st);
  }
  ~ProfScope() {
    if (!on) return;
    cudaEventRecord(rec.b, st);
    net->prof.push_back(rec);
  }
};

static int run_conv(b200sep_mdxnet* net, int cat, const ConvW& cw, const float* x, float* y, const float* mul, int B, int H, int W, int relu, int epilogue, cudaStream_t st,
                    const void* x_lo = nullptr, void* y_lo = nullptr, const void* mul_lo = nullptr) {
  const double pix = (double)B * (H / cw.stride) * (W / cw.stride);
  const double out_elems = pix * cw.n;
  ProfScope ps(net, st, cat, 2.0 * pix * cw.n * cw.cin * cw.kh * cw.kw,
               4.0 * ((double)B * cw.cin * H * W + out_elems * (mul ? 2 : 1) + (double)cw.cin * cw.kh * cw.kw * cw.n));
  ConvParams p;
  p.x = x; p.w = cw.w; p.scale = cw.scale; p.shift = cw.shift; p.mul = mul; p.y = y;
  p.x_lo = x_lo; p.mul_lo = mul_lo; p.y_lo = y_lo;
  p.B = B; p.Cin = cw.cin; p.H = H; p.W = W; p.Cout = cw.n; p.CoutPad = cw.n_pad;
  p.Ho = H / cw.stride; p.Wo = W / cw.stride; p.relu = relu; p.epilogue = epilogue;
  return conv2d_simt(p, cw.kh, cw.kw, cw.stride, st);
}

// lo plane of a per-scale activation buffer in pair mode (nullptr in fp32 mode)
static inline void* lo_of(const b200sep_mdxnet* net, const float* buf, int scale) {
  return net->pair ? (void*)((uint16_t*)buf + net->buf_elems[scale]) : nullptr;
}

// TFC (l x conv3x3+BN+ReLU) then x + TDF(x) (modules.py:20-23, :63-74).  in: bufA, result left in bufB.
static int run_block(b200sep_mdxnet* net, BlockW& bw, int scale, int B, int c, int T, int F, cudaStream_t st) {
  float* A = net->bufA[scale];
  float* Bf = net->bufB[scale];
  float* src = A;
  float* dst = Bf;
  int rc;
  for (size_t i = 0; i < bw.tfc.size(); ++i) {
    const ConvW& cw = bw.tfc[i];
    if (net->pair && cw.umma && net->plan_ok[scale]) {
      const UmmaConvPlan& pl = (src == A) ? net->planA[scale] : net->planB[scale];
      const double pix = (double)B * T * F;
      ProfScope ps(net, st, scale == 0 ? CAT_CONV3X3_S0 : CAT_CONV3X3, 2.0 * pix * cw.n * cw.cin * 9, 4.0 * (pix * cw.cin + pix * cw.n + 9.0 * cw.cin * cw.n));
      rc = umma_conv_run(pl, cw.wb_hi, cw.wb_lo, B, cw.n, cw.n_tile, cw.kh, cw.scale, cw.shift, 1, dst, lo_of(net, dst, scale), st);
    } else {
      rc = run_conv(net, scale == 0 ? CAT_CONV3X3_S0 : CAT_CONV3X3, cw, src, dst, nullptr, B, T, F, 1, EPI_NORMAL, st, lo_of(net, src, scale), lo_of(net, dst, scale));
    }
    if (rc) return rc;
    float* t = src; src = dst; dst = t;
  }
  float* x = src;  // after an odd number of convs the result is in Bf; after an even number it is back in A
  const int M = B * c * T;
  void* tmp_lo = net->pair ? (void*)((uint16_t*)net->tdf_tmp + net->tdf_tmp_elems) : nullptr;
  // t1 = relu(bn(x @ W1^T))
  if (net->pair && bw.tdf1.umma) {
    ProfScope ps(net, st, CAT_TDF, 2.0 * M * bw.tdf1.n * (double)F, 4.0 * ((double)M * F + (double)M * bw.tdf1.n + (double)bw.tdf1.n * F));
    rc = umma_gemm_run(x == Bf ? bw.tdf1.plan : bw.tdf1.plan, bw.tdf1.scale, bw.tdf1.shift, T, c, 1, net->tdf_tmp, tmp_lo, nullptr, nullptr, M, st);
  } else {
    GemmParams g;
    g.A = x; g.A_lo = lo_of(net, x, scale); g.Bw = bw.tdf1.w; g.scale = bw.tdf1.scale; g.shift = bw.tdf1.shift; g.res = nullptr;
    g.C = net->tdf_tmp; g.C_lo = tmp_lo;
    g.M = M; g.N = bw.tdf1.n; g.K = F; g.rows_per_channel = T; g.channels = c; g.relu = 1;
    ProfScope ps(net, st, CAT_TDF, 2.0 * g.M * g.N * (double)g.K, 4.0 * ((double)g.M * g.K + (double)g.M * g.N + (double)g.N * g.K));
    rc = gemm_tn_simt(g, st);
  }
  if (rc) return rc;
  // Bf = x + relu(bn(t1 @ W2^T))   (x == Bf when l is odd: in-place residual, each element read then written by one thread)
  if (net->pair && bw.tdf2.umma) {
    ProfScope ps(net, st, CAT_TDF, 2.0 * M * (double)F * bw.tdf2.k, 4.0 * ((double)M * bw.tdf2.k + 2.0 * M * F + (double)F * bw.tdf2.k));
    rc = umma_gemm_run(bw.tdf2.plan, bw.tdf2.scale, bw.tdf2.shift, T, c, 1, Bf, lo_of(net, Bf, scale), x, lo_of(net, x, scale), M, st);
  } else {
    GemmParams g;
    g.A = net->tdf_tmp; g.A_lo = tmp_lo; g.Bw = bw.tdf2.w; g.scale = bw.tdf2.scale; g.shift = bw.tdf2.shift;
    g.res = x; g.res_lo = lo_of(net, x, scale); g.C = Bf; g.C_lo = lo_of(net, Bf, scale);
    g.M = M; g.N = F; g.K = bw.tdf2.k; g.rows_per_channel = T; g.channels = c; g.relu = 1;
    ProfScope ps(net, st, CAT_TDF, 2.0 * g.M * g.N * (double)g.K, 4.0 * ((double)g.M * g.K + 2.0 * (double)g.M * g.N + (double)g.N * g.K));
    rc = gemm_tn_simt(g, st);
  }
  return rc;
}

// bind the TMA plans of one block's TDF linears: A operands are the block's output buffer and the shared tdf_tmp
static int bind_block_plans(b200sep_mdxnet* net, BlockW& bw, int scale, int c, int T, int F) {
  if (!net->pair) return B200SEP_OK;
  const int M = net->cfg.max_batch * c * T;
  float* x = (bw.tfc.size() & 1) ? net->bufB[scale] : net->bufA[scale];
  int rc = B200SEP_OK;
  if (bw.tdf1.umma) rc = umma_gemm_plan_create(&bw.tdf1.plan, x, lo_of(net, x, scale), bw.tdf1.w_hi, bw.tdf1.w_lo, M, bw.tdf1.n, F);
  if (!rc && bw.tdf2.umma)
    rc = umma_gemm_plan_create(&bw.tdf2.plan, net->tdf_tmp, (uint16_t*)net->tdf_tmp + net->tdf_tmp_elems, bw.tdf2.w_hi, bw.tdf2.w_lo, M, F, bw.tdf2.k);
  return rc;
}

}  // namespace b200sep

extern "C" int64_t b200sep_mdxnet_param_count(const b200sep_mdxnet_config* c) {
  if (!c || c->num_blocks < 1 || (c->num_blocks & 1) == 0 || c->bn < 1) return -1;
  const int n = c->num_blocks / 2;
  int64_t total = (int64_t)c->g * c->dim_c + c->g + 4 * c->g;
  int64_t f = c->dim_f, ch = c->g;
  for (int i = 0; i < n; ++i) {
    total += block_params(*c, ch, f);
    total += (ch + c->g) * ch * 4 + (ch + c->g) + 4 * (ch + c->g);
    f /= 2;
    ch += c->g;
  }
  total += block_params(*c, ch, f);
  for (int i = 0; i < n; ++i) {
    total += ch * (ch - c->g) * 4 + (ch - c->g) + 4 * (ch - c->g);
    f *= 2;
    ch -= c->g;
    total += block_params(*c, ch, f);
  }
  total += (int64_t)c->dim_c * ch + c->dim_c;
  return total;
}

extern "C" int b200sep_mdxnet_create(b200sep_mdxnet** out, const b200sep_mdxnet_config* cfg, const float* params_host, int64_t n_params) {
  B2_CHECK_ARG(out && cfg && params_host, "mdxnet_create: NULL argument");
  B2_CHECK_ARG(cfg->num_blocks >= 1 && (cfg->num_blocks & 1), "mdxnet_create: num_blocks=%d must be odd", cfg->num_blocks);
  B2_CHECK_ARG(cfg->k == 3, "mdxnet_create: only k=3 TFC kernels are supported (got %d)", cfg->k);
  B2_CHECK_ARG(cfg->l >= 1 && cfg->g >= 1 && cfg->bn >= 1 && cfg->dim_c >= 1 && cfg->max_batch >= 1, "mdxnet_create: bad config");
  const int n = cfg->num_blocks / 2;
  B2_CHECK_ARG(cfg->dim_f % (1 << n) == 0 && cfg->dim_t % (1 << n) == 0, "mdxnet_create: dim_f=%d / dim_t=%d must be divisible by 2^%d", cfg->dim_f,
               cfg->dim_t, n);
  B2_CHECK_ARG((cfg->dim_f >> n) % cfg->bn == 0, "mdxnet_create: dim_f/2^%d must be divisible by bn=%d", n, cfg->bn);
  const int64_t expect = b200sep_mdxnet_param_count(cfg);
  B2_CHECK_ARG(expect == n_params, "mdxnet_create: expected %lld parameters for this config, got %lld", (long long)expect, (long long)n_params);
  int dev_count = 0;
  B2_CUDA(cudaGetDeviceCount(&dev_count));

  b200sep_mdxnet* net = new b200sep_mdxnet();
  net->cfg = *cfg;
  net->n_scales = n;
  net->pair = cfg->precision != 0;
  ParamReader rd{params_host, n_params};
  int rc = make_conv(net, rd, net->first, cfg->dim_c, cfg->g, 1, 1, true);
  int f = cfg->dim_f, c = cfg->g;
  net->enc.resize(n); net->dec.resize(n); net->ds.resize(n); net->us.resize(n);
  for (int i = 0; i < n && !rc; ++i) {
    rc = make_block(net, rd, net->enc[i], c, f);
    if (!rc) rc = make_conv(net, rd, net->ds[i], c, c + cfg->g, 2, 2, true);
    f /= 2; c += cfg->g;
  }
  if (!rc) rc = make_block(net, rd, net->bottleneck, c, f);
  for (int i = 0; i < n && !rc; ++i) {
    rc = make_convt(net, rd, net->us[i], c, c - cfg->g);
    f *= 2; c -= cfg->g;
    if (!rc) rc = make_block(net, rd, net->dec[i], c, f);
  }
  if (!rc) rc = make_conv(net, rd, net->final, c, cfg->dim_c, 1, 1, false);
  if (!rc && (!rd.ok || rd.pos != n_params)) {
    set_error("mdxnet_create: parameter blob size mismatch (consumed %lld of %lld)", (long long)rd.pos, (long long)n_params);
    rc = B200SEP_ERR_ARG;
  }
  // activation arena
  net->bufA.assign(n + 1, nullptr);
  net->bufB.assign(n + 1, nullptr);
  net->buf_elems.assign(n + 1, 0);
  net->planA.resize(n + 1);
  net->planB.resize(n + 1);
  net->plan_ok.assign(n + 1, 0);
  int64_t tmp_max = 0;
  for (int i = 0; i <= n && !rc; ++i) {
    const int64_t ci = (int64_t)cfg->g * (i + 1), ti = cfg->dim_t >> i, fi = cfg->dim_f >> i;
    net->buf_elems[i] = (int64_t)cfg->max_batch * ci * ti * fi;
    const int64_t bytes = net->buf_elems[i] * sizeof(float);
    rc = dev_alloc(net, (void**)&net->bufA[i], bytes);
    if (!rc) rc = dev_alloc(net, (void**)&net->bufB[i], bytes);
    tmp_max = std::max<int64_t>(tmp_max, (int64_t)cfg->max_batch * ci * ti * (fi / cfg->bn));
    if (!rc && net->pair && umma_conv_supported((int)ci, (int)ci, (int)fi, 3, 3)) {
      int kc, nt;
      umma_conv_choose((int)ci, (int)ci, &kc, &nt);
      rc = umma_conv_plan_create(&net->planA[i], net->bufA[i], lo_of(net, net->bufA[i], i), cfg->max_batch, (int)ci, (int)ti, (int)fi, kc);
      if (!rc) rc = umma_conv_plan_create(&net->planB[i], net->bufB[i], lo_of(net, net->bufB[i], i), cfg->max_batch, (int)ci, (int)ti, (int)fi, kc);
      net->plan_ok[i] = rc == 0;
    }
  }
  net->tdf_tmp_elems = tmp_max;
  if (!rc) rc = dev_alloc(net, (void**)&net->tdf_tmp, tmp_max * sizeof(float));
  for (int i = 0; i <= n && !rc; ++i) {
    const int ci = cfg->g * (i + 1), ti = cfg->dim_t >> i, fi = cfg->dim_f >> i;
    if (i < n) {
      rc = bind_block_plans(net, net->enc[i], i, ci, ti, fi);
      if (!rc) rc = bind_block_plans(net, net->dec[n - 1 - i], i, ci, ti, fi);
    } else {
      rc = bind_block_plans(net, net->bottleneck, i, ci, ti, fi);
    }
  }
  if (!rc) rc = dev_alloc(net, (void**)&net->io_tmp, (int64_t)cfg->max_batch * cfg->dim_c * cfg->dim_t * cfg->dim_f * sizeof(float));
  if (rc) {
    b200sep_mdxnet_destroy(net);
    return rc;
  }
  *out = net;
  return B200SEP_OK;
}

extern "C" void b200sep_mdxnet_destroy(b200sep_mdxnet* net) {
  if (!net) return;
  for (auto& r : net->prof) { cudaEventDestroy(r.a); cudaEventDestroy(r.b); }
  for (void* p : net->allocs) cudaFree(p);
  delete net;
}

extern "C" int64_t b200sep_mdxnet_device_bytes(const b200sep_mdxnet* net) { return net ? net->device_bytes : 0; }

extern "C" int b200sep_mdxnet_forward(b200sep_mdxnet* net, const float* spec_in, float* spec_out, int batch, int layout, void* stream) {
  B2_CHECK_ARG(net && spec_in && spec_out, "mdxnet_forward: NULL argument");
  B2_CHECK_ARG(batch >= 0 && batch <= net->cfg.max_batch, "mdxnet_forward: batch=%d exceeds max_batch=%d", batch, net->cfg.max_batch);
  B2_CHECK_ARG(layout == B200SEP_LAYOUT_CFT || layout == B200SEP_LAYOUT_CTF, "mdxnet_forward: bad layout %d", layout);
  if (batch == 0) return B200SEP_OK;
  cudaStream_t st = (cudaStream_t)stream;
  const b200sep_mdxnet_config& cfg = net->cfg;
  const int n = net->n_scales, B = batch;
  int T = cfg.dim_t, F = cfg.dim_f, c = cfg.g;
  int rc;
  const float* in = spec_in;
  if (layout == B200SEP_LAYOUT_CFT) {  // (B,4,F,T) -> (B,4,T,F); the 1x1 first conv commutes with the transpose (mdxnet.py:99-101)
    ProfScope ps(net, st, CAT_TRANSPOSE, 0.0, 8.0 * B * cfg.dim_c * T * F);
    rc = transpose_hw(spec_in, net->io_tmp, B * cfg.dim_c, F, T, st);
    if (rc) return rc;
    in = net->io_tmp;
  }
  if (net->pair && pointwise_pair_supported(cfg.dim_c, cfg.g, (int64_t)T * F, 1)) {
    const double pix = (double)B * T * F;
    ProfScope ps(net, st, CAT_POINTWISE, 2.0 * pix * cfg.dim_c * cfg.g, 4.0 * pix * (cfg.dim_c + cfg.g));
    rc = pointwise_first_pair(in, net->first.w, net->first.n_pad, net->first.scale, net->first.shift, 1, net->bufA[0], lo_of(net, net->bufA[0], 0), B, cfg.dim_c,
                              cfg.g, (int64_t)T * F, st);
  } else {
    rc = run_conv(net, CAT_POINTWISE, net->first, in, net->bufA[0], nullptr, B, T, F, 1, EPI_NORMAL, st, nullptr, lo_of(net, net->bufA[0], 0));
  }
  if (rc) return rc;
  for (int i = 0; i < n; ++i) {  // encoder (mdxnet.py:103-107)
    rc = run_block(net, net->enc[i], i, B, c, T, F, st);
    if (rc) return rc;
    if (net->pair && net->ds[i].umma && net->plan_ok[i]) {
      const ConvW& cw = net->ds[i];
      const double pix = (double)B * (T / 2) * (F / 2);
      ProfScope ps(net, st, CAT_DOWN, 2.0 * pix * cw.n * cw.cin * 4, 4.0 * ((double)B * cw.cin * T * F + pix * cw.n + 4.0 * cw.cin * cw.n));
      rc = umma_down_run(net->planB[i], cw.wb_hi, cw.wb_lo, B, cw.n, cw.n_tile, cw.scale, cw.shift, 1, net->bufA[i + 1], lo_of(net, net->bufA[i + 1], i + 1), st);
    } else {
      rc = run_conv(net, CAT_DOWN, net->ds[i], net->bufB[i], net->bufA[i + 1], nullptr, B, T, F, 1, EPI_NORMAL, st, lo_of(net, net->bufB[i], i),
                    lo_of(net, net->bufA[i + 1], i + 1));
    }
    if (rc) return rc;
    T /= 2; F /= 2; c += cfg.g;
  }
  rc = run_block(net, net->bottleneck, n, B, c, T, F, st);  // mdxnet.py:109
  if (rc) return rc;
  for (int i = 0; i < n; ++i) {  // decoder (mdxnet.py:111-114): convT+BN+ReLU, multiply by the skip, TFC_TDF
    const int s = n - 1 - i;
    if (net->pair && net->us[i].umma && net->plan_ok[s + 1]) {
      const ConvW& cw = net->us[i];
      const int cr = cw.n / 4;
      const double pix = (double)B * T * F;
      ProfScope ps(net, st, CAT_UP, 2.0 * pix * cw.n * cw.cin, 4.0 * (pix * cw.cin + 2.0 * pix * cw.n + (double)cw.cin * cw.n));
      rc = umma_up_run(net->planB[s + 1], cw.wb_hi, cw.wb_lo, B, cr, cw.n_tile, cw.scale, cw.shift, 1, net->bufB[s], lo_of(net, net->bufB[s], s), net->bufA[s],
                       lo_of(net, net->bufA[s], s), st);
    } else {
      rc = run_conv(net, CAT_UP, net->us[i], net->bufB[s + 1], net->bufA[s], net->bufB[s], B, T, F, 1, EPI_CONVT2X2, st, lo_of(net, net->bufB[s + 1], s + 1),
                    lo_of(net, net->bufA[s], s), lo_of(net, net->bufB[s], s));
    }
    if (rc) return rc;
    T *= 2; F *= 2; c -= cfg.g;
    rc = run_block(net, net->dec[i], s, B, c, T, F, st);
    if (rc) return rc;
  }
  float* out = (layout == B200SEP_LAYOUT_CFT) ? net->io_tmp : spec_out;
  if (net->pair && pointwise_pair_supported(cfg.g, cfg.dim_c, (int64_t)T * F, 0)) {
    const double pix = (double)B * T * F;
    ProfScope ps(net, st, CAT_POINTWISE, 2.0 * pix * cfg.dim_c * cfg.g, 4.0 * pix * (cfg.dim_c + cfg.g));
    rc = pointwise_last_pair(net->bufB[0], lo_of(net, net->bufB[0], 0), net->final.w, net->final.n_pad, net->final.scale, net->final.shift, 0, out, B, cfg.g,
                             cfg.dim_c, (int64_t)T * F, st);
  } else {
    rc = run_conv(net, CAT_POINTWISE, net->final, net->bufB[0], out, nullptr, B, T, F, 0, EPI_NORMAL, st, lo_of(net, net->bufB[0], 0), nullptr);
  }
  if (rc) return rc;
  if (layout == B200SEP_LAYOUT_CFT) {
    ProfScope ps(net, st, CAT_TRANSPOSE, 0.0, 8.0 * B * cfg.dim_c * T * F);
    rc = transpose_hw(net->io_tmp, spec_out, B * cfg.dim_c, T, F, st);
  }
  return rc;
}

extern "C" int b200sep_mdxnet_profile_enable(b200sep_mdxnet* net, int enable) {
  B2_CHECK_ARG(net, "mdxnet_profile_enable: NULL handle");
  for (auto& r : net->prof) { cudaEventDestroy(r.a); cudaEventDestroy(r.b); }
  net->prof.clear();
  net->profiling = enable != 0;
  return B200SEP_OK;
}

extern "C" int b200sep_mdxnet_profile_read(b200sep_mdxnet* net, int max_categories, float* ms, int64_t* launches, double* flops, double* bytes) {
  B2_CHECK_ARG(net && ms && launches && flops && bytes && max_categories >= CAT_COUNT, "mdxnet_profile_read: need room for %d categories", CAT_COUNT);
  for (int c = 0; c < CAT_COUNT; ++c) { ms[c] = 0.f; launches[c] = 0; flops[c] = 0.0; bytes[c] = 0.0; }
  for (auto& r : net->prof) {
    B2_CUDA(cudaEventSynchronize(r.b));
    float t = 0.f;
    B2_CUDA(cudaEventElapsedTime(&t, r.a, r.b));
    ms[r.cat] += t; launches[r.cat] += 1; flops[r.cat] += r.flops; bytes[r.cat] += r.bytes;
  }
  return CAT_COUNT;
}

extern "C" const char* b200sep_mdxnet_profile_name(int category) { return (category >= 0 && category < CAT_COUNT) ? kCatNames[category] : ""; }
