// FID Inception-v3 pool3 features (clean-fid's `clean` mode detector as pytorch-fid restates it): torchvision's
// Inception3 layout (aux_logits off) with the FID blocks -- the branch_pool average pools of Mixed_5b-d, 6b-e and 7b
// exclude the padding (count_include_pad=False) and Mixed_7c's branch_pool is a 3 x 3 / stride 1 / pad 1 max pool --
// up to the global 8 x 8 average: [B, 2048] fp32.
//
// Activations are NHWC rows (image, y, x) x channels.  Every BasicConv2d (conv without bias, BatchNorm with eps 1e-3,
// ReLU) runs with the BatchNorm folded into its packed weights and a bias at ds_inception_set_weights.  Each branch
// writes straight into its channel slice of the block's concatenated output (pitch = the block's width), so there is
// no concatenation copy; stores are masked to the branch's channels.
//
// bf16 mode: stride-1 convolutions with 8 | cin run as k_vgg_conv's implicit GEMM on wgmma, one TMA box of the input
// per (ky, kx, 64-channel block) shifted by (ky - ph, kx - pw), TMA's zero fill as the padding and as the channel tail
// (the packed weights carry zeros in each tap's channels past cin).  The stride-2 convolutions and the first one
// (cin = 3) run over an im2col of their input (K padded to a multiple of 64) as a 1 x 1 convolution of the same
// kernel.  fp32 mode: im2col (skipped for 1 x 1) and the exact SIMT GEMM with the bias and ReLU.  Both run in passes
// of `capacity` images.  Pools and the global average sum in a fixed order, so an image's features do not depend on
// the other images of the batch.
#include "engine_internal.h"
#include "tc_common.cuh"

namespace ds {
namespace {

constexpr int IC_IMG = 299;
constexpr double IC_BN_EPS = 1e-3;
enum { T_IN = 0, T_A, T_B, T_T1, T_T2, T_COLS, T_NBUF };
enum { OP_CONV = 0, OP_MAXPOOL_S2, OP_AVGPOOL_S1, OP_MAXPOOL_S1 };

// images [B, 3, 299, 299] fp32 in [0, 255] -> x [B, 299, 299, 3] = (v - 128) / 128
template <typename T>
__global__ void k_inc_pack(const float* __restrict__ img, T* __restrict__ x, int64_t n) {
  const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int c = int(i % 3);
  const int64_t p = i / 3, b = p / (IC_IMG * IC_IMG), q = p % (IC_IMG * IC_IMG);
  stf(x + i, __fdiv_rn(__fsub_rn(img[(b * 3 + c) * (IC_IMG * IC_IMG) + q], 128.f), 128.f));
}

// cols[(b, oy, ox)][(ky * kw + kx) * cin + ci], zero in the padding and in the columns [kh * kw * cin, ld)
template <typename T>
__global__ void k_inc_im2col(const T* __restrict__ in, int cin, int H, int W, int kh, int kw, int st, int ph, int pw,
                             int Ho, int Wo, int ld, T* __restrict__ cols, int64_t n) {
  const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int j = int(i % ld);
  const int64_t r = i / ld;
  float v = 0.f;
  if (j < kh * kw * cin) {
    const int ci = j % cin, tap = j / cin, ky = tap / kw, kx = tap % kw;
    const int ox = int(r % Wo), oy = int((r / Wo) % Ho);
    const int64_t b = r / ((int64_t)Wo * Ho);
    const int y = oy * st + ky - ph, x = ox * st + kx - pw;
    if (y >= 0 && y < H && x >= 0 && x < W) v = ldf(in + ((b * H + y) * W + x) * cin + ci);
  }
  stf(cols + i, v);
}

// BasicConv2d fold, one CTA per output channel: wp[co * ld + tap * cs + ci] = W[co][ci][ky][kx] * s (zero elsewhere),
// bias[co] = beta - mean * s with s = gamma / sqrt(var + 1e-3), in fp64.  bn == nullptr: s = 1 and bias = b_raw.
template <typename T>
__global__ void k_inc_fold(const float* __restrict__ w, const float* __restrict__ bn, const float* __restrict__ b_raw,
                           int cin, int cout, int taps, int cs, int ld, T* __restrict__ wp, float* __restrict__ bias) {
  const int co = blockIdx.x;
  double s = 1.0;
  if (bn) s = (double)bn[co] / sqrt((double)bn[3 * cout + co] + IC_BN_EPS);
  for (int j = threadIdx.x; j < ld; j += blockDim.x) {
    const int tap = j / cs, ci = j % cs;
    float v = 0.f;
    if (tap < taps && ci < cin) v = (float)((double)w[((int64_t)co * cin + ci) * taps + tap] * s);
    stf(wp + (int64_t)co * ld + j, v);
  }
  if (threadIdx.x == 0)
    bias[co] = bn ? (float)((double)bn[cout + co] - (double)bn[2 * cout + co] * s) : b_raw[co];
}

// 3 x 3 / stride 2 valid max pool: in [B, H, W, C] -> out[(b, oy, ox) * ldo + co_off + c]
template <typename T>
__global__ void k_inc_maxpool_s2(const T* __restrict__ in, int C, int H, int W, int Ho, int Wo, T* __restrict__ out,
                                 int ldo, int co_off, int64_t n) {
  const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int c = int(i % C);
  const int64_t r = i / C;
  const int ox = int(r % Wo), oy = int((r / Wo) % Ho);
  const int64_t b = r / ((int64_t)Wo * Ho);
  float m = -INFINITY;
  for (int ky = 0; ky < 3; ++ky)
    for (int kx = 0; kx < 3; ++kx) m = fmaxf(m, ldf(in + ((b * H + 2 * oy + ky) * W + 2 * ox + kx) * C + c));
  stf(out + r * ldo + co_off + c, m);
}

// 3 x 3 / stride 1 / pad 1 pool of [B, H, W, C] into the same shape: the average over the taps inside the image
// (count_include_pad=False), summed in (ky, kx) order, or the maximum
template <bool MAX, typename T>
__global__ void k_inc_pool3(const T* __restrict__ in, int C, int H, int W, T* __restrict__ out, int64_t n) {
  const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int c = int(i % C);
  const int64_t r = i / C;
  const int x = int(r % W), y = int((r / W) % H);
  const int64_t b = r / ((int64_t)W * H);
  float acc = MAX ? -INFINITY : 0.f;
  int cnt = 0;
  for (int yy = y - 1; yy <= y + 1; ++yy)
    for (int xx = x - 1; xx <= x + 1; ++xx) {
      if (yy < 0 || yy >= H || xx < 0 || xx >= W) continue;
      const float v = ldf(in + ((b * H + yy) * W + xx) * C + c);
      acc = MAX ? fmaxf(acc, v) : acc + v;
      ++cnt;
    }
  stf(out + i, MAX ? acc : acc / float(cnt));
}

struct Tens { int slot, H, W, C; };

struct IncConv {
  int cin, cout, kh, kw, st, ph, pw, H, W, Ho, Wo;
  bool tc_im2col;      // bf16: over an im2col (stride 2 or cin = 3); fp32: every convolution but the 1 x 1 ones
  int cs, ld;          // packed weight: [cout][ld], tap t's channels at t * cs
  size_t wp_off, b_off;
  int w_idx;           // expected-weight index of conv.weight (bn.weight, bn.bias, running_mean, running_var follow)
  int bn;              // bf16 tile width
  CUtensorMap tm_in, tm_w;
};

struct IncOp {
  int kind, conv;
  Tens in, out;        // out.C is the output pitch
  int co_off;
};

// shared geometry rules of one convolution
void conv_layout(IncConv& c, bool bf16) {
  c.Ho = (c.H + 2 * c.ph - c.kh) / c.st + 1;
  c.Wo = (c.W + 2 * c.pw - c.kw) / c.st + 1;
  const int taps = c.kh * c.kw;
  if (bf16) {
    c.tc_im2col = c.st != 1 || c.cin % 8 != 0;
    if (c.tc_im2col) {
      c.cs = c.cin;
      c.ld = (taps * c.cin + BK - 1) / BK * BK;
    } else {
      c.cs = (c.cin + BK - 1) / BK * BK;
      c.ld = taps * c.cs;
    }
    c.bn = c.cout % 128 == 0 ? 128 : 64;
  } else {
    c.tc_im2col = taps != 1 || c.st != 1;
    c.cs = c.cin;
    c.ld = taps * c.cin;
  }
}

}  // namespace
}  // namespace ds

struct ds_inception {
  ds_inception_config cfg;
  bool bf16 = false;
  size_t esz = 4;
  WeightTable w;
  std::vector<IncConv> convs;
  std::vector<IncOp> ops;
  size_t wp_total = 0, b_total = 0;
  size_t buf_n[T_NBUF] = {};        // elements per image (T_COLS: per pass)
  void* buf[T_NBUF] = {};
  void* wp = nullptr;
  float* bias = nullptr;
  Tens last{};
  bool weights_set = false;
};

namespace {

void ic_free(ds_inception* h) {
  for (void* b : h->buf) cudaFree(b);
  cudaFree(h->wp);
  cudaFree(h->bias);
}


void need(ds_inception* h, const Tens& t) {
  size_t& n = h->buf_n[t.slot];
  n = std::max(n, (size_t)t.H * t.W * t.C);
}

// network builder: each call appends one op in torchvision's module (= state-dict) order
struct Net {
  ds_inception* h;
  Tens conv(const std::string& name, const Tens& in, int cout, int kh, int kw, int st, int ph, int pw, int out_slot,
            int co_off = 0, int pitch = 0) {
    IncConv c = {};
    c.cin = in.C; c.cout = cout; c.kh = kh; c.kw = kw; c.st = st; c.ph = ph; c.pw = pw; c.H = in.H; c.W = in.W;
    conv_layout(c, h->bf16);
    c.wp_off = h->wp_total;
    h->wp_total += (size_t)c.cout * c.ld;
    c.b_off = h->b_total;
    h->b_total += c.cout;
    c.w_idx = int(h->w.names.size());
    h->w.add(name + ".conv.weight", (int64_t)cout * c.cin * kh * kw);
    for (const char* s : {".bn.weight", ".bn.bias", ".bn.running_mean", ".bn.running_var"}) h->w.add(name + s, cout);
    if (c.tc_im2col) h->buf_n[T_COLS] = std::max(h->buf_n[T_COLS], (size_t)c.Ho * c.Wo * c.ld);
    const Tens out = {out_slot, c.Ho, c.Wo, pitch ? pitch : cout};
    need(h, out);
    h->ops.push_back({OP_CONV, int(h->convs.size()), in, out, co_off});
    h->convs.push_back(c);
    return out;
  }
  Tens pool(int kind, const Tens& in, int out_slot, int co_off = 0, int pitch = 0) {
    const bool s2 = kind == OP_MAXPOOL_S2;
    const Tens out = {out_slot, s2 ? (in.H - 3) / 2 + 1 : in.H, s2 ? (in.W - 3) / 2 + 1 : in.W, pitch ? pitch : in.C};
    need(h, out);
    h->ops.push_back({kind, -1, in, out, co_off});
    return out;
  }
};

// Mixed_5b-d (InceptionA), 35 x 35: [64 | 64 | 96 | pool_features]
Tens block_a(Net& n, const std::string& p, const Tens& x, int pf, int out) {
  const int C = 224 + pf;
  n.conv(p + ".branch1x1", x, 64, 1, 1, 1, 0, 0, out, 0, C);
  Tens t = n.conv(p + ".branch5x5_1", x, 48, 1, 1, 1, 0, 0, T_T1);
  n.conv(p + ".branch5x5_2", t, 64, 5, 5, 1, 2, 2, out, 64, C);
  t = n.conv(p + ".branch3x3dbl_1", x, 64, 1, 1, 1, 0, 0, T_T1);
  t = n.conv(p + ".branch3x3dbl_2", t, 96, 3, 3, 1, 1, 1, T_T2);
  n.conv(p + ".branch3x3dbl_3", t, 96, 3, 3, 1, 1, 1, out, 128, C);
  t = n.pool(OP_AVGPOOL_S1, x, T_T1);
  return n.conv(p + ".branch_pool", t, pf, 1, 1, 1, 0, 0, out, 224, C);
}
// Mixed_6a (InceptionB), 35 -> 17: [384 | 96 | in]
Tens block_b(Net& n, const std::string& p, const Tens& x, int out) {
  const int C = 480 + x.C;
  n.conv(p + ".branch3x3", x, 384, 3, 3, 2, 0, 0, out, 0, C);
  Tens t = n.conv(p + ".branch3x3dbl_1", x, 64, 1, 1, 1, 0, 0, T_T1);
  t = n.conv(p + ".branch3x3dbl_2", t, 96, 3, 3, 1, 1, 1, T_T2);
  n.conv(p + ".branch3x3dbl_3", t, 96, 3, 3, 2, 0, 0, out, 384, C);
  return n.pool(OP_MAXPOOL_S2, x, out, 480, C);
}
// Mixed_6b-e (InceptionC), 17 x 17: [192 | 192 | 192 | 192]
Tens block_c(Net& n, const std::string& p, const Tens& x, int c7, int out) {
  n.conv(p + ".branch1x1", x, 192, 1, 1, 1, 0, 0, out, 0, 768);
  Tens t = n.conv(p + ".branch7x7_1", x, c7, 1, 1, 1, 0, 0, T_T1);
  t = n.conv(p + ".branch7x7_2", t, c7, 1, 7, 1, 0, 3, T_T2);
  n.conv(p + ".branch7x7_3", t, 192, 7, 1, 1, 3, 0, out, 192, 768);
  t = n.conv(p + ".branch7x7dbl_1", x, c7, 1, 1, 1, 0, 0, T_T1);
  t = n.conv(p + ".branch7x7dbl_2", t, c7, 7, 1, 1, 3, 0, T_T2);
  t = n.conv(p + ".branch7x7dbl_3", t, c7, 1, 7, 1, 0, 3, T_T1);
  t = n.conv(p + ".branch7x7dbl_4", t, c7, 7, 1, 1, 3, 0, T_T2);
  n.conv(p + ".branch7x7dbl_5", t, 192, 1, 7, 1, 0, 3, out, 384, 768);
  t = n.pool(OP_AVGPOOL_S1, x, T_T1);
  return n.conv(p + ".branch_pool", t, 192, 1, 1, 1, 0, 0, out, 576, 768);
}
// Mixed_7a (InceptionD), 17 -> 8: [320 | 192 | in]
Tens block_d(Net& n, const std::string& p, const Tens& x, int out) {
  const int C = 512 + x.C;
  Tens t = n.conv(p + ".branch3x3_1", x, 192, 1, 1, 1, 0, 0, T_T1);
  n.conv(p + ".branch3x3_2", t, 320, 3, 3, 2, 0, 0, out, 0, C);
  t = n.conv(p + ".branch7x7x3_1", x, 192, 1, 1, 1, 0, 0, T_T1);
  t = n.conv(p + ".branch7x7x3_2", t, 192, 1, 7, 1, 0, 3, T_T2);
  t = n.conv(p + ".branch7x7x3_3", t, 192, 7, 1, 1, 3, 0, T_T1);
  n.conv(p + ".branch7x7x3_4", t, 192, 3, 3, 2, 0, 0, out, 320, C);
  return n.pool(OP_MAXPOOL_S2, x, out, 512, C);
}
// Mixed_7b-c (InceptionE), 8 x 8: [320 | 384 | 384 | 384 | 384 | 192]; branch_pool is an average (7b) or max (7c)
Tens block_e(Net& n, const std::string& p, const Tens& x, int pool_kind, int out) {
  n.conv(p + ".branch1x1", x, 320, 1, 1, 1, 0, 0, out, 0, 2048);
  Tens t = n.conv(p + ".branch3x3_1", x, 384, 1, 1, 1, 0, 0, T_T1);
  n.conv(p + ".branch3x3_2a", t, 384, 1, 3, 1, 0, 1, out, 320, 2048);
  n.conv(p + ".branch3x3_2b", t, 384, 3, 1, 1, 1, 0, out, 704, 2048);
  t = n.conv(p + ".branch3x3dbl_1", x, 448, 1, 1, 1, 0, 0, T_T1);
  t = n.conv(p + ".branch3x3dbl_2", t, 384, 3, 3, 1, 1, 1, T_T2);
  n.conv(p + ".branch3x3dbl_3a", t, 384, 1, 3, 1, 0, 1, out, 1088, 2048);
  n.conv(p + ".branch3x3dbl_3b", t, 384, 3, 1, 1, 1, 0, out, 1472, 2048);
  t = n.pool(pool_kind, x, T_T1);
  return n.conv(p + ".branch_pool", t, 192, 1, 1, 1, 0, 0, out, 1856, 2048);
}

void build_net(ds_inception* h) {
  Net n{h};
  Tens x = {T_IN, IC_IMG, IC_IMG, 3};
  need(h, x);
  x = n.conv("Conv2d_1a_3x3", x, 32, 3, 3, 2, 0, 0, T_T1);
  x = n.conv("Conv2d_2a_3x3", x, 32, 3, 3, 1, 0, 0, T_T2);
  x = n.conv("Conv2d_2b_3x3", x, 64, 3, 3, 1, 1, 1, T_T1);
  x = n.pool(OP_MAXPOOL_S2, x, T_T2);
  x = n.conv("Conv2d_3b_1x1", x, 80, 1, 1, 1, 0, 0, T_T1);
  x = n.conv("Conv2d_4a_3x3", x, 192, 3, 3, 1, 0, 0, T_T2);
  x = n.pool(OP_MAXPOOL_S2, x, T_A);
  x = block_a(n, "Mixed_5b", x, 32, T_B);
  x = block_a(n, "Mixed_5c", x, 64, T_A);
  x = block_a(n, "Mixed_5d", x, 64, T_B);
  x = block_b(n, "Mixed_6a", x, T_A);
  x = block_c(n, "Mixed_6b", x, 128, T_B);
  x = block_c(n, "Mixed_6c", x, 160, T_A);
  x = block_c(n, "Mixed_6d", x, 160, T_B);
  x = block_c(n, "Mixed_6e", x, 192, T_A);
  x = block_d(n, "Mixed_7a", x, T_B);
  x = block_e(n, "Mixed_7b", x, OP_AVGPOOL_S1, T_A);
  x = block_e(n, "Mixed_7c", x, OP_MAXPOOL_S1, T_B);
  h->last = x;
}

// one convolution of B images: in (NHWC, pitch cin) -> out + co_off (pitch ldo)
template <typename T>
void conv_fwd(const IncConv& c, const T* in, T* cols, const T* wp, const float* bias, T* out, int ldo, int co_off,
              int B, cudaStream_t s) {
  const int64_t M = (int64_t)B * c.Ho * c.Wo;
  if (c.tc_im2col) {
    const int64_t n = M * c.ld;
    k_inc_im2col<T><<<ceil_div(n, 256), 256, 0, s>>>(in, c.cin, c.H, c.W, c.kh, c.kw, c.st, c.ph, c.pw, c.Ho, c.Wo,
                                                    c.ld, cols, n);
  }
  if constexpr (std::is_same<T, float>::value) {
    launch_gemm_simt_chunked(c.tc_im2col ? cols : in, c.ld, wp, bias, out + co_off, ldo, (int)M, c.cout, ACT_RELU, s);
  } else {
    VgConvEpi e;
    memset(&e, 0, sizeof e);
    e.bias = bias; e.out = out; e.cout = c.cout; e.Ho = c.Ho; e.Wo = c.Wo; e.ldo = ldo; e.co_off = co_off;
    if (c.tc_im2col) {      // a 1 x 1 convolution over the columns, an "image" of Ho x Wo pixels with ld channels
      e.H = c.Ho; e.W = c.Wo; e.C = c.ld; e.taps = 1; e.kw = 1;
    } else {
      e.H = c.H; e.W = c.W; e.C = c.cs; e.taps = c.kh * c.kw; e.kw = c.kw; e.ph = c.ph; e.pw = c.pw;
    }
    conv_tc_launch(c.tm_in, c.tm_w, e, c.bn, false, B, s);
  }
}

int conv_maps(IncConv& c, const void* in, const void* cols, const bf16* wp, int images, char* err, int len) {
  if (c.tc_im2col) return conv_tc_maps(&c.tm_in, &c.tm_w, cols, c.ld, c.Ho, c.Wo, images, wp, c.ld, c.cout, c.bn, err, len);
  return conv_tc_maps(&c.tm_in, &c.tm_w, in, c.cin, c.H, c.W, images, wp, c.ld, c.cout, c.bn, err, len);
}

template <typename T>
void run_pass(ds_inception* h, int B, float* feat, cudaStream_t s) {
  T* const* buf = (T* const*)h->buf;
  for (const IncOp& op : h->ops) {
    const T* in = buf[op.in.slot];
    T* out = buf[op.out.slot];
    if (op.kind == OP_CONV) {
      const IncConv& c = h->convs[op.conv];
      conv_fwd<T>(c, in, buf[T_COLS], (const T*)h->wp + c.wp_off, h->bias + c.b_off, out, op.out.C, op.co_off, B, s);
    } else if (op.kind == OP_MAXPOOL_S2) {
      const int64_t n = (int64_t)B * op.out.H * op.out.W * op.in.C;
      k_inc_maxpool_s2<T><<<ceil_div(n, 256), 256, 0, s>>>(in, op.in.C, op.in.H, op.in.W, op.out.H, op.out.W, out,
                                                           op.out.C, op.co_off, n);
    } else {
      const int64_t n = (int64_t)B * op.in.H * op.in.W * op.in.C;
      if (op.kind == OP_MAXPOOL_S1) k_inc_pool3<true, T><<<ceil_div(n, 256), 256, 0, s>>>(in, op.in.C, op.in.H, op.in.W, out, n);
      else k_inc_pool3<false, T><<<ceil_div(n, 256), 256, 0, s>>>(in, op.in.C, op.in.H, op.in.W, out, n);
    }
  }
  launch_re_avgpool<T>(buf[h->last.slot], feat, B, h->last.C, h->last.H * h->last.W, s);
}

}  // namespace

extern "C" int ds_inception_create(const ds_inception_config* cfg, ds_inception** out) {
  if (!cfg || !out) return fail(DS_ERR_INVALID, "null argument");
  *out = nullptr;
  if (cfg->precision != DS_PREC_FP32 && cfg->precision != DS_PREC_BF16)
    return fail(DS_ERR_INVALID, "inception: precision %d unknown", cfg->precision);
  if (cfg->capacity < 1 || cfg->capacity > 256)
    return fail(DS_ERR_INVALID, "inception: capacity %d outside [1, 256]", cfg->capacity);
  if (const int rc = open_device(cfg->device)) return rc;
  if (cfg->precision == DS_PREC_BF16) {
    const int rc = conv_tc_set_attrs();
    if (rc) return rc;
  }
  ds_inception* h = new ds_inception();
  h->cfg = *cfg;
  h->bf16 = cfg->precision == DS_PREC_BF16;
  h->esz = h->bf16 ? 2 : 4;
  build_net(h);
  const size_t cap = cfg->capacity;
  cudaError_t ce = cudaSuccess;
  auto alloc = [&](void** p, size_t bytes) { if (ce == cudaSuccess && bytes) ce = cudaMalloc(p, bytes); };
  alloc(&h->wp, h->wp_total * h->esz);
  alloc((void**)&h->bias, h->b_total * 4);
  for (int b = 0; b < T_NBUF; ++b) alloc(&h->buf[b], cap * h->buf_n[b] * h->esz);
  if (ce != cudaSuccess) {
    ic_free(h);
    delete h;
    return fail(DS_ERR_CUDA, "inception: buffers for %d images: %s", cfg->capacity, cudaGetErrorString(ce));
  }
  if (h->bf16) {
    char err[256] = "";
    for (const IncOp& op : h->ops) {
      if (op.kind != OP_CONV) continue;
      IncConv& c = h->convs[op.conv];
      if (conv_maps(c, h->buf[op.in.slot], h->buf[T_COLS], (const bf16*)h->wp + c.wp_off, cfg->capacity, err,
                    sizeof err)) {
        ic_free(h);
        delete h;
        return fail(DS_ERR_CUDA, "inception: tensor maps of %s: %s", h->w.names[c.w_idx].c_str(), err);
      }
    }
  }
  *out = h;
  return 0;
}

extern "C" int ds_inception_destroy(ds_inception* h) {
  if (!h) return 0;
  cudaSetDevice(h->cfg.device);
  ic_free(h);
  delete h;
  return 0;
}

extern "C" int ds_inception_expected_weight_count(ds_inception* h) {
  if (!h) return fail(DS_ERR_INVALID, "null handle");
  return h->w.count();
}

extern "C" int ds_inception_expected_weight(ds_inception* h, int index, const char** name, int64_t* numel) {
  if (!h) return fail(DS_ERR_INVALID, "null argument");
  return h->w.get(index, name, numel);
}

extern "C" int ds_inception_set_weights(ds_inception* h, const float* flat_params_dev, int64_t count, void* stream) {
  if (!h || !flat_params_dev) return fail(DS_ERR_INVALID, "null argument");
  if (count != h->w.total)
    return fail(DS_ERR_INVALID, "inception: %lld parameters given, %lld expected", (long long)count,
                (long long)h->w.total);
  CK(cudaSetDevice(h->cfg.device));
  cudaStream_t s = (cudaStream_t)stream;
  float* bn = nullptr;
  CK(cudaMallocAsync((void**)&bn, (size_t)4 * 448 * 4, s));      // [gamma | beta | mean | var] of one convolution
  for (const IncConv& c : h->convs) {
    const float* w = flat_params_dev + h->w.off[c.w_idx];
    for (int k = 0; k < 4; ++k)
      CK(cudaMemcpyAsync(bn + k * c.cout, flat_params_dev + h->w.off[c.w_idx + 1 + k], c.cout * 4,
                         cudaMemcpyDeviceToDevice, s));
    if (h->bf16)
      k_inc_fold<bf16><<<c.cout, 256, 0, s>>>(w, bn, nullptr, c.cin, c.cout, c.kh * c.kw, c.cs, c.ld,
                                               (bf16*)h->wp + c.wp_off, h->bias + c.b_off);
    else
      k_inc_fold<float><<<c.cout, 256, 0, s>>>(w, bn, nullptr, c.cin, c.cout, c.kh * c.kw, c.cs, c.ld,
                                                (float*)h->wp + c.wp_off, h->bias + c.b_off);
  }
  cudaFreeAsync(bn, s);
  CK(cudaGetLastError());
  h->weights_set = true;
  return 0;
}

extern "C" int ds_inception_features(ds_inception* h, const float* images_dev, int32_t batch, int32_t height,
                                     int32_t width, float* features_dev, void* stream) {
  if (!h || !images_dev || !features_dev) return fail(DS_ERR_INVALID, "null argument");
  if (batch < 0) return fail(DS_ERR_INVALID, "inception: batch %d < 0", batch);
  if (height != IC_IMG || width != IC_IMG)
    return fail(DS_ERR_INVALID, "inception: images are %d x %d, the detector takes 299 x 299 (resize first)", height,
                width);
  if (!h->weights_set) return fail(DS_ERR_STATE, "inception: ds_inception_set_weights first");
  CK(cudaSetDevice(h->cfg.device));
  cudaStream_t s = (cudaStream_t)stream;
  const int64_t img_n = (int64_t)3 * IC_IMG * IC_IMG;
  for (int b0 = 0; b0 < batch; b0 += h->cfg.capacity) {
    const int B = std::min(h->cfg.capacity, batch - b0);
    const int64_t n = (int64_t)B * img_n;
    float* feat = features_dev + (int64_t)b0 * DS_INCEPTION_FEATURES;
    if (h->bf16) {
      k_inc_pack<bf16><<<ceil_div(n, 256), 256, 0, s>>>(images_dev + b0 * img_n, (bf16*)h->buf[T_IN], n);
      run_pass<bf16>(h, B, feat, s);
    } else {
      k_inc_pack<float><<<ceil_div(n, 256), 256, 0, s>>>(images_dev + b0 * img_n, (float*)h->buf[T_IN], n);
      run_pass<float>(h, B, feat, s);
    }
    CK(cudaGetLastError());
  }
  return 0;
}

extern "C" int ds_inception_test_conv(int32_t precision, const float* in_dev, int32_t batch, int32_t height,
                                      int32_t width, int32_t cin, int32_t cout, int32_t kh, int32_t kw,
                                      int32_t stride, int32_t pad_h, int32_t pad_w, const float* weight_dev,
                                      const float* bias_dev, float* out_dev, int32_t out_pitch, int32_t out_offset,
                                      void* stream) {
  if (!in_dev || !weight_dev || !bias_dev || !out_dev) return fail(DS_ERR_INVALID, "null argument");
  if (precision != DS_PREC_FP32 && precision != DS_PREC_BF16)
    return fail(DS_ERR_INVALID, "inception conv: precision %d unknown", precision);
  if (batch < 1 || height < 1 || width < 1 || height > 512 || width > 512 || cin < 1 || cin > 4096 || cout < 1 ||
      cout > 4096 || kh < 1 || kw < 1 || kh > 7 || kw > 7 || stride < 1 || stride > 2 || pad_h < 0 || pad_w < 0 ||
      2 * pad_h >= kh + 1 || 2 * pad_w >= kw + 1)
    return fail(DS_ERR_INVALID, "inception conv: unsupported geometry");
  if (height + 2 * pad_h < kh || width + 2 * pad_w < kw) return fail(DS_ERR_INVALID, "inception conv: empty output");
  if (out_offset < 0 || out_pitch < out_offset + cout || out_pitch % 8 || out_offset % 8 || cout % 8)
    return fail(DS_ERR_INVALID, "inception conv: output slice [%d, %d) of pitch %d (multiples of 8)", out_offset,
                out_offset + cout, out_pitch);
  if (const int rc = require_device()) return rc;
  const bool tc = precision == DS_PREC_BF16;
  if (tc) {
    const int rc = conv_tc_set_attrs();
    if (rc) return rc;
  }
  cudaStream_t s = (cudaStream_t)stream;
  IncConv c = {};
  c.cin = cin; c.cout = cout; c.kh = kh; c.kw = kw; c.st = stride; c.ph = pad_h; c.pw = pad_w; c.H = height; c.W = width;
  conv_layout(c, tc);
  const size_t esz = tc ? 2 : 4;
  const int64_t px = (int64_t)batch * height * width, n_out = (int64_t)batch * c.Ho * c.Wo * out_pitch;
  void *x = nullptr, *cols = nullptr, *wp = nullptr, *y = nullptr;
  float* bias = nullptr;
  CK(cudaMallocAsync(&wp, (size_t)cout * c.ld * esz, s));
  CK(cudaMallocAsync((void**)&bias, (size_t)cout * 4, s));
  if (c.tc_im2col) CK(cudaMallocAsync(&cols, (size_t)batch * c.Ho * c.Wo * c.ld * esz, s));
  int rc = 0;
  if (tc) {
    CK(cudaMallocAsync(&x, px * cin * 2, s));
    CK(cudaMallocAsync(&y, n_out * 2, s));
    launch_te_convert<bf16>(in_dev, (bf16*)x, px * cin, s);
    launch_te_convert<bf16>(out_dev, (bf16*)y, n_out, s);      // the output buffer, sentinels included
    k_inc_fold<bf16><<<cout, 256, 0, s>>>(weight_dev, nullptr, bias_dev, cin, cout, kh * kw, c.cs, c.ld, (bf16*)wp, bias);
    char err[256] = "";
    if (conv_maps(c, x, cols, (const bf16*)wp, batch, err, sizeof err)) {
      rc = fail(DS_ERR_CUDA, "inception conv: tensor maps: %s", err);
    } else {
      conv_fwd<bf16>(c, (const bf16*)x, (bf16*)cols, (const bf16*)wp, bias, (bf16*)y, out_pitch, out_offset, batch, s);
      launch_widen_bf16((const bf16*)y, out_dev, n_out, s);
    }
    cudaFreeAsync(x, s);
    cudaFreeAsync(y, s);
  } else {
    k_inc_fold<float><<<cout, 256, 0, s>>>(weight_dev, nullptr, bias_dev, cin, cout, kh * kw, c.cs, c.ld, (float*)wp,
                                           bias);
    conv_fwd<float>(c, in_dev, (float*)cols, (const float*)wp, bias, out_dev, out_pitch, out_offset, batch, s);
  }
  cudaFreeAsync(wp, s);
  cudaFreeAsync(bias, s);
  if (cols) cudaFreeAsync(cols, s);
  if (rc) return rc;
  CK(cudaGetLastError());
  CK(cudaStreamSynchronize(s));
  return 0;
}
