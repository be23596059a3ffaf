// Floor-plan encoder: the ResNet-18 trunk of the reference's `ResNet18` feature extractor
// (scene_synthesis/networks/feature_extractors.py:19-47, FrozenBatchNorm2d of frozen_batchnorm.py), forward and
// backward, behind its own small handle (ds_room_enc_*).  It shares no state with the denoiser's handle.
//
// Activations are NHWC and token-major like the rest of the library: row = (scene, y, x), columns = channels.
// Every convolution is an im2col (columns ordered (ky, kx, cin), zero-padded to a multiple of 64) followed by one of
// the library's GEMMs: k_gemm_wg through a TcGemmPlan in bf16 where the output width is a multiple of 128, the SIMT
// GEMM otherwise and in the fp32 parity mode.  FrozenBatchNorm is folded into the packed weights and a bias
// (W' = W * s[co], bias = b - running_mean * s, s = weight / sqrt(running_var)); the block tails (+ residual, ReLU) are
// one pointwise kernel because the GEMM epilogue adds its residual after the activation.
//
// The backward pass runs the adjoints in reverse: ReLU (zero where the kept output is <= 0, torch's
// threshold_backward), residual split, dW' = dY^T cols (k_gemm_tn), dbias = column sums, dcols = dY W' followed by a
// gather col2im (fixed order, no atomics), the max-pool and average-pool adjoints as gathers, and finally the adjoint
// of the BatchNorm fold into the reference's parameter layout.
#include "engine_internal.h"

namespace ds {
// backward.cu
template <typename TA, typename TB, typename TD>
void launch_gemm_nn(const TA* A, int lda, const TB* B, int ldb, TD* D, int ldd, int M, int N, int K, int accumulate, cudaStream_t s);
template <typename TA, typename TB>
void launch_gemm_tn(const TA* A, int lda, const TB* B, int ldb, float* D, int ldd, int M, int Ka, int Kb, cudaStream_t s);
template <typename T> void launch_colsum(const T* A, int lda, float* out, int M, int N, cudaStream_t s);

// mask [B, C, HW] fp32 (NCHW) -> [B * HW, C] activation rows
template <typename T>
__global__ void k_re_pack_mask(const float* __restrict__ m, T* __restrict__ out, int C, int HW, int64_t n) {
  const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int c = int(i % C);
  const int64_t r = i / C;
  const int64_t b = r / HW, p = r % HW;
  stf(out + i, m[(b * C + c) * HW + p]);
}
template <typename T>
void launch_re_pack_mask(const float* mask, T* out, int B, int C, int H, int W, cudaStream_t s) {
  const int64_t n = (int64_t)B * H * W * C;
  if (n > 0) k_re_pack_mask<T><<<ceil_div(n, 256), 256, 0, s>>>(mask, out, C, H * W, n);
}

// cols[r][(ky * k + kx) * Cin + ci] = in[b, oy * stride - pad + ky, ox * stride - pad + kx, ci] (0 outside / in the pad)
template <typename T>
__global__ void k_re_im2col(const T* __restrict__ in, RoomConvGeom g, T* __restrict__ cols, int64_t n) {
  const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int j = int(i % g.Kp);
  const int64_t r = i / g.Kp;
  float v = 0.f;
  if (j < g.k * g.k * g.cin) {
    const int ci = j % g.cin, kk = j / g.cin, ky = kk / g.k, kx = kk % g.k;
    const int ox = int(r % g.wout), oy = int((r / g.wout) % g.hout);
    const int64_t b = r / ((int64_t)g.wout * g.hout);
    const int iy = oy * g.stride - g.pad + ky, ix = ox * g.stride - g.pad + kx;
    if (iy >= 0 && iy < g.hin && ix >= 0 && ix < g.win) v = ldf(in + ((b * g.hin + iy) * g.win + ix) * g.cin + ci);
  }
  stf(cols + i, v);
}
template <typename T>
void launch_re_im2col(const T* in, const RoomConvGeom& g, int B, T* cols, cudaStream_t s) {
  const int64_t n = (int64_t)B * g.hout * g.wout * g.Kp;
  if (n > 0) k_re_im2col<T><<<ceil_div(n, 256), 256, 0, s>>>(in, g, cols, n);
}

// Adjoint of im2col as a gather: out[b, iy, ix, ci] = sum over the (ky, kx) taps that read it of dcols, in ascending
// (ky, kx) order; then (+ out if accumulate) (+ add) and zeroed where mask <= 0 (the ReLU adjoint of the producer).
template <typename T>
__global__ void k_re_col2im(const T* __restrict__ dcols, RoomConvGeom g, T* __restrict__ out, int accumulate,
                            const T* __restrict__ add, const T* __restrict__ mask, int64_t n) {
  const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int ci = int(i % g.cin);
  const int64_t r = i / g.cin;
  const int ix = int(r % g.win), iy = int((r / g.win) % g.hin);
  const int64_t b = r / ((int64_t)g.win * g.hin);
  float acc = 0.f;
  for (int ky = 0; ky < g.k; ++ky) {
    const int ty = iy + g.pad - ky;
    if (ty < 0 || ty % g.stride) continue;
    const int oy = ty / g.stride;
    if (oy >= g.hout) continue;
    for (int kx = 0; kx < g.k; ++kx) {
      const int tx = ix + g.pad - kx;
      if (tx < 0 || tx % g.stride) continue;
      const int ox = tx / g.stride;
      if (ox >= g.wout) continue;
      acc += ldf(dcols + ((b * g.hout + oy) * g.wout + ox) * g.Kp + (ky * g.k + kx) * g.cin + ci);
    }
  }
  if (accumulate) acc += ldf(out + i);
  if (add) acc += ldf(add + i);
  if (mask && !(ldf(mask + i) > 0.f)) acc = 0.f;
  stf(out + i, acc);
}
template <typename T>
void launch_re_col2im(const T* dcols, const RoomConvGeom& g, int B, T* out, int accumulate, const T* add, const T* mask,
                      cudaStream_t s) {
  const int64_t n = (int64_t)B * g.hin * g.win * g.cin;
  if (n > 0) k_re_col2im<T><<<ceil_div(n, 256), 256, 0, s>>>(dcols, g, out, accumulate, add, mask, n);
}

// out = relu(z (+ res)); in place allowed (out == z).  NaN passes through, as torch's relu lets it.
template <typename T>
__global__ void k_re_add_relu(const T* z, const T* __restrict__ res, T* out, int64_t n) {
  const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (i >= n) return;
  float v = ldf(z + i);
  if (res) v += ldf(res + i);
  stf(out + i, (v > 0.f || v != v) ? v : 0.f);
}
template <typename T>
void launch_re_add_relu(const T* z, const T* res, T* out, int64_t n, cudaStream_t s) {
  if (n > 0) k_re_add_relu<T><<<ceil_div(n, 256), 256, 0, s>>>(z, res, out, n);
}

// 3x3 / stride 2 / pad 1 max pool window of output (oy, ox): torch's argmax, i.e. the first maximum in row-major
// window order (strict >), the padding acting as -inf.  A NaN is taken as a new maximum, as torch's max_pool2d takes
// it, so a window holding NaN pools to NaN.  Returns the flat input pixel index within the scene.
template <typename T>
__device__ __forceinline__ int re_pool_argmax(const T* in, int64_t b, int oy, int ox, int C, int c, int hin, int win,
                                              float* best_out) {
  float best = -INFINITY;
  int arg = -1;
  for (int ky = 0; ky < 3; ++ky) {
    const int iy = oy * 2 - 1 + ky;
    if (iy < 0 || iy >= hin) continue;
    for (int kx = 0; kx < 3; ++kx) {
      const int ix = ox * 2 - 1 + kx;
      if (ix < 0 || ix >= win) continue;
      const float v = ldf(in + ((b * hin + iy) * win + ix) * C + c);
      if (v > best || isnan(v) || arg < 0) {
        best = v;
        arg = iy * win + ix;
      }
    }
  }
  *best_out = best;
  return arg;
}
template <typename T>
__global__ void k_re_maxpool(const T* __restrict__ in, T* __restrict__ out, int C, int hin, int win, int hout, int wout,
                             int64_t n) {
  const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int c = int(i % C);
  const int64_t r = i / C;
  const int ox = int(r % wout), oy = int((r / wout) % hout);
  const int64_t b = r / ((int64_t)wout * hout);
  float best;
  re_pool_argmax(in, b, oy, ox, C, c, hin, win, &best);
  stf(out + i, best);
}
template <typename T>
void launch_re_maxpool(const T* in, T* out, int B, int C, int hin, int win, int hout, int wout, cudaStream_t s) {
  const int64_t n = (int64_t)B * hout * wout * C;
  if (n > 0) k_re_maxpool<T><<<ceil_div(n, 256), 256, 0, s>>>(in, out, C, hin, win, hout, wout, n);
}
// max-pool adjoint as a gather: din[b, iy, ix, c] = sum of dout over the windows whose argmax is (iy, ix) (windows in
// row-major order), zeroed where the pooled input (a ReLU output) is <= 0
template <typename T>
__global__ void k_re_maxpool_bwd(const T* __restrict__ in, const T* __restrict__ dout, T* __restrict__ din, int C,
                                 int hin, int win, int hout, int wout, int64_t n) {
  const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int c = int(i % C);
  const int64_t r = i / C;
  const int ix = int(r % win), iy = int((r / win) % hin);
  const int64_t b = r / ((int64_t)win * hin);
  float acc = 0.f;
  if (ldf(in + i) > 0.f) {
    const int me = iy * win + ix;
    for (int oy = iy / 2; oy <= min((iy + 1) / 2, hout - 1); ++oy)      // windows 2 oy - 1 .. 2 oy + 1 holding iy
      for (int ox = ix / 2; ox <= min((ix + 1) / 2, wout - 1); ++ox) {
        float best;
        if (re_pool_argmax(in, b, oy, ox, C, c, hin, win, &best) == me)
          acc += ldf(dout + ((b * hout + oy) * wout + ox) * C + c);
      }
  }
  stf(din + i, acc);
}
template <typename T>
void launch_re_maxpool_bwd(const T* in, const T* dout, T* din, int B, int C, int hin, int win, int hout, int wout,
                           cudaStream_t s) {
  const int64_t n = (int64_t)B * hin * win * C;
  if (n > 0) k_re_maxpool_bwd<T><<<ceil_div(n, 256), 256, 0, s>>>(in, dout, din, C, hin, win, hout, wout, n);
}

// global average pool: feat[b][c] = (sum over the scene's pixels in row-major order) / hw, fp32
template <typename T>
__global__ void k_re_avgpool(const T* __restrict__ in, float* __restrict__ feat, int C, int hw, int64_t n) {
  const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int c = int(i % C);
  const int64_t b = i / C;
  float s = 0.f;
  for (int p = 0; p < hw; ++p) s += ldf(in + (b * hw + p) * C + c);
  feat[i] = s / float(hw);
}
template <typename T>
void launch_re_avgpool(const T* in, float* feat, int B, int C, int hw, cudaStream_t s) {
  const int64_t n = (int64_t)B * C;
  if (n > 0) k_re_avgpool<T><<<ceil_div(n, 256), 256, 0, s>>>(in, feat, C, hw, n);
}
// its adjoint fused with the ReLU adjoint of the last block: d[b, p, c] = (out > 0) * dfeat[b][c] / hw
template <typename T>
__global__ void k_re_avgpool_bwd(const float* __restrict__ dfeat, const T* __restrict__ out, T* __restrict__ d, int C,
                                 int hw, int64_t n) {
  const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int c = int(i % C);
  const int64_t b = i / ((int64_t)C * hw);
  stf(d + i, ldf(out + i) > 0.f ? dfeat[b * C + c] / float(hw) : 0.f);
}
template <typename T>
void launch_re_avgpool_bwd(const float* dfeat, const T* out, T* d, int B, int C, int hw, cudaStream_t s) {
  const int64_t n = (int64_t)B * hw * C;
  if (n > 0) k_re_avgpool_bwd<T><<<ceil_div(n, 256), 256, 0, s>>>(dfeat, out, d, C, hw, n);
}

// FrozenBatchNorm fold, one CTA per output channel: wp[co][(ky, kx, ci)] = W[co][ci][ky][kx] * s (0 in the padding),
// bias[co] = b - rm * s with s = weight / sqrt(running_var)
template <typename T>
__global__ void k_re_fold(const float* __restrict__ W, const float* __restrict__ bn, RoomConvGeom g, T* __restrict__ wp,
                          float* __restrict__ bias) {
  const int co = blockIdx.x, cout = gridDim.x;
  const float* bw = bn;
  const float* bb = bn + cout;
  const float* rm = bn + 2 * cout;
  const float* rv = bn + 3 * cout;
  const float s = bw[co] * (1.0f / sqrtf(rv[co]));
  const int kin = g.k * g.k * g.cin;
  for (int j = threadIdx.x; j < g.Kp; j += blockDim.x) {
    float v = 0.f;
    if (j < kin) {
      const int ci = j % g.cin, kk = j / g.cin, ky = kk / g.k, kx = kk % g.k;
      v = W[(((int64_t)co * g.cin + ci) * g.k + ky) * g.k + kx] * s;
    }
    stf(wp + (int64_t)co * g.Kp + j, v);
  }
  if (threadIdx.x == 0) bias[co] = bb[co] - rm[co] * s;
}
// adjoint of the fold: dW = dW' s, dbias_bn = dbias, dweight_bn = (sum_k dW'[co,k] W[co,k] - rm dbias) / sqrt(rv)
__global__ void k_re_fold_bwd(const float* __restrict__ dwp, const float* __restrict__ dbias, const float* __restrict__ W,
                              const float* __restrict__ bn, RoomConvGeom g, float* __restrict__ dW, float* __restrict__ dbn) {
  __shared__ float part[8];
  const int co = blockIdx.x, cout = gridDim.x;
  const float* rm = bn + 2 * cout;
  const float r = 1.0f / sqrtf(bn[3 * cout + co]);
  const float s = bn[co] * r;
  const int kin = g.k * g.k * g.cin;
  float acc = 0.f;
  for (int j = threadIdx.x; j < kin; j += blockDim.x) {
    const int ci = j % g.cin, kk = j / g.cin, ky = kk / g.k, kx = kk % g.k;
    const int64_t wi = (((int64_t)co * g.cin + ci) * g.k + ky) * g.k + kx;
    const float d = dwp[(int64_t)co * g.Kp + j];
    dW[wi] = d * s;
    acc = fmaf(d, W[wi], acc);
  }
  acc = warp_sum(acc);
  if ((threadIdx.x & 31) == 0) part[threadIdx.x >> 5] = acc;
  __syncthreads();
  if (threadIdx.x == 0) {
    float t = 0.f;
    for (int w = 0; w < (int)(blockDim.x >> 5); ++w) t += part[w];
    dbn[co] = r * (t - rm[co] * dbias[co]);      // d weight
    dbn[cout + co] = dbias[co];                   // d bias
  }
}

template <typename T>
void launch_re_fold(const float* W, const float* bn, const RoomConvGeom& g, T* wp, float* bias, cudaStream_t s) {
  k_re_fold<T><<<g.cout, 256, 0, s>>>(W, bn, g, wp, bias);
}
void launch_re_fold_bwd(const float* dwp, const float* dbias, const float* W, const float* bn, const RoomConvGeom& g,
                        float* dW, float* dbn, cudaStream_t s) {
  k_re_fold_bwd<<<g.cout, 256, 0, s>>>(dwp, dbias, W, bn, g, dW, dbn);
}

#define INST_RE(T)                                                                                                   \
  template void launch_re_pack_mask<T>(const float*, T*, int, int, int, int, cudaStream_t);                         \
  template void launch_re_im2col<T>(const T*, const RoomConvGeom&, int, T*, cudaStream_t);                          \
  template void launch_re_col2im<T>(const T*, const RoomConvGeom&, int, T*, int, const T*, const T*, cudaStream_t); \
  template void launch_re_add_relu<T>(const T*, const T*, T*, int64_t, cudaStream_t);                               \
  template void launch_re_maxpool<T>(const T*, T*, int, int, int, int, int, int, cudaStream_t);                     \
  template void launch_re_maxpool_bwd<T>(const T*, const T*, T*, int, int, int, int, int, int, cudaStream_t);       \
  template void launch_re_avgpool<T>(const T*, float*, int, int, int, cudaStream_t);                                \
  template void launch_re_avgpool_bwd<T>(const float*, const T*, T*, int, int, int, cudaStream_t);                  \
  template void launch_re_fold<T>(const float*, const float*, const RoomConvGeom&, T*, float*, cudaStream_t);
INST_RE(float)
INST_RE(bf16)
}  // namespace ds

// ------------------------------------------------------------------------------------------------
// handle and C ABI
// ------------------------------------------------------------------------------------------------
namespace {
struct RConv {
  RoomConvGeom g;
  int w_idx, bn_idx;      // expected-weight index of the conv weight and of the BatchNorm's `weight`
  size_t wp_off;          // element offset into the packed-weight arena (multiple of 64)
  size_t b_off;           // float offset into the bias / dbias arenas
  size_t dw_off;          // float offset into the dW' arena
};
}  // namespace

struct ds_room_enc {
  ds_room_enc_config cfg;
  bool bf16 = false;
  size_t esz = 4;
  WeightTable w;
  std::vector<RConv> conv;      // stem, then per block: conv1, conv2 (, downsample)
  int blk_first[8];             // index into conv of each block's conv1; downsample follows conv2 when present
  bool blk_ds[8];
  int H2, W2, H4, W4;           // stem output, max-pool output
  // device buffers
  int cap = 0;
  void *x0 = nullptr, *a1 = nullptr, *p = nullptr, *h[8] = {nullptr}, *o[8] = {nullptr};
  void *cols = nullptr, *z = nullptr, *dsb = nullptr;
  // input gradients of the backward pass, one buffer per array (ds_room_enc_read): per block the gradient of the
  // pre-ReLU block sum (dz) and of conv1's pre-ReLU output (dh); the max-pool output (dp) and input (da1)
  void *dz[8] = {nullptr}, *dh[8] = {nullptr}, *dp = nullptr, *da1 = nullptr;
  void* wp = nullptr;
  float *bias = nullptr, *dwp = nullptr, *dbias = nullptr;
  size_t wp_total = 0, b_total = 0, dw_total = 0;
  std::vector<TcGemmPlan*> tc;      // forward GEMM plans (bf16, output width % 128 == 0), per conv
  int last_B = 0;                   // batch of the last forward (0: none since the buffers were allocated)
  bool have_grads = false;          // a backward ran after the last forward
  // state kept by a forward with keep_for_backward
  bool kept = false;
  int kept_B = 0;
  const float* kept_params = nullptr;
};

namespace {
template <typename T> T* P(void* v, size_t off = 0) { return (T*)v + off; }
constexpr int RE_ROW_CHUNK = 32768 * 64;

void re_free(ds_room_enc* h) {
  for (auto* p : h->tc) if (p) tc_plan_destroy(p);
  h->tc.assign(h->conv.size(), nullptr);
  void** bufs[] = {&h->x0, &h->a1, &h->p, &h->cols, &h->z, &h->dsb, &h->dp, &h->da1};
  for (void** b : bufs) { cudaFree(*b); *b = nullptr; }
  for (int i = 0; i < 8; ++i)
    for (void** b : {&h->h[i], &h->o[i], &h->dz[i], &h->dh[i]}) { cudaFree(*b); *b = nullptr; }
  h->cap = 0;
  h->last_B = 0;
  h->have_grads = false;
  h->kept = false;
}

int add_conv(ds_room_enc* h, const std::string& conv_name, const std::string& bn_name, int cin, int cout, int k, int stride,
             int pad, int hin, int win) {
  RConv c;
  c.g.cin = cin; c.g.cout = cout; c.g.k = k; c.g.stride = stride; c.g.pad = pad; c.g.hin = hin; c.g.win = win;
  c.g.hout = (hin + 2 * pad - k) / stride + 1;
  c.g.wout = (win + 2 * pad - k) / stride + 1;
  c.g.Kp = (k * k * cin + 63) / 64 * 64;
  c.w_idx = int(h->w.names.size());
  h->w.add(conv_name + ".weight", (int64_t)cout * cin * k * k);
  c.bn_idx = int(h->w.names.size());
  for (const char* s : {".weight", ".bias", ".running_mean", ".running_var"}) h->w.add(bn_name + s, cout);
  c.wp_off = h->wp_total;
  h->wp_total += (size_t)cout * c.g.Kp;
  c.b_off = h->b_total;
  h->b_total += cout;
  c.dw_off = h->dw_total;
  h->dw_total += (size_t)cout * c.g.Kp;
  h->conv.push_back(c);
  return int(h->conv.size()) - 1;
}

int64_t rows_of(const RoomConvGeom& g, int B) { return (int64_t)B * g.hout * g.wout; }

int re_ensure(ds_room_enc* h, int B) {
  if (B <= h->cap) return 0;
  re_free(h);
  const size_t e = h->esz;
  const int Cin = h->cfg.input_channels;
  const int64_t HW = (int64_t)h->cfg.height * h->cfg.width;
  int64_t cols_max = 0, z_max = 0;
  for (const RConv& c : h->conv) {
    cols_max = std::max(cols_max, rows_of(c.g, B) * c.g.Kp);
    z_max = std::max(z_max, rows_of(c.g, B) * c.g.cout);
  }
  const int64_t a1n = (int64_t)B * h->H2 * h->W2 * 64;
  CK(cudaMalloc(&h->x0, (size_t)B * HW * Cin * e));
  CK(cudaMalloc(&h->a1, (size_t)a1n * e));
  CK(cudaMalloc(&h->p, (size_t)B * h->H4 * h->W4 * 64 * e));
  for (int i = 0; i < 8; ++i) {
    const RoomConvGeom& g = h->conv[h->blk_first[i]].g;
    for (void** b : {&h->h[i], &h->o[i], &h->dz[i], &h->dh[i]}) CK(cudaMalloc(b, (size_t)rows_of(g, B) * g.cout * e));
  }
  CK(cudaMalloc(&h->cols, (size_t)cols_max * e));
  CK(cudaMalloc(&h->z, (size_t)z_max * e));
  CK(cudaMalloc(&h->dsb, (size_t)z_max * e));
  CK(cudaMalloc(&h->dp, (size_t)B * h->H4 * h->W4 * 64 * e));
  CK(cudaMalloc(&h->da1, (size_t)a1n * e));
  h->cap = B;
  if (h->bf16) {
    char err[256] = "";
    for (size_t i = 0; i < h->conv.size(); ++i) {
      const RConv& c = h->conv[i];
      if (c.g.cout % 128) continue;
      GemmArgs g;
      memset(&g, 0, sizeof g);
      g.a0 = h->cols; g.lda0 = c.g.Kp; g.k0 = c.g.Kp;
      g.w = P<bf16>(h->wp, c.wp_off); g.ldw = c.g.Kp;
      g.bias = h->bias + c.b_off;
      g.d = nullptr; g.ldd = c.g.cout;
      g.M = int(rows_of(c.g, B)); g.N = c.g.cout;
      // destination: conv1 of a block writes h[i], conv2 writes z, the downsample writes dsb
      for (int b = 0; b < 8; ++b) {
        const int f = h->blk_first[b];
        if ((int)i == f) g.d = h->h[b];
        else if ((int)i == f + 1) g.d = h->z;
        else if ((int)i == f + 2 && h->blk_ds[b]) g.d = h->dsb;
      }
      h->tc[i] = tc_plan_create(g, g.M, err, sizeof err);
      if (!h->tc[i]) return fail(DS_ERR_CUDA, "room encoder: tensor-core GEMM plan for conv %d failed: %s", (int)i, err);
    }
  }
  return 0;
}

template <typename T>
int conv_fwd(ds_room_enc* h, int ci, const T* in, T* out, int B, cudaStream_t s) {
  const RConv& c = h->conv[ci];
  launch_re_im2col<T>(in, c.g, B, P<T>(h->cols), s);
  const int M = int(rows_of(c.g, B));
  if (h->tc[ci]) {
    const int e = launch_gemm_tc(h->tc[ci], M, s);
    if (e) return fail(DS_ERR_CUDA, "room encoder: GEMM of conv %d failed: %s", ci, cudaGetErrorString((cudaError_t)e));
    return 0;
  }
  // row chunks keep the SIMT GEMMs' grids (64 rows per CTA row) inside the 65535 limit of gridDim.y
  for (int m0 = 0; m0 < M; m0 += RE_ROW_CHUNK) {
    GemmArgs g;
    memset(&g, 0, sizeof g);
    g.a0 = P<T>(h->cols, (size_t)m0 * c.g.Kp); g.lda0 = c.g.Kp; g.k0 = c.g.Kp;
    g.w = P<T>(h->wp, c.wp_off); g.ldw = c.g.Kp;
    g.bias = h->bias + c.b_off;
    g.d = out + (size_t)m0 * c.g.cout; g.ldd = c.g.cout;
    g.M = std::min(RE_ROW_CHUNK, M - m0); g.N = c.g.cout;
    launch_gemm_simt<T>(g, !h->bf16, s);
  }
  return 0;
}

template <typename T>
int re_forward(ds_room_enc* h, const float* prm, const float* mask, int B, float* feat, cudaStream_t s) {
  for (const RConv& c : h->conv)
    launch_re_fold<T>(prm + h->w.off[c.w_idx], prm + h->w.off[c.bn_idx], c.g, P<T>(h->wp, c.wp_off), h->bias + c.b_off, s);
  launch_re_pack_mask<T>(mask, P<T>(h->x0), B, h->cfg.input_channels, h->cfg.height, h->cfg.width, s);
  int rc;
  if ((rc = conv_fwd<T>(h, 0, P<T>(h->x0), P<T>(h->a1), B, s))) return rc;
  launch_re_add_relu<T>(P<T>(h->a1), nullptr, P<T>(h->a1), (int64_t)B * h->H2 * h->W2 * 64, s);
  launch_re_maxpool<T>(P<T>(h->a1), P<T>(h->p), B, 64, h->H2, h->W2, h->H4, h->W4, s);
  const T* x = P<T>(h->p);
  for (int b = 0; b < 8; ++b) {
    const int f = h->blk_first[b];
    const RoomConvGeom& g2 = h->conv[f + 1].g;
    if ((rc = conv_fwd<T>(h, f, x, P<T>(h->h[b]), B, s))) return rc;
    launch_re_add_relu<T>(P<T>(h->h[b]), nullptr, P<T>(h->h[b]), rows_of(g2, B) * g2.cout, s);
    if ((rc = conv_fwd<T>(h, f + 1, P<T>(h->h[b]), P<T>(h->z), B, s))) return rc;
    const T* res = x;
    if (h->blk_ds[b]) {
      if ((rc = conv_fwd<T>(h, f + 2, x, P<T>(h->dsb), B, s))) return rc;
      res = P<T>(h->dsb);
    }
    launch_re_add_relu<T>(P<T>(h->z), res, P<T>(h->o[b]), rows_of(g2, B) * g2.cout, s);
    x = P<T>(h->o[b]);
  }
  const RoomConvGeom& gl = h->conv[h->blk_first[7] + 1].g;
  launch_re_avgpool<T>(x, feat, B, 512, gl.hout * gl.wout, s);
  return 0;
}

// dW' += dy^T cols(in), dbias += colsum(dy), then (optionally) dcols = dy W' into the cols scratch
template <typename T>
void conv_bwd_w(ds_room_enc* h, int ci, const T* in, const T* dy, int B, bool want_dcols, cudaStream_t s) {
  const RConv& c = h->conv[ci];
  const int M = int(rows_of(c.g, B));
  launch_re_im2col<T>(in, c.g, B, P<T>(h->cols), s);
  launch_gemm_tn<T, T>(dy, c.g.cout, P<T>(h->cols), c.g.Kp, h->dwp + c.dw_off, c.g.Kp, M, c.g.cout, c.g.Kp, s);
  for (int m0 = 0; m0 < M; m0 += RE_ROW_CHUNK)      // k_colsum's gridDim.y is rows / 256
    launch_colsum<T>(dy + (size_t)m0 * c.g.cout, c.g.cout, h->dbias + c.b_off, std::min(RE_ROW_CHUNK, M - m0), c.g.cout, s);
  if (want_dcols)
    for (int m0 = 0; m0 < M; m0 += RE_ROW_CHUNK)
      launch_gemm_nn<T, T, T>(dy + (size_t)m0 * c.g.cout, c.g.cout, P<T>(h->wp, c.wp_off), c.g.Kp,
                              P<T>(h->cols, (size_t)m0 * c.g.Kp), c.g.Kp, std::min(RE_ROW_CHUNK, M - m0), c.g.Kp,
                              c.g.cout, 0, s);
}

template <typename T>
int re_backward(ds_room_enc* h, const float* dfeat, float* grads, cudaStream_t s) {
  const int B = h->kept_B;
  const float* prm = h->kept_params;
  CK(cudaMemsetAsync(grads, 0, (size_t)h->w.total * 4, s));
  CK(cudaMemsetAsync(h->dwp, 0, h->dw_total * 4, s));
  CK(cudaMemsetAsync(h->dbias, 0, h->b_total * 4, s));
  {
    const RoomConvGeom& gl = h->conv[h->blk_first[7] + 1].g;
    launch_re_avgpool_bwd<T>(dfeat, P<T>(h->o[7]), P<T>(h->dz[7]), B, 512, gl.hout * gl.wout, s);
  }
  for (int b = 7; b >= 0; --b) {
    const int f = h->blk_first[b];
    const T* x = b > 0 ? P<T>(h->o[b - 1]) : P<T>(h->p);
    const T* xmask = b > 0 ? x : nullptr;      // the max-pool output gets its ReLU adjoint after the pool adjoint
    T* dz = P<T>(h->dz[b]);
    T* dh = P<T>(h->dh[b]);
    T* dx = b > 0 ? P<T>(h->dz[b - 1]) : P<T>(h->dp);
    conv_bwd_w<T>(h, f + 1, P<T>(h->h[b]), dz, B, true, s);
    launch_re_col2im<T>(P<T>(h->cols), h->conv[f + 1].g, B, dh, 0, nullptr, P<T>(h->h[b]), s);
    conv_bwd_w<T>(h, f, x, dh, B, true, s);
    if (h->blk_ds[b]) {
      launch_re_col2im<T>(P<T>(h->cols), h->conv[f].g, B, dx, 0, nullptr, nullptr, s);
      conv_bwd_w<T>(h, f + 2, x, dz, B, true, s);
      launch_re_col2im<T>(P<T>(h->cols), h->conv[f + 2].g, B, dx, 1, nullptr, xmask, s);
    } else {
      launch_re_col2im<T>(P<T>(h->cols), h->conv[f].g, B, dx, 0, dz, xmask, s);
    }
  }
  launch_re_maxpool_bwd<T>(P<T>(h->a1), P<T>(h->dp), P<T>(h->da1), B, 64, h->H2, h->W2, h->H4, h->W4, s);
  conv_bwd_w<T>(h, 0, P<T>(h->x0), P<T>(h->da1), B, false, s);
  for (const RConv& c : h->conv)
    launch_re_fold_bwd(h->dwp + c.dw_off, h->dbias + c.b_off, prm + h->w.off[c.w_idx], prm + h->w.off[c.bn_idx], c.g,
                       grads + h->w.off[c.w_idx], grads + h->w.off[c.bn_idx], s);
  return 0;
}
}  // namespace

extern "C" int ds_room_enc_create(const ds_room_enc_config* cfg, ds_room_enc** out) {
  if (!cfg || !out) return fail(DS_ERR_INVALID, "null argument");
  *out = nullptr;
  if (cfg->precision != DS_PREC_FP32 && cfg->precision != DS_PREC_BF16)
    return fail(DS_ERR_INVALID, "room encoder: precision %d unknown", cfg->precision);
  if (cfg->input_channels < 1 || cfg->input_channels > 8)
    return fail(DS_ERR_INVALID, "room encoder: input_channels %d outside [1, 8]", cfg->input_channels);
  if (cfg->height < 32 || cfg->width < 32 || cfg->height % 32 || cfg->width % 32)
    return fail(DS_ERR_INVALID, "room encoder: mask %d x %d must be at least 32 x 32 and a multiple of 32", cfg->height,
                cfg->width);
  if (const int rc = open_device(cfg->device)) return rc;
  if (cfg->precision == DS_PREC_BF16) {
    char err[256] = "";
    if (!tc_runtime_available(err, sizeof err)) return fail(DS_ERR_CUDA, "%s", err);
  }
  ds_room_enc* h = new ds_room_enc();
  h->cfg = *cfg;
  h->bf16 = cfg->precision == DS_PREC_BF16;
  h->esz = h->bf16 ? 2 : 4;
  h->H2 = cfg->height / 2; h->W2 = cfg->width / 2;
  h->H4 = cfg->height / 4; h->W4 = cfg->width / 4;
  add_conv(h, "conv1", "bn1", cfg->input_channels, 64, 7, 2, 3, cfg->height, cfg->width);
  int hin = h->H4, win = h->W4, cin = 64;
  for (int L = 0; L < 4; ++L) {
    const int cout = 64 << L;
    for (int j = 0; j < 2; ++j) {
      const int b = 2 * L + j, stride = (L > 0 && j == 0) ? 2 : 1;
      const std::string pre = "layer" + std::to_string(L + 1) + "." + std::to_string(j) + ".";
      h->blk_first[b] = add_conv(h, pre + "conv1", pre + "bn1", cin, cout, 3, stride, 1, hin, win);
      const RoomConvGeom g1 = h->conv[h->blk_first[b]].g;
      add_conv(h, pre + "conv2", pre + "bn2", cout, cout, 3, 1, 1, g1.hout, g1.wout);
      h->blk_ds[b] = stride != 1 || cin != cout;
      if (h->blk_ds[b]) add_conv(h, pre + "downsample.0", pre + "downsample.1", cin, cout, 1, stride, 0, hin, win);
      hin = g1.hout; win = g1.wout; cin = cout;
    }
  }
  h->tc.assign(h->conv.size(), nullptr);
  cudaError_t e = cudaMalloc(&h->wp, h->wp_total * h->esz);
  if (e == cudaSuccess) e = cudaMalloc(&h->bias, h->b_total * 4);
  if (e == cudaSuccess) e = cudaMalloc(&h->dwp, h->dw_total * 4);
  if (e == cudaSuccess) e = cudaMalloc(&h->dbias, h->b_total * 4);
  if (e != cudaSuccess) {
    cudaFree(h->wp); cudaFree(h->bias); cudaFree(h->dwp); cudaFree(h->dbias);
    delete h;
    return fail(DS_ERR_CUDA, "room encoder: weight arena allocation failed: %s", cudaGetErrorString(e));
  }
  *out = h;
  return 0;
}

extern "C" int ds_room_enc_destroy(ds_room_enc* h) {
  if (!h) return 0;
  cudaSetDevice(h->cfg.device);
  re_free(h);
  cudaFree(h->wp); cudaFree(h->bias); cudaFree(h->dwp); cudaFree(h->dbias);
  delete h;
  return 0;
}

extern "C" int ds_room_enc_expected_weight_count(ds_room_enc* h) {
  if (!h) return fail(DS_ERR_INVALID, "null handle");
  return h->w.count();
}

extern "C" int ds_room_enc_expected_weight(ds_room_enc* h, int index, const char** name, int64_t* numel) {
  if (!h) return fail(DS_ERR_INVALID, "null argument");
  return h->w.get(index, name, numel);
}

extern "C" int ds_room_enc_forward(ds_room_enc* h, const float* flat_params_dev, const float* mask_dev, int32_t batch,
                                   float* feat_dev, int32_t keep_for_backward, void* stream) {
  if (!h || !flat_params_dev || !mask_dev || !feat_dev) return fail(DS_ERR_INVALID, "null argument");
  if (batch < 1) return fail(DS_ERR_INVALID, "room encoder: batch %d < 1", batch);
  CK(cudaSetDevice(h->cfg.device));
  cudaStream_t s = (cudaStream_t)stream;
  int rc = re_ensure(h, batch);
  if (rc) return rc;
  h->kept = false;
  rc = h->bf16 ? re_forward<bf16>(h, flat_params_dev, mask_dev, batch, feat_dev, s)
               : re_forward<float>(h, flat_params_dev, mask_dev, batch, feat_dev, s);
  if (rc) return rc;
  CK(cudaGetLastError());
  h->last_B = batch;
  h->have_grads = false;
  if (keep_for_backward) {
    h->kept = true;
    h->kept_B = batch;
    h->kept_params = flat_params_dev;
  }
  return 0;
}

extern "C" int ds_room_enc_backward(ds_room_enc* h, const float* dfeat_dev, float* flat_grads_dev, void* stream) {
  if (!h || !dfeat_dev || !flat_grads_dev) return fail(DS_ERR_INVALID, "null argument");
  if (!h->kept) return fail(DS_ERR_INVALID, "room encoder: backward needs a forward with keep_for_backward");
  CK(cudaSetDevice(h->cfg.device));
  cudaStream_t s = (cudaStream_t)stream;
  const int rc = h->bf16 ? re_backward<bf16>(h, dfeat_dev, flat_grads_dev, s)
                         : re_backward<float>(h, dfeat_dev, flat_grads_dev, s);
  if (rc) return rc;
  CK(cudaGetLastError());
  h->have_grads = true;
  return 0;
}

extern "C" int ds_room_enc_read(ds_room_enc* h, int32_t kind, int32_t index, float* dev_out, int64_t capacity,
                                int32_t* rows, int32_t* width, void* stream) {
  if (!h) return fail(DS_ERR_INVALID, "null argument");
  if (!h->last_B) return fail(DS_ERR_STATE, "room encoder: no forward has run");
  const bool grad_kind = kind >= DS_RE_DWP && kind <= DS_RE_DA1;
  if (grad_kind && !h->have_grads) return fail(DS_ERR_STATE, "room encoder: no backward since the last forward");
  const int B = h->last_B;      // a backward always follows the forward it differentiates
  const int n_conv = int(h->conv.size());
  const void* src = nullptr;
  bool wide = false;      // fp32 source; otherwise the handle's activation dtype
  int64_t r = 0;
  int w = 0;
  switch (kind) {
    case DS_RE_X0:
      src = h->x0; r = (int64_t)B * h->cfg.height * h->cfg.width; w = h->cfg.input_channels; break;
    case DS_RE_A1: case DS_RE_DA1:
      src = kind == DS_RE_A1 ? h->a1 : h->da1; r = (int64_t)B * h->H2 * h->W2; w = 64; break;
    case DS_RE_P: case DS_RE_DP:
      src = kind == DS_RE_P ? h->p : h->dp; r = (int64_t)B * h->H4 * h->W4; w = 64; break;
    case DS_RE_H: case DS_RE_O: case DS_RE_DZ: case DS_RE_DH: {
      if (index < 0 || index >= 8) return fail(DS_ERR_INVALID, "room encoder: block index %d out of range", index);
      const RoomConvGeom& g = h->conv[h->blk_first[index]].g;
      src = kind == DS_RE_H ? h->h[index] : kind == DS_RE_O ? h->o[index] : kind == DS_RE_DZ ? h->dz[index] : h->dh[index];
      r = rows_of(g, B); w = g.cout;
      break;
    }
    case DS_RE_WP: case DS_RE_BIAS: case DS_RE_DWP: case DS_RE_DBIAS: {
      if (index < 0 || index >= n_conv) return fail(DS_ERR_INVALID, "room encoder: conv index %d out of range", index);
      const RConv& c = h->conv[index];
      const bool vec = kind == DS_RE_BIAS || kind == DS_RE_DBIAS;
      src = kind == DS_RE_WP ? P<char>(h->wp, c.wp_off * h->esz) : kind == DS_RE_BIAS ? (void*)(h->bias + c.b_off)
            : kind == DS_RE_DWP ? (void*)(h->dwp + c.dw_off) : (void*)(h->dbias + c.b_off);
      wide = kind != DS_RE_WP;
      r = vec ? 1 : c.g.cout; w = vec ? c.g.cout : c.g.Kp;
      break;
    }
    default:
      return fail(DS_ERR_INVALID, "room encoder: bad state kind %d", kind);
  }
  if (!h->bf16) wide = true;
  if (r > INT32_MAX) return fail(DS_ERR_INVALID, "room encoder: %lld rows do not fit the row count", (long long)r);
  if (rows) *rows = int32_t(r);
  if (width) *width = w;
  const int64_t n = r * w;
  if (!dev_out) return 0;      // size query
  if (n > capacity) return fail(DS_ERR_INVALID, "output capacity %lld < %lld", (long long)capacity, (long long)n);
  CK(cudaSetDevice(h->cfg.device));
  cudaStream_t s = (cudaStream_t)stream;
  if (wide) CK(cudaMemcpyAsync(dev_out, src, (size_t)n * 4, cudaMemcpyDeviceToDevice, s));
  else launch_widen_bf16((const bf16*)src, dev_out, n, s);
  CK(cudaGetLastError());
  return 0;
}
