// Pillow's separable resize (libImaging/Resample.c) on the device, for feeding renders to the image metrics without
// a host round trip: clean-fid's `clean` resize (each channel a float32 'F' image, bicubic, fp64 coefficients) and
// the improved-precision-recall transform (uint8 RGB, bilinear, 22-bit fixed-point coefficients) followed by
// ToTensor + Normalize.  The coefficient tables are Pillow's precompute_coeffs, computed on the host
// (diffuscene_b200/render.py); these kernels apply them in Pillow's order and rounding: the horizontal pass into an
// intermediate image of the input's height, then the vertical pass.  Sums run serially in Pillow's order with
// explicit _rn operations, so no FMA contraction changes a bit.
#include "engine_internal.h"

namespace ds {
namespace {

constexpr int PRECISION_BITS = 32 - 8 - 2;      // Pillow's 8-bpc fixed point
constexpr int MAX_KSIZE = 1024;

__device__ __forceinline__ bool bounds_ok(const int* bd, int o, int ks, int in) {
  const int lo = bd[2 * o], n = bd[2 * o + 1];
  return lo >= 0 && n >= 0 && n <= ks && lo + n <= in;
}

__device__ __forceinline__ uint8_t clip8(int v) {
  const int s = v >> PRECISION_BITS;
  return (uint8_t)(s < 0 ? 0 : s > 255 ? 255 : s);
}

// Horizontal pass: [B, H, W, 3] -> [B, H, OW, 3].  T_IN uint8, T_OUT float ('F' mode) or uint8 (8 bpc).
template <bool F>
__global__ void k_resize_h(const uint8_t* __restrict__ in, int B, int H, int W, int OW, const int* __restrict__ bd,
                           const void* __restrict__ coeffs, int ks, void* __restrict__ tmp, int* __restrict__ err) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (int64_t)B * H * OW) return;
  const int ox = int(i % OW);
  const int64_t row = i / OW;                   // b * H + y
  if (!bounds_ok(bd, ox, ks, W)) {
    atomicOr(err, 1);
    return;
  }
  const int x0 = bd[2 * ox], n = bd[2 * ox + 1];
  const uint8_t* src = in + (row * W + x0) * 3;
  if (F) {
    const double* k = (const double*)coeffs + (int64_t)ox * ks;
    double ss[3] = {0.0, 0.0, 0.0};
    for (int x = 0; x < n; ++x)
#pragma unroll
      for (int c = 0; c < 3; ++c) ss[c] = __dadd_rn(ss[c], __dmul_rn((double)src[x * 3 + c], k[x]));
    float* o = (float*)tmp + i * 3;
#pragma unroll
    for (int c = 0; c < 3; ++c) o[c] = __double2float_rn(ss[c]);
  } else {
    const int* k = (const int*)coeffs + (int64_t)ox * ks;
    int ss[3] = {1 << (PRECISION_BITS - 1), 1 << (PRECISION_BITS - 1), 1 << (PRECISION_BITS - 1)};
    for (int x = 0; x < n; ++x)
#pragma unroll
      for (int c = 0; c < 3; ++c) ss[c] += (int)src[x * 3 + c] * k[x];
    uint8_t* o = (uint8_t*)tmp + i * 3;
#pragma unroll
    for (int c = 0; c < 3; ++c) o[c] = clip8(ss[c]);
  }
}

// Vertical pass: [B, H, OW, 3] -> planar [B, 3, OH, OW] fp32 with the metric's post-processing.
template <bool F>
__global__ void k_resize_v(const void* __restrict__ tmp, int B, int H, int OH, int OW, const int* __restrict__ bd,
                           const void* __restrict__ coeffs, int ks, float m0, float m1, float m2, float s0, float s1,
                           float s2, float* __restrict__ out, int* __restrict__ err) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (int64_t)B * OH * OW) return;
  const int ox = int(i % OW), oy = int((i / OW) % OH), b = int(i / ((int64_t)OW * OH));
  if (!bounds_ok(bd, oy, ks, H)) {
    atomicOr(err, 2);
    return;
  }
  const int y0 = bd[2 * oy], n = bd[2 * oy + 1];
  const int64_t plane = (int64_t)OH * OW, dst = (int64_t)b * 3 * plane + (int64_t)oy * OW + ox;
  if (F) {
    const double* k = (const double*)coeffs + (int64_t)oy * ks;
    const float* src = (const float*)tmp + (((int64_t)b * H + y0) * OW + ox) * 3;
    double ss[3] = {0.0, 0.0, 0.0};
    for (int y = 0; y < n; ++y)
#pragma unroll
      for (int c = 0; c < 3; ++c) ss[c] = __dadd_rn(ss[c], __dmul_rn((double)src[(int64_t)y * OW * 3 + c], k[y]));
#pragma unroll
    for (int c = 0; c < 3; ++c) out[dst + c * plane] = fminf(fmaxf(__double2float_rn(ss[c]), 0.f), 255.f);
  } else {
    const int* k = (const int*)coeffs + (int64_t)oy * ks;
    const uint8_t* src = (const uint8_t*)tmp + (((int64_t)b * H + y0) * OW + ox) * 3;
    int ss[3] = {1 << (PRECISION_BITS - 1), 1 << (PRECISION_BITS - 1), 1 << (PRECISION_BITS - 1)};
    for (int y = 0; y < n; ++y)
#pragma unroll
      for (int c = 0; c < 3; ++c) ss[c] += (int)src[(int64_t)y * OW * 3 + c] * k[y];
    const float mean[3] = {m0, m1, m2}, stdv[3] = {s0, s1, s2};
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      const float x = __fdiv_rn((float)clip8(ss[c]), 255.f);
      out[dst + c * plane] = __fdiv_rn(__fsub_rn(x, mean[c]), stdv[c]);
    }
  }
}

template <bool F>
int resize(const char* name, const uint8_t* in, int B, int H, int W, int OH, int OW, const int* hb, const void* hk,
           int hks, const int* vb, const void* vk, int vks, const float* ms, float* out, void* stream) {
  if (!in || !hb || !hk || !vb || !vk || !out || (!F && !ms))
    return fail(DS_ERR_INVALID, "%s: NULL input, table or output pointer", name);
  if (B < 0) return fail(DS_ERR_INVALID, "%s: batch %d < 0", name, B);
  if (H < 1 || H > 4096 || W < 1 || W > 4096 || OH < 1 || OH > 4096 || OW < 1 || OW > 4096)
    return fail(DS_ERR_INVALID, "%s: sizes %d x %d -> %d x %d outside [1, 4096]", name, H, W, OH, OW);
  if (hks < 1 || hks > MAX_KSIZE || vks < 1 || vks > MAX_KSIZE)
    return fail(DS_ERR_INVALID, "%s: kernel sizes %d, %d outside [1, %d]", name, hks, vks, MAX_KSIZE);
  if (const int rc = require_device()) return rc;
  if (B == 0) return 0;
  cudaStream_t s = (cudaStream_t)stream;
  void* tmp = nullptr;
  int* err_dev = nullptr;
  CK(cudaMallocAsync(&tmp, (size_t)B * H * OW * 3 * (F ? sizeof(float) : 1), s));
  CK(cudaMallocAsync(&err_dev, sizeof(int), s));
  CK(cudaMemsetAsync(err_dev, 0, sizeof(int), s));
  k_resize_h<F><<<ceil_div((int64_t)B * H * OW, 256), 256, 0, s>>>(in, B, H, W, OW, hb, hk, hks, tmp, err_dev);
  cudaError_t e = cudaGetLastError();
  if (e == cudaSuccess) {
    const float z[6] = {0, 0, 0, 1, 1, 1};
    const float* m = F ? z : ms;
    k_resize_v<F><<<ceil_div((int64_t)B * OH * OW, 256), 256, 0, s>>>(tmp, B, H, OH, OW, vb, vk, vks, m[0], m[1], m[2],
                                                                  m[3], m[4], m[5], out, err_dev);
    e = cudaGetLastError();
  }
  int err = 0;
  if (e == cudaSuccess) e = cudaMemcpyAsync(&err, err_dev, sizeof(int), cudaMemcpyDeviceToHost, s);
  cudaFreeAsync(tmp, s);
  cudaFreeAsync(err_dev, s);
  if (e == cudaSuccess) e = cudaStreamSynchronize(s);
  if (e != cudaSuccess) return fail(DS_ERR_CUDA, "%s: %s", name, cudaGetErrorString(e));
  if (err) return fail(DS_ERR_INVALID, "%s: a %s coefficient bound lies outside the input or the kernel size", name,
                       err & 1 ? "horizontal" : "vertical");
  return 0;
}

}  // namespace
}  // namespace ds

extern "C" int ds_resize_f32(const uint8_t* in_dev, int32_t batch, int32_t in_h, int32_t in_w, int32_t out_h,
                             int32_t out_w, const int32_t* h_bounds_dev, const double* h_coeffs_dev, int32_t h_ksize,
                             const int32_t* v_bounds_dev, const double* v_coeffs_dev, int32_t v_ksize, float* out_dev,
                             void* stream) {
  return resize<true>("ds_resize_f32", in_dev, batch, in_h, in_w, out_h, out_w, h_bounds_dev, h_coeffs_dev, h_ksize,
                      v_bounds_dev, v_coeffs_dev, v_ksize, nullptr, out_dev, stream);
}

extern "C" int ds_resize_u8(const uint8_t* in_dev, int32_t batch, int32_t in_h, int32_t in_w, int32_t out_h,
                            int32_t out_w, const int32_t* h_bounds_dev, const int32_t* h_coeffs_dev, int32_t h_ksize,
                            const int32_t* v_bounds_dev, const int32_t* v_coeffs_dev, int32_t v_ksize,
                            const float* mean_std, float* out_dev, void* stream) {
  return resize<false>("ds_resize_u8", in_dev, batch, in_h, in_w, out_h, out_w, h_bounds_dev, h_coeffs_dev, h_ksize,
                       v_bounds_dev, v_coeffs_dev, v_ksize, mean_std, out_dev, stream);
}
