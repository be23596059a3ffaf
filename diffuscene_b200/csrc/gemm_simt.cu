// CUDA-core GEMM: D[M,N] = act([A0|A1][M,K] * W[N,K]^T + bias) (+ residual), fp32 accumulate.
//
// This is the fp32 parity path (storage float: FMA order differs from the reference only in summation
// order) and the cross-check backend for the bf16 tensor-core kernel in gemm_tc.cu.  It replaces the
// reference's F.conv1d(k=1) / nn.Linear calls (scene_synthesis/networks/denoise_net.py:91,183,214-217).
// 64x64 output tile per 256-thread CTA, 16-deep k-slices staged transposed in shared memory, 4x4
// register micro-tile per thread.
#include <algorithm>

#include "kernels.cuh"

namespace ds {

template <typename T, bool EXACT>
__global__ void __launch_bounds__(256) k_gemm_simt(GemmArgs g) {
  __shared__ __align__(16) float As[16][64 + 4];
  __shared__ __align__(16) float Bs[16][64 + 4];
  const int tid = threadIdx.x;
  const int tx = tid & 15, ty = tid >> 4;
  const int m0 = blockIdx.y * 64, n0 = blockIdx.x * 64;
  const int K = g.k0 + g.k1;
  const T* a0 = (const T*)g.a0;
  const T* a1 = (const T*)g.a1;
  const T* w = (const T*)g.w;
  const int lrow = tid >> 2, lk = (tid & 3) * 4;

  float acc[4][4];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;

  for (int kb = 0; kb < K; kb += 16) {
    {
      const int m = m0 + lrow;
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const int kk = kb + lk + i;
        float v = 0.f;
        if (m < g.M && kk < K)
          v = kk < g.k0 ? ldf(a0 + (int64_t)m * g.lda0 + kk) : ldf(a1 + (int64_t)m * g.lda1 + (kk - g.k0));
        As[lk + i][lrow] = v;
      }
      const int n = n0 + lrow;
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const int kk = kb + lk + i;
        float v = 0.f;
        if (n < g.N && kk < K) v = ldf(w + (int64_t)n * g.ldw + kk);
        Bs[lk + i][lrow] = v;
      }
    }
    __syncthreads();
#pragma unroll
    for (int k = 0; k < 16; ++k) {
      const float4 av = *reinterpret_cast<const float4*>(&As[k][ty * 4]);
      const float4 bv = *reinterpret_cast<const float4*>(&Bs[k][tx * 4]);
      const float a[4] = {av.x, av.y, av.z, av.w};
      const float b[4] = {bv.x, bv.y, bv.z, bv.w};
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(a[i], b[j], acc[i][j]);
    }
    __syncthreads();
  }

  T* d = (T*)g.d;
  const T* res = (const T*)g.res;
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int m = m0 + ty * 4 + i;
    if (m >= g.M) continue;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int n = n0 + tx * 4 + j;
      if (n >= g.N) continue;
      float v = acc[i][j];
      if (g.bias) v += g.bias[n];
      v = apply_act<EXACT>(v, g.act);
      if (res) v += ldf(res + (int64_t)m * g.ldres + n);
      stf(d + (int64_t)m * g.ldd + n, v);
    }
  }
}

template <typename T>
void launch_gemm_simt(const GemmArgs& g, bool exact, cudaStream_t s) {
  dim3 grid((g.N + 63) / 64, (g.M + 63) / 64);
  if (exact) k_gemm_simt<T, true><<<grid, 256, 0, s>>>(g);
  else k_gemm_simt<T, false><<<grid, 256, 0, s>>>(g);
}
void launch_gemm_f32(const GemmArgs& g, cudaStream_t s) { launch_gemm_simt<float>(g, true, s); }

void launch_gemm_simt_chunked(const float* a, int K, const float* w, const float* bias, float* d, int ldd, int M, int N,
                              int act, cudaStream_t s) {
  constexpr int CHUNK = 32768 * 64;
  for (int m0 = 0; m0 < M; m0 += CHUNK) {
    GemmArgs g = {};
    g.a0 = a + (size_t)m0 * K; g.lda0 = K; g.k0 = K;
    g.w = w; g.ldw = K;
    g.bias = bias;
    g.d = d + (size_t)m0 * ldd; g.ldd = ldd;
    g.M = std::min(CHUNK, M - m0); g.N = N; g.act = act;
    launch_gemm_simt<float>(g, true, s);
  }
}

template void launch_gemm_simt<float>(const GemmArgs&, bool, cudaStream_t);
template void launch_gemm_simt<bf16>(const GemmArgs&, bool, cudaStream_t);

}  // namespace ds
