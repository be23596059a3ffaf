// Feature statistics of FID and the kernel terms of KID, fp64 on the fp64 tensor cores (mma.sync m16n8k16 .f64, the
// tile path of manifold.cu), from fp32 features [rows, d] row-major.
//
//   mean   per column, 8 strided partial sums combined in a fixed order, / n;
//   cov    (X - mu)^T (X - mu) * (1 / (n - 1)), as np.cov does on float64-promoted features: 64 x 64 tiles of the
//          upper triangle, K = n walked in order by one CTA each, mirrored on store (no n x n matrix);
//   KID    per subset s, the three m x m Gram products x x^T, y y^T and x y^T of rows gathered by index, each element
//          taken through (g / d + 1)^3 in the tile epilogue (the diagonal left out of the first two) and summed per tile
//          in a fixed order; a second kernel adds the tiles in order: t_s = (sum a) / (m - 1) - 2 (sum b) / m.
// No floating-point atomics: every output is independent of scheduling and of how many subsets share the launch.
#include "engine_internal.h"

namespace ds {
namespace {

constexpr int FS_T = 64, FS_K = 16, FS_PITCH = FS_K + 4, FS_THREADS = 128;
constexpr int FS_SMEM = 2 * FS_T * FS_PITCH * 8;
enum { FS_COV = 0, FS_KID = 1 };

__device__ __forceinline__ void dmma16816(double (&d)[4], const double (&a)[8], const double (&b)[4]) {
  asm volatile(
      "mma.sync.aligned.m16n8k16.row.col.f64.f64.f64.f64 {%0, %1, %2, %3}, {%4, %5, %6, %7, %8, %9, %10, %11}, "
      "{%12, %13, %14, %15}, {%0, %1, %2, %3};"
      : "+d"(d[0]), "+d"(d[1]), "+d"(d[2]), "+d"(d[3])
      : "d"(a[0]), "d"(a[1]), "d"(a[2]), "d"(a[3]), "d"(a[4]), "d"(a[5]), "d"(a[6]), "d"(a[7]), "d"(b[0]), "d"(b[1]),
        "d"(b[2]), "d"(b[3]));
}

__global__ void k_fs_mean(const float* __restrict__ x, int n, int d, double* __restrict__ mean) {
  __shared__ double part[8][32];
  const int c = blockIdx.x * 32 + (threadIdx.x & 31), r0 = threadIdx.x >> 5;
  double s = 0.0;
  if (c < d)
    for (int r = r0; r < n; r += 8) s = __dadd_rn(s, (double)x[(int64_t)r * d + c]);
  part[r0][threadIdx.x & 31] = s;
  __syncthreads();
  if (r0 == 0 && c < d) {
    double t = part[0][threadIdx.x];
    for (int q = 1; q < 8; ++q) t = __dadd_rn(t, part[q][threadIdx.x]);
    mean[c] = __ddiv_rn(t, (double)n);
  }
}

struct FsArgs {
  const float *x, *y;            // COV: x = y = features [n, d]; KID: fake [n_x, d], real [n_y, d]
  const double* mu;              // COV
  const int64_t *ix, *iy;        // KID: [subsets, m] row indices into x / y
  int n, d, m, tiles;            // COV: K = n, output d x d; KID: K = d, output m x m, tiles = ceil(m / 64)
  double* cov;                   // COV: [d, d]
  double* part;                  // KID: [subsets, 3, tiles, tiles]
};

// COV: blockIdx.x enumerates the upper-triangle tiles (ti <= tj).  KID: blockIdx.x = ti * tiles + tj, blockIdx.y =
// subset * 3 + kind (0: x x^T, 1: y y^T, 2: x y^T)
template <int MODE>
__global__ void __launch_bounds__(FS_THREADS) k_fs_tiles(FsArgs a) {
  extern __shared__ double sm[];
  double* As = sm;
  double* Bs = As + FS_T * FS_PITCH;
  __shared__ double red[FS_THREADS / 32];
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, g = lane >> 2, t = lane & 3;
  const int wr = (warp >> 1) * 32, wc = (warp & 1) * 32;
  int ti, tj, kind = 0, sub = 0;
  if (MODE == FS_COV) {
    int b = blockIdx.x;
    ti = 0;
    while (b >= a.tiles - ti) b -= a.tiles - ti++;
    tj = ti + b;
  } else {
    ti = blockIdx.x / a.tiles;
    tj = blockIdx.x % a.tiles;
    sub = blockIdx.y / 3;
    kind = blockIdx.y % 3;
  }
  const int i0 = ti * FS_T, j0 = tj * FS_T;
  const int K = MODE == FS_COV ? a.n : a.d;
  const int rows = MODE == FS_COV ? a.d : a.m;
  const float* xa = (MODE == FS_KID && kind == 1) ? a.y : a.x;
  const float* xb = (MODE == FS_KID && kind != 0) ? a.y : a.x;
  const int64_t* ia = MODE == FS_KID ? (kind == 1 ? a.iy : a.ix) + (int64_t)sub * a.m : nullptr;
  const int64_t* ib = MODE == FS_KID ? (kind == 0 ? a.ix : a.iy) + (int64_t)sub * a.m : nullptr;

  double acc[2][4][4];
#pragma unroll
  for (int mi = 0; mi < 2; ++mi)
#pragma unroll
    for (int ni = 0; ni < 4; ++ni)
#pragma unroll
      for (int e = 0; e < 4; ++e) acc[mi][ni][e] = 0.0;

  // 8 elements of each operand per thread per K step.  COV: element (row r of the tile, k) is x[k0 + k][i0 + r] - mu,
  // read along r (coalesced); KID: x[idx[i0 + r]][k0 + k], read along k
  double ra[8], rb[8];
  int64_t rowa[8], rowb[8];
  if (MODE == FS_KID) {
#pragma unroll
    for (int q = 0; q < 8; ++q) {
      const int r = (tid + FS_THREADS * q) >> 4;
      rowa[q] = i0 + r < rows ? ia[i0 + r] : -1;
      rowb[q] = j0 + r < rows ? ib[j0 + r] : -1;
    }
  }
  auto load = [&](int k0) {
#pragma unroll
    for (int q = 0; q < 8; ++q) {
      const int idx = tid + FS_THREADS * q;
      if (MODE == FS_COV) {
        const int r = idx & 63, k = k0 + (idx >> 6);
        ra[q] = (i0 + r < rows && k < K) ? __dsub_rn((double)__ldg(xa + (int64_t)k * a.d + i0 + r), a.mu[i0 + r]) : 0.0;
        rb[q] = (j0 + r < rows && k < K) ? __dsub_rn((double)__ldg(xb + (int64_t)k * a.d + j0 + r), a.mu[j0 + r]) : 0.0;
      } else {
        const int k = k0 + (idx & 15);
        ra[q] = (rowa[q] >= 0 && k < K) ? (double)__ldg(xa + rowa[q] * a.d + k) : 0.0;
        rb[q] = (rowb[q] >= 0 && k < K) ? (double)__ldg(xb + rowb[q] * a.d + k) : 0.0;
      }
    }
  };
  load(0);
  for (int k0 = 0; k0 < K; k0 += FS_K) {
    __syncthreads();
#pragma unroll
    for (int q = 0; q < 8; ++q) {
      const int idx = tid + FS_THREADS * q;
      const int r = MODE == FS_COV ? (idx & 63) : (idx >> 4), c = MODE == FS_COV ? (idx >> 6) : (idx & 15);
      As[r * FS_PITCH + c] = ra[q];
      Bs[r * FS_PITCH + c] = rb[q];
    }
    __syncthreads();
    if (k0 + FS_K < K) load(k0 + FS_K);
    double fa[2][8], fb[4][4];
#pragma unroll
    for (int mi = 0; mi < 2; ++mi)
#pragma unroll
      for (int v = 0; v < 8; ++v) fa[mi][v] = As[(wr + mi * 16 + g + 8 * (v & 1)) * FS_PITCH + t + 4 * (v >> 1)];
#pragma unroll
    for (int ni = 0; ni < 4; ++ni)
#pragma unroll
      for (int v = 0; v < 4; ++v) fb[ni][v] = Bs[(wc + ni * 8 + g) * FS_PITCH + t + 4 * v];
#pragma unroll
    for (int mi = 0; mi < 2; ++mi)
#pragma unroll
      for (int ni = 0; ni < 4; ++ni) dmma16816(acc[mi][ni], fa[mi], fb[ni]);
  }

  // accumulator element e of tile (mi, ni): row g + 8 (e >> 1), column 2 t + (e & 1)
  if (MODE == FS_COV) {
    const double inv = 1.0 / (double)(a.n - 1);
#pragma unroll
    for (int mi = 0; mi < 2; ++mi)
#pragma unroll
      for (int ni = 0; ni < 4; ++ni)
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          const int i = i0 + wr + mi * 16 + g + 8 * (e >> 1), j = j0 + wc + ni * 8 + 2 * t + (e & 1);
          if (i >= rows || j >= rows) continue;
          const double v = __dmul_rn(acc[mi][ni][e], inv);
          a.cov[(int64_t)i * a.d + j] = v;
          a.cov[(int64_t)j * a.d + i] = v;
        }
  } else {
    const double inv_d = 1.0 / (double)a.d;
    double s = 0.0;
#pragma unroll
    for (int mi = 0; mi < 2; ++mi)
#pragma unroll
      for (int ni = 0; ni < 4; ++ni)
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          const int i = i0 + wr + mi * 16 + g + 8 * (e >> 1), j = j0 + wc + ni * 8 + 2 * t + (e & 1);
          if (i >= rows || j >= rows || (kind != 2 && i == j)) continue;
          const double u = __dadd_rn(__dmul_rn(acc[mi][ni][e], inv_d), 1.0);
          s = __dadd_rn(s, __dmul_rn(__dmul_rn(u, u), u));
        }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) s = __dadd_rn(s, __shfl_xor_sync(0xffffffffu, s, o));
    if (lane == 0) red[warp] = s;
    __syncthreads();
    if (tid == 0)
      a.part[((int64_t)blockIdx.y * a.tiles + ti) * a.tiles + tj] =
          __dadd_rn(__dadd_rn(red[0], red[1]), __dadd_rn(red[2], red[3]));
  }
}

// t_s = (sum of the x x^T and y y^T tiles) / (m - 1) - 2 (sum of the x y^T tiles) / m, tiles added in order
__global__ void k_kid_reduce(const double* __restrict__ part, int tiles, int m, int subsets, double* __restrict__ terms) {
  const int s = blockIdx.x * blockDim.x + threadIdx.x;
  if (s >= subsets) return;
  const int tt = tiles * tiles;
  const double* p = part + (int64_t)s * 3 * tt;
  double sa = 0.0, sb = 0.0;
  for (int q = 0; q < 2 * tt; ++q) sa = __dadd_rn(sa, p[q]);
  for (int q = 0; q < tt; ++q) sb = __dadd_rn(sb, p[2 * tt + q]);
  terms[s] = __dsub_rn(__ddiv_rn(sa, (double)(m - 1)), __ddiv_rn(__dmul_rn(2.0, sb), (double)m));
}

__global__ void k_kid_check(const int64_t* __restrict__ idx, int64_t count, int64_t n, int* __restrict__ bad) {
  const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (i < count && (idx[i] < 0 || idx[i] >= n)) atomicOr(bad, 1);
}

bool has_device() {
  int ndev = 0;
  if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) {
    cudaGetLastError();
    return false;
  }
  return true;
}

}  // namespace
}  // namespace ds

extern "C" int ds_feature_stats(const float* feats_dev, int32_t n, int32_t d, double* mean_dev, double* cov_dev,
                                void* stream) {
  if (!feats_dev || !mean_dev || !cov_dev) return fail(DS_ERR_INVALID, "ds_feature_stats: NULL pointer");
  if (n < 2 || d < 1) return fail(DS_ERR_INVALID, "ds_feature_stats: n %d must be >= 2 and d %d >= 1", n, d);
  if (!has_device()) return fail(DS_ERR_NO_DEVICE, "no CUDA device: diffuscene_b200 has no CPU fallback");
  cudaStream_t s = (cudaStream_t)stream;
  k_fs_mean<<<(d + 31) / 32, 256, 0, s>>>(feats_dev, n, d, mean_dev);
  CK(cudaFuncSetAttribute(k_fs_tiles<FS_COV>, cudaFuncAttributeMaxDynamicSharedMemorySize, FS_SMEM));
  FsArgs a = {};
  a.x = a.y = feats_dev; a.mu = mean_dev; a.n = n; a.d = d;
  a.tiles = (d + FS_T - 1) / FS_T;
  a.cov = cov_dev;
  k_fs_tiles<FS_COV><<<a.tiles * (a.tiles + 1) / 2, FS_THREADS, FS_SMEM, s>>>(a);
  CK(cudaGetLastError());
  return 0;
}

extern "C" int ds_kid_terms(const float* real_dev, int32_t n_real, const float* fake_dev, int32_t n_fake, int32_t d,
                            const int64_t* idx_fake_dev, const int64_t* idx_real_dev, int32_t subsets, int32_t m,
                            double* terms_dev, void* stream) {
  if (!real_dev || !fake_dev || !idx_fake_dev || !idx_real_dev || !terms_dev)
    return fail(DS_ERR_INVALID, "ds_kid_terms: NULL pointer");
  if (m < 2 || subsets < 1 || d < 1 || n_real < m || n_fake < m)
    return fail(DS_ERR_INVALID, "ds_kid_terms: m %d must be >= 2 and <= n_real %d, n_fake %d; subsets %d, d %d >= 1", m,
                n_real, n_fake, subsets, d);
  if ((int64_t)subsets * 3 > 65535) return fail(DS_ERR_INVALID, "ds_kid_terms: %d subsets > 21845", subsets);
  if (!has_device()) return fail(DS_ERR_NO_DEVICE, "no CUDA device: diffuscene_b200 has no CPU fallback");
  cudaStream_t s = (cudaStream_t)stream;
  const int64_t cnt = (int64_t)subsets * m;
  const int tiles = (m + FS_T - 1) / FS_T;
  int* bad = nullptr;
  double* part = nullptr;
  CK(cudaMallocAsync((void**)&bad, 4, s));
  cudaError_t e = cudaMallocAsync((void**)&part, (size_t)subsets * 3 * tiles * tiles * 8, s);
  if (e != cudaSuccess) {
    cudaFreeAsync(bad, s);
    return fail(DS_ERR_CUDA, "ds_kid_terms: tile sums of %d subsets: %s", subsets, cudaGetErrorString(e));
  }
  int rc = 0, h_bad = 0;
  e = cudaMemsetAsync(bad, 0, 4, s);
  if (e == cudaSuccess) {
    k_kid_check<<<(unsigned)((cnt + 255) / 256), 256, 0, s>>>(idx_fake_dev, cnt, n_fake, bad);
    k_kid_check<<<(unsigned)((cnt + 255) / 256), 256, 0, s>>>(idx_real_dev, cnt, n_real, bad);
    e = cudaMemcpyAsync(&h_bad, bad, 4, cudaMemcpyDeviceToHost, s);
  }
  if (e == cudaSuccess) e = cudaStreamSynchronize(s);
  if (e != cudaSuccess) rc = fail(DS_ERR_CUDA, "ds_kid_terms: index check: %s", cudaGetErrorString(e));
  else if (h_bad) rc = fail(DS_ERR_INVALID, "ds_kid_terms: a subset index lies outside its feature set");
  if (!rc) {
    e = cudaFuncSetAttribute(k_fs_tiles<FS_KID>, cudaFuncAttributeMaxDynamicSharedMemorySize, FS_SMEM);
    if (e == cudaSuccess) {
      FsArgs a = {};
      a.x = fake_dev; a.y = real_dev; a.ix = idx_fake_dev; a.iy = idx_real_dev;
      a.d = d; a.m = m; a.tiles = tiles; a.part = part;
      k_fs_tiles<FS_KID><<<dim3(tiles * tiles, subsets * 3), FS_THREADS, FS_SMEM, s>>>(a);
      k_kid_reduce<<<(subsets + 127) / 128, 128, 0, s>>>(part, tiles, m, subsets, terms_dev);
      e = cudaGetLastError();
    }
    if (e != cudaSuccess) rc = fail(DS_ERR_CUDA, "ds_kid_terms: %s", cudaGetErrorString(e));
  }
  cudaFreeAsync(part, s);
  cudaFreeAsync(bad, s);
  return rc;
}
