// k-NN manifold metrics of improved precision and recall (reference scripts/improved_precision_recall.py:228-305):
// pairwise Euclidean distances of feature vectors in fp64, never held as an N x N matrix.
//
// One kernel computes 64 x 64 tiles of X Y^T on the fp64 tensor cores (mma.sync m16n8k16 .f64, DMMA.16x8x16 on
// sm_90a), turns them into distances exactly as compute_pairwise_distances does (d2 = (|x|^2 - 2 x.y) + |y|^2, negative
// d2 counted and set to 0, d = sqrt(d2), every step rounded to nearest in fp64, no contraction), stages the tile in
// shared memory and hands it to one of three epilogues:
//   DIST   writes the distances (small inputs and tests only);
//   RADII  keeps, per row, the 17 smallest distances seen over the CTA's column range; a second kernel merges the
//          column splits and returns the (k+1)-th smallest (distances2radii / get_kth_value, the row's ~0 self
//          distance counted);
//   COVER  one pass over reference x subject pairs: subject j is covered when some reference i has d < radius_i
//          (compute_metric, strict), reference i is covered when some subject j has d < radius_j (the other
//          direction), and realism_j = max_i radius_i / (d + 1e-6), d taken from the difference itself for
//          near-duplicate pairs (the reference's realism uses norm(real_i - f), not the expansion).
// Flags are plain stores of 1 and the realism maximum is an integer atomic max on the bits of a non-negative double,
// so every output is independent of scheduling.  Operands are read as given (fp64, any D >= 1): the K and row tails
// are zero-filled while the tiles are loaded.
#include "engine_internal.h"

namespace ds {
namespace {

constexpr int MF_T = 64;                  // tile rows and columns
constexpr int MF_K = 16;                  // K step (one DMMA)
constexpr int MF_PITCH = MF_K + 4;        // doubles; half-warp fragment loads hit distinct banks
constexpr int MF_DPITCH = MF_T + 1;       // distance tile pitch
constexpr int MF_THREADS = 128;           // 4 warps, 2 x 2, 32 x 32 each
constexpr int MF_LIST = DS_MANIFOLD_MAX_K + 1;
constexpr int MF_SMEM = (2 * MF_T * MF_PITCH + MF_T * MF_DPITCH + 2 * MF_T) * 8;
enum { EPI_DIST = 0, EPI_RADII = 1, EPI_COVER = 2 };

__device__ __forceinline__ void dmma16816(double (&d)[4], const double (&a)[8], const double (&b)[4]) {
  asm volatile(
      "mma.sync.aligned.m16n8k16.row.col.f64.f64.f64.f64 {%0, %1, %2, %3}, {%4, %5, %6, %7, %8, %9, %10, %11}, "
      "{%12, %13, %14, %15}, {%0, %1, %2, %3};"
      : "+d"(d[0]), "+d"(d[1]), "+d"(d[2]), "+d"(d[3])
      : "d"(a[0]), "d"(a[1]), "d"(a[2]), "d"(a[3]), "d"(a[4]), "d"(a[5]), "d"(a[6]), "d"(a[7]), "d"(b[0]), "d"(b[1]),
        "d"(b[2]), "d"(b[3]));
}

// ascending list of the MF_LIST smallest values inserted so far (a multiset: ties are kept)
__device__ __forceinline__ void list_insert(double (&l)[MF_LIST], double v) {
  if (!(v < l[MF_LIST - 1])) return;
#pragma unroll
  for (int q = MF_LIST - 1; q >= 1; --q) l[q] = v < l[q - 1] ? l[q - 1] : (v < l[q] ? v : l[q]);
  l[0] = v < l[0] ? v : l[0];
}

__global__ void k_mf_sqnorm(const double* __restrict__ x, int n, int d, double* __restrict__ out) {
  const int row = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (row >= n) return;
  const double* xr = x + (int64_t)row * d;
  double s = 0.0;
  for (int k = lane; k < d; k += 32) s = __dadd_rn(s, __dmul_rn(xr[k], xr[k]));
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) s = __dadd_rn(s, __shfl_xor_sync(0xffffffffu, s, o));
  if (lane == 0) out[row] = s;
}

// |x_i - y_j| from the difference, fp64 (one thread; only for the rare near-duplicate pairs of the realism ratio)
__device__ double direct_dist(const double* x, const double* y, int i, int j, int d) {
  const double* xi = x + (int64_t)i * d;
  const double* yj = y + (int64_t)j * d;
  double s = 0.0;
  for (int k = 0; k < d; ++k) {
    const double t = __dsub_rn(__ldg(xi + k), __ldg(yj + k));
    s = __fma_rn(t, t, s);
  }
  return __dsqrt_rn(s);
}

struct MfArgs {
  const double *x, *y, *nx, *ny;        // rows of the tile come from x, columns from y
  int n, m, d;
  int col_tiles_per_split;
  double* dist;                          // DIST: [n][m]
  double* part;                          // RADII: [splits * 2][n][MF_LIST]
  const double *rx, *ry;                 // COVER: radii of x rows / of y rows (ry may be null)
  uint8_t *y_cov, *x_cov;                // COVER: y_cov[j] = some x row covers j; x_cov[i] = some y row covers i
  double* realism;                       // COVER: [m] (bits of non-negative doubles, atomic max), may be null
  unsigned long long* clamped;           // negative d2 count, may be null
};

template <int EPI>
__global__ void __launch_bounds__(MF_THREADS) k_mf_tiles(MfArgs a) {
  extern __shared__ double sm[];
  double* As = sm;                                   // [64][MF_PITCH]
  double* Bs = As + MF_T * MF_PITCH;                 // [64][MF_PITCH]
  double* Ds = Bs + MF_T * MF_PITCH;                 // [64][MF_DPITCH]
  double* snx = Ds + MF_T * MF_DPITCH;               // [64]
  double* sny = snx + MF_T;                          // [64]
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, g = lane >> 2, t = lane & 3;
  const int wr = (warp >> 1) * 32, wc = (warp & 1) * 32;
  const int i0 = blockIdx.x * MF_T;
  const int ct_total = (a.m + MF_T - 1) / MF_T;
  const int ct_lo = blockIdx.y * a.col_tiles_per_split;
  const int ct_hi = min(ct_total, ct_lo + a.col_tiles_per_split);
  unsigned long long clamped = 0;

  // RADII: two threads per row, each over 32 columns of every tile
  const int er = tid >> 1, eh = tid & 1;
  double lst[MF_LIST];
  if (EPI == EPI_RADII) {
#pragma unroll
    for (int q = 0; q < MF_LIST; ++q) lst[q] = INFINITY;
  }
  int x_hit = 0;                                     // COVER: row er is covered (this thread's half of the columns)

  if (tid < MF_T) snx[tid] = i0 + tid < a.n ? a.nx[i0 + tid] : 0.0;

  for (int ct = ct_lo; ct < ct_hi; ++ct) {
    const int j0 = ct * MF_T;
    __syncthreads();                                 // previous tile's epilogue is done with Ds / sny
    if (tid < MF_T) sny[tid] = j0 + tid < a.m ? a.ny[j0 + tid] : 0.0;
    double acc[2][4][4];
#pragma unroll
    for (int mi = 0; mi < 2; ++mi)
#pragma unroll
      for (int ni = 0; ni < 4; ++ni)
#pragma unroll
        for (int e = 0; e < 4; ++e) acc[mi][ni][e] = 0.0;

    // each thread loads 8 elements of each operand per K step: idx = tid + 128 q, row idx / 16, column idx % 16
    double ra[8], rb[8];
    auto load = [&](int k0) {
#pragma unroll
      for (int q = 0; q < 8; ++q) {
        const int idx = tid + MF_THREADS * q, r = idx >> 4, c = k0 + (idx & 15);
        ra[q] = (i0 + r < a.n && c < a.d) ? __ldg(a.x + (int64_t)(i0 + r) * a.d + c) : 0.0;
        rb[q] = (j0 + r < a.m && c < a.d) ? __ldg(a.y + (int64_t)(j0 + r) * a.d + c) : 0.0;
      }
    };
    load(0);
    for (int k0 = 0; k0 < a.d; k0 += MF_K) {
      __syncthreads();
#pragma unroll
      for (int q = 0; q < 8; ++q) {
        const int idx = tid + MF_THREADS * q, r = idx >> 4, c = idx & 15;
        As[r * MF_PITCH + c] = ra[q];
        Bs[r * MF_PITCH + c] = rb[q];
      }
      __syncthreads();
      if (k0 + MF_K < a.d) load(k0 + MF_K);          // next step's loads in flight during the MMAs
      double fa[2][8], fb[4][4];
#pragma unroll
      for (int mi = 0; mi < 2; ++mi)
#pragma unroll
        for (int v = 0; v < 8; ++v)
          fa[mi][v] = As[(wr + mi * 16 + g + 8 * (v & 1)) * MF_PITCH + t + 4 * (v >> 1)];
#pragma unroll
      for (int ni = 0; ni < 4; ++ni)
#pragma unroll
        for (int v = 0; v < 4; ++v) fb[ni][v] = Bs[(wc + ni * 8 + g) * MF_PITCH + t + 4 * v];
#pragma unroll
      for (int mi = 0; mi < 2; ++mi)
#pragma unroll
        for (int ni = 0; ni < 4; ++ni) dmma16816(acc[mi][ni], fa[mi], fb[ni]);
    }

    // distances: accumulator element e of tile (mi, ni) is row g + 8 (e >> 1), column 2 t + (e & 1)
#pragma unroll
    for (int mi = 0; mi < 2; ++mi)
#pragma unroll
      for (int ni = 0; ni < 4; ++ni)
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          const int r = wr + mi * 16 + g + 8 * (e >> 1), c = wc + ni * 8 + 2 * t + (e & 1);
          double d2 = __dadd_rn(__dsub_rn(snx[r], __dmul_rn(2.0, acc[mi][ni][e])), sny[c]);
          if (d2 < 0.0) {
            if (i0 + r < a.n && j0 + c < a.m) ++clamped;
            d2 = 0.0;
          }
          Ds[r * MF_DPITCH + c] = __dsqrt_rn(d2);
        }
    __syncthreads();

    if (EPI == EPI_DIST) {
      for (int idx = tid; idx < MF_T * MF_T; idx += MF_THREADS) {
        const int r = idx / MF_T, c = idx % MF_T;
        if (i0 + r < a.n && j0 + c < a.m) a.dist[(int64_t)(i0 + r) * a.m + j0 + c] = Ds[r * MF_DPITCH + c];
      }
    } else if (EPI == EPI_RADII) {
      const int cn = min(32, a.m - j0 - 32 * eh);
      for (int c = 0; c < cn; ++c) list_insert(lst, Ds[er * MF_DPITCH + 32 * eh + c]);
    } else {
      // columns: subject j = j0 + er is covered by some reference row among this thread's 32 rows
      const int jj = j0 + er;
      if (jj < a.m) {
        const int rn = min(32, a.n - i0 - 32 * eh);
        bool hit = false;
        double best = 0.0;
        for (int r = 0; r < rn; ++r) {
          const int rr = 32 * eh + r;
          const double dd = Ds[rr * MF_DPITCH + er], rad = a.rx[i0 + rr];
          hit |= dd < rad;
          if (a.realism) {
            // near-duplicate pairs: the expansion leaves sqrt(rounding of |x|^2 + |y|^2) instead of ~0, which the
            // 1e-6 of the ratio would not absorb; the reference's norm(real_i - f) is recomputed directly there
            double dr = dd;
            if (__dmul_rn(dd, dd) < 0x1p-20 * (snx[rr] + sny[er])) dr = direct_dist(a.x, a.y, i0 + rr, jj, a.d);
            best = fmax(best, __ddiv_rn(rad, __dadd_rn(dr, 1e-6)));
          }
        }
        if (hit && a.y_cov) a.y_cov[jj] = 1;
        if (a.realism && rn > 0)
          atomicMax(reinterpret_cast<unsigned long long*>(a.realism + jj), (unsigned long long)__double_as_longlong(best));
      }
      // rows: reference i = i0 + er is covered by some subject column among this thread's 32 columns
      if (a.ry && i0 + er < a.n) {
        const int cn = min(32, a.m - j0 - 32 * eh);
        for (int c = 0; c < cn; ++c) x_hit |= Ds[er * MF_DPITCH + 32 * eh + c] < a.ry[j0 + 32 * eh + c];
      }
    }
  }

  if (EPI == EPI_RADII && i0 + er < a.n) {
    double* p = a.part + ((int64_t)(blockIdx.y * 2 + eh) * a.n + i0 + er) * MF_LIST;
#pragma unroll
    for (int q = 0; q < MF_LIST; ++q) p[q] = lst[q];
  }
  if (EPI == EPI_COVER && x_hit && a.x_cov) a.x_cov[i0 + er] = 1;
  if (a.clamped) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) clamped += __shfl_xor_sync(0xffffffffu, clamped, o);
    if (lane == 0 && clamped) atomicAdd(a.clamped, clamped);
  }
}

// radii[i] = the (k+1)-th smallest of the 2 x splits partial lists of row i
__global__ void k_mf_radii_merge(const double* __restrict__ part, int n, int lists, int k, double* __restrict__ radii) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  double lst[MF_LIST];
#pragma unroll
  for (int q = 0; q < MF_LIST; ++q) lst[q] = INFINITY;
  for (int s = 0; s < lists; ++s) {
    const double* p = part + ((int64_t)s * n + i) * MF_LIST;
    for (int q = 0; q < MF_LIST; ++q) list_insert(lst, p[q]);
  }
  radii[i] = lst[k];
}

template <int EPI>
int run_tiles(MfArgs a, int splits, cudaStream_t s) {
  // set on every call: the attribute is per device, and the call may run on any device
  CK(cudaFuncSetAttribute(k_mf_tiles<EPI>, cudaFuncAttributeMaxDynamicSharedMemorySize, MF_SMEM));
  const int ct_total = (a.m + MF_T - 1) / MF_T;
  a.col_tiles_per_split = (ct_total + splits - 1) / splits;
  k_mf_tiles<EPI><<<dim3((a.n + MF_T - 1) / MF_T, splits), MF_THREADS, MF_SMEM, s>>>(a);
  CK(cudaGetLastError());
  return 0;
}

// norms of x (and y) into a scratch block [n (+ m)] allocated on the stream
int norms(const double* x, int n, const double* y, int m, int d, double** out, cudaStream_t s) {
  CK(cudaMallocAsync((void**)out, (size_t)(n + m) * 8, s));
  k_mf_sqnorm<<<(n + 7) / 8, 256, 0, s>>>(x, n, d, *out);
  if (y) k_mf_sqnorm<<<(m + 7) / 8, 256, 0, s>>>(y, m, d, *out + n);
  CK(cudaGetLastError());
  return 0;
}

}  // namespace
}  // namespace ds

extern "C" int ds_manifold_distances(const double* x_dev, int32_t n, const double* y_dev, int32_t m, int32_t d,
                                     double* out_dev, int64_t* clamped_dev, void* stream) {
  if (!x_dev || !y_dev || !out_dev) return fail(DS_ERR_INVALID, "ds_manifold_distances: NULL x, y or out pointer");
  if (n < 1 || m < 1 || d < 1)
    return fail(DS_ERR_INVALID, "ds_manifold_distances: n %d, m %d and d %d must be >= 1", n, m, d);
  if (const int rc = require_device()) return rc;
  cudaStream_t s = (cudaStream_t)stream;
  if (clamped_dev) CK(cudaMemsetAsync(clamped_dev, 0, 8, s));
  double* nrm = nullptr;
  int rc = norms(x_dev, n, y_dev, m, d, &nrm, s);
  if (rc) return rc;
  MfArgs a = {};
  a.x = x_dev; a.y = y_dev; a.nx = nrm; a.ny = nrm + n; a.n = n; a.m = m; a.d = d;
  a.dist = out_dev;
  a.clamped = (unsigned long long*)clamped_dev;
  rc = run_tiles<EPI_DIST>(a, 1, s);
  cudaFreeAsync(nrm, s);
  return rc;
}

extern "C" int ds_manifold_radii(const double* x_dev, int32_t n, int32_t d, int32_t k, double* radii_dev,
                                 int64_t* clamped_dev, void* stream) {
  if (!x_dev || !radii_dev) return fail(DS_ERR_INVALID, "ds_manifold_radii: NULL features or radii pointer");
  if (k < 1 || k > DS_MANIFOLD_MAX_K) return fail(DS_ERR_INVALID, "ds_manifold_radii: k %d outside [1, %d]", k, DS_MANIFOLD_MAX_K);
  if (n <= k) return fail(DS_ERR_INVALID, "ds_manifold_radii: %d features, need more than k = %d", n, k);
  if (d < 1) return fail(DS_ERR_INVALID, "ds_manifold_radii: feature size %d < 1", d);
  if (const int rc = require_device()) return rc;
  cudaStream_t s = (cudaStream_t)stream;
  if (clamped_dev) CK(cudaMemsetAsync(clamped_dev, 0, 8, s));
  int dev = 0, sms = 132;
  cudaGetDevice(&dev);
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  // column splits so that small N still fills the device: k_mf_tiles holds 2 CTAs per SM (about 224 registers x
  // 128 threads)
  const int rt = (n + MF_T - 1) / MF_T;
  const int splits = std::max(1, std::min(rt, (2 * sms + rt - 1) / rt));
  double* nrm = nullptr;
  int rc = norms(x_dev, n, nullptr, 0, d, &nrm, s);
  if (rc) return rc;
  double* part = nullptr;
  cudaError_t e = cudaMallocAsync((void**)&part, (size_t)splits * 2 * n * MF_LIST * 8, s);
  if (e != cudaSuccess) {
    cudaFreeAsync(nrm, s);
    return fail(DS_ERR_CUDA, "ds_manifold_radii: partial lists (%d splits): %s", splits, cudaGetErrorString(e));
  }
  MfArgs a = {};
  a.x = x_dev; a.y = x_dev; a.nx = nrm; a.ny = nrm; a.n = n; a.m = n; a.d = d;
  a.part = part;
  a.clamped = (unsigned long long*)clamped_dev;
  rc = run_tiles<EPI_RADII>(a, splits, s);
  if (!rc) {
    k_mf_radii_merge<<<(n + 127) / 128, 128, 0, s>>>(part, n, 2 * splits, k, radii_dev);
    e = cudaGetLastError();
    if (e != cudaSuccess) rc = fail(DS_ERR_CUDA, "ds_manifold_radii: %s", cudaGetErrorString(e));
  }
  cudaFreeAsync(part, s);
  cudaFreeAsync(nrm, s);
  return rc;
}

extern "C" int ds_manifold_cover(const double* ref_dev, const double* ref_radii_dev, int32_t n_ref,
                                 const double* subj_dev, const double* subj_radii_dev, int32_t n_subj, int32_t d,
                                 uint8_t* subj_covered_dev, uint8_t* ref_covered_dev, double* realism_dev,
                                 int64_t* clamped_dev, void* stream) {
  if (!ref_dev || !ref_radii_dev || !subj_dev)
    return fail(DS_ERR_INVALID, "ds_manifold_cover: NULL reference features, reference radii or subject features");
  if (ref_covered_dev && !subj_radii_dev)
    return fail(DS_ERR_INVALID, "ds_manifold_cover: reference coverage needs the subject radii");
  if (n_ref < 1 || n_subj < 1 || d < 1)
    return fail(DS_ERR_INVALID, "ds_manifold_cover: n_ref %d, n_subj %d and d %d must be >= 1", n_ref, n_subj, d);
  if (const int rc = require_device()) return rc;
  cudaStream_t s = (cudaStream_t)stream;
  if (clamped_dev) CK(cudaMemsetAsync(clamped_dev, 0, 8, s));
  if (subj_covered_dev) CK(cudaMemsetAsync(subj_covered_dev, 0, n_subj, s));
  if (ref_covered_dev) CK(cudaMemsetAsync(ref_covered_dev, 0, n_ref, s));
  if (realism_dev) CK(cudaMemsetAsync(realism_dev, 0, (size_t)n_subj * 8, s));      // +0.0: below every ratio
  double* nrm = nullptr;
  int rc = norms(ref_dev, n_ref, subj_dev, n_subj, d, &nrm, s);
  if (rc) return rc;
  MfArgs a = {};
  a.x = ref_dev; a.y = subj_dev; a.nx = nrm; a.ny = nrm + n_ref; a.n = n_ref; a.m = n_subj; a.d = d;
  a.rx = ref_radii_dev; a.ry = ref_covered_dev ? subj_radii_dev : nullptr;
  a.y_cov = subj_covered_dev; a.x_cov = ref_covered_dev; a.realism = realism_dev;
  a.clamped = (unsigned long long*)clamped_dev;
  rc = run_tiles<EPI_COVER>(a, 1, s);
  cudaFreeAsync(nrm, s);
  return rc;
}
