// Object shape auto-encoder: the reference's `KLAutoEncoder` (scene_synthesis/networks/foldingnet_autoencoder.py:131-390,
// a FoldingNet with a KL latent head) and its Chamfer loss (ChamferDistancePytorch/chamfer3D), forward and backward,
// fp32, behind its own handle (ds_shape_ae_*).  It shares no state with the denoiser's handle.
//
// Activations are point-major rows like the rest of the library: row = (object, point), columns = channels.  Every
// 1x1 conv and linear layer is one of the library's fp32 GEMMs (k_gemm_simt forward, k_gemm_nn / k_gemm_tn / k_colsum
// backward).  The kernels here are the rest:
//   kNN           k_sae_knn: fused distance + top-16, candidates streamed through shared memory, the list on chip
//   covariances   k_sae_cov: the 12-channel encoder input (xyz + 3x3 neighbourhood scatter)
//   local max     k_sae_nbr_max and its adjoint k_sae_nbr_max_bwd, a gather over the reverse kNN graph (CSR)
//   BatchNorm1d   k_bn_partial / k_bn_final / k_bn_apply (train: batch statistics in fixed order, running update;
//                 eval: running statistics) and the train-mode adjoint k_bn_bwd_partial / k_bn_bwd_final / k_bn_bwd_apply
//   global max    k_sae_gmax (first maximum over the points) and its adjoint
//   latent head   k_sae_latent (clamp, reparameterisation with caller-supplied eps, KL) and its adjoint
//   folding       k_sae_fold_in: W [g; code] + b = W_g g + (W_c code + b) without the 514 / 515-wide concat;
//                 k_sae_objsum sums dY over an object's rows for the adjoint
//   Chamfer       k_chamfer_nn (first minimum, strict <) and k_chamfer_grad (gather, fixed order, no atomics)
//   loss          k_sae_loss
// Every reduction runs in a fixed order, so an object's outputs and the gradients do not depend on scheduling (the
// dW GEMMs excepted: k_gemm_tn splits its row sum over CTAs with fp32 atomics).
#include "engine_internal.h"

namespace ds {
// backward.cu
template <typename TA, typename TB, typename TD>
void launch_gemm_nn(const TA* A, int lda, const TB* B, int ldb, TD* D, int ldd, int M, int N, int K, int accumulate, cudaStream_t s);
template <typename TA, typename TB>
void launch_gemm_tn(const TA* A, int lda, const TB* B, int ldb, float* D, int ldd, int M, int Ka, int Kb, cudaStream_t s);
template <typename T> void launch_colsum(const T* A, int lda, float* out, int M, int N, cudaStream_t s);
}  // namespace ds

namespace {
constexpr int KNN = 16;              // neighbours per point in all three kNN stages
constexpr int GRID_SIDE = 45;
constexpr int GRID_M = GRID_SIDE * GRID_SIDE;      // decoder points per object
constexpr float BN_EPS = 1e-5f, BN_MOMENTUM = 0.1f;
constexpr int BN_ROWS = 256;         // rows per partial-statistics chunk

// ---- kNN ------------------------------------------------------------------------------------------------------------
// One thread per query point, QT queries per CTA; candidate tiles of JT points are staged in shared memory.  Distances
// are sum_c (q_c - x_c)^2 accumulated in channel order with fmaf; CP is C rounded up to 4 (padding channels are 0).
// The list is kept sorted ascending; a candidate enters only when strictly closer than the 16th, and candidates arrive
// in index order, so equal distances keep the lower index first.
template <int CP, int QT, int JT>
__global__ void __launch_bounds__(QT) k_sae_knn(const float* __restrict__ x, int P, int C, int* __restrict__ idx) {
  constexpr int QP = CP + 4;
  __shared__ __align__(16) float qs[QT * QP];
  __shared__ __align__(16) float cs[JT * CP];
  const int b = blockIdx.y, q0 = blockIdx.x * QT, t = threadIdx.x;
  const float* xb = x + (int64_t)b * P * C;
  for (int e = t; e < QT * CP; e += QT) {
    const int r = e / CP, c = e % CP;
    qs[r * QP + c] = (q0 + r < P && c < C) ? xb[(int64_t)(q0 + r) * C + c] : 0.f;
  }
  float bd[KNN];
  int bi[KNN];
#pragma unroll
  for (int k = 0; k < KNN; ++k) { bd[k] = INFINITY; bi[k] = 0; }
  for (int j0 = 0; j0 < P; j0 += JT) {
    __syncthreads();
    for (int e = t; e < JT * CP; e += QT) {
      const int r = e / CP, c = e % CP;
      cs[e] = (j0 + r < P && c < C) ? xb[(int64_t)(j0 + r) * C + c] : 0.f;
    }
    __syncthreads();
    float d[JT];
#pragma unroll
    for (int jj = 0; jj < JT; ++jj) d[jj] = 0.f;
#pragma unroll 2
    for (int c = 0; c < CP; c += 4) {
      const float4 q = *reinterpret_cast<const float4*>(&qs[t * QP + c]);
#pragma unroll
      for (int jj = 0; jj < JT; ++jj) {
        const float4 v = *reinterpret_cast<const float4*>(&cs[jj * CP + c]);
        float u = q.x - v.x; d[jj] = fmaf(u, u, d[jj]);
        u = q.y - v.y; d[jj] = fmaf(u, u, d[jj]);
        u = q.z - v.z; d[jj] = fmaf(u, u, d[jj]);
        u = q.w - v.w; d[jj] = fmaf(u, u, d[jj]);
      }
    }
    const int jn = min(JT, P - j0);
#pragma unroll
    for (int jj = 0; jj < JT; ++jj) {
      if (jj < jn && d[jj] < bd[KNN - 1]) {
        bd[KNN - 1] = d[jj];
        bi[KNN - 1] = j0 + jj;
#pragma unroll
        for (int k = KNN - 1; k > 0; --k)
          if (bd[k] < bd[k - 1]) {
            const float td = bd[k]; bd[k] = bd[k - 1]; bd[k - 1] = td;
            const int ti = bi[k]; bi[k] = bi[k - 1]; bi[k - 1] = ti;
          }
      }
    }
  }
  if (q0 + t < P) {
    int* o = idx + ((int64_t)b * P + q0 + t) * KNN;
#pragma unroll
    for (int k = 0; k < KNN; ++k) o[k] = bi[k];
  }
}

void launch_knn(const float* x, int B, int P, int C, int* idx, cudaStream_t s) {
  if (C <= 4) {
    k_sae_knn<4, 128, 32><<<dim3(ceil_div(P, 128), B), 128, 0, s>>>(x, P, C, idx);
  } else if (C <= 64) {
    k_sae_knn<64, 64, 16><<<dim3(ceil_div(P, 64), B), 64, 0, s>>>(x, P, C, idx);
  } else {
    k_sae_knn<128, 64, 16><<<dim3(ceil_div(P, 64), B), 64, 0, s>>>(x, P, C, idx);
  }
}

// ---- encoder input: xyz + the 3x3 scatter of the centred neighbourhood (foldingnet_autoencoder.py:186-192) -----------
__global__ void k_sae_cov(const float* __restrict__ pts, const int* __restrict__ idx, int P, float* __restrict__ out,
                          int64_t R) {
  const int64_t r = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (r >= R) return;
  const float* pb = pts + (r / P) * P * 3;
  float nb[KNN][3];
  float mean[3] = {0.f, 0.f, 0.f};
#pragma unroll
  for (int k = 0; k < KNN; ++k) {
    const int j = idx[r * KNN + k];
#pragma unroll
    for (int c = 0; c < 3; ++c) { nb[k][c] = pb[j * 3 + c]; mean[c] += nb[k][c]; }
  }
#pragma unroll
  for (int c = 0; c < 3; ++c) mean[c] /= float(KNN);
#pragma unroll
  for (int k = 0; k < KNN; ++k)
#pragma unroll
    for (int c = 0; c < 3; ++c) nb[k][c] -= mean[c];
  float* o = out + r * 12;
#pragma unroll
  for (int c = 0; c < 3; ++c) o[c] = pts[r * 3 + c];
#pragma unroll
  for (int i = 0; i < 3; ++i)
#pragma unroll
    for (int j = 0; j < 3; ++j) {
      float acc = 0.f;
#pragma unroll
      for (int k = 0; k < KNN; ++k) acc = fmaf(nb[k][i], nb[k][j], acc);
      o[3 + i * 3 + j] = acc;
    }
}

// ---- local max pooling over the kNN neighbourhood (GraphLayer, :150-154) ----------------------------------------------
// out[i, c] = max_k y[idx[i, k], c]; am[i, c] = the first k holding the maximum (torch's rule for the adjoint)
__global__ void k_sae_nbr_max(const float* __restrict__ y, const int* __restrict__ idx, int P, int C,
                              float* __restrict__ out, uint8_t* __restrict__ am, int64_t n) {
  const int64_t e = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (e >= n) return;
  const int c = int(e % C);
  const int64_t r = e / C;
  const float* yb = y + (r / P) * P * (int64_t)C + c;
  const int* nb = idx + r * KNN;
  float best = yb[(int64_t)nb[0] * C];
  int arg = 0;
#pragma unroll
  for (int k = 1; k < KNN; ++k) {
    const float v = yb[(int64_t)nb[k] * C];
    if (v > best) { best = v; arg = k; }
  }
  out[e] = best;
  am[e] = (uint8_t)arg;
}
// adjoint as a gather over the reverse kNN graph: dy[j, c] = sum over the entries (i, k) with idx[i, k] = j (ascending)
// whose argmax is k, of dm[i, c]
__global__ void k_sae_nbr_max_bwd(const float* __restrict__ dm, const uint8_t* __restrict__ am,
                                  const int* __restrict__ start, const int* __restrict__ list, int P, int C,
                                  float* __restrict__ dy, int64_t n) {
  const int64_t e = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (e >= n) return;
  const int c = int(e % C);
  const int64_t j = e / C;
  const int64_t base = (j / P) * P;
  float acc = 0.f;
  for (int q = start[j]; q < start[j + 1]; ++q) {
    const int src = list[q];
    const int64_t i = base + (src >> 4);
    if (am[i * C + c] == (src & (KNN - 1))) acc += dm[i * C + c];
  }
  dy[e] = acc;
}

// ---- reverse kNN graph: CSR over the targets, entries sorted by source (i * 16 + k) -----------------------------------
__global__ void k_csr_count(const int* __restrict__ idx, int per_obj, int m, int* __restrict__ cnt, int64_t n) {
  const int64_t e = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (e >= n) return;
  atomicAdd(cnt + (e / per_obj) * m + idx[e], 1);
}
// one CTA (1024 threads) per object: exclusive scan of the object's m counts; start[] holds global entry offsets
__global__ void __launch_bounds__(1024) k_csr_scan(const int* __restrict__ cnt, int m, int per_obj, int n_obj,
                                                   int* __restrict__ start, int* __restrict__ cursor) {
  __shared__ int part[1024];
  const int b = blockIdx.x, t = threadIdx.x;
  const int chunk = (m + 1023) / 1024;
  const int lo = min(m, t * chunk), hi = min(m, lo + chunk);
  const int* cb = cnt + (int64_t)b * m;
  int s = 0;
  for (int j = lo; j < hi; ++j) s += cb[j];
  part[t] = s;
  __syncthreads();
  for (int o = 1; o < 1024; o <<= 1) {
    const int v = t >= o ? part[t - o] : 0;
    __syncthreads();
    part[t] += v;
    __syncthreads();
  }
  int run = (int)((int64_t)b * per_obj) + part[t] - s;
  for (int j = lo; j < hi; ++j) {
    start[(int64_t)b * m + j] = run;
    cursor[(int64_t)b * m + j] = run;
    run += cb[j];
  }
  if (b == n_obj - 1 && t == 0) start[(int64_t)n_obj * m] = n_obj * per_obj;
}
__global__ void k_csr_fill(const int* __restrict__ idx, int per_obj, int m, int* __restrict__ cursor,
                           int* __restrict__ list, int64_t n) {
  const int64_t e = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (e >= n) return;
  const int64_t b = e / per_obj;
  const int pos = atomicAdd(cursor + b * m + idx[e], 1);
  list[pos] = int(e - b * per_obj);
}
__global__ void k_csr_sort(const int* __restrict__ start, int* __restrict__ list, int64_t n_targets) {
  const int64_t j = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (j >= n_targets) return;
  const int lo = start[j], hi = start[j + 1];
  for (int a = lo + 1; a < hi; ++a) {
    const int v = list[a];
    int q = a - 1;
    while (q >= lo && list[q] > v) { list[q + 1] = list[q]; --q; }
    list[q + 1] = v;
  }
}

// ---- BatchNorm1d ----------------------------------------------------------------------------------------------------
// partial column sums over chunks of BN_ROWS rows: part[chunk][c] = sum (x - shift[c]) (sq: squared); block 32 x 8
__global__ void __launch_bounds__(256) k_bn_partial(const float* __restrict__ x, int64_t R, int C,
                                                    const float* __restrict__ shift, int sq, float* __restrict__ part) {
  __shared__ float red[8][33];
  const int c = blockIdx.x * 32 + threadIdx.x, ty = threadIdx.y;
  const int64_t r0 = (int64_t)blockIdx.y * BN_ROWS, r1 = min(R, r0 + BN_ROWS);
  float s = 0.f;
  if (c < C) {
    const float sh = shift ? shift[c] : 0.f;
    for (int64_t r = r0 + ty; r < r1; r += 8) {
      const float v = x[r * C + c] - sh;
      s = sq ? fmaf(v, v, s) : s + v;
    }
  }
  red[ty][threadIdx.x] = s;
  __syncthreads();
  if (ty == 0 && c < C) {
    float t = 0.f;
    for (int k = 0; k < 8; ++k) t += red[k][threadIdx.x];
    part[(int64_t)blockIdx.y * C + c] = t;
  }
}
// mode 0: mean[c] = sum / R.  mode 1: var = sum of squares / R -> rstd, and the running statistics (unbiased variance)
// are updated in place.  mode 2 (eval): mean = running_mean, rstd from running_var.
__global__ void k_bn_final(const float* __restrict__ part, int nchunks, int C, int64_t R, int mode, float* mean,
                           float* rstd, float* running_mean, float* running_var) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= C) return;
  if (mode == 2) {
    mean[c] = running_mean[c];
    rstd[c] = 1.0f / sqrtf(running_var[c] + BN_EPS);
    return;
  }
  float s = 0.f;
  for (int k = 0; k < nchunks; ++k) s += part[(int64_t)k * C + c];
  if (mode == 0) {
    mean[c] = s / float(R);
    return;
  }
  const float var = s / float(R);
  rstd[c] = 1.0f / sqrtf(var + BN_EPS);
  running_mean[c] = (1.f - BN_MOMENTUM) * running_mean[c] + BN_MOMENTUM * mean[c];
  const float unbiased = R > 1 ? var * (float(R) / float(R - 1)) : var;
  running_var[c] = (1.f - BN_MOMENTUM) * running_var[c] + BN_MOMENTUM * unbiased;
}
__global__ void k_bn_apply(const float* __restrict__ z, int C, const float* __restrict__ mean,
                           const float* __restrict__ rstd, const float* __restrict__ gamma, const float* __restrict__ beta,
                           int relu, float* __restrict__ y, int64_t n) {
  const int64_t e = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (e >= n) return;
  const int c = int(e % C);
  float v = (z[e] - mean[c]) * rstd[c] * gamma[c] + beta[c];
  if (relu) v = v > 0.f ? v : 0.f;
  y[e] = v;
}
// adjoint partials: part[chunk][c] = sum g, part[chunk][C + c] = sum g * xhat, with g = dy masked by the ReLU (y > 0)
__global__ void __launch_bounds__(256) k_bn_bwd_partial(const float* __restrict__ dy, const float* __restrict__ y,
                                                        const float* __restrict__ z, const float* __restrict__ mean,
                                                        const float* __restrict__ rstd, int64_t R, int C, int relu,
                                                        float* __restrict__ part) {
  __shared__ float red[2][8][33];
  const int c = blockIdx.x * 32 + threadIdx.x, ty = threadIdx.y;
  const int64_t r0 = (int64_t)blockIdx.y * BN_ROWS, r1 = min(R, r0 + BN_ROWS);
  float sg = 0.f, sgx = 0.f;
  if (c < C) {
    const float mu = mean[c], rs = rstd[c];
    for (int64_t r = r0 + ty; r < r1; r += 8) {
      const int64_t e = r * C + c;
      const float g = (!relu || y[e] > 0.f) ? dy[e] : 0.f;
      sg += g;
      sgx = fmaf(g, (z[e] - mu) * rs, sgx);
    }
  }
  red[0][ty][threadIdx.x] = sg;
  red[1][ty][threadIdx.x] = sgx;
  __syncthreads();
  if (ty == 0 && c < C) {
    float a = 0.f, bsum = 0.f;
    for (int k = 0; k < 8; ++k) { a += red[0][k][threadIdx.x]; bsum += red[1][k][threadIdx.x]; }
    part[(int64_t)blockIdx.y * 2 * C + c] = a;
    part[(int64_t)blockIdx.y * 2 * C + C + c] = bsum;
  }
}
// dgamma = sum g xhat, dbeta = sum g (into the flat gradient buffer)
__global__ void k_bn_bwd_final(const float* __restrict__ part, int nchunks, int C, float* __restrict__ dgamma,
                               float* __restrict__ dbeta) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= C) return;
  float a = 0.f, bsum = 0.f;
  for (int k = 0; k < nchunks; ++k) {
    a += part[(int64_t)k * 2 * C + c];
    bsum += part[(int64_t)k * 2 * C + C + c];
  }
  dbeta[c] = a;
  dgamma[c] = bsum;
}
// dx = gamma rstd (g - dbeta / R - xhat dgamma / R); dx may alias dy
__global__ void k_bn_bwd_apply(const float* dy, const float* __restrict__ y, const float* __restrict__ z,
                               const float* __restrict__ mean, const float* __restrict__ rstd,
                               const float* __restrict__ gamma, const float* __restrict__ dgamma,
                               const float* __restrict__ dbeta, int64_t R, int C, int relu, float* dx, int64_t n) {
  const int64_t e = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (e >= n) return;
  const int c = int(e % C);
  const float g = (!relu || y[e] > 0.f) ? dy[e] : 0.f;
  const float rs = rstd[c];
  const float xhat = (z[e] - mean[c]) * rs;
  const float inv_r = 1.0f / float(R);
  dx[e] = gamma[c] * rs * (g - dbeta[c] * inv_r - xhat * dgamma[c] * inv_r);
}

// ---- global max over the points (Encoder, :206): block 32 channels x 8 point strides per object ----------------------
__global__ void __launch_bounds__(256) k_sae_gmax(const float* __restrict__ y, int P, int C, float* __restrict__ code,
                                                  int* __restrict__ arg) {
  __shared__ float bv[8][33];
  __shared__ int ba[8][33];
  const int c = blockIdx.x * 32 + threadIdx.x, ty = threadIdx.y, b = blockIdx.y;
  float best = -INFINITY;
  int a = -1;
  if (c < C)
    for (int p = ty; p < P; p += 8) {
      const float v = y[((int64_t)b * P + p) * C + c];
      if (v > best || a < 0) { best = v; a = p; }
    }
  bv[ty][threadIdx.x] = best;
  ba[ty][threadIdx.x] = a;
  __syncthreads();
  if (ty == 0 && c < C) {
    for (int k = 1; k < 8; ++k) {
      const float v = bv[k][threadIdx.x];
      const int q = ba[k][threadIdx.x];
      if (q >= 0 && (v > best || (v == best && q < a))) { best = v; a = q; }
    }
    code[(int64_t)b * C + c] = best;
    arg[(int64_t)b * C + c] = a;
  }
}
__global__ void k_sae_gmax_bwd(const float* __restrict__ dcode, const int* __restrict__ arg, int P, int C,
                               float* __restrict__ dy, int n) {
  const int e = blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= n) return;
  const int b = e / C, c = e % C;
  dy[((int64_t)b * P + arg[e]) * C + c] = dcode[e];
}

// ---- latent head (DiagonalGaussianDistribution, :297-324): one warp per object --------------------------------------
__global__ void k_sae_latent(const float* __restrict__ mean, const float* __restrict__ lvraw,
                             const float* __restrict__ eps, int B, int F, float* __restrict__ lat, float* __restrict__ kl) {
  const int b = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (b >= B) return;
  float s = 0.f;
  for (int f = lane; f < F; f += 32) {
    const int64_t e = (int64_t)b * F + f;
    const float lv = fminf(fmaxf(lvraw[e], -30.f), 20.f);
    const float m = mean[e];
    lat[e] = m + expf(0.5f * lv) * eps[e];
    s += m * m + expf(lv) - 1.0f - lv;
  }
  s = warp_sum(s);
  if (lane == 0) kl[b] = 0.5f * (s / float(F));
}
// d(mean), d(logvar) of loss = ... + kl_weight * sum_b kl_b / B with dlat from the decoder; the clamp passes the
// gradient on [-30, 20] inclusive (torch.clamp)
__global__ void k_sae_latent_bwd(const float* __restrict__ mean, const float* __restrict__ lvraw,
                                 const float* __restrict__ eps, const float* __restrict__ dlat, int F, float klw_over_b,
                                 float* __restrict__ dmean, float* __restrict__ dlv, int64_t n) {
  const int64_t e = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (e >= n) return;
  const float raw = lvraw[e];
  const float lv = fminf(fmaxf(raw, -30.f), 20.f);
  const float c = klw_over_b * 0.5f / float(F);
  dmean[e] = dlat[e] + c * 2.0f * mean[e];
  const float g = dlat[e] * eps[e] * 0.5f * expf(0.5f * lv) + c * (expf(lv) - 1.0f);
  dlv[e] = (raw >= -30.f && raw <= 20.f) ? g : 0.f;
}

// ---- folding layers -------------------------------------------------------------------------------------------------
// out[r, n] = sum_{j<K} a[r, j] W[n, j] + cobj[r / rows_per_obj, n]   (cobj = W_c code + b, one row per object)
__global__ void k_sae_fold_in(const float* __restrict__ a, int K, const float* __restrict__ W, int ldw,
                              const float* __restrict__ cobj, int rows_per_obj, int N, float* __restrict__ out,
                              int64_t n) {
  const int64_t e = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (e >= n) return;
  const int c = int(e % N);
  const int64_t r = e / N;
  float v = cobj[(r / rows_per_obj) * N + c];
  for (int j = 0; j < K; ++j) v = fmaf(a[r * K + j], W[(int64_t)c * ldw + j], v);
  out[e] = v;
}
// out[b, n] = sum over the object's rows of d[r, n], fixed order; block 32 x 8, grid (N / 32, B)
__global__ void __launch_bounds__(256) k_sae_objsum(const float* __restrict__ d, int rows_per_obj, int N,
                                                    float* __restrict__ out) {
  __shared__ float red[8][33];
  const int c = blockIdx.x * 32 + threadIdx.x, ty = threadIdx.y, b = blockIdx.y;
  float s = 0.f;
  if (c < N)
    for (int r = ty; r < rows_per_obj; r += 8) s += d[((int64_t)b * rows_per_obj + r) * N + c];
  red[ty][threadIdx.x] = s;
  __syncthreads();
  if (ty == 0 && c < N) {
    float t = 0.f;
    for (int k = 0; k < 8; ++k) t += red[k][threadIdx.x];
    out[(int64_t)b * N + c] = t;
  }
}
// decoder grid: np.meshgrid(linspace(-0.3, 0.3, 45) x 2) flattened, repeated per object: row (b, m) = (xx[m], yy[m])
__global__ void k_sae_grid(float* __restrict__ g, int64_t R) {
  const int64_t r = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (r >= R) return;
  const int m = int(r % GRID_M);
  // np.linspace(float32): i * step + start in float64 (separately rounded, no fma), then rounded to float32
  const double step = 0.6 / (GRID_SIDE - 1);
  g[r * 2 + 0] = float(__dadd_rn(__dmul_rn(double(m % GRID_SIDE), step), -0.3));
  g[r * 2 + 1] = float(__dadd_rn(__dmul_rn(double(m / GRID_SIDE), step), -0.3));
}

// ---- Chamfer distance (chamfer3D.cu semantics) ----------------------------------------------------------------------
// dist[b, i] = min_j |a_i - b_j|^2, idx the first minimum (strict <, index order); one thread per point of a
constexpr int CH_TILE = 512;
__global__ void __launch_bounds__(256) k_chamfer_nn(const float* __restrict__ a, int n, const float* __restrict__ b,
                                                    int m, float* __restrict__ dist, int* __restrict__ idx) {
  __shared__ float bs[CH_TILE * 3];
  const int o = blockIdx.y, i = blockIdx.x * blockDim.x + threadIdx.x;
  const float* bb = b + (int64_t)o * m * 3;
  float x = 0.f, y = 0.f, z = 0.f;
  if (i < n) {
    const float* p = a + ((int64_t)o * n + i) * 3;
    x = p[0]; y = p[1]; z = p[2];
  }
  float best = INFINITY;
  int arg = 0;
  for (int j0 = 0; j0 < m; j0 += CH_TILE) {
    const int jn = min(CH_TILE, m - j0);
    __syncthreads();
    for (int e = threadIdx.x; e < jn * 3; e += blockDim.x) bs[e] = bb[(int64_t)j0 * 3 + e];
    __syncthreads();
    for (int j = 0; j < jn; ++j) {
      const float dx = bs[j * 3] - x, dy = bs[j * 3 + 1] - y, dz = bs[j * 3 + 2] - z;
      const float d = fmaf(dz, dz, fmaf(dy, dy, dx * dx));
      if (d < best) { best = d; arg = j0 + j; }
    }
  }
  if (i < n) {
    dist[(int64_t)o * n + i] = best;
    idx[(int64_t)o * n + i] = arg;
  }
}
// grad_p[i] = 2 (p_i - q_{idx_pq[i]}) g_pq[i] - sum over j with idx_qp[j] = i (ascending j) of 2 (q_j - p_i) g_qp[j].
// A NULL g_pq / g_qp stands for the constant gc_pq / gc_qp.  One thread per point of p; q tiles in shared memory.
__global__ void __launch_bounds__(256) k_chamfer_grad(const float* __restrict__ p, int n, const float* __restrict__ q,
                                                      int m, const int* __restrict__ idx_pq, const float* __restrict__ g_pq,
                                                      float gc_pq, const int* __restrict__ idx_qp,
                                                      const float* __restrict__ g_qp, float gc_qp,
                                                      float* __restrict__ grad_p) {
  __shared__ float qs[CH_TILE * 3];
  __shared__ float gs[CH_TILE];
  __shared__ int is[CH_TILE];
  const int o = blockIdx.y, i = blockIdx.x * blockDim.x + threadIdx.x;
  const float* qb = q + (int64_t)o * m * 3;
  float px = 0.f, py = 0.f, pz = 0.f, ax = 0.f, ay = 0.f, az = 0.f;
  if (i < n) {
    const int64_t r = (int64_t)o * n + i;
    px = p[r * 3]; py = p[r * 3 + 1]; pz = p[r * 3 + 2];
    const int j = idx_pq[r];
    const float g = 2.0f * (g_pq ? g_pq[r] : gc_pq);
    ax = (px - qb[j * 3]) * g;
    ay = (py - qb[j * 3 + 1]) * g;
    az = (pz - qb[j * 3 + 2]) * g;
  }
  for (int j0 = 0; j0 < m; j0 += CH_TILE) {
    const int jn = min(CH_TILE, m - j0);
    __syncthreads();
    for (int e = threadIdx.x; e < jn; e += blockDim.x) {
      const int64_t r = (int64_t)o * m + j0 + e;
      is[e] = idx_qp[r];
      gs[e] = 2.0f * (g_qp ? g_qp[r] : gc_qp);
      qs[e * 3] = qb[(j0 + e) * 3];
      qs[e * 3 + 1] = qb[(j0 + e) * 3 + 1];
      qs[e * 3 + 2] = qb[(j0 + e) * 3 + 2];
    }
    __syncthreads();
    for (int j = 0; j < jn; ++j)
      if (is[j] == i) {
        const float g = gs[j];
        ax -= (qs[j * 3] - px) * g;
        ay -= (qs[j * 3 + 1] - py) * g;
        az -= (qs[j * 3 + 2] - pz) * g;
      }
  }
  if (i < n) {
    float* gp = grad_p + ((int64_t)o * n + i) * 3;
    gp[0] = ax; gp[1] = ay; gp[2] = az;
  }
}

// ---- loss (get_loss, :374-390): losses = {loss, loss_cd, loss_kl}; one CTA, fixed order ------------------------------
__device__ float block_sum256(float v, float* red) {
  v = warp_sum(v);
  __syncthreads();
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
  __syncthreads();
  float t = 0.f;
  for (int w = 0; w < 8; ++w) t += red[w];
  return t;
}
__global__ void __launch_bounds__(256) k_sae_loss(const float* __restrict__ d1, int n, const float* __restrict__ d2,
                                                  int m, const float* __restrict__ kl, int B, float kl_weight,
                                                  float* __restrict__ losses) {
  __shared__ float red[8];
  float cd = 0.f, ks = 0.f;
  for (int b = 0; b < B; ++b) {
    float s1 = 0.f, s2 = 0.f;
    for (int i = threadIdx.x; i < n; i += 256) s1 += d1[(int64_t)b * n + i];
    for (int j = threadIdx.x; j < m; j += 256) s2 += d2[(int64_t)b * m + j];
    s1 = block_sum256(s1, red);
    s2 = block_sum256(s2, red);
    cd += s1 / float(n) + s2 / float(m);
    ks += kl[b];
  }
  if (threadIdx.x == 0) {
    cd /= float(B);
    ks /= float(B);
    losses[0] = cd + ks * kl_weight;
    losses[1] = cd;
    losses[2] = ks;
  }
}
}  // namespace

// ------------------------------------------------------------------------------------------------
// handle and C ABI
// ------------------------------------------------------------------------------------------------
namespace {
struct SaeLinear { int64_t w, b; int in, out; };
struct SaeBn { int64_t w; int C; };      // weight, bias, running_mean, running_var at w, w + C, w + 2C, w + 3C
enum { BN_E1, BN_E2, BN_E3, BN_G1, BN_G2, BN_E4, BN_F1A, BN_F1B, BN_F2A, BN_F2B, BN_COUNT };
}  // namespace

struct ds_shape_ae {
  ds_shape_ae_config cfg;
  int P = 0, F = 0;
  WeightTable w;
  SaeLinear conv1, conv2, conv3, gl1, gl2, conv4, mean_fc, logvar_fc, fc, f1[3], f2[3];
  SaeBn bn[BN_COUNT];
  // device buffers (capacity `cap` objects)
  int cap = 0;
  float *pts = nullptr, *f12 = nullptr, *grid = nullptr;
  float *z[BN_COUNT] = {nullptr}, *y[BN_COUNT] = {nullptr};
  float *m1 = nullptr, *m2 = nullptr;
  uint8_t *am1 = nullptr, *am2 = nullptr;
  int* knn[3] = {nullptr};
  float *code_e = nullptr, *mean = nullptr, *lvraw = nullptr, *lat = nullptr, *kl = nullptr, *code_d = nullptr;
  float *c1 = nullptr, *c2 = nullptr, *r1 = nullptr, *rec = nullptr, *drec = nullptr, *dr1 = nullptr;
  int* garg = nullptr;
  float *stats = nullptr, *part = nullptr;      // per-BN mean / rstd (2 x 1024 each); partial sums
  float *dist1 = nullptr, *dist2 = nullptr;
  int *cidx1 = nullptr, *cidx2 = nullptr;
  float *gA = nullptr, *gB = nullptr, *gsmall = nullptr;
  int *csr_cnt = nullptr, *csr_start = nullptr, *csr_cur = nullptr, *csr_list = nullptr;
  const int* inject = nullptr;
  bool kept = false;
  int kept_B = 0;
};

namespace {
void sae_free(ds_shape_ae* h) {
  float** fb[] = {&h->pts, &h->f12, &h->grid, &h->m1, &h->m2, &h->code_e, &h->mean, &h->lvraw, &h->lat, &h->kl,
                  &h->code_d, &h->c1, &h->c2, &h->r1, &h->rec, &h->drec, &h->dr1, &h->stats, &h->part, &h->dist1, &h->dist2, &h->gA,
                  &h->gB, &h->gsmall};
  for (float** b : fb) { cudaFree(*b); *b = nullptr; }
  for (int i = 0; i < BN_COUNT; ++i) { cudaFree(h->z[i]); cudaFree(h->y[i]); h->z[i] = h->y[i] = nullptr; }
  int** ib[] = {&h->knn[0], &h->knn[1], &h->knn[2], &h->garg, &h->cidx1, &h->cidx2, &h->csr_cnt, &h->csr_start,
                &h->csr_cur, &h->csr_list};
  for (int** b : ib) { cudaFree(*b); *b = nullptr; }
  cudaFree(h->am1); cudaFree(h->am2);
  h->am1 = h->am2 = nullptr;
  h->cap = 0;
  h->kept = false;
}

SaeLinear add_linear(ds_shape_ae* h, const std::string& n, int in, int out) {
  SaeLinear l;
  l.in = in; l.out = out;
  l.w = h->w.total;
  h->w.add(n + ".weight", (int64_t)in * out);
  l.b = h->w.total;
  h->w.add(n + ".bias", out);
  return l;
}
SaeBn add_bn(ds_shape_ae* h, const std::string& n, int C) {
  SaeBn b;
  b.C = C;
  b.w = h->w.total;
  for (const char* s : {".weight", ".bias", ".running_mean", ".running_var"}) h->w.add(n + s, C);
  return b;
}

int64_t enc_rows(const ds_shape_ae* h, int B) { return (int64_t)B * h->P; }
int64_t dec_rows(int B) { return (int64_t)B * GRID_M; }
int bn_width(int i) {
  static const int w[BN_COUNT] = {64, 64, 64, 128, 1024, 512, 512, 512, 512, 512};
  return w[i];
}
bool bn_is_dec(int i) { return i >= BN_F1A; }

int sae_ensure(ds_shape_ae* h, int B) {
  if (B <= h->cap) return 0;
  sae_free(h);
  const int64_t R = enc_rows(h, B), Rm = dec_rows(B), F = h->F;
  const int64_t big = std::max(R * 1024, Rm * 512);
  auto fm = [](float** p, int64_t n) { return cudaMalloc(p, (size_t)std::max<int64_t>(n, 1) * 4); };
  auto im = [](int** p, int64_t n) { return cudaMalloc(p, (size_t)std::max<int64_t>(n, 1) * 4); };
  CK(fm(&h->pts, R * 3));
  CK(fm(&h->f12, R * 12));
  CK(fm(&h->grid, Rm * 2));
  for (int i = 0; i < BN_COUNT; ++i) {
    const int64_t rows = bn_is_dec(i) ? Rm : R;
    CK(fm(&h->z[i], rows * bn_width(i)));
    CK(fm(&h->y[i], rows * bn_width(i)));
  }
  CK(fm(&h->m1, R * 64));
  CK(fm(&h->m2, R * 128));
  CK(cudaMalloc(&h->am1, (size_t)R * 64));
  CK(cudaMalloc(&h->am2, (size_t)R * 128));
  for (int i = 0; i < 3; ++i) CK(im(&h->knn[i], R * KNN));
  CK(fm(&h->code_e, (int64_t)B * 512));
  CK(fm(&h->mean, B * F));
  CK(fm(&h->lvraw, B * F));
  CK(fm(&h->lat, B * F));
  CK(fm(&h->kl, B));
  CK(fm(&h->code_d, (int64_t)B * 512));
  CK(fm(&h->c1, (int64_t)B * 512));
  CK(fm(&h->c2, (int64_t)B * 512));
  CK(fm(&h->r1, Rm * 3));
  CK(fm(&h->rec, Rm * 3));
  CK(fm(&h->drec, Rm * 3));
  CK(fm(&h->dr1, Rm * 3));
  CK(im(&h->garg, (int64_t)B * 512));
  CK(fm(&h->stats, BN_COUNT * 2 * 1024));
  CK(fm(&h->part, (std::max(R, Rm) / BN_ROWS + 1) * 2 * 1024));
  CK(fm(&h->dist1, R));
  CK(fm(&h->dist2, Rm));
  CK(im(&h->cidx1, R));
  CK(im(&h->cidx2, Rm));
  CK(fm(&h->gA, big));
  CK(fm(&h->gB, big));
  CK(fm(&h->gsmall, (int64_t)B * 512 * 4 + 4 * B * F));
  CK(im(&h->csr_cnt, R));
  CK(im(&h->csr_start, R + 1));
  CK(im(&h->csr_cur, R));
  CK(im(&h->csr_list, R * KNN));
  h->cap = B;
  return 0;
}

float* bn_mean(ds_shape_ae* h, int i) { return h->stats + (int64_t)i * 2048; }
float* bn_rstd(ds_shape_ae* h, int i) { return h->stats + (int64_t)i * 2048 + 1024; }

// out[R, N] = in[R, K] W^T + b with the exact fp32 SIMT GEMM (W [N, K] row pitch ldw)
void linear_fwd(const float* in, int K, const float* W, int ldw, const float* bias, float* out, int64_t R, int N,
                cudaStream_t s) {
  GemmArgs g;
  memset(&g, 0, sizeof g);
  g.a0 = in; g.lda0 = K; g.k0 = K;
  g.w = W; g.ldw = ldw;
  g.bias = bias;
  g.d = out; g.ldd = N;
  g.M = int(R); g.N = N;
  launch_gemm_simt<float>(g, true, s);
}
// dW += dY^T X, db += colsum dY, dX = dY W (when dx != NULL)
void linear_bwd(const float* x, const float* dy, const SaeLinear& l, const float* prm, float* grads, float* dx,
                int64_t R, cudaStream_t s) {
  launch_gemm_tn<float, float>(dy, l.out, x, l.in, grads + l.w, l.in, int(R), l.out, l.in, s);
  launch_colsum<float>(dy, l.out, grads + l.b, int(R), l.out, s);
  if (dx) launch_gemm_nn<float, float, float>(dy, l.out, prm + l.w, l.in, dx, l.in, int(R), l.in, l.out, 0, s);
}

void bn_fwd(ds_shape_ae* h, int i, float* prm, int64_t R, bool train, bool relu, cudaStream_t s) {
  const SaeBn& b = h->bn[i];
  const int C = b.C;
  float* mean = bn_mean(h, i);
  float* rstd = bn_rstd(h, i);
  float* rm = prm + b.w + 2 * C;
  float* rv = prm + b.w + 3 * C;
  const int nch = int((R + BN_ROWS - 1) / BN_ROWS);
  if (train) {
    const dim3 grid(ceil_div(C, 32), nch), blk(32, 8);
    k_bn_partial<<<grid, blk, 0, s>>>(h->z[i], R, C, nullptr, 0, h->part);
    k_bn_final<<<ceil_div(C, 256), 256, 0, s>>>(h->part, nch, C, R, 0, mean, rstd, rm, rv);
    k_bn_partial<<<grid, blk, 0, s>>>(h->z[i], R, C, mean, 1, h->part);
    k_bn_final<<<ceil_div(C, 256), 256, 0, s>>>(h->part, nch, C, R, 1, mean, rstd, rm, rv);
  } else {
    k_bn_final<<<ceil_div(C, 256), 256, 0, s>>>(nullptr, 0, C, R, 2, mean, rstd, rm, rv);
  }
  k_bn_apply<<<ceil_div(R * C, 256), 256, 0, s>>>(h->z[i], C, mean, rstd, prm + b.w, prm + b.w + C, relu ? 1 : 0, h->y[i],
                                              R * C);
}
// dy (masked by the ReLU when relu) -> dx in place; dgamma / dbeta into grads
void bn_bwd(ds_shape_ae* h, int i, const float* prm, float* grads, float* d, int64_t R, bool relu, cudaStream_t s) {
  const SaeBn& b = h->bn[i];
  const int C = b.C;
  const int nch = int((R + BN_ROWS - 1) / BN_ROWS);
  k_bn_bwd_partial<<<dim3(ceil_div(C, 32), nch), dim3(32, 8), 0, s>>>(d, h->y[i], h->z[i], bn_mean(h, i), bn_rstd(h, i),
                                                                  R, C, relu ? 1 : 0, h->part);
  k_bn_bwd_final<<<ceil_div(C, 256), 256, 0, s>>>(h->part, nch, C, grads + b.w, grads + b.w + C);
  k_bn_bwd_apply<<<ceil_div(R * C, 256), 256, 0, s>>>(d, h->y[i], h->z[i], bn_mean(h, i), bn_rstd(h, i), prm + b.w,
                                                  grads + b.w, grads + b.w + C, R, C, relu ? 1 : 0, d, R * C);
}

void nbr_max(ds_shape_ae* h, const float* y, const int* idx, int C, float* out, uint8_t* am, int B, cudaStream_t s) {
  const int64_t n = enc_rows(h, B) * C;
  k_sae_nbr_max<<<ceil_div(n, 256), 256, 0, s>>>(y, idx, h->P, C, out, am, n);
}
void build_csr(ds_shape_ae* h, const int* idx, int B, cudaStream_t s) {
  const int64_t R = enc_rows(h, B), n = R * KNN;
  cudaMemsetAsync(h->csr_cnt, 0, (size_t)R * 4, s);
  k_csr_count<<<ceil_div(n, 256), 256, 0, s>>>(idx, h->P * KNN, h->P, h->csr_cnt, n);
  k_csr_scan<<<B, 1024, 0, s>>>(h->csr_cnt, h->P, h->P * KNN, B, h->csr_start, h->csr_cur);
  k_csr_fill<<<ceil_div(n, 256), 256, 0, s>>>(idx, h->P * KNN, h->P, h->csr_cur, h->csr_list, n);
  k_csr_sort<<<ceil_div(R, 128), 128, 0, s>>>(h->csr_start, h->csr_list, R);
}

void fold_layer_fwd(ds_shape_ae* h, const SaeLinear* L, int bn0, const float* in, int K, float* cobj, float* out, float* prm,
                    int B, bool train, cudaStream_t s) {
  const int64_t Rm = dec_rows(B);
  const int ldw = L[0].in;      // 2 + 512 or 3 + 512
  linear_fwd(h->code_d, 512, prm + L[0].w + K, ldw, prm + L[0].b, cobj, B, 512, s);
  k_sae_fold_in<<<ceil_div(Rm * 512, 256), 256, 0, s>>>(in, K, prm + L[0].w, ldw, cobj, GRID_M, 512, h->z[bn0], Rm * 512);
  bn_fwd(h, bn0, prm, Rm, train, true, s);
  linear_fwd(h->y[bn0], 512, prm + L[1].w, 512, prm + L[1].b, h->z[bn0 + 1], Rm, 512, s);
  bn_fwd(h, bn0 + 1, prm, Rm, train, true, s);
  linear_fwd(h->y[bn0 + 1], 512, prm + L[2].w, 512, prm + L[2].b, out, Rm, 3, s);
}
// backward of one folding layer from d(out) [Rm, 3]: parameter gradients, d(in) [Rm, K] (when din), and
// d(code) (= | +=) into dcode [B, 512]
void fold_layer_bwd(ds_shape_ae* h, const SaeLinear* L, int bn0, const float* in, int K, const float* dout, float* din,
                    float* dcode, int accumulate, const float* prm, float* grads, int B, cudaStream_t s) {
  const int64_t Rm = dec_rows(B);
  const int ldw = L[0].in;
  linear_bwd(h->y[bn0 + 1], dout, L[2], prm, grads, h->gA, Rm, s);
  bn_bwd(h, bn0 + 1, prm, grads, h->gA, Rm, true, s);
  linear_bwd(h->y[bn0], h->gA, L[1], prm, grads, h->gB, Rm, s);
  bn_bwd(h, bn0, prm, grads, h->gB, Rm, true, s);
  float* dc = h->gsmall;      // [B, 512] per-object sums of dz
  k_sae_objsum<<<dim3(512 / 32, B), dim3(32, 8), 0, s>>>(h->gB, GRID_M, 512, dc);
  launch_gemm_tn<float, float>(h->gB, 512, in, K, grads + L[0].w, ldw, int(Rm), 512, K, s);
  launch_gemm_tn<float, float>(dc, 512, h->code_d, 512, grads + L[0].w + K, ldw, B, 512, 512, s);
  launch_colsum<float>(dc, 512, grads + L[0].b, B, 512, s);
  if (din) launch_gemm_nn<float, float, float>(h->gB, 512, prm + L[0].w, ldw, din, K, int(Rm), K, 512, 0, s);
  launch_gemm_nn<float, float, float>(dc, 512, prm + L[0].w + K, ldw, dcode, 512, B, 512, 512, accumulate, s);
}

int sae_forward(ds_shape_ae* h, float* prm, const float* points, int B, const float* eps, bool train, cudaStream_t s) {
  const int P = h->P, F = h->F;
  const int64_t R = enc_rows(h, B), Rm = dec_rows(B);
  CK(cudaMemcpyAsync(h->pts, points, (size_t)R * 3 * 4, cudaMemcpyDeviceToDevice, s));
  k_sae_grid<<<ceil_div(Rm, 256), 256, 0, s>>>(h->grid, Rm);
  if (h->inject)
    for (int i = 0; i < 3; ++i)
      CK(cudaMemcpyAsync(h->knn[i], h->inject + (int64_t)i * R * KNN, (size_t)R * KNN * 4, cudaMemcpyDeviceToDevice, s));
  // encoder (:182-207)
  if (!h->inject) launch_knn(h->pts, B, P, 3, h->knn[0], s);
  k_sae_cov<<<ceil_div(R, 128), 128, 0, s>>>(h->pts, h->knn[0], P, h->f12, R);
  linear_fwd(h->f12, 12, prm + h->conv1.w, 12, prm + h->conv1.b, h->z[BN_E1], R, 64, s);
  bn_fwd(h, BN_E1, prm, R, train, true, s);
  linear_fwd(h->y[BN_E1], 64, prm + h->conv2.w, 64, prm + h->conv2.b, h->z[BN_E2], R, 64, s);
  bn_fwd(h, BN_E2, prm, R, train, true, s);
  linear_fwd(h->y[BN_E2], 64, prm + h->conv3.w, 64, prm + h->conv3.b, h->z[BN_E3], R, 64, s);
  bn_fwd(h, BN_E3, prm, R, train, true, s);
  if (!h->inject) launch_knn(h->y[BN_E3], B, P, 64, h->knn[1], s);
  nbr_max(h, h->y[BN_E3], h->knn[1], 64, h->m1, h->am1, B, s);
  linear_fwd(h->m1, 64, prm + h->gl1.w, 64, prm + h->gl1.b, h->z[BN_G1], R, 128, s);
  bn_fwd(h, BN_G1, prm, R, train, true, s);
  if (!h->inject) launch_knn(h->y[BN_G1], B, P, 128, h->knn[2], s);
  nbr_max(h, h->y[BN_G1], h->knn[2], 128, h->m2, h->am2, B, s);
  linear_fwd(h->m2, 128, prm + h->gl2.w, 128, prm + h->gl2.b, h->z[BN_G2], R, 1024, s);
  bn_fwd(h, BN_G2, prm, R, train, true, s);
  linear_fwd(h->y[BN_G2], 1024, prm + h->conv4.w, 1024, prm + h->conv4.b, h->z[BN_E4], R, 512, s);
  bn_fwd(h, BN_E4, prm, R, train, false, s);
  k_sae_gmax<<<dim3(512 / 32, B), dim3(32, 8), 0, s>>>(h->y[BN_E4], P, 512, h->code_e, h->garg);
  // latent head (:349-358) and decoder (:265-282)
  linear_fwd(h->code_e, 512, prm + h->mean_fc.w, 512, prm + h->mean_fc.b, h->mean, B, F, s);
  linear_fwd(h->code_e, 512, prm + h->logvar_fc.w, 512, prm + h->logvar_fc.b, h->lvraw, B, F, s);
  k_sae_latent<<<ceil_div(B, 8), 256, 0, s>>>(h->mean, h->lvraw, eps, B, F, h->lat, h->kl);
  linear_fwd(h->lat, F, prm + h->fc.w, F, prm + h->fc.b, h->code_d, B, 512, s);
  fold_layer_fwd(h, h->f1, BN_F1A, h->grid, 2, h->c1, h->r1, prm, B, train, s);
  fold_layer_fwd(h, h->f2, BN_F2A, h->r1, 3, h->c2, h->rec, prm, B, train, s);
  return 0;
}


void chamfer_fwd(const float* a, int n, const float* b, int m, int B, float* d1, float* d2, int* i1, int* i2,
                 cudaStream_t s) {
  k_chamfer_nn<<<dim3(ceil_div(n, 256), B), 256, 0, s>>>(a, n, b, m, d1, i1);
  k_chamfer_nn<<<dim3(ceil_div(m, 256), B), 256, 0, s>>>(b, m, a, n, d2, i2);
}

// backward of the training loss into grads; the kept forward of the same call provides every activation
int sae_backward(ds_shape_ae* h, const float* prm, float* grads, int B, float kl_weight, const float* eps,
                 cudaStream_t s) {
  const int P = h->P, F = h->F;
  const int64_t R = enc_rows(h, B), Rm = dec_rows(B);
  float* dcode = h->gsmall + (int64_t)B * 512;
  float* dce = h->gsmall + (int64_t)B * 512 * 2;
  float* dlat = h->gsmall + (int64_t)B * 512 * 3;
  float* dmean = dlat + (int64_t)B * F;
  float* dlv = dmean + (int64_t)B * F;
  CK(cudaMemsetAsync(grads, 0, (size_t)h->w.total * 4, s));
  // Chamfer adjoint into the reconstruction, d(dist1) = 1 / (B P), d(dist2) = 1 / (B M)
  k_chamfer_grad<<<dim3(ceil_div(GRID_M, 256), B), 256, 0, s>>>(h->rec, GRID_M, h->pts, P, h->cidx2, nullptr,
                                                            1.0f / float(Rm), h->cidx1, nullptr, 1.0f / float(R),
                                                            h->drec);
  fold_layer_bwd(h, h->f2, BN_F2A, h->r1, 3, h->drec, h->dr1, dcode, 0, prm, grads, B, s);
  fold_layer_bwd(h, h->f1, BN_F1A, h->grid, 2, h->dr1, nullptr, dcode, 1, prm, grads, B, s);
  linear_bwd(h->lat, dcode, h->fc, prm, grads, dlat, B, s);
  k_sae_latent_bwd<<<ceil_div((int64_t)B * F, 256), 256, 0, s>>>(h->mean, h->lvraw, eps, dlat, F, kl_weight / float(B),
                                                             dmean, dlv, (int64_t)B * F);
  linear_bwd(h->code_e, dmean, h->mean_fc, prm, grads, dce, B, s);
  launch_gemm_tn<float, float>(dlv, F, h->code_e, 512, grads + h->logvar_fc.w, 512, B, F, 512, s);
  launch_colsum<float>(dlv, F, grads + h->logvar_fc.b, B, F, s);
  launch_gemm_nn<float, float, float>(dlv, F, prm + h->logvar_fc.w, 512, dce, 512, B, 512, F, 1, s);
  // encoder, last layer first
  CK(cudaMemsetAsync(h->gA, 0, (size_t)R * 512 * 4, s));
  k_sae_gmax_bwd<<<ceil_div(B * 512, 256), 256, 0, s>>>(dce, h->garg, P, 512, h->gA, B * 512);
  bn_bwd(h, BN_E4, prm, grads, h->gA, R, false, s);
  linear_bwd(h->y[BN_G2], h->gA, h->conv4, prm, grads, h->gB, R, s);
  bn_bwd(h, BN_G2, prm, grads, h->gB, R, true, s);
  linear_bwd(h->m2, h->gB, h->gl2, prm, grads, h->gA, R, s);
  build_csr(h, h->knn[2], B, s);
  k_sae_nbr_max_bwd<<<ceil_div(R * 128, 256), 256, 0, s>>>(h->gA, h->am2, h->csr_start, h->csr_list, P, 128, h->gB, R * 128);
  bn_bwd(h, BN_G1, prm, grads, h->gB, R, true, s);
  linear_bwd(h->m1, h->gB, h->gl1, prm, grads, h->gA, R, s);
  build_csr(h, h->knn[1], B, s);
  k_sae_nbr_max_bwd<<<ceil_div(R * 64, 256), 256, 0, s>>>(h->gA, h->am1, h->csr_start, h->csr_list, P, 64, h->gB, R * 64);
  bn_bwd(h, BN_E3, prm, grads, h->gB, R, true, s);
  linear_bwd(h->y[BN_E2], h->gB, h->conv3, prm, grads, h->gA, R, s);
  bn_bwd(h, BN_E2, prm, grads, h->gA, R, true, s);
  linear_bwd(h->y[BN_E1], h->gA, h->conv2, prm, grads, h->gB, R, s);
  bn_bwd(h, BN_E1, prm, grads, h->gB, R, true, s);
  linear_bwd(h->f12, h->gB, h->conv1, prm, grads, nullptr, R, s);
  // the running statistics get no gradient: their slots were zeroed above and nothing writes them
  return 0;
}
}  // namespace

extern "C" int ds_shape_ae_create(const ds_shape_ae_config* cfg, ds_shape_ae** out) {
  if (!cfg || !out) return fail(DS_ERR_INVALID, "null argument");
  *out = nullptr;
  if (cfg->latent_dim < 1 || cfg->latent_dim > 512)
    return fail(DS_ERR_INVALID, "shape auto-encoder: latent_dim %d outside [1, 512]", cfg->latent_dim);
  if (cfg->num_points < KNN)
    return fail(DS_ERR_INVALID, "shape auto-encoder: num_points %d < %d (the kNN size)", cfg->num_points, KNN);
  if (const int rc = open_device(cfg->device)) return rc;
  ds_shape_ae* h = new ds_shape_ae();
  h->cfg = *cfg;
  h->P = cfg->num_points;
  h->F = cfg->latent_dim;
  const int F = h->F;
  // the reference's state-dict order (module registration order; num_batches_tracked stays with the caller)
  h->conv1 = add_linear(h, "encoder.conv1", 12, 64);
  h->conv2 = add_linear(h, "encoder.conv2", 64, 64);
  h->conv3 = add_linear(h, "encoder.conv3", 64, 64);
  h->bn[BN_E1] = add_bn(h, "encoder.bn1", 64);
  h->bn[BN_E2] = add_bn(h, "encoder.bn2", 64);
  h->bn[BN_E3] = add_bn(h, "encoder.bn3", 64);
  h->gl1 = add_linear(h, "encoder.graph_layer1.conv", 64, 128);
  h->bn[BN_G1] = add_bn(h, "encoder.graph_layer1.bn", 128);
  h->gl2 = add_linear(h, "encoder.graph_layer2.conv", 128, 1024);
  h->bn[BN_G2] = add_bn(h, "encoder.graph_layer2.bn", 1024);
  h->conv4 = add_linear(h, "encoder.conv4", 1024, 512);
  h->bn[BN_E4] = add_bn(h, "encoder.bn4", 512);
  h->mean_fc = add_linear(h, "mean_fc", 512, F);
  h->logvar_fc = add_linear(h, "logvar_fc", 512, F);
  h->fc = add_linear(h, "fc", F, 512);
  for (int f = 0; f < 2; ++f) {
    const std::string pre = f == 0 ? "decoder.fold1.layers." : "decoder.fold2.layers.";
    SaeLinear* L = f == 0 ? h->f1 : h->f2;
    const int bn0 = f == 0 ? BN_F1A : BN_F2A;
    L[0] = add_linear(h, pre + "0", 512 + 2 + f, 512);
    h->bn[bn0] = add_bn(h, pre + "1", 512);
    L[1] = add_linear(h, pre + "3", 512, 512);
    h->bn[bn0 + 1] = add_bn(h, pre + "4", 512);
    L[2] = add_linear(h, pre + "6", 512, 3);
  }
  *out = h;
  return 0;
}

extern "C" int ds_shape_ae_destroy(ds_shape_ae* h) {
  if (!h) return 0;
  cudaSetDevice(h->cfg.device);
  sae_free(h);
  delete h;
  return 0;
}

extern "C" int ds_shape_ae_expected_weight_count(ds_shape_ae* h) {
  if (!h) return fail(DS_ERR_INVALID, "null handle");
  return h->w.count();
}

extern "C" int ds_shape_ae_expected_weight(ds_shape_ae* h, int index, const char** name, int64_t* numel) {
  if (!h) return fail(DS_ERR_INVALID, "null argument");
  return h->w.get(index, name, numel);
}

extern "C" int ds_shape_ae_forward(ds_shape_ae* h, float* flat_params_dev, const float* points_dev, int32_t batch,
                                   const float* eps_dev, int32_t train, int32_t keep, float* latent_dev, float* kl_dev,
                                   float* recon_dev, void* stream) {
  if (!h || !flat_params_dev || !points_dev || !eps_dev) return fail(DS_ERR_INVALID, "null argument");
  if (batch < 1) return fail(DS_ERR_INVALID, "shape auto-encoder: batch %d < 1", batch);
  CK(cudaSetDevice(h->cfg.device));
  cudaStream_t s = (cudaStream_t)stream;
  int rc = sae_ensure(h, batch);
  if (rc) return rc;
  h->kept = false;
  if ((rc = sae_forward(h, flat_params_dev, points_dev, batch, eps_dev, train != 0, s))) return rc;
  const int64_t F = h->F;
  if (latent_dev) CK(cudaMemcpyAsync(latent_dev, h->lat, (size_t)batch * F * 4, cudaMemcpyDeviceToDevice, s));
  if (kl_dev) CK(cudaMemcpyAsync(kl_dev, h->kl, (size_t)batch * 4, cudaMemcpyDeviceToDevice, s));
  if (recon_dev) CK(cudaMemcpyAsync(recon_dev, h->rec, (size_t)dec_rows(batch) * 3 * 4, cudaMemcpyDeviceToDevice, s));
  CK(cudaGetLastError());
  if (keep) {
    h->kept = true;
    h->kept_B = batch;
  }
  return 0;
}

extern "C" int ds_shape_ae_train_step(ds_shape_ae* h, float* flat_params_dev, const float* points_dev, int32_t batch,
                                      const float* eps_dev, float kl_weight, float* flat_grads_dev, float* losses_dev,
                                      void* stream) {
  if (!h || !flat_params_dev || !points_dev || !eps_dev || !flat_grads_dev || !losses_dev)
    return fail(DS_ERR_INVALID, "null argument");
  if (batch < 1) return fail(DS_ERR_INVALID, "shape auto-encoder: batch %d < 1", batch);
  CK(cudaSetDevice(h->cfg.device));
  cudaStream_t s = (cudaStream_t)stream;
  int rc = sae_ensure(h, batch);
  if (rc) return rc;
  h->kept = false;
  if ((rc = sae_forward(h, flat_params_dev, points_dev, batch, eps_dev, true, s))) return rc;
  chamfer_fwd(h->pts, h->P, h->rec, GRID_M, batch, h->dist1, h->dist2, h->cidx1, h->cidx2, s);
  k_sae_loss<<<1, 256, 0, s>>>(h->dist1, h->P, h->dist2, GRID_M, h->kl, batch, kl_weight, losses_dev);
  if ((rc = sae_backward(h, flat_params_dev, flat_grads_dev, batch, kl_weight, eps_dev, s))) return rc;
  CK(cudaGetLastError());
  h->kept = true;
  h->kept_B = batch;
  return 0;
}

extern "C" int ds_shape_ae_set_knn(ds_shape_ae* h, const int32_t* idx_dev) {
  if (!h) return fail(DS_ERR_INVALID, "null handle");
  h->inject = idx_dev;
  return 0;
}

extern "C" int ds_shape_ae_get_knn(ds_shape_ae* h, int32_t* idx_dev, void* stream) {
  if (!h || !idx_dev) return fail(DS_ERR_INVALID, "null argument");
  if (!h->kept) return fail(DS_ERR_INVALID, "shape auto-encoder: no kept forward pass to read the kNN indices of");
  CK(cudaSetDevice(h->cfg.device));
  const size_t n = (size_t)enc_rows(h, h->kept_B) * KNN;
  for (int i = 0; i < 3; ++i)
    CK(cudaMemcpyAsync(idx_dev + i * n, h->knn[i], n * 4, cudaMemcpyDeviceToDevice, (cudaStream_t)stream));
  return 0;
}

extern "C" int ds_knn(const float* x_dev, int32_t batch, int32_t num_points, int32_t channels, int32_t* idx_dev,
                      void* stream) {
  if (!x_dev || !idx_dev) return fail(DS_ERR_INVALID, "null argument");
  if (channels != 3 && channels != 64 && channels != 128)
    return fail(DS_ERR_INVALID, "knn: channels %d not in {3, 64, 128}", channels);
  if (num_points < KNN) return fail(DS_ERR_INVALID, "knn: num_points %d < %d", num_points, KNN);
  if (batch < 1) return fail(DS_ERR_INVALID, "knn: batch %d < 1", batch);
  launch_knn(x_dev, batch, num_points, channels, idx_dev, (cudaStream_t)stream);
  CK(cudaGetLastError());
  return 0;
}

extern "C" int ds_chamfer_forward(const float* a_dev, int32_t n, const float* b_dev, int32_t m, int32_t batch,
                                  float* dist1_dev, float* dist2_dev, int32_t* idx1_dev, int32_t* idx2_dev,
                                  void* stream) {
  if (!a_dev || !b_dev || !dist1_dev || !dist2_dev || !idx1_dev || !idx2_dev) return fail(DS_ERR_INVALID, "null argument");
  if (n < 1 || m < 1 || batch < 1) return fail(DS_ERR_INVALID, "chamfer: empty input (n %d, m %d, batch %d)", n, m, batch);
  chamfer_fwd(a_dev, n, b_dev, m, batch, dist1_dev, dist2_dev, idx1_dev, idx2_dev, (cudaStream_t)stream);
  CK(cudaGetLastError());
  return 0;
}

extern "C" int ds_chamfer_backward(const float* a_dev, int32_t n, const float* b_dev, int32_t m, int32_t batch,
                                   const int32_t* idx1_dev, const int32_t* idx2_dev, const float* g1_dev,
                                   const float* g2_dev, float* grad_a_dev, float* grad_b_dev, void* stream) {
  if (!a_dev || !b_dev || !idx1_dev || !idx2_dev || !g1_dev || !g2_dev || (!grad_a_dev && !grad_b_dev))
    return fail(DS_ERR_INVALID, "null argument");
  if (n < 1 || m < 1 || batch < 1) return fail(DS_ERR_INVALID, "chamfer: empty input (n %d, m %d, batch %d)", n, m, batch);
  cudaStream_t s = (cudaStream_t)stream;
  if (grad_a_dev)
    k_chamfer_grad<<<dim3(ceil_div(n, 256), batch), 256, 0, s>>>(a_dev, n, b_dev, m, idx1_dev, g1_dev, 0.f, idx2_dev, g2_dev,
                                                             0.f, grad_a_dev);
  if (grad_b_dev)
    k_chamfer_grad<<<dim3(ceil_div(m, 256), batch), 256, 0, s>>>(b_dev, m, a_dev, n, idx2_dev, g2_dev, 0.f, idx1_dev, g1_dev,
                                                             0.f, grad_b_dev);
  CK(cudaGetLastError());
  return 0;
}
