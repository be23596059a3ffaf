// Scene evaluation of generated layouts (the reference's `--compute_intersec` statistics, scripts/utils.py:560-745):
// the world-space axis-aligned bounds of each placed model (k_scene_boxes) and, per scene, the pairwise 3D box IoU,
// the intersecting pairs, the overlap ratio and the symmetric pairs (k_scene_stats).  Stateless C ABI at the bottom.
//
// Every operation is an explicit _rn intrinsic, so no FMA contraction changes a result, and every sum runs in a fixed
// order without atomics: a scene's numbers do not depend on the batch it is evaluated in.
#include "engine_internal.h"
#include "placement.cuh"

namespace ds {
namespace {

constexpr int SE_MAX_N = 64;                    // objects per scene (one warp, two slots per lane)
constexpr int SE_MAX_PAIRS = SE_MAX_N * (SE_MAX_N - 1) / 2;
constexpr int SE_WARPS = 4;                     // scenes per CTA of k_scene_stats

enum { SE_ERR_OFFSETS = 1, SE_ERR_INDEX = 2 };

inline int cdiv(int64_t a, int64_t b) { return int((a + b - 1) / b); }

__device__ const double k_unit_half[3] = {1, 1, 1}, k_zero_aabb[6] = {0, 0, 0, 0, 0, 0};

// One object: place the model (or the object's own box) and take the bounds of the placed hull.  The placement is
// make_placement (placement.cuh), shared with the renderer.  x and z are linear in (v.x, v.z), so their extremes over
// the mesh lie on the xz convex hull; y needs only the raw y range.
__global__ void k_scene_boxes(const float* __restrict__ trans, const float* __restrict__ size,
                              const float* __restrict__ angle, const int64_t* __restrict__ model, int Q,
                              const int* __restrict__ hull_off, const double* __restrict__ hull_xz, int H,
                              const double* __restrict__ raw_half, const double* __restrict__ raw_aabb, int M,
                              double* __restrict__ out, int* __restrict__ err) {
  const int q = blockIdx.x * blockDim.x + threadIdx.x;
  if (q < M && hull_off) {                      // the whole CSR table is checked, used rows or not
    const int a = hull_off[q], b = hull_off[q + 1];
    if (a < 0 || b < a || b > H) atomicOr(err, SE_ERR_OFFSETS);
  }
  if (q >= Q) return;
  const int64_t m = model ? model[q] : -1;
  double* o = out + (int64_t)q * 6;
  if (m < -1 || m >= M) {
    atomicOr(err, SE_ERR_INDEX);
    for (int k = 0; k < 6; ++k) o[k] = __longlong_as_double(0x7ff8000000000000ll);
    return;
  }
  int beg = 0, end = 0;
  if (m >= 0) {
    beg = hull_off[m];
    end = hull_off[m + 1];
    if (beg < 0 || end < beg || end > H) {      // flagged above; read nothing
      for (int k = 0; k < 6; ++k) o[k] = __longlong_as_double(0x7ff8000000000000ll);
      return;
    }
  }
  const bool own_box = beg == end;              // only the rotation and translation of p are used then
  const Placement p = make_placement(size + q * 3, trans + q * 3, angle[q], own_box ? k_unit_half : raw_half + m * 3,
                                     own_box ? k_zero_aabb : raw_aabb + m * 6);
  double ylo, yhi, x1 = INFINITY, x2 = -INFINITY, z1 = INFINITY, z2 = -INFINITY;
  auto put = [&](double px, double pz) {
    double x, z;
    rotate_xz(p, px, pz, x, z);
    x1 = fmin(x1, x); x2 = fmax(x2, x);
    z1 = fmin(z1, z); z2 = fmax(z2, z);
  };
  if (own_box) {                                // no footprint: the object is its own box, centred, half sizes = size
    const double sx = size[q * 3 + 0], sy = size[q * 3 + 1], sz = size[q * 3 + 2];
    ylo = __dadd_rn(-sy, p.ty);
    yhi = __dadd_rn(sy, p.ty);
    put(-sx, -sz); put(-sx, sz); put(sx, -sz); put(sx, sz);
  } else {
    const double* bb = raw_aabb + m * 6;
    ylo = __dadd_rn(__dsub_rn(__dmul_rn(bb[1], p.ky), p.cy), p.ty);
    yhi = __dadd_rn(__dsub_rn(__dmul_rn(bb[4], p.ky), p.cy), p.ty);
    for (int v = beg; v < end; ++v)
      put(__dsub_rn(__dmul_rn(hull_xz[2 * v], p.kx), p.cx), __dsub_rn(__dmul_rn(hull_xz[2 * v + 1], p.kz), p.cz));
  }
  o[0] = x1; o[1] = fmin(ylo, yhi); o[2] = z1;  // a negative size mirrors the object: min <= max still holds
  o[3] = x2; o[4] = fmax(ylo, yhi); o[5] = z2;
}

struct PairIou { float iou, overlap; };

// axis_aligned_bbox_overlaps_3d (scripts/utils.py:560-662) for one pair, in torch's evaluation order.
__device__ __forceinline__ PairIou pair_iou(const float* a, const float* b, float area_a, float area_b) {
  float wh[3];
#pragma unroll
  for (int k = 0; k < 3; ++k) wh[k] = fmaxf(__fsub_rn(fminf(a[3 + k], b[3 + k]), fmaxf(a[k], b[k])), 0.f);
  PairIou r;
  r.overlap = __fmul_rn(__fmul_rn(wh[0], wh[1]), wh[2]);
  const float uni = fmaxf(__fsub_rn(__fadd_rn(area_a, area_b), r.overlap), 1e-6f);
  r.iou = __fdiv_rn(r.overlap, uni);
  return r;
}

// judge_if_symmetry (scripts/utils.py:703-714) on the fp64 bounds, size_diff = pos_diff = 0.1.
__device__ __forceinline__ bool symmetric(const double* a, const double* b) {
  double dmax = 0.0;
  bool nan = false;
  for (int k = 0; k < 3; ++k) {
    const double d = fabs(__dsub_rn(__dmul_rn(__dsub_rn(a[3 + k], a[k]), 0.5), __dmul_rn(__dsub_rn(b[3 + k], b[k]), 0.5)));
    nan |= d != d;
    dmax = fmax(dmax, d);
  }
  if (nan || !(dmax < 0.1)) return false;
  const double dx = fabs(__dsub_rn(__dmul_rn(__dadd_rn(a[3], a[0]), 0.5), __dmul_rn(__dadd_rn(b[3], b[0]), 0.5)));
  const double dz = fabs(__dsub_rn(__dmul_rn(__dadd_rn(a[5], a[2]), 0.5), __dmul_rn(__dadd_rn(b[5], b[2]), 0.5)));
  return dx < 0.1 || dz < 0.1;
}

// One warp per scene over its kept objects, in slot order.  Outputs follow computer_intersection /
// computer_symmetry (scripts/utils.py:664-745): the IoU sum over pairs i < j in lexicographic order, accumulated
// serially in fp32 as the reference's sum() over numpy float32 scalars does; the count of pairs with IoU > 0; the
// overlap ratio sum(overlap) / (sum(area) - sum(overlap)) over distinct pairs; the symmetric pairs among those with
// equal class and, when model ids are given, equal model.  0 or 1 kept objects give (n, 1, 0, 0, 0) and 0.
__global__ void __launch_bounds__(SE_WARPS * 32)
k_scene_stats(const double* __restrict__ bounds, const uint8_t* __restrict__ keep, const int64_t* __restrict__ cls,
              const int64_t* __restrict__ model_id, int B, int N, int32_t* __restrict__ o_nobj,
              int32_t* __restrict__ o_npairs, float* __restrict__ o_iou_sum, int32_t* __restrict__ o_insec,
              float* __restrict__ o_ratio, int32_t* __restrict__ o_nsym, float* __restrict__ o_pair_iou) {
  __shared__ float s_box[SE_WARPS][SE_MAX_N][6];
  __shared__ float s_area[SE_WARPS][SE_MAX_N];
  __shared__ int s_slot[SE_WARPS][SE_MAX_N];
  __shared__ int s_rank[SE_WARPS][SE_MAX_N];
  __shared__ float s_iou[SE_WARPS][SE_MAX_PAIRS];
  const int w = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int b = blockIdx.x * SE_WARPS + w;
  if (b >= B) return;
  const int64_t base = (int64_t)b * N;

  // compaction of the kept slots (ranks in slot order)
  int n = 0;
  for (int s0 = 0; s0 < N; s0 += 32) {
    const int s = s0 + lane;
    const bool k = s < N && (keep == nullptr || keep[base + s] != 0);
    const unsigned bal = __ballot_sync(0xffffffffu, k);
    const int r = n + __popc(bal & ((1u << lane) - 1u));
    if (s < N) s_rank[w][s] = k ? r : -1;
    if (k) s_slot[w][r] = s;
    n += __popc(bal);
  }
  __syncwarp();
  // fp32 boxes (the reference's astype(np.float32)) and volumes ((dx * dy) * dz)
  for (int r = lane; r < n; r += 32) {
    const double* src = bounds + (base + s_slot[w][r]) * 6;
    float* bx = s_box[w][r];
    for (int k = 0; k < 6; ++k) bx[k] = __double2float_rn(src[k]);
    s_area[w][r] = __fmul_rn(__fmul_rn(__fsub_rn(bx[3], bx[0]), __fsub_rn(bx[4], bx[1])), __fsub_rn(bx[5], bx[2]));
  }
  __syncwarp();
  if (o_pair_iou) {                             // the full [N, N] matrix by slot, 0 where a slot is not kept
    float* dst = o_pair_iou + (int64_t)b * N * N;
    for (int e = lane; e < N * N; e += 32) {
      const int ri = s_rank[w][e / N], rj = s_rank[w][e % N];
      dst[e] = ri < 0 || rj < 0 ? 0.f : pair_iou(s_box[w][ri], s_box[w][rj], s_area[w][ri], s_area[w][rj]).iou;
    }
  }
  if (n <= 1) {
    if (lane == 0) {
      o_nobj[b] = n; o_npairs[b] = 1; o_iou_sum[b] = 0.f; o_insec[b] = 0; o_ratio[b] = 0.f; o_nsym[b] = 0;
    }
    return;
  }

  int insec = 0, nsym = 0;
  double ov = 0.0;
  for (int i = 0; i < n - 1; ++i) {
    const int row = i * n - i * (i + 1) / 2 - i - 1;      // pair (i, j) is s_iou[row + j]
    const int si = s_slot[w][i];
    for (int j = i + 1 + lane; j < n; j += 32) {
      const PairIou p = pair_iou(s_box[w][i], s_box[w][j], s_area[w][i], s_area[w][j]);
      s_iou[w][row + j] = p.iou;
      insec += p.iou > 0.f;
      ov = __dadd_rn(ov, (double)p.overlap);
      const int sj = s_slot[w][j];
      if (cls[base + si] == cls[base + sj] && (model_id == nullptr || model_id[base + si] == model_id[base + sj]))
        nsym += symmetric(bounds + (base + si) * 6, bounds + (base + sj) * 6);
    }
  }
  double area = 0.0;
  for (int r = lane; r < n; r += 32) area = __dadd_rn(area, (double)s_area[w][r]);
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    ov = __dadd_rn(ov, __shfl_xor_sync(0xffffffffu, ov, o));
    area = __dadd_rn(area, __shfl_xor_sync(0xffffffffu, area, o));
    insec += __shfl_xor_sync(0xffffffffu, insec, o);
    nsym += __shfl_xor_sync(0xffffffffu, nsym, o);
  }
  __syncwarp();
  if (lane == 0) {
    const int P = n * (n - 1) / 2;
    float sum = 0.f;
    for (int p = 0; p < P; ++p) {
      const float v = s_iou[w][p];
      sum = __fadd_rn(sum, v > 0.f ? v : 0.f);
    }
    // overlap.sum() / 2 over the symmetric matrix with a zero diagonal is the sum over distinct pairs, and
    // (area1.sum() + area2.sum()) / 2 is the volume sum.  Both sums are taken in fp64 and rounded once, so they
    // differ from torch's fp32 reductions only by those reductions' own rounding; the rest is the reference's fp32
    // arithmetic, with its 0 / 0 = NaN.
    const float ov32 = __double2float_rn(ov), area32 = __double2float_rn(area);
    const float area_sum = __fsub_rn(__fmul_rn(__fadd_rn(area32, area32), 0.5f), ov32);
    o_nobj[b] = n; o_npairs[b] = P; o_iou_sum[b] = sum; o_insec[b] = insec;
    o_ratio[b] = __fdiv_rn(ov32, area_sum); o_nsym[b] = nsym;
  }
}

}  // namespace
}  // namespace ds

extern "C" int ds_scene_boxes(const float* translation_dev, const float* size_dev, const float* angle_dev,
                              const int64_t* model_index_dev, int32_t num_objects, const int32_t* hull_offsets_dev,
                              const double* hull_xz_dev, int32_t num_hull_vertices, const double* raw_half_dev,
                              const double* raw_aabb_dev, int32_t num_models, double* bounds_dev, void* stream) {
  if (!translation_dev || !size_dev || !angle_dev || !bounds_dev)
    return fail(DS_ERR_INVALID, "ds_scene_boxes: NULL translation, size, angle or bounds pointer");
  if (num_objects < 0 || num_models < 0 || num_hull_vertices < 0)
    return fail(DS_ERR_INVALID, "ds_scene_boxes: negative count (objects %d, models %d, hull vertices %d)",
                num_objects, num_models, num_hull_vertices);
  if (num_models > 0 && (!hull_offsets_dev || !raw_half_dev || !raw_aabb_dev || (num_hull_vertices > 0 && !hull_xz_dev)))
    return fail(DS_ERR_INVALID, "ds_scene_boxes: NULL footprint table for %d models", num_models);
  int ndev = 0;
  if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) {
    cudaGetLastError();
    return fail(DS_ERR_NO_DEVICE, "no CUDA device: diffuscene_b200 has no CPU fallback");
  }
  const int work = std::max(num_objects, num_models);
  if (work == 0) return 0;
  cudaStream_t s = (cudaStream_t)stream;
  int* err_dev = nullptr;
  CK(cudaMallocAsync(&err_dev, sizeof(int), s));
  CK(cudaMemsetAsync(err_dev, 0, sizeof(int), s));
  k_scene_boxes<<<cdiv(work, 128), 128, 0, s>>>(translation_dev, size_dev, angle_dev, model_index_dev, num_objects,
                                                num_models ? hull_offsets_dev : nullptr, hull_xz_dev,
                                                num_hull_vertices, raw_half_dev, raw_aabb_dev, num_models, bounds_dev,
                                                err_dev);
  int err = 0;
  cudaError_t e = cudaGetLastError();
  if (e == cudaSuccess) e = cudaMemcpyAsync(&err, err_dev, sizeof(int), cudaMemcpyDeviceToHost, s);
  cudaFreeAsync(err_dev, s);
  if (e == cudaSuccess) e = cudaStreamSynchronize(s);
  if (e != cudaSuccess) return fail(DS_ERR_CUDA, "ds_scene_boxes: %s", cudaGetErrorString(e));
  if (err & SE_ERR_OFFSETS)
    return fail(DS_ERR_INVALID, "ds_scene_boxes: hull offsets must start at >= 0, not decrease and end at <= %d",
                num_hull_vertices);
  if (err & SE_ERR_INDEX)
    return fail(DS_ERR_INVALID, "ds_scene_boxes: model index outside [-1, %d)", num_models);
  return 0;
}

extern "C" int ds_scene_stats(const double* bounds_dev, const uint8_t* keep_dev, const int64_t* class_dev,
                              const int64_t* model_id_dev, int32_t batch, int32_t num_objects,
                              int32_t* num_objects_dev, int32_t* num_pairs_dev, float* iou_sum_dev,
                              int32_t* insec_count_dev, float* overlap_ratio_dev, int32_t* num_symmetry_dev,
                              float* pair_iou_dev, void* stream) {
  if (!num_objects_dev || !num_pairs_dev || !iou_sum_dev || !insec_count_dev || !overlap_ratio_dev ||
      !num_symmetry_dev || (num_objects > 0 && (!bounds_dev || !class_dev)))
    return fail(DS_ERR_INVALID, "ds_scene_stats: NULL bounds, class or output pointer");
  if (batch < 0) return fail(DS_ERR_INVALID, "ds_scene_stats: batch %d < 0", batch);
  if (num_objects < 0 || num_objects > SE_MAX_N)
    return fail(DS_ERR_INVALID, "ds_scene_stats: %d objects per scene outside [0, %d]", num_objects, SE_MAX_N);
  int ndev = 0;
  if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) {
    cudaGetLastError();
    return fail(DS_ERR_NO_DEVICE, "no CUDA device: diffuscene_b200 has no CPU fallback");
  }
  if (batch == 0) return 0;
  k_scene_stats<<<cdiv(batch, SE_WARPS), SE_WARPS * 32, 0, (cudaStream_t)stream>>>(
      bounds_dev, keep_dev, class_dev, model_id_dev, batch, num_objects, num_objects_dev, num_pairs_dev, iou_sum_dev,
      insec_count_dev, overlap_ratio_dev, num_symmetry_dev, pair_iou_dev);
  CK(cudaGetLastError());
  return 0;
}
