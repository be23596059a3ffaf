// Training batches of preprocessed rooms (DESIGN.md, "Training data"): one launch turns B scene indices and their
// per-scene draws into the tensors the reference's `Diffusion.__getitem__` + default collate give
// (scene_synthesis/datasets/threed_front_dataset.py:313-584, 888-925).  One warp per scene and one lane per object
// (N <= 32): each lane carries its object through the augmentations in the configured order, the scaling, and then
// writes its row at the slot the permutation gives it; lanes L..N-1 write the padding rows.  blockIdx.y == 1 copies
// (and, under a fixed rotation, rotates by a quarter-turn index permutation) the same scenes' room layouts.
//
// Precision follows numpy's promotion in the reference chain: a rotation turns translations and angles into fp64
// (R is float64), a jitter on an fp32 key is an fp32 add, scaling casts to fp32 once and normalises against fp64
// bounds, and the result is cast to fp32.  Every operation is an explicit _rn intrinsic, so no FMA contraction
// changes a rounding.
#include "engine_internal.h"

namespace ds {
namespace {

constexpr int WARPS = 4;
constexpr double TWO_PI = 6.283185307179586;           // 2 * np.pi
constexpr double HALF_PI = 1.5707963267948966;         // np.pi * 0.5

struct Bounds {
  double t_lo[3], t_hi[3], s_lo[3], s_hi[3], a_lo, a_hi, f_lo, f_hi;
};

struct Aug {
  int n, op[2];
};

__device__ __forceinline__ float f32add(double a, double b) { return __fadd_rn((float)a, (float)b); }

// numpy's float64 remainder (npy_divmod): fmod, then moved into the divisor's sign; an exact zero becomes +0.
__device__ __forceinline__ double pymod(double a, double b) {
  double m = fmod(a, b);
  if (m != 0.0) {
    if ((b < 0.0) != (m < 0.0)) m = __dadd_rn(m, b);
  } else {
    m = copysign(0.0, b);
  }
  return m;
}

// Scale.scale: X = x.astype(float32); clip to [lo, hi] (fp64); 2 * (X - lo) / (hi - lo) - 1 in fp64; then fp32.
__device__ __forceinline__ float scale01(double x, double lo, double hi) {
  double X = (double)(float)x;
  X = X < lo ? lo : (X > hi ? hi : X);       // np.clip = minimum(maximum(X, lo), hi); NaN stays NaN
  const double q = __ddiv_rn(__dsub_rn(X, lo), __dsub_rn(hi, lo));
  return (float)__dsub_rn(__dmul_rn(2.0, q), 1.0);
}

__global__ void __launch_bounds__(WARPS * 32) k_scene_batch(
    const int32_t* __restrict__ offsets, const int32_t* __restrict__ lengths, const int32_t* __restrict__ cls,
    const float* __restrict__ tr, const float* __restrict__ sz, const float* __restrict__ an,
    const float* __restrict__ of, const float* __restrict__ layouts, int num_scenes, int ncols, int F, int H, int W,
    Bounds bd, int cosin, int angle_dim, int permute, Aug aug, int B, int N, const int64_t* __restrict__ scene_index,
    const double* __restrict__ rot_angle, const double* __restrict__ jitter, const float* __restrict__ perm_key,
    float* __restrict__ o_cls, float* __restrict__ o_tr, float* __restrict__ o_sz, float* __restrict__ o_an,
    float* __restrict__ o_of, int64_t* __restrict__ o_len, float* __restrict__ o_layout) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int b = blockIdx.x * WARPS + warp;
  if (blockIdx.y == 1) {
    // room layouts: the block's WARPS scenes, every thread over every pixel of each
    const int64_t HW = (int64_t)H * W;
    for (int w = 0; w < WARPS; ++w) {
      const int bb = blockIdx.x * WARPS + w;
      if (bb >= B) break;
      const int64_t s = scene_index[bb];
      if (s < 0 || s >= num_scenes) continue;
      int k = 0;
      for (int a = 0; a < aug.n; ++a)
        if (aug.op[a] == DS_SCENE_AUG_FIXED_ROTATION) k = (int)llrint(__ddiv_rn(rot_angle[bb], HALF_PI)) & 3;
      const float* src = layouts + s * HW;
      float* dst = o_layout + (int64_t)bb * HW;
      for (int64_t p = threadIdx.x; p < HW; p += blockDim.x) {
        const int i = int(p / W), j = int(p % W);
        int si = i, sj = j;                      // np.rot90(img, k)[i, j] (square when k is odd)
        if (k == 1) { si = j; sj = W - 1 - i; }
        else if (k == 2) { si = H - 1 - i; sj = W - 1 - j; }
        else if (k == 3) { si = H - 1 - j; sj = i; }
        dst[p] = src[(int64_t)si * W + sj];
      }
    }
    return;
  }
  if (b >= B) return;
  const int64_t s = scene_index[b];
  if (s < 0 || s >= num_scenes) return;
  const int L = min((int)lengths[s], N);
  const bool real = lane < L;
  const int64_t o = (int64_t)offsets[s] + (real ? lane : 0);

  // the object as the reference holds it: values with their numpy dtype (fp32 until a rotation makes them fp64)
  double t[3] = {0.0, 0.0, 0.0}, a = 0.0;
  float sv[3] = {0.f, 0.f, 0.f};
  bool t64 = false, a64 = false;
  if (real) {
    for (int c = 0; c < 3; ++c) {
      t[c] = tr[o * 3 + c];
      sv[c] = sz[o * 3 + c];
    }
    a = an[o];
  }
  for (int q = 0; q < aug.n; ++q) {
    if (aug.op[q] == DS_SCENE_AUG_JITTER) {
      const double* j = jitter + (int64_t)b * 3;          // one draw per key, in the keys' order
      for (int c = 0; c < 3; ++c) {
        t[c] = t64 ? __dadd_rn(t[c], j[0]) : (double)f32add(t[c], j[0]);
        sv[c] = f32add(sv[c], j[1]);
      }
      a = a64 ? __dadd_rn(a, j[2]) : (double)f32add(a, j[2]);
    } else {
      // translations @ R(theta) (x' = x cos + z sin, z' = -x sin + z cos); angles (a + theta - lo) % 2 pi + lo
      const double th = rot_angle[b];
      double sn, cs;
      sincos(th, &sn, &cs);
      const double x = t[0], y = t[1], z = t[2];
      t[0] = __dadd_rn(__dadd_rn(__dmul_rn(x, cs), __dmul_rn(y, 0.0)), __dmul_rn(z, sn));
      t[1] = __dadd_rn(__dadd_rn(__dmul_rn(x, 0.0), __dmul_rn(y, 1.0)), __dmul_rn(z, 0.0));
      t[2] = __dadd_rn(__dadd_rn(__dmul_rn(x, -sn), __dmul_rn(y, 0.0)), __dmul_rn(z, cs));
      t64 = true;
      const double v = a64 ? __dadd_rn(a, th) : (double)f32add(a, th);
      a = __dadd_rn(pymod(__dsub_rn(v, bd.a_lo), TWO_PI), bd.a_lo);
      a64 = true;
    }
  }

  int slot = lane;
  if (permute) {      // rank of the key within the scene, ties broken by index
    const float key = lane < L ? perm_key[(int64_t)b * N + lane] : 0.f;
    int r = 0;
    for (int j = 0; j < L; ++j) {
      const float kj = __shfl_sync(0xffffffffu, key, j);
      r += (kj < key) || (kj == key && j < lane);
    }
    if (real) slot = r;
  }
  if (lane >= N) return;

  const int C = ncols - 1;
  const int64_t row = (int64_t)b * N + slot;
  // class labels: start column dropped, the end label on padding rows, in +-1
  int hot = C - 1;
  if (real) {
    const int c = cls[o];
    hot = c < ncols - 2 ? c : (c == ncols - 1 ? C - 1 : -1);
  }
  for (int c = 0; c < C; ++c) o_cls[row * C + c] = c == hot ? 1.f : -1.f;
  for (int c = 0; c < 3; ++c) {
    o_tr[row * 3 + c] = real ? scale01(t[c], bd.t_lo[c], bd.t_hi[c]) : 0.f;
    o_sz[row * 3 + c] = real ? scale01(sv[c], bd.s_lo[c], bd.s_hi[c]) : 0.f;
  }
  if (cosin) {
    double sn, cs;
    sincos(a, &sn, &cs);
    o_an[row * 2 + 0] = real ? (float)cs : 0.f;
    o_an[row * 2 + 1] = real ? (float)sn : 0.f;
  } else {
    o_an[row * angle_dim] = real ? scale01(a, bd.a_lo, bd.a_hi) : 0.f;
  }
  if (F > 0) {
    const float4* src = reinterpret_cast<const float4*>(of + o * F);
    float4* dst = reinterpret_cast<float4*>(o_of + row * F);
    for (int c = 0; c < F / 4; ++c) {
      float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
      if (real) {
        v = src[c];
        if (cosin) {
          v.x = scale01(v.x, bd.f_lo, bd.f_hi);
          v.y = scale01(v.y, bd.f_lo, bd.f_hi);
          v.z = scale01(v.z, bd.f_lo, bd.f_hi);
          v.w = scale01(v.w, bd.f_lo, bd.f_hi);
        }
      }
      dst[c] = v;
    }
  }
  if (lane == 0) o_len[b] = L;
}

bool aligned16(const void* p) { return ((uintptr_t)p & 15) == 0; }

}  // namespace
}  // namespace ds

extern "C" int ds_scene_batch(const ds_scene_batch_args* a, void* stream) {
  using namespace ds;
  if (!a) return fail(DS_ERR_INVALID, "ds_scene_batch: NULL args");
  const int B = a->batch, N = a->num_slots, F = a->objfeat_dim;
  const bool layouts = a->layout_h > 0 || a->layout_w > 0;
  if (B < 0) return fail(DS_ERR_INVALID, "ds_scene_batch: batch %d < 0", B);
  if (N < 1 || N > 32) return fail(DS_ERR_INVALID, "ds_scene_batch: num_slots %d outside [1, 32]", N);
  if (a->num_scenes < 1) return fail(DS_ERR_INVALID, "ds_scene_batch: num_scenes %d < 1", a->num_scenes);
  if (a->num_class_columns < 2)
    return fail(DS_ERR_INVALID, "ds_scene_batch: num_class_columns %d < 2 (classes + start + end)",
                a->num_class_columns);
  if (F < 0 || F > 256 || F % 4 != 0)
    return fail(DS_ERR_INVALID, "ds_scene_batch: objfeat_dim %d is not a multiple of 4 in [0, 256]", F);
  if (a->scaling != DS_SCENE_SCALE && a->scaling != DS_SCENE_SCALE_COSIN_OBJFEATSNORM)
    return fail(DS_ERR_INVALID, "ds_scene_batch: unknown scaling %d", a->scaling);
  const int want_angle_dim = a->scaling == DS_SCENE_SCALE ? 1 : 2;
  if (a->angle_dim != want_angle_dim)
    return fail(DS_ERR_INVALID, "ds_scene_batch: angle_dim %d, the scaling writes %d", a->angle_dim, want_angle_dim);
  if (layouts && (a->layout_h < 1 || a->layout_h > 4096 || a->layout_w < 1 || a->layout_w > 4096))
    return fail(DS_ERR_INVALID, "ds_scene_batch: layout size %d x %d outside [1, 4096]", a->layout_h, a->layout_w);
  if (a->num_augmentations < 0 || a->num_augmentations > 2)
    return fail(DS_ERR_INVALID, "ds_scene_batch: %d augmentations, at most one rotation and one jitter",
                a->num_augmentations);
  Aug aug{a->num_augmentations, {0, 0}};
  int n_rot = 0, n_jit = 0;
  for (int q = 0; q < aug.n; ++q) {
    const int op = a->augmentations[q];
    aug.op[q] = op;
    if (op == DS_SCENE_AUG_FIXED_ROTATION || op == DS_SCENE_AUG_ROTATION) {
      ++n_rot;
      if (layouts && op == DS_SCENE_AUG_ROTATION)
        return fail(DS_ERR_INVALID, "ds_scene_batch: continuous rotations of room layouts are not supported");
      if (layouts && a->layout_h != a->layout_w)
        return fail(DS_ERR_INVALID, "ds_scene_batch: rotated layouts must be square, not %d x %d", a->layout_h,
                    a->layout_w);
    } else if (op == DS_SCENE_AUG_JITTER) {
      ++n_jit;
    } else {
      return fail(DS_ERR_INVALID, "ds_scene_batch: unknown augmentation %d", op);
    }
  }
  if (n_rot > 1 || n_jit > 1)
    return fail(DS_ERR_INVALID, "ds_scene_batch: at most one rotation and one jitter");
  if (!a->offsets_dev || !a->lengths_dev || !a->class_dev || !a->translations_dev || !a->sizes_dev ||
      !a->angles_dev || !a->scene_index_dev || !a->class_labels_out_dev || !a->translations_out_dev ||
      !a->sizes_out_dev || !a->angles_out_dev || !a->length_out_dev)
    return fail(DS_ERR_INVALID, "ds_scene_batch: NULL store, index or output pointer");
  if (F > 0 && (!a->objfeats_dev || !a->objfeats_out_dev))
    return fail(DS_ERR_INVALID, "ds_scene_batch: objfeat_dim %d needs objfeats and objfeats_out", F);
  if (F > 0 && (!aligned16(a->objfeats_dev) || !aligned16(a->objfeats_out_dev)))
    return fail(DS_ERR_INVALID, "ds_scene_batch: objfeats pointers must be 16-byte aligned");
  if (layouts && (!a->layouts_dev || !a->room_layout_out_dev))
    return fail(DS_ERR_INVALID, "ds_scene_batch: a layout size needs layouts and room_layout_out");
  if (n_rot && !a->rot_angle_dev) return fail(DS_ERR_INVALID, "ds_scene_batch: a rotation needs rot_angle");
  if (n_jit && !a->jitter_dev) return fail(DS_ERR_INVALID, "ds_scene_batch: a jitter needs jitter draws");
  if (a->permute && !a->perm_key_dev) return fail(DS_ERR_INVALID, "ds_scene_batch: permute needs perm_key");
  if (const int rc = require_device()) return rc;
  if (B == 0) return 0;
  Bounds bd;
  for (int c = 0; c < 3; ++c) {
    bd.t_lo[c] = a->bounds_translations[c];
    bd.t_hi[c] = a->bounds_translations[3 + c];
    bd.s_lo[c] = a->bounds_sizes[c];
    bd.s_hi[c] = a->bounds_sizes[3 + c];
  }
  bd.a_lo = a->bounds_angles[0];
  bd.a_hi = a->bounds_angles[1];
  bd.f_lo = a->bounds_objfeats[0];
  bd.f_hi = a->bounds_objfeats[1];
  const dim3 grid((B + WARPS - 1) / WARPS, layouts ? 2 : 1);
  k_scene_batch<<<grid, WARPS * 32, 0, (cudaStream_t)stream>>>(
      a->offsets_dev, a->lengths_dev, a->class_dev, a->translations_dev, a->sizes_dev, a->angles_dev,
      a->objfeats_dev, a->layouts_dev, a->num_scenes, a->num_class_columns, F, layouts ? a->layout_h : 0,
      layouts ? a->layout_w : 0, bd, a->scaling == DS_SCENE_SCALE_COSIN_OBJFEATSNORM, a->angle_dim,
      a->permute != 0, aug, B, N, a->scene_index_dev, a->rot_angle_dev, a->jitter_dev, a->perm_key_dev,
      a->class_labels_out_dev, a->translations_out_dev, a->sizes_out_dev, a->angles_out_dev, a->objfeats_out_dev,
      a->length_out_dev, a->room_layout_out_dev);
  const cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return fail(DS_ERR_CUDA, "ds_scene_batch: %s", cudaGetErrorString(e));
  return 0;
}
