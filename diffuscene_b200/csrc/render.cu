// Top-down rendering of placed furniture meshes (the reference's render_top2down through simple-3dviz,
// scripts/generate_diffusion.py:251-264 / preprocess_data.py:297-350) and the perspective views of its
// completion / rearrangement driver (scripts/utils.py:431-458): a batched rasterizer writing uint8 [B, H, W, 3]
// images on the device.  Stateful catalogue handle (ds_mesh_catalog_*) and one render call.
//
// Pipeline per call (both kernels are templated on the projection; the orthographic instantiation is the original):
//   k_render_prep    one thread per (scene, slot): the shared placement (placement.cuh) composed with the camera into
//                    fp32 affine maps raw vertex -> (pixel x, pixel y, depth) (perspective: (pixel x * depth,
//                    pixel y * depth, depth), divided per vertex) and raw vertex -> world, and the object's
//                    conservative pixel bounds; slot N is the scene's floor.
//   k_render_tiles   one CTA per (scene, 64 x 64 tile): visibility by atomicMin of (depth bits, slot, face) into a
//                    shared-memory tile, then a resolve pass per pixel that recomputes barycentrics and shades.
//                    Perspective faces are clipped at depth = near in view space into at most two triangles first;
//                    depth and barycentrics are interpolated perspective-correctly.
// atomicMin is order independent, so an image depends neither on scheduling nor on the rest of the batch.
#include <mutex>
#include <set>

#include "engine_internal.h"
#include "placement.cuh"

namespace ds {
namespace {

constexpr int RT = 64;                          // tile side in pixels
constexpr int RT_THREADS = 256;
constexpr int SMALL_TRI_PIXELS = 64;            // larger bounding boxes are rasterised by the whole CTA
constexpr int FACE_BITS = 25;                   // id = slot << 25 | face; slot <= 64 (the floor is slot N)
constexpr int MAX_SLOTS = 64;
constexpr unsigned long long EMPTY_KEY = ~0ull;
constexpr float AMBIENT = 0.35f, DIFFUSE = 0.65f;  // shade = AMBIENT + DIFFUSE * |n . l|
constexpr float FLOOR_UV_PERIOD = 0.3f;         // floor texture repeats every 30 cm (scripts/utils.py:99-114)

enum { RE_MODEL = 1, RE_CLASS = 2, RE_FLOOR_OFF = 4, RE_FLOOR_TEX = 8, RE_FLOOR_COUNT = 16 };
enum { RF_NO_TEXTURE = 1, RF_WHITE_BACKGROUND = 2 };

struct Catalog {
  int device = 0, M = 0, T = 0;
  int64_t V = 0, F = 0;
  int* vert_off = nullptr;      // [M + 1]
  float* verts = nullptr;       // [V, 3] raw vertices
  int* face_off = nullptr;      // [M + 1]
  int* faces = nullptr;         // [F, 3] model-local vertex indices
  float* uvs = nullptr;         // [F, 3, 2] per-corner UVs, NaN: the face has none
  double* half = nullptr;       // [M, 3]
  double* aabb = nullptr;       // [M, 6]
  float* kd = nullptr;          // [M, 3]
  uint8_t* tex = nullptr;       // [M, T, T, 3]
};

std::mutex g_cat_mu;
std::set<void*> g_cats;         // live handles: anything else passed as a catalogue is rejected

// Per (scene, slot): pixel-space map rows 0..2 (x, y, depth) and world rows 3..5, each (a, b, c, d): a*vx+b*vy+c*vz+d.
struct ObjXf { float m[6][4]; int x0, y0, x1, y1; float umin, vmin; int faces, pad; };

struct Cam { double m[3][4]; float near_p, far_p, eye[3]; int W, H; };

__device__ __forceinline__ float apply(const float* r, float x, float y, float z) {
  return __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(r[0], x), __fmul_rn(r[1], y)), __fmul_rn(r[2], z)), r[3]);
}

// Writes the 3 x 4 composition cam * (R (K v - c) + t) as fp32 rows; K = diag(k), R rotates about y.
__device__ void compose(const Cam& cam, const Placement& p, float (*px)[4], float (*wx)[4]) {
  // world = W v + w0 with W = R K: x = c kx vx + s kz vz, y = ky vy, z = -s kx vx + c kz vz
  double W[3][4];
  W[0][0] = p.c * p.kx; W[0][1] = 0; W[0][2] = p.s * p.kz;
  W[1][0] = 0; W[1][1] = p.ky; W[1][2] = 0;
  W[2][0] = -p.s * p.kx; W[2][1] = 0; W[2][2] = p.c * p.kz;
  W[0][3] = -(p.c * p.cx + p.s * p.cz) + p.tx;
  W[1][3] = -p.cy + p.ty;
  W[2][3] = -(-p.s * p.cx + p.c * p.cz) + p.tz;
  for (int r = 0; r < 3; ++r) {
    for (int c = 0; c < 4; ++c) {
      wx[r][c] = (float)W[r][c];
      double a = c == 3 ? cam.m[r][3] : 0.0;
      for (int k = 0; k < 3; ++k) a += cam.m[r][k] * W[k][c];
      px[r][c] = (float)a;
    }
  }
}

template <bool PERSP>
__global__ void k_render_prep(Cam cam, const float* __restrict__ trans, const float* __restrict__ size,
                              const float* __restrict__ angle, const int64_t* __restrict__ model,
                              const int64_t* __restrict__ cls, int num_colors, int check_cls,
                              const int* __restrict__ vert_off, const float* __restrict__ verts,
                              const int* __restrict__ face_off, const double* __restrict__ half,
                              const double* __restrict__ aabb, int M, const int* __restrict__ floor_off,
                              const float* __restrict__ floor_tris, int floor_total,
                              const int* __restrict__ floor_tex_idx, int num_floor_tex, int B, int N,
                              ObjXf* __restrict__ xf, int* __restrict__ err) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= B * (N + 1)) return;
  const int b = i / (N + 1), slot = i % (N + 1);
  ObjXf o;
  o.x0 = o.y0 = 1; o.x1 = o.y1 = 0; o.faces = 0; o.umin = o.vmin = 0.f; o.pad = 0;
  float lo[3] = {INFINITY, INFINITY, INFINITY}, hi[3] = {-INFINITY, -INFINITY, -INFINITY};
  if (slot < N) {
    const int64_t q = (int64_t)b * N + slot;
    const int64_t m = model[q];
    if (m < -1 || m >= M) { atomicOr(err, RE_MODEL); xf[i] = o; return; }
    if (m < 0) { xf[i] = o; return; }
    if (check_cls && (cls[q] < 0 || cls[q] >= num_colors)) { atomicOr(err, RE_CLASS); xf[i] = o; return; }
    const Placement p = make_placement(size + q * 3, trans + q * 3, angle[q], half + m * 3, aabb + m * 6);
    compose(cam, p, o.m, o.m + 3);
    o.faces = face_off[m + 1] - face_off[m];
    // the placed mesh lies in the placed raw AABB: its 8 corners bound the screen footprint
    const double* bb = aabb + m * 6;
    for (int c = 0; c < 8; ++c) {
      const float vx = (float)bb[(c & 1) ? 3 : 0], vy = (float)bb[(c & 2) ? 4 : 1], vz = (float)bb[(c & 4) ? 5 : 2];
      for (int r = 0; r < 3; ++r) {
        const float v = apply(o.m[r], vx, vy, vz);
        lo[r] = fminf(lo[r], v); hi[r] = fmaxf(hi[r], v);
      }
    }
  } else {
    if (!floor_off) { xf[i] = o; return; }
    const int a = floor_off[b], e = floor_off[b + 1];
    if (a < 0 || e < a || e > floor_total) { atomicOr(err, RE_FLOOR_OFF); xf[i] = o; return; }
    if (e - a >= (1 << FACE_BITS)) { atomicOr(err, RE_FLOOR_COUNT); xf[i] = o; return; }
    if (floor_tex_idx && (floor_tex_idx[b] < -1 || floor_tex_idx[b] >= num_floor_tex)) {
      atomicOr(err, RE_FLOOR_TEX); xf[i] = o; return;
    }
    for (int r = 0; r < 3; ++r)
      for (int c = 0; c < 4; ++c) {
        o.m[r][c] = (float)cam.m[r][c];
        o.m[3 + r][c] = r == c ? 1.f : 0.f;
      }
    o.faces = e - a;
    float umin = INFINITY, vmin = INFINITY;
    for (int t = a; t < e; ++t)
      for (int k = 0; k < 3; ++k) {
        const float* v = floor_tris + (int64_t)t * 9 + k * 3;
        umin = fminf(umin, v[0]); vmin = fminf(vmin, v[2]);
        for (int r = 0; r < 3; ++r) {
          const float s = apply(o.m[r], v[0], v[1], v[2]);
          lo[r] = fminf(lo[r], s); hi[r] = fmaxf(hi[r], s);
        }
      }
    o.umin = umin; o.vmin = vmin;
  }
  if constexpr (PERSP) {
    // rows 0 and 1 are pixel coordinates times depth: the pixel range of a box wholly in front of the near plane is
    // that of its divided corners (a projective map keeps convex hulls there); a box that reaches the near plane
    // may cover any pixel
    if (o.faces > 0 && hi[2] >= cam.near_p * 0.999f && lo[2] <= cam.far_p * 1.001f) {
      if (lo[2] >= cam.near_p * 1.001f) {
        float sl[2] = {INFINITY, INFINITY}, sh[2] = {-INFINITY, -INFINITY};
        if (slot < N) {
          const double* bb = aabb + model[(int64_t)b * N + slot] * 6;
          for (int c = 0; c < 8; ++c) {
            const float vx = (float)bb[(c & 1) ? 3 : 0], vy = (float)bb[(c & 2) ? 4 : 1], vz = (float)bb[(c & 4) ? 5 : 2];
            const float d = apply(o.m[2], vx, vy, vz);
            for (int r = 0; r < 2; ++r) {
              const float v = __fdiv_rn(apply(o.m[r], vx, vy, vz), d);
              sl[r] = fminf(sl[r], v); sh[r] = fmaxf(sh[r], v);
            }
          }
        } else {
          for (int t = floor_off[b]; t < floor_off[b + 1]; ++t)
            for (int k = 0; k < 3; ++k) {
              const float* v = floor_tris + (int64_t)t * 9 + k * 3;
              const float d = apply(o.m[2], v[0], v[1], v[2]);
              for (int r = 0; r < 2; ++r) {
                const float s = __fdiv_rn(apply(o.m[r], v[0], v[1], v[2]), d);
                sl[r] = fminf(sl[r], s); sh[r] = fmaxf(sh[r], s);
              }
            }
        }
        lo[0] = sl[0]; hi[0] = sh[0]; lo[1] = sl[1]; hi[1] = sh[1];
      } else {
        lo[0] = lo[1] = -INFINITY; hi[0] = hi[1] = INFINITY;
      }
    } else {
      lo[0] = 1.f; hi[0] = 0.f;                    // culled
    }
  }
  // conservative pixel range (one pixel of slack for the fp32 rounding of the composed map), depth culled only when
  // the whole box lies beyond the clip range
  if (o.faces > 0 && hi[2] >= cam.near_p * 0.999f && lo[2] <= cam.far_p * 1.001f && lo[0] <= hi[0]) {
    o.x0 = max(0, (int)floorf(lo[0]) - 1); o.x1 = min(cam.W - 1, (int)ceilf(hi[0]) + 1);
    o.y0 = max(0, (int)floorf(lo[1]) - 1); o.y1 = min(cam.H - 1, (int)ceilf(hi[1]) + 1);
    if (!(lo[0] > -1e9f && hi[0] < 1e9f && lo[1] > -1e9f && hi[1] < 1e9f)) { o.x0 = 0; o.x1 = cam.W - 1; o.y0 = 0; o.y1 = cam.H - 1; }
  }
  xf[i] = o;
}

struct Tri { float x[3], y[3], d[3]; };

// Edge function of (a -> b) at p, evaluated with the endpoints in a canonical order so that an edge shared by two
// triangles gives exactly opposite values in both (watertight).
__device__ __forceinline__ float edge_fn(float ax, float ay, float bx, float by, float px, float py) {
  const bool sw = bx < ax || (bx == ax && by < ay);
  const float x0 = sw ? bx : ax, y0 = sw ? by : ay, x1 = sw ? ax : bx, y1 = sw ? ay : by;
  const float e = __fsub_rn(__fmul_rn(__fsub_rn(px, x0), __fsub_rn(y1, y0)), __fmul_rn(__fsub_rn(py, y0), __fsub_rn(x1, x0)));
  return sw ? -e : e;
}

// Coverage of pixel centre (px, py) with the top-left rule (y grows downwards): with the triangle oriented so its area
// is positive, a centre on an edge a -> b belongs to the triangle when b.y > a.y, or b.y == a.y and b.x < a.x.
// Returns false for degenerate triangles; w receives the barycentrics.
__device__ __forceinline__ bool cover(const Tri& t, float px, float py, float* w) {
  const float area = edge_fn(t.x[0], t.y[0], t.x[1], t.y[1], t.x[2], t.y[2]);
  if (!(area != 0.f) || !isfinite(area)) return false;
  const float sg = area > 0.f ? 1.f : -1.f;
  float e[3];
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    const int a = (k + 1) % 3, b = (k + 2) % 3;          // w_k belongs to the edge opposite vertex k
    e[k] = sg * edge_fn(t.x[a], t.y[a], t.x[b], t.y[b], px, py);
    float dx = __fsub_rn(t.x[b], t.x[a]), dy = __fsub_rn(t.y[b], t.y[a]);
    if (sg < 0.f) { dx = -dx; dy = -dy; }
    const bool owns = dy > 0.f || (dy == 0.f && dx < 0.f);
    if (!(e[k] > 0.f || (e[k] == 0.f && owns))) return false;
  }
  const float aa = fabsf(area);
#pragma unroll
  for (int k = 0; k < 3; ++k) w[k] = __fdiv_rn(e[k], aa);
  return true;
}

__device__ __forceinline__ float interp(const float* v, const float* w) {
  return __fadd_rn(__fadd_rn(__fmul_rn(w[0], v[0]), __fmul_rn(w[1], v[1])), __fmul_rn(w[2], v[2]));
}

// Corner k of face f of (scene, slot): raw (model) or world (floor) coordinates.
__device__ __forceinline__ void corner(int slot, int N, int f, int k, const int* faces, const int* face_off,
                                       const int* vert_off, const float* verts, int64_t m, const float* ftris,
                                       int fbeg, float& x, float& y, float& z) {
  if (slot < N) {
    const int v = vert_off[m] + faces[(int64_t)(face_off[m] + f) * 3 + k];
    x = verts[(int64_t)v * 3]; y = verts[(int64_t)v * 3 + 1]; z = verts[(int64_t)v * 3 + 2];
  } else {
    const float* p = ftris + (int64_t)(fbeg + f) * 9 + k * 3;
    x = p[0]; y = p[1]; z = p[2];
  }
}

__device__ __forceinline__ void sample_rgb(const uint8_t* tex, int T, float u, float v, float* rgb) {
  // bilinear, repeat wrap; v = 0 is the image's bottom row (OBJ convention), texel centres at (i + 0.5) / T
  const float tx = __fsub_rn(__fmul_rn(u, (float)T), 0.5f);
  const float ty = __fsub_rn(__fmul_rn(__fsub_rn(1.f, v), (float)T), 0.5f);
  const float fx0 = floorf(tx), fy0 = floorf(ty);
  const float ax = __fsub_rn(tx, fx0), ay = __fsub_rn(ty, fy0);
  const long long ix = (long long)fx0, iy = (long long)fy0;
  const int x0 = (int)(((ix % T) + T) % T), y0 = (int)(((iy % T) + T) % T);
  const int x1 = (x0 + 1) % T, y1 = (y0 + 1) % T;
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    const float t00 = tex[((int64_t)y0 * T + x0) * 3 + c], t01 = tex[((int64_t)y0 * T + x1) * 3 + c];
    const float t10 = tex[((int64_t)y1 * T + x0) * 3 + c], t11 = tex[((int64_t)y1 * T + x1) * 3 + c];
    const float top = __fadd_rn(t00, __fmul_rn(ax, __fsub_rn(t01, t00)));
    const float bot = __fadd_rn(t10, __fmul_rn(ax, __fsub_rn(t11, t10)));
    rgb[c] = __fdiv_rn(__fadd_rn(top, __fmul_rn(ay, __fsub_rn(bot, top))), 255.f);
  }
}

struct BigTri { Tri t; int face, x0, y0, x1, y1; };

// Point of edge a -> b (a in front of the near plane, b behind) at depth = near, from the homogeneous (X, Y, depth)
// corners.  The front endpoint always comes first, so two faces sharing the edge get the same bits (watertight).
__device__ __forceinline__ void clip_point(const float* X, const float* Y, const float* D, int a, int b, float near,
                                           float& x, float& y) {
  const float t = __fdiv_rn(__fsub_rn(near, D[a]), __fsub_rn(D[b], D[a]));
  x = __fdiv_rn(__fadd_rn(X[a], __fmul_rn(t, __fsub_rn(X[b], X[a]))), near);
  y = __fdiv_rn(__fadd_rn(Y[a], __fmul_rn(t, __fsub_rn(Y[b], Y[a]))), near);
}

// The part of a face with view depth >= near as at most two screen triangles whose d[] holds 1 / depth; both keep
// the face's winding.  Returns their count.
__device__ __forceinline__ int clip_near(const float* X, const float* Y, const float* D, float near, Tri* out) {
  const float rn = __frcp_rn(near);
  int nin = 0, i_in = 0, i_out = 0;
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    if (D[k] >= near) { ++nin; i_in = k; } else { i_out = k; }
  }
  if (nin == 0) return 0;
  if (nin == 3) {
#pragma unroll
    for (int k = 0; k < 3; ++k) {
      out[0].x[k] = __fdiv_rn(X[k], D[k]); out[0].y[k] = __fdiv_rn(Y[k], D[k]); out[0].d[k] = __frcp_rn(D[k]);
    }
    return 1;
  }
  if (nin == 1) {                                   // (i, i -> j at near, i -> k at near)
    const int i = i_in, j = (i + 1) % 3, k = (i + 2) % 3;
    out[0].x[0] = __fdiv_rn(X[i], D[i]); out[0].y[0] = __fdiv_rn(Y[i], D[i]); out[0].d[0] = __frcp_rn(D[i]);
    clip_point(X, Y, D, i, j, near, out[0].x[1], out[0].y[1]);
    clip_point(X, Y, D, i, k, near, out[0].x[2], out[0].y[2]);
    out[0].d[1] = out[0].d[2] = rn;
    return 1;
  }
  // two in front (i, j), k behind: the quad (i, j, j -> k, i -> k) as (i, j, p) and (i, p, q)
  const int k = i_out, i = (k + 1) % 3, j = (k + 2) % 3;
  float px, py, qx, qy;
  clip_point(X, Y, D, j, k, near, px, py);
  clip_point(X, Y, D, i, k, near, qx, qy);
  const float xi = __fdiv_rn(X[i], D[i]), yi = __fdiv_rn(Y[i], D[i]), ri = __frcp_rn(D[i]);
  out[0].x[0] = xi; out[0].y[0] = yi; out[0].d[0] = ri;
  out[0].x[1] = __fdiv_rn(X[j], D[j]); out[0].y[1] = __fdiv_rn(Y[j], D[j]); out[0].d[1] = __frcp_rn(D[j]);
  out[0].x[2] = px; out[0].y[2] = py; out[0].d[2] = rn;
  out[1].x[0] = xi; out[1].y[0] = yi; out[1].d[0] = ri;
  out[1].x[1] = px; out[1].y[1] = py; out[1].d[1] = rn;
  out[1].x[2] = qx; out[1].y[2] = qy; out[1].d[2] = rn;
  return 2;
}

// Perspective-correct barycentrics of pixel centre (px, py) on the plane of a face with homogeneous corners
// (X, Y, depth): w_k is proportional to the 2-D cross product of corners k + 1 and k + 2 taken relative to the pixel's
// ray, which needs no clipping.
__device__ __forceinline__ void persp_bary(const float* X, const float* Y, const float* D, float px, float py,
                                           float* w) {
  float rx[3], ry[3];
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    rx[k] = __fsub_rn(X[k], __fmul_rn(px, D[k]));
    ry[k] = __fsub_rn(Y[k], __fmul_rn(py, D[k]));
  }
  float e[3];
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    const int a = (k + 1) % 3, b = (k + 2) % 3;
    e[k] = __fsub_rn(__fmul_rn(rx[a], ry[b]), __fmul_rn(ry[a], rx[b]));
  }
  const float s = __fadd_rn(__fadd_rn(e[0], e[1]), e[2]);
#pragma unroll
  for (int k = 0; k < 3; ++k) w[k] = s != 0.f ? __fdiv_rn(e[k], s) : 1.f / 3.f;
}

template <bool PERSP>
__global__ void __launch_bounds__(RT_THREADS)
k_render_tiles(Cam cam, const ObjXf* __restrict__ xf, const int64_t* __restrict__ model,
               const int64_t* __restrict__ cls, const float* __restrict__ palette, int flags,
               const int* __restrict__ vert_off, const float* __restrict__ verts, const int* __restrict__ face_off,
               const int* __restrict__ faces, const float* __restrict__ uvs, const float* __restrict__ kd,
               const uint8_t* __restrict__ tex, int T, const int* __restrict__ floor_off,
               const float* __restrict__ floor_tris, const uint8_t* __restrict__ floor_tex,
               const int* __restrict__ floor_tex_idx, int floor_T, int N, int tiles_x,
               uint8_t* __restrict__ image, int64_t* __restrict__ ids) {
  __shared__ unsigned long long s_key[RT * RT];
  __shared__ BigTri s_big[RT_THREADS];
  __shared__ int s_nbig;
  const int b = blockIdx.y;
  const int tx0 = (blockIdx.x % tiles_x) * RT, ty0 = (blockIdx.x / tiles_x) * RT;
  const int tx1 = min(tx0 + RT, cam.W) - 1, ty1 = min(ty0 + RT, cam.H) - 1;
  for (int p = threadIdx.x; p < RT * RT; p += RT_THREADS) s_key[p] = EMPTY_KEY;
  if (threadIdx.x == 0) s_nbig = 0;
  __syncthreads();

  auto plot = [&](const Tri& t, unsigned id, int x, int y) {
    float w[3];
    if (!cover(t, __fadd_rn((float)x, 0.5f), __fadd_rn((float)y, 0.5f), w)) return;
    float d = interp(t.d, w);
    if constexpr (PERSP) d = __fdiv_rn(1.f, d);          // t.d holds 1 / depth, linear in screen space
    if (!(d >= cam.near_p && d <= cam.far_p)) return;   // per-pixel near / far clipping; NaN is never drawn
    const unsigned long long key = ((unsigned long long)__float_as_uint(fmaxf(d, 0.f)) << 32) | id;
    atomicMin(&s_key[(y - ty0) * RT + (x - tx0)], key);
  };

  const int fbeg = floor_off ? floor_off[b] : 0;
  for (int slot = 0; slot <= N; ++slot) {
    const ObjXf& o = xf[(int64_t)b * (N + 1) + slot];
    if (o.x0 > o.x1 || o.x1 < tx0 || o.x0 > tx1 || o.y1 < ty0 || o.y0 > ty1) continue;   // uniform over the CTA
    const int64_t m = slot < N ? model[(int64_t)b * N + slot] : -1;
    const int nf = o.faces;
    for (int f0 = 0; f0 < nf; f0 += RT_THREADS) {
      const int f = f0 + threadIdx.x;
      if (f < nf) {
        const unsigned id = ((unsigned)slot << FACE_BITS) | (unsigned)f;
        auto emit = [&](const Tri& t) {
          float lx = INFINITY, hx = -INFINITY, ly = INFINITY, hy = -INFINITY;
#pragma unroll
          for (int k = 0; k < 3; ++k) {
            lx = fminf(lx, t.x[k]); hx = fmaxf(hx, t.x[k]); ly = fminf(ly, t.y[k]); hy = fmaxf(hy, t.y[k]);
          }
          // pixels whose centres can lie in the triangle, clipped to the tile
          const int x0 = (int)fmaxf((float)tx0, ceilf(__fsub_rn(lx, 0.5f)));
          const int x1 = (int)fminf((float)tx1, floorf(__fsub_rn(hx, 0.5f)));
          const int y0 = (int)fmaxf((float)ty0, ceilf(__fsub_rn(ly, 0.5f)));
          const int y1 = (int)fminf((float)ty1, floorf(__fsub_rn(hy, 0.5f)));
          if (x0 <= x1 && y0 <= y1) {
            if ((x1 - x0 + 1) * (y1 - y0 + 1) <= SMALL_TRI_PIXELS) {
              for (int y = y0; y <= y1; ++y)
                for (int x = x0; x <= x1; ++x) plot(t, id, x, y);
            } else {
              const int q = atomicAdd(&s_nbig, 1);
              if (q < RT_THREADS) {
                s_big[q] = BigTri{t, f, x0, y0, x1, y1};
              } else {                              // a clipped face's second half found the list full
                for (int y = y0; y <= y1; ++y)
                  for (int x = x0; x <= x1; ++x) plot(t, id, x, y);
              }
            }
          }
        };
        float X[3], Y[3], D[3];
#pragma unroll
        for (int k = 0; k < 3; ++k) {
          float vx, vy, vz;
          corner(slot, N, f, k, faces, face_off, vert_off, verts, m, floor_tris, fbeg, vx, vy, vz);
          X[k] = apply(o.m[0], vx, vy, vz);
          Y[k] = apply(o.m[1], vx, vy, vz);
          D[k] = apply(o.m[2], vx, vy, vz);
        }
        if constexpr (PERSP) {
          Tri sub[2];
          const int ns = clip_near(X, Y, D, cam.near_p, sub);
          if (ns > 0) emit(sub[0]);
          if (ns > 1) emit(sub[1]);
        } else {
          Tri t;
#pragma unroll
          for (int k = 0; k < 3; ++k) { t.x[k] = X[k]; t.y[k] = Y[k]; t.d[k] = D[k]; }
          emit(t);
        }
      }
      __syncthreads();
      const int nbig = min(s_nbig, RT_THREADS);
      for (int q = 0; q < nbig; ++q) {              // large triangles: the CTA splits their pixels
        const BigTri& bt = s_big[q];
        const int w = bt.x1 - bt.x0 + 1, n = w * (bt.y1 - bt.y0 + 1);
        const unsigned id = ((unsigned)slot << FACE_BITS) | (unsigned)bt.face;
        for (int p = threadIdx.x; p < n; p += RT_THREADS) plot(bt.t, id, bt.x0 + p % w, bt.y0 + p / w);
      }
      __syncthreads();
      if (threadIdx.x == 0) s_nbig = 0;
      __syncthreads();
    }
  }

  // resolve: recompute the winner's barycentrics and shade
  const bool white_bg = flags & RF_WHITE_BACKGROUND;
  for (int p = threadIdx.x; p < RT * RT; p += RT_THREADS) {
    const int x = tx0 + p % RT, y = ty0 + p / RT;
    if (x > tx1 || y > ty1) continue;
    const unsigned long long key = s_key[p];
    const int64_t pix = ((int64_t)b * cam.H + y) * cam.W + x;
    uint8_t rgb8[3];
    if (key == EMPTY_KEY) {
      rgb8[0] = rgb8[1] = rgb8[2] = white_bg ? 255 : 0;
      if (ids) ids[pix] = -1;
    } else {
      const unsigned id = (unsigned)key;
      const int slot = id >> FACE_BITS, f = id & ((1u << FACE_BITS) - 1);
      const ObjXf& o = xf[(int64_t)b * (N + 1) + slot];
      const int64_t m = slot < N ? model[(int64_t)b * N + slot] : -1;
      Tri t;
      float wv[3][3];
      for (int k = 0; k < 3; ++k) {
        float vx, vy, vz;
        corner(slot, N, f, k, faces, face_off, vert_off, verts, m, floor_tris, fbeg, vx, vy, vz);
        t.x[k] = apply(o.m[0], vx, vy, vz);
        t.y[k] = apply(o.m[1], vx, vy, vz);
        t.d[k] = apply(o.m[2], vx, vy, vz);
        for (int r = 0; r < 3; ++r) wv[r][k] = apply(o.m[3 + r], vx, vy, vz);
      }
      float w[3];
      if constexpr (PERSP)
        persp_bary(t.x, t.y, t.d, __fadd_rn((float)x, 0.5f), __fadd_rn((float)y, 0.5f), w);
      else
        cover(t, __fadd_rn((float)x, 0.5f), __fadd_rn((float)y, 0.5f), w);
      float base[3] = {1.f, 1.f, 1.f};
      if (slot < N) {
        if (flags & RF_NO_TEXTURE) {
          const float* c = palette + cls[(int64_t)b * N + slot] * 3;
          base[0] = c[0]; base[1] = c[1]; base[2] = c[2];
        } else {
          const float* uv = uvs + (int64_t)(face_off[m] + f) * 6;
          const float* k = kd + m * 3;
          if (uv[0] == uv[0]) {
            const float u3[3] = {uv[0], uv[2], uv[4]}, v3[3] = {uv[1], uv[3], uv[5]};
            sample_rgb(tex + (int64_t)m * T * T * 3, T, interp(u3, w), interp(v3, w), base);
          }
          for (int c = 0; c < 3; ++c) base[c] = __fmul_rn(base[c], k[c]);
        }
      } else if (floor_tex_idx && floor_tex_idx[b] >= 0) {
        const float u = __fdiv_rn(__fsub_rn(interp(wv[0], w), o.umin), FLOOR_UV_PERIOD);
        const float v = __fdiv_rn(__fsub_rn(interp(wv[2], w), o.vmin), FLOOR_UV_PERIOD);
        sample_rgb(floor_tex + (int64_t)floor_tex_idx[b] * floor_T * floor_T * 3, floor_T, u, v, base);
      }
      // point light at the camera: ambient + diffuse * |n . l| on the placed triangle's geometric normal
      float e1[3], e2[3], pw[3], l[3];
      for (int r = 0; r < 3; ++r) {
        e1[r] = __fsub_rn(wv[r][1], wv[r][0]);
        e2[r] = __fsub_rn(wv[r][2], wv[r][0]);
        pw[r] = interp(wv[r], w);
        l[r] = __fsub_rn(cam.eye[r], pw[r]);
      }
      const float n[3] = {__fsub_rn(__fmul_rn(e1[1], e2[2]), __fmul_rn(e1[2], e2[1])),
                          __fsub_rn(__fmul_rn(e1[2], e2[0]), __fmul_rn(e1[0], e2[2])),
                          __fsub_rn(__fmul_rn(e1[0], e2[1]), __fmul_rn(e1[1], e2[0]))};
      const float nn = __fadd_rn(__fadd_rn(__fmul_rn(n[0], n[0]), __fmul_rn(n[1], n[1])), __fmul_rn(n[2], n[2]));
      const float ll = __fadd_rn(__fadd_rn(__fmul_rn(l[0], l[0]), __fmul_rn(l[1], l[1])), __fmul_rn(l[2], l[2]));
      const float dot = __fadd_rn(__fadd_rn(__fmul_rn(n[0], l[0]), __fmul_rn(n[1], l[1])), __fmul_rn(n[2], l[2]));
      const float den = __fsqrt_rn(__fmul_rn(nn, ll));
      const float cosang = den > 0.f ? fminf(__fdiv_rn(fabsf(dot), den), 1.f) : 0.f;
      const float shade = __fadd_rn(AMBIENT, __fmul_rn(DIFFUSE, cosang));
      for (int c = 0; c < 3; ++c)
        rgb8[c] = (uint8_t)__float2int_rn(__fmul_rn(__saturatef(__fmul_rn(base[c], shade)), 255.f));
      if (ids) ids[pix] = ((int64_t)slot << 32) | f;
    }
    image[pix * 3 + 0] = rgb8[0];
    image[pix * 3 + 1] = rgb8[1];
    image[pix * 3 + 2] = rgb8[2];
  }
}

void catalog_free(Catalog* c) {
  void* ptrs[] = {c->vert_off, c->verts, c->face_off, c->faces, c->uvs, c->half, c->aabb, c->kd, c->tex};
  for (void* p : ptrs)
    if (p) cudaFree(p);
  delete c;
}

template <class T>
int upload(T** dst, const T* src, int64_t n, const char* what) {
  if (n == 0) return 0;
  if (!src) return fail(DS_ERR_INVALID, "ds_mesh_catalog_create: NULL %s", what);
  CK(cudaMalloc(dst, sizeof(T) * n));
  CK(cudaMemcpy(*dst, src, sizeof(T) * n, cudaMemcpyHostToDevice));
  return 0;
}

}  // namespace
}  // namespace ds

extern "C" int ds_mesh_catalog_create(int32_t num_models, const int32_t* vertex_offsets, const float* vertices,
                                      const int32_t* face_offsets, const int32_t* faces, const float* uvs,
                                      const double* raw_half, const double* raw_aabb, const float* kd,
                                      const uint8_t* textures, int32_t texture_size, int32_t device, void** handle) {
  if (!handle) return fail(DS_ERR_INVALID, "ds_mesh_catalog_create: NULL handle pointer");
  *handle = nullptr;
  if (num_models < 0) return fail(DS_ERR_INVALID, "ds_mesh_catalog_create: num_models %d < 0", num_models);
  if (num_models > 0 && (!vertex_offsets || !face_offsets || !raw_half || !raw_aabb || !kd || !textures))
    return fail(DS_ERR_INVALID, "ds_mesh_catalog_create: NULL offsets, bounds, Kd or texture array");
  if (texture_size < 1 || texture_size > 4096)
    return fail(DS_ERR_INVALID, "ds_mesh_catalog_create: texture size %d outside [1, 4096]", texture_size);
  if (num_models > 0 && (vertex_offsets[0] != 0 || face_offsets[0] != 0))
    return fail(DS_ERR_INVALID, "ds_mesh_catalog_create: offsets must start at 0");
  for (int m = 0; m < num_models; ++m) {
    const int nv = vertex_offsets[m + 1] - vertex_offsets[m], nf = face_offsets[m + 1] - face_offsets[m];
    if (nv < 0 || nf < 0)
      return fail(DS_ERR_INVALID, "ds_mesh_catalog_create: offsets decrease at model %d", m);
    if (nf >= (1 << FACE_BITS))
      return fail(DS_ERR_INVALID, "ds_mesh_catalog_create: model %d has %d faces, at most %d", m, nf,
                  (1 << FACE_BITS) - 1);
    for (int64_t i = (int64_t)face_offsets[m] * 3; i < (int64_t)face_offsets[m + 1] * 3; ++i)
      if (faces[i] < 0 || faces[i] >= nv)
        return fail(DS_ERR_INVALID, "ds_mesh_catalog_create: model %d has a vertex index %d outside [0, %d)", m,
                    faces[i], nv);
    for (int k = 0; k < 3; ++k)
      if (!(raw_half[m * 3 + k] > 0.0))
        return fail(DS_ERR_INVALID, "ds_mesh_catalog_create: model %d has a half size <= 0", m);
  }
  if (const int rc = require_device()) return rc;
  CK(cudaSetDevice(device));
  Catalog* c = new Catalog();
  c->device = device;
  c->M = num_models;
  c->T = texture_size;
  c->V = num_models ? vertex_offsets[num_models] : 0;
  c->F = num_models ? face_offsets[num_models] : 0;
  const int64_t M = num_models, T = texture_size;
  int rc = 0;
  if (!rc) rc = upload(&c->vert_off, vertex_offsets, M ? M + 1 : 0, "vertex offsets");
  if (!rc) rc = upload(&c->face_off, face_offsets, M ? M + 1 : 0, "face offsets");
  if (!rc) rc = upload(&c->verts, vertices, c->V * 3, "vertices");
  if (!rc) rc = upload(&c->faces, faces, c->F * 3, "faces");
  if (!rc) rc = upload(&c->uvs, uvs, c->F * 6, "uvs");
  if (!rc) rc = upload(&c->half, raw_half, M * 3, "raw_half");
  if (!rc) rc = upload(&c->aabb, raw_aabb, M * 6, "raw_aabb");
  if (!rc) rc = upload(&c->kd, kd, M * 3, "Kd");
  if (!rc) rc = upload(&c->tex, textures, M * T * T * 3, "textures");
  if (rc) {
    catalog_free(c);
    return rc;
  }
  std::lock_guard<std::mutex> lk(g_cat_mu);
  g_cats.insert(c);
  *handle = c;
  return 0;
}

extern "C" int ds_mesh_catalog_destroy(void* handle) {
  std::lock_guard<std::mutex> lk(g_cat_mu);
  if (!g_cats.count(handle))
    return fail(DS_ERR_INVALID, "ds_mesh_catalog_destroy: not a live mesh catalogue handle");
  g_cats.erase(handle);
  catalog_free((Catalog*)handle);
  return 0;
}

extern "C" int ds_render_scenes(void* handle, const ds_render_camera* camera, const ds_render_args* a, void* stream) {
  {
    std::lock_guard<std::mutex> lk(g_cat_mu);
    if (!g_cats.count(handle))
      return fail(DS_ERR_INVALID, "ds_render_scenes: not a live mesh catalogue handle");
  }
  const Catalog* c = (const Catalog*)handle;
  if (!camera || !a) return fail(DS_ERR_INVALID, "ds_render_scenes: NULL camera or arguments");
  if (a->batch < 0 || a->num_objects < 0 || a->num_objects > MAX_SLOTS)
    return fail(DS_ERR_INVALID, "ds_render_scenes: batch %d < 0 or %d objects per scene outside [0, %d]", a->batch,
                a->num_objects, MAX_SLOTS);
  if (camera->width < 1 || camera->width > 4096 || camera->height < 1 || camera->height > 4096)
    return fail(DS_ERR_INVALID, "ds_render_scenes: image size %d x %d outside [1, 4096]", camera->width,
                camera->height);
  const int proj = camera->projection;
  if (proj != DS_RENDER_ORTHOGRAPHIC && proj != DS_RENDER_PERSPECTIVE)
    return fail(DS_ERR_INVALID, "ds_render_scenes: unknown projection %d", proj);
  if (!(camera->near_plane >= 0.f) || !(camera->far_plane > camera->near_plane) || camera->left == camera->right ||
      camera->bottom == camera->top)
    return fail(DS_ERR_INVALID, "ds_render_scenes: need 0 <= near < far and a non-empty view volume");
  if (proj == DS_RENDER_PERSPECTIVE && !(camera->near_plane > 0.f))
    return fail(DS_ERR_INVALID, "ds_render_scenes: a perspective view volume needs near > 0");
  if (!a->image_dev) return fail(DS_ERR_INVALID, "ds_render_scenes: NULL image pointer");
  if (a->num_objects > 0 && a->batch > 0 &&
      (!a->translation_dev || !a->size_dev || !a->angle_dev || !a->model_index_dev))
    return fail(DS_ERR_INVALID, "ds_render_scenes: NULL translation, size, angle or model index pointer");
  const bool no_tex = a->flags & RF_NO_TEXTURE;
  if (no_tex && a->num_objects > 0 && a->batch > 0 && (!a->class_index_dev || !a->palette_dev || a->num_colors < 1))
    return fail(DS_ERR_INVALID, "ds_render_scenes: untextured rendering needs class indices and a palette");
  if (a->floor_offsets_dev && a->num_floor_tris > 0 && !a->floor_tris_dev)
    return fail(DS_ERR_INVALID, "ds_render_scenes: NULL floor triangles");
  if (a->num_floor_tris < 0) return fail(DS_ERR_INVALID, "ds_render_scenes: negative floor triangle count");
  if (a->floor_texture_index_dev &&
      (!a->floor_textures_dev || a->num_floor_textures < 1 || a->floor_texture_size < 1 ||
       a->floor_texture_size > 4096))
    return fail(DS_ERR_INVALID, "ds_render_scenes: floor texture indices need floor textures of size [1, 4096]");
  if (const int rc = require_device()) return rc;
  int cur = -1;
  CK(cudaGetDevice(&cur));
  if (cur != c->device)
    return fail(DS_ERR_INVALID, "ds_render_scenes: the catalogue lives on device %d, the current device is %d",
                c->device, cur);
  if (a->batch == 0) return 0;

  // camera: pyrr's create_look_at and orthogonal_projection (or create_perspective_projection_from_bounds), then the
  // viewport (DESIGN.md, rendering)
  Cam cam;
  double e[3], f[3], u[3], sd[3];
  for (int k = 0; k < 3; ++k) { e[k] = camera->eye[k]; f[k] = (double)camera->target[k] - e[k]; u[k] = camera->up[k]; }
  auto norm = [](double* v) {
    const double n = sqrt(v[0] * v[0] + v[1] * v[1] + v[2] * v[2]);
    if (n > 0) for (int k = 0; k < 3; ++k) v[k] /= n;
    return n;
  };
  if (norm(f) == 0.0) return fail(DS_ERR_INVALID, "ds_render_scenes: eye and target coincide");
  sd[0] = f[1] * u[2] - f[2] * u[1]; sd[1] = f[2] * u[0] - f[0] * u[2]; sd[2] = f[0] * u[1] - f[1] * u[0];
  if (norm(sd) == 0.0) return fail(DS_ERR_INVALID, "ds_render_scenes: up is parallel to the view direction");
  double up2[3] = {sd[1] * f[2] - sd[2] * f[1], sd[2] * f[0] - sd[0] * f[2], sd[0] * f[1] - sd[1] * f[0]};
  norm(up2);
  const double L = camera->left, R = camera->right, Bo = camera->bottom, To = camera->top;
  const double W = camera->width, H = camera->height;
  // pixel x = W / 2 (x_ndc + 1), pixel y (array row) = H / 2 (y_ndc + 1), depth = distance along the view direction
  const double sx = W / (R - L), ox = -W / 2 * (R + L) / (R - L) + W / 2;
  const double sy = H / (To - Bo), oy = -H / 2 * (To + Bo) / (To - Bo) + H / 2;
  for (int k = 0; k < 3; ++k) {
    cam.m[0][k] = sx * sd[k];
    cam.m[1][k] = sy * up2[k];
    cam.m[2][k] = f[k];
  }
  cam.m[0][3] = ox - sx * (sd[0] * e[0] + sd[1] * e[1] + sd[2] * e[2]);
  cam.m[1][3] = oy - sy * (up2[0] * e[0] + up2[1] * e[1] + up2[2] * e[2]);
  cam.m[2][3] = -(f[0] * e[0] + f[1] * e[1] + f[2] * e[2]);
  if (proj == DS_RENDER_PERSPECTIVE) {
    // clip x = 2 n / (R - L) x_view - (R + L) / (R - L) depth with w = depth, so pixel x * depth = W / 2 (clip x +
    // depth) is affine in the vertex; likewise pixel y * depth
    const double n = camera->near_plane;
    const double px = W * n / (R - L), pd = W / 2 * (1.0 - (R + L) / (R - L));
    const double qy = H * n / (To - Bo), qd = H / 2 * (1.0 - (To + Bo) / (To - Bo));
    for (int c = 0; c < 4; ++c) {
      const double vx = c < 3 ? sd[c] : -(sd[0] * e[0] + sd[1] * e[1] + sd[2] * e[2]);
      const double vy = c < 3 ? up2[c] : -(up2[0] * e[0] + up2[1] * e[1] + up2[2] * e[2]);
      cam.m[0][c] = px * vx + pd * cam.m[2][c];
      cam.m[1][c] = qy * vy + qd * cam.m[2][c];
    }
  }
  cam.near_p = camera->near_plane;
  cam.far_p = camera->far_plane;
  for (int k = 0; k < 3; ++k) cam.eye[k] = camera->eye[k];
  cam.W = camera->width;
  cam.H = camera->height;

  cudaStream_t s = (cudaStream_t)stream;
  const int B = a->batch, N = a->num_objects;
  ObjXf* xf = nullptr;
  int* err_dev = nullptr;
  CK(cudaMallocAsync(&xf, sizeof(ObjXf) * (int64_t)B * (N + 1), s));
  CK(cudaMallocAsync(&err_dev, sizeof(int), s));
  CK(cudaMemsetAsync(err_dev, 0, sizeof(int), s));
  const bool persp = proj == DS_RENDER_PERSPECTIVE;
  (persp ? k_render_prep<true> : k_render_prep<false>)<<<ceil_div((int64_t)B * (N + 1), 128), 128, 0, s>>>(
      cam, a->translation_dev, a->size_dev, a->angle_dev, a->model_index_dev, a->class_index_dev, a->num_colors,
      no_tex, c->vert_off, c->verts, c->face_off, c->half, c->aabb, c->M, a->floor_offsets_dev, a->floor_tris_dev,
      a->num_floor_tris, a->floor_texture_index_dev, a->num_floor_textures, B, N, xf, err_dev);
  cudaError_t ce = cudaGetLastError();
  const int tiles_x = ceil_div(cam.W, RT), tiles_y = ceil_div(cam.H, RT);
  if (ce == cudaSuccess) {
    (persp ? k_render_tiles<true> : k_render_tiles<false>)<<<dim3(tiles_x * tiles_y, B), RT_THREADS, 0, s>>>(
        cam, xf, a->model_index_dev, a->class_index_dev, a->palette_dev, a->flags, c->vert_off, c->verts, c->face_off,
        c->faces, c->uvs, c->kd, c->tex, c->T, a->floor_offsets_dev, a->floor_tris_dev, a->floor_textures_dev,
        a->floor_texture_index_dev, a->floor_texture_size, N, tiles_x, (uint8_t*)a->image_dev, (int64_t*)a->id_dev);
    ce = cudaGetLastError();
  }
  int err = 0;
  if (ce == cudaSuccess) ce = cudaMemcpyAsync(&err, err_dev, sizeof(int), cudaMemcpyDeviceToHost, s);
  cudaFreeAsync(xf, s);
  cudaFreeAsync(err_dev, s);
  if (ce == cudaSuccess) ce = cudaStreamSynchronize(s);
  if (ce != cudaSuccess) return fail(DS_ERR_CUDA, "ds_render_scenes: %s", cudaGetErrorString(ce));
  if (err & RE_MODEL) return fail(DS_ERR_INVALID, "ds_render_scenes: model index outside [-1, %d)", c->M);
  if (err & RE_CLASS)
    return fail(DS_ERR_INVALID, "ds_render_scenes: class index outside [0, %d) of the palette", a->num_colors);
  if (err & RE_FLOOR_OFF)
    return fail(DS_ERR_INVALID, "ds_render_scenes: floor offsets must start at >= 0, not decrease and end at <= %d",
                a->num_floor_tris);
  if (err & RE_FLOOR_COUNT)
    return fail(DS_ERR_INVALID, "ds_render_scenes: a floor has %d or more triangles", 1 << FACE_BITS);
  if (err & RE_FLOOR_TEX)
    return fail(DS_ERR_INVALID, "ds_render_scenes: floor texture index outside [-1, %d)", a->num_floor_textures);
  return 0;
}
