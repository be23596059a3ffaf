// VGG16 feature extractor of improved precision and recall (reference scripts/improved_precision_recall.py:159-163,
// torchvision `vgg16`): classifier[:4](features(x).view(-1, 7 * 7 * 512)), the fc2 output before its ReLU.
//
// Activations are NHWC rows (image, y, x) x channels.  The input pack kernel applies F.interpolate's nearest pixel
// choice and writes [B, 224, 224, 3]; the first convolution (cin = 3) runs over a 64-column im2col of it
// (launch_re_im2col, 27 taps zero-padded to one 64-wide K block).
//
// bf16 mode: every convolution is k_vgg_conv, an implicit GEMM on wgmma.  A CTA owns an 8 x 16 patch of output pixels
// (128 GEMM rows) and 64 or 128 output channels.  For each (ky, kx, 64-channel block) its A operand is ONE TMA load of
// the 4-D box {64 ch, 16 x, 8 y, 1 image} of the NHWC input at (x0 + kx - 1, y0 + ky - 1): TMA's out-of-bounds zero
// fill is the convolution's padding, so no im2col buffer exists.  The box lands in shared memory exactly like a
// 128 x 64 K-major GEMM tile (128-byte swizzle), so the wgmma descriptors are those of k_gemm_wg.  The weights are
// [cout, (ky, kx, ci)] bf16, K-major.  The epilogue adds the bias, applies the ReLU, rounds to bf16 and, after conv
// layers 2, 4, 7, 10 and 13, takes the 2 x 2 max-pool inside the tile (tiles start at even pixels; max commutes with
// ReLU and with rounding) before the NHWC store.  fc1 (ReLU epilogue) and fc2 run on k_gemm_wg; fc2 adds its products
// to an fp32 output pre-filled with the bias (one addition per element, so the features are fp32 and deterministic).
//
// fp32 mode: im2col (launch_re_im2col) + the exact SIMT GEMM with the bias and ReLU, a separate 2 x 2 max-pool, and the
// SIMT GEMM for fc1 / fc2.  The im2col buffer is bounded by the pass size (ds_vgg_config.capacity).
//
// fc1's columns are permuted when packed: the reference flattens NCHW (c, y, x), the activations here are (y, x, c).
#include "engine_internal.h"
#include "tc_common.cuh"

namespace ds {
int* tc_error_flag_dev();      // gemm_tc.cu
namespace {

constexpr int VG_IMG = 224;
constexpr int VG_TX = 16, VG_TY = 8;                 // output patch of one CTA (128 pixels)
constexpr int VG_STAGES = 3;
constexpr int VG_THREADS = 256;
constexpr int VG_NCONV = 13;
const int kCin[VG_NCONV] = {3, 64, 64, 128, 128, 256, 256, 256, 512, 512, 512, 512, 512};
const int kCout[VG_NCONV] = {64, 64, 128, 128, 256, 256, 256, 512, 512, 512, 512, 512, 512};
const bool kPool[VG_NCONV] = {false, true, false, true, false, false, true, false, false, true, false, false, true};
const int kFeatIdx[VG_NCONV] = {0, 2, 5, 7, 10, 12, 14, 17, 19, 21, 24, 26, 28};
constexpr int VG_FC1_K = 7 * 7 * 512;

template <int BN> struct VgSmem {
  static constexpr int STAGE = A_BYTES + BN * BK * 2;
  static constexpr int BAR_OFF = VG_STAGES * STAGE;
  static constexpr int BIAS_OFF = BAR_OFF + 64;
  static constexpr int BYTES = 1024 + BIAS_OFF + BN * 4;
  static constexpr int STG_PITCH = BN + 8;           // bf16 staging tile [128][BN + 8] in the drained ring
  static_assert(BM * STG_PITCH * 2 <= VG_STAGES * STAGE, "staging tile fits in the ring");
};

// D[64 x 64] (+)= A[64 x 16] * B[64 x 16]^T, operands as wgmma_m64n128k16
__device__ __forceinline__ void wgmma_m64n64k16(float (&d)[32], uint64_t a_desc, uint64_t b_desc, uint32_t accumulate) {
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "setp.ne.b32 p, %34, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
      "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, "
      "%32, %33, p, 1, 1, 0, 0;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
        "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
        "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
        "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
      : "l"(a_desc), "l"(b_desc), "r"(accumulate)
      : "memory");
}
template <int BN> __device__ __forceinline__ void wgmma_tile(float (&d)[BN / 2], uint64_t a, uint64_t b, uint32_t acc) {
  if constexpr (BN == 128) wgmma_m64n128k16(d, a, b, acc);
  else wgmma_m64n64k16(d, a, b, acc);
}

__device__ __forceinline__ void tma_load_4d(uint32_t dst, const CUtensorMap* map, int c0, int c1, int c2, int c3,
                                            uint32_t bar) {
  asm volatile(
      "cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3, %4, %5}], [%6];"
      ::"r"(dst), "l"(map), "r"(c0), "r"(c1), "r"(c2), "r"(c3), "r"(bar)
      : "memory");
}

template <int BN, bool POOL>
__global__ void __launch_bounds__(VG_THREADS, 2)
k_vgg_conv(const __grid_constant__ CUtensorMap tm_in, const __grid_constant__ CUtensorMap tm_w, VgConvEpi e,
           int* err_flag) {
  using S = VgSmem<BN>;
  extern __shared__ uint8_t smem_raw[];
  const uint32_t raw = smem_u32(smem_raw);
  const uint32_t base = (raw + 1023u) & ~1023u;
  uint8_t* const base_ptr = smem_raw + (base - raw);
  const uint32_t bar_base = base + S::BAR_OFF;
  auto full_bar = [&](int s) { return bar_base + 8u * s; };
  auto empty_bar = [&](int s) { return bar_base + 8u * (VG_STAGES + s); };
  float* const sbias = reinterpret_cast<float*>(base_ptr + S::BIAS_OFF);

  const int tid = threadIdx.x, wg = tid >> 7, wq = (tid >> 5) & 3, lane = tid & 31;
  const int n_tiles = (e.cout + BN - 1) / BN;
  int t = blockIdx.x;
  const int nt = t % n_tiles; t /= n_tiles;
  const int tx = t % e.tiles_x; t /= e.tiles_x;
  const int ty = t % e.tiles_y;
  const int img = t / e.tiles_y;
  const int x0 = tx * VG_TX, y0 = ty * VG_TY, n0 = nt * BN;
  const int cblocks = e.C / BK;
  const int nk = e.taps * cblocks;

  if (tid == 0) {
    tma_prefetch_desc(&tm_in);
    tma_prefetch_desc(&tm_w);
    for (int s = 0; s < VG_STAGES; ++s) {
      mbar_init(full_bar(s), 1);
      mbar_init(empty_bar(s), VG_THREADS);
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
  }
  for (int c = tid; c < BN; c += VG_THREADS) sbias[c] = n0 + c < e.cout ? __ldg(e.bias + n0 + c) : 0.f;
  __syncthreads();

  auto issue = [&](int i) {
    const int s = i % VG_STAGES, tap = i / cblocks, cb = i % cblocks;
    const int dy = tap / e.kw - e.ph, dx = tap % e.kw - e.pw;
    const uint32_t sa = base + uint32_t(s * S::STAGE);
    mbar_expect_tx(full_bar(s), S::STAGE);
    tma_load_4d(sa, &tm_in, cb * BK, x0 + dx, y0 + dy, img, full_bar(s));
    tma_load_2d(sa + A_BYTES, &tm_w, i * BK, n0, full_bar(s));
  };
  if (tid == 0)
    for (int i = 0; i < VG_STAGES && i < nk; ++i) issue(i);

  float acc[BN / 2];
#pragma unroll
  for (int j = 0; j < BN / 2; ++j) acc[j] = 0.f;
  for (int i = 0; i < nk; ++i) {
    const int s = i % VG_STAGES;
    const uint32_t ph = uint32_t(i / VG_STAGES) & 1u;
    mbar_wait(full_bar(s), ph, err_flag, 3);
    const uint32_t sa = base + uint32_t(s * S::STAGE);
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < BK / 16; ++k)
      wgmma_tile<BN>(acc, wgmma_desc_sw128(sa + uint32_t(wg * 64 * 128 + k * 32)),
                     wgmma_desc_sw128(sa + uint32_t(A_BYTES + k * 32)), uint32_t(i | k));
    wgmma_commit();
    wgmma_wait0();
    mbar_arrive(empty_bar(s));
    if (tid == 0 && i + VG_STAGES < nk) {
      mbar_wait(empty_bar(s), ph, err_flag, 4);
      issue(i + VG_STAGES);
    }
    __syncwarp();
  }
  __syncthreads();      // the other warpgroup's MMAs may still read the ring the tile is staged in

  // accumulator of wgmma m64nBN: rows r0, r0 + 8 of the warpgroup's 64, columns 8 j + cq + {0, 1} in acc[4 j + 2 h + e]
  bf16* const stg = reinterpret_cast<bf16*>(base_ptr);
  const int r0 = wg * 64 + wq * 16 + (lane >> 2), cq = 2 * (lane & 3);
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    bf16* sp = stg + (r0 + 8 * h) * S::STG_PITCH + cq;
#pragma unroll
    for (int j = 0; j < BN / 8; ++j) {
      float v0 = acc[4 * j + 2 * h] + sbias[8 * j + cq], v1 = acc[4 * j + 2 * h + 1] + sbias[8 * j + cq + 1];
      v0 = v0 < 0.f ? 0.f : v0;
      v1 = v1 < 0.f ? 0.f : v1;
      *reinterpret_cast<__nv_bfloat162*>(sp + 8 * j) = __floats2bfloat162_rn(v0, v1);
    }
  }
  __syncthreads();
  // tile row r = (y - y0) * 16 + (x - x0), the TMA box order; 16-byte chunks of 8 channels
  constexpr int CH = BN / 8;
  if constexpr (POOL) {
    const int Ho = e.H / 2, Wo = e.W / 2;
    for (int idx = tid; idx < (VG_TY / 2) * (VG_TX / 2) * CH; idx += VG_THREADS) {
      const int c = (idx % CH) * 8, p = idx / CH, py = p / (VG_TX / 2), px = p % (VG_TX / 2);
      const int oy = y0 / 2 + py, ox = x0 / 2 + px;
      if (oy >= Ho || ox >= Wo) continue;
      const bf16* q = stg + ((2 * py) * VG_TX + 2 * px) * S::STG_PITCH + c;
      __align__(16) __nv_bfloat162 m[4];
#pragma unroll
      for (int u = 0; u < 4; ++u) m[u] = reinterpret_cast<const __nv_bfloat162*>(q)[u];
#pragma unroll
      for (int w = 1; w < 4; ++w) {
        const bf16* qq = q + ((w >> 1) * VG_TX + (w & 1)) * S::STG_PITCH;
#pragma unroll
        for (int u = 0; u < 4; ++u) m[u] = __hmax2(m[u], reinterpret_cast<const __nv_bfloat162*>(qq)[u]);
      }
      *reinterpret_cast<uint4*>(e.out + (((int64_t)img * Ho + oy) * Wo + ox) * e.cout + n0 + c) =
          *reinterpret_cast<const uint4*>(m);
    }
  } else {
    for (int idx = tid; idx < BM * CH; idx += VG_THREADS) {
      const int c = (idx % CH) * 8, r = idx / CH, y = y0 + r / VG_TX, x = x0 + r % VG_TX;
      if (y >= e.Ho || x >= e.Wo || n0 + c >= e.cout) continue;
      *reinterpret_cast<uint4*>(e.out + (((int64_t)img * e.Ho + y) * e.Wo + x) * e.ldo + e.co_off + n0 + c) =
          *reinterpret_cast<const uint4*>(stg + r * S::STG_PITCH + c);
    }
  }
}

// images [B, 3, H, W] fp32 -> x [B, 224, 224, 3]; F.interpolate(size=(224, 224), mode='nearest') pixel choice
template <typename T>
__global__ void k_vgg_pack(const float* __restrict__ img, int H, int W, T* __restrict__ x, int64_t n) {
  const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int c = int(i % 3);
  const int64_t r = i / 3;
  const int ox = int(r % VG_IMG), oy = int((r / VG_IMG) % VG_IMG);
  const int64_t b = r / (VG_IMG * VG_IMG);
  const float sy = float(H) / float(VG_IMG), sx = float(W) / float(VG_IMG);
  const int iy = H == VG_IMG ? oy : min(int(floorf(__fmul_rn(float(oy), sy))), H - 1);
  const int ix = W == VG_IMG ? ox : min(int(floorf(__fmul_rn(float(ox), sx))), W - 1);
  stf(x + i, img[((b * 3 + c) * H + iy) * W + ix]);
}

// conv weight [cout, cin, 3, 3] -> wp[co][(ky * 3 + kx) * cin + ci], zero up to Kp
template <typename T>
__global__ void k_vgg_pack_conv(const float* __restrict__ w, int cin, int Kp, T* __restrict__ wp) {
  const int co = blockIdx.x;
  for (int j = threadIdx.x; j < Kp; j += blockDim.x) {
    float v = 0.f;
    if (j < 9 * cin) {
      const int ci = j % cin, kk = j / cin;
      v = w[((int64_t)co * cin + ci) * 9 + kk];
    }
    stf(wp + (int64_t)co * Kp + j, v);
  }
}
// fc weight [N, K]: permute == 1 maps the reference's (c, y, x) flatten of the 7 x 7 x 512 map to (y, x, c)
template <typename T>
__global__ void k_vgg_pack_fc(const float* __restrict__ w, int K, int permute, T* __restrict__ wp) {
  const int n = blockIdx.x;
  for (int j = threadIdx.x; j < K; j += blockDim.x) {
    int src = j;
    if (permute) {
      const int c = j % 512, p = j / 512;
      src = c * 49 + p;
    }
    stf(wp + (int64_t)n * K + j, w[(int64_t)n * K + src]);
  }
}

// 2 x 2 / stride 2 max-pool of NHWC rows (fp32 mode)
template <typename T>
__global__ void k_vgg_pool(const T* __restrict__ in, T* __restrict__ out, int C, int H, int W, int64_t n) {
  const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int Ho = H / 2, Wo = W / 2, c = int(i % C);
  const int64_t r = i / C;
  const int ox = int(r % Wo), oy = int((r / Wo) % Ho);
  const int64_t b = r / ((int64_t)Wo * Ho);
  const T* p = in + ((b * H + 2 * oy) * W + 2 * ox) * C + c;
  const float v = fmaxf(fmaxf(ldf(p), ldf(p + C)), fmaxf(ldf(p + (int64_t)W * C), ldf(p + (int64_t)W * C + C)));
  stf(out + i, v);
}

__global__ void k_vgg_fill_bias(const float* __restrict__ bias, float* __restrict__ out, int N, int64_t n) {
  const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (i < n) out[i] = bias[i % N];
}

__global__ void k_vgg_bf16_to_f32(const bf16* __restrict__ in, float* __restrict__ out, int64_t n) {
  const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (i < n) out[i] = __bfloat162float(in[i]);
}

inline unsigned blocks(int64_t n, int t) { return (unsigned)((n + t - 1) / t); }

typedef CUresult (*PFN_encodeTiled)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                    const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                    CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
PFN_encodeTiled vg_encode() {
  static PFN_encodeTiled fn = nullptr;
  if (!fn) {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess &&
        q == cudaDriverEntryPointSuccess)
      fn = (PFN_encodeTiled)p;
  }
  return fn;
}

struct VgConv {
  RoomConvGeom g;         // stride 1, pad 1 (the first layer: its 3 x 3 x 3 im2col as a 1 x 1 convolution of 64 columns)
  int H, W, cin, cout;
  bool pool;
  size_t wp_off, b_off;   // into the packed-weight arena (elements) and the bias arena (floats)
  int w_idx;              // expected-weight index of the conv weight (the bias follows)
  CUtensorMap tm_in, tm_w;
};

}  // namespace
}  // namespace ds

struct ds_vgg {
  ds_vgg_config cfg;
  bool bf16 = false;
  size_t esz = 4;
  std::vector<std::string> names;
  std::vector<int64_t> numel, off;
  int64_t n_params = 0;
  VgConv conv[VG_NCONV];
  size_t fc1_off = 0, fc2_off = 0, wp_total = 0;     // packed-weight arena offsets
  int fc1_idx = 0, fc2_idx = 0;
  void* wp = nullptr;
  float* bias = nullptr;      // [conv biases | fc1 bias (4096) | fc2 bias (4096)]
  size_t fc1_b = 0, fc2_b = 0;
  bool weights_set = false;
  // pass buffers for `capacity` images
  void *x0 = nullptr, *cols = nullptr, *act[2] = {nullptr, nullptr}, *z = nullptr, *h1 = nullptr;
  TcGemmPlan *fc1 = nullptr, *fc2 = nullptr;
};

namespace {

void vg_free(ds_vgg* h) {
  if (h->fc1) tc_plan_destroy(h->fc1);
  if (h->fc2) tc_plan_destroy(h->fc2);
  void* bufs[] = {h->x0, h->cols, h->act[0], h->act[1], h->z, h->h1, h->wp, h->bias};
  for (void* b : bufs) cudaFree(b);
}

void add_name(ds_vgg* h, const std::string& n, int64_t numel) {
  h->names.push_back(n);
  h->numel.push_back(numel);
  h->off.push_back(h->n_params);
  h->n_params += numel;
}

bool encode(CUtensorMap* map, const void* base, int rank, const cuuint64_t* dims, const cuuint64_t* strides_bytes,
            const cuuint32_t* box, char* err, int err_len) {
  PFN_encodeTiled enc = vg_encode();
  if (!enc) {
    snprintf(err, err_len, "cuTensorMapEncodeTiled unavailable");
    return false;
  }
  cuuint32_t estr[4] = {1, 1, 1, 1};
  CUresult r = enc(map, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, rank, const_cast<void*>(base), dims, strides_bytes, box, estr,
                   CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                   CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    snprintf(err, err_len, "cuTensorMapEncodeTiled failed (%d), rank %d", (int)r, rank);
    return false;
  }
  return true;
}

// geometry of one 3 x 3 / pad 1 convolution (cin = 3: the first layer, run over its 64-column im2col)
void conv_geom(VgConv& c, int cin, int cout, int H, int W, bool pool) {
  c.cin = cin; c.cout = cout; c.pool = pool; c.H = H; c.W = W;
  c.g.cin = cin; c.g.cout = cout; c.g.k = 3; c.g.stride = 1; c.g.pad = 1;
  c.g.hin = c.g.hout = H;
  c.g.win = c.g.wout = W;
  c.g.Kp = (9 * cin + 63) / 64 * 64;
}

// tensor maps of one bf16 convolution: its NHWC input (the im2col columns for cin = 3) for `cap` images, and its
// packed weights at wp + c.wp_off
int conv_maps(VgConv& c, const void* in, const bf16* wp, int cap, int l) {
  char err[256] = "";
  if (conv_tc_maps(&c.tm_in, &c.tm_w, in, c.cin == 3 ? 64 : c.cin, c.H, c.W, cap, wp + c.wp_off, c.g.Kp, c.cout,
                   c.cout == 64 ? 64 : 128, err, sizeof err))
    return fail(DS_ERR_CUDA, "vgg16: tensor maps of conv %d: %s", l, err);
  return 0;
}

int vg_set_attrs() { return conv_tc_set_attrs(); }

// tensor maps and GEMM plans of the bf16 path over the pass buffers
int vg_plan_bf16(ds_vgg* h) {
  const int cap = h->cfg.capacity;
  char err[256] = "";
  for (int l = 0; l < VG_NCONV; ++l) {
    const int rc = conv_maps(h->conv[l], l == 0 ? h->cols : h->act[(l - 1) & 1], (const bf16*)h->wp, cap, l);
    if (rc) return rc;
  }
  GemmArgs g;
  memset(&g, 0, sizeof g);
  g.a0 = h->act[0]; g.lda0 = VG_FC1_K; g.k0 = VG_FC1_K;      // conv 13 (index 12) writes act[0]
  g.w = (const bf16*)h->wp + h->fc1_off; g.ldw = VG_FC1_K;
  g.bias = h->bias + h->fc1_b;
  g.d = h->h1; g.ldd = DS_VGG_FEATURES;
  g.M = cap; g.N = DS_VGG_FEATURES; g.act = ACT_RELU;
  if (!(h->fc1 = tc_plan_create(g, cap, err, sizeof err))) return fail(DS_ERR_CUDA, "vgg16: fc1 GEMM plan: %s", err);
  memset(&g, 0, sizeof g);
  g.a0 = h->h1; g.lda0 = DS_VGG_FEATURES; g.k0 = DS_VGG_FEATURES;
  g.w = (const bf16*)h->wp + h->fc2_off; g.ldw = DS_VGG_FEATURES;
  g.ldd = DS_VGG_FEATURES;
  g.M = cap; g.N = DS_VGG_FEATURES;
  if (!(h->fc2 = tc_plan_create(g, cap, err, sizeof err))) return fail(DS_ERR_CUDA, "vgg16: fc2 GEMM plan: %s", err);
  return 0;
}

void conv_fwd_bf16(const VgConv& c, bf16* out, const float* bias, int B, cudaStream_t s) {
  VgConvEpi e;
  const bool first = c.cin == 3;
  e.bias = bias; e.out = out; e.H = c.H; e.W = c.W; e.C = c.g.Kp / (first ? 1 : 9); e.cout = c.cout;
  e.taps = first ? 1 : 9;
  e.kw = first ? 1 : 3;
  e.ph = e.pw = first ? 0 : 1;
  e.Ho = c.H; e.Wo = c.W; e.ldo = c.cout; e.co_off = 0;
  conv_tc_launch(c.tm_in, c.tm_w, e, c.cout == 64 ? 64 : 128, c.pool, B, s);
}


int vg_pass_bf16(ds_vgg* h, int B, float* feat, cudaStream_t s) {
  const VgConv& c0 = h->conv[0];
  launch_re_im2col<bf16>((const bf16*)h->x0, c0.g, B, (bf16*)h->cols, s);
  for (int l = 0; l < VG_NCONV; ++l) {
    const VgConv& c = h->conv[l];
    bf16* out = (bf16*)h->act[l & 1];
    conv_fwd_bf16(c, out, h->bias + c.b_off, B, s);
  }
  CK(cudaGetLastError());
  int e = launch_gemm_tc(h->fc1, B, s);
  if (e) return fail(DS_ERR_CUDA, "vgg16: fc1 GEMM failed: %s", cudaGetErrorString((cudaError_t)e));
  const int64_t n = (int64_t)B * DS_VGG_FEATURES;
  k_vgg_fill_bias<<<blocks(n, 256), 256, 0, s>>>(h->bias + h->fc2_b, feat, DS_VGG_FEATURES, n);
  tc_plan_set_atomic_out(h->fc2, feat, DS_VGG_FEATURES, 1);
  e = launch_gemm_tc(h->fc2, B, s);
  if (e) return fail(DS_ERR_CUDA, "vgg16: fc2 GEMM failed: %s", cudaGetErrorString((cudaError_t)e));
  return 0;
}

void simt(const float* a, int K, const float* w, const float* bias, float* d, int M, int N, int act, cudaStream_t s) {
  constexpr int CHUNK = 32768 * 64;      // gridDim.y of the SIMT GEMM (64 rows per CTA row) stays below 65535
  for (int m0 = 0; m0 < M; m0 += CHUNK) {
    GemmArgs g;
    memset(&g, 0, sizeof g);
    g.a0 = a + (size_t)m0 * K; g.lda0 = K; g.k0 = K;
    g.w = w; g.ldw = K;
    g.bias = bias;
    g.d = d + (size_t)m0 * N; g.ldd = N;
    g.M = std::min(CHUNK, M - m0); g.N = N; g.act = act;
    launch_gemm_simt<float>(g, true, s);
  }
}

int vg_pass_fp32(ds_vgg* h, int B, float* feat, cudaStream_t s) {
  const float* x = (const float*)h->x0;
  for (int l = 0; l < VG_NCONV; ++l) {
    const VgConv& c = h->conv[l];
    float* out = (float*)h->act[l & 1];
    launch_re_im2col<float>(x, c.g, B, (float*)h->cols, s);
    const int M = B * c.H * c.W;
    simt((const float*)h->cols, c.g.Kp, (const float*)h->wp + c.wp_off, h->bias + c.b_off, c.pool ? (float*)h->z : out,
         M, c.cout, ACT_RELU, s);
    if (c.pool) {
      const int64_t n = (int64_t)B * (c.H / 2) * (c.W / 2) * c.cout;
      k_vgg_pool<float><<<blocks(n, 256), 256, 0, s>>>((const float*)h->z, out, c.cout, c.H, c.W, n);
    }
    x = out;
  }
  simt(x, VG_FC1_K, (const float*)h->wp + h->fc1_off, h->bias + h->fc1_b, (float*)h->h1, B, DS_VGG_FEATURES, ACT_RELU, s);
  simt((const float*)h->h1, DS_VGG_FEATURES, (const float*)h->wp + h->fc2_off, h->bias + h->fc2_b, feat, B,
       DS_VGG_FEATURES, ACT_NONE, s);
  CK(cudaGetLastError());
  return 0;
}

}  // namespace

namespace ds {
int conv_tc_set_attrs() {
  char err[256] = "";
  if (!tc_runtime_available(err, sizeof err)) return fail(DS_ERR_CUDA, "%s", err);
  CK(cudaFuncSetAttribute(k_vgg_conv<64, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, VgSmem<64>::BYTES));
  CK(cudaFuncSetAttribute(k_vgg_conv<64, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, VgSmem<64>::BYTES));
  CK(cudaFuncSetAttribute(k_vgg_conv<128, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, VgSmem<128>::BYTES));
  CK(cudaFuncSetAttribute(k_vgg_conv<128, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, VgSmem<128>::BYTES));
  return 0;
}

int conv_tc_maps(CUtensorMap* tm_in, CUtensorMap* tm_w, const void* in, int C, int H, int W, int images,
                 const bf16* wp, int K, int cout, int bn, char* err, int err_len) {
  const cuuint64_t dims[4] = {(cuuint64_t)C, (cuuint64_t)W, (cuuint64_t)H, (cuuint64_t)images};
  const cuuint64_t str[3] = {(cuuint64_t)C * 2, (cuuint64_t)W * C * 2, (cuuint64_t)H * W * C * 2};
  const cuuint32_t box[4] = {BK, VG_TX, VG_TY, 1};
  if (!encode(tm_in, in, 4, dims, str, box, err, err_len)) return -1;
  const cuuint64_t wd[2] = {(cuuint64_t)K, (cuuint64_t)cout};
  const cuuint64_t ws[1] = {(cuuint64_t)K * 2};
  const cuuint32_t wb[2] = {BK, (cuuint32_t)bn};
  if (!encode(tm_w, wp, 2, wd, ws, wb, err, err_len)) return -1;
  return 0;
}

void conv_tc_launch(const CUtensorMap& tm_in, const CUtensorMap& tm_w, const VgConvEpi& e0, int bn, bool pool, int B,
                    cudaStream_t s) {
  VgConvEpi e = e0;
  e.tiles_x = (e.Wo + VG_TX - 1) / VG_TX;
  e.tiles_y = (e.Ho + VG_TY - 1) / VG_TY;
  const int64_t grid = (int64_t)B * e.tiles_x * e.tiles_y * ((e.cout + bn - 1) / bn);
  int* flag = tc_error_flag_dev();
  if (bn == 64) {
    if (pool) k_vgg_conv<64, true><<<(unsigned)grid, VG_THREADS, VgSmem<64>::BYTES, s>>>(tm_in, tm_w, e, flag);
    else k_vgg_conv<64, false><<<(unsigned)grid, VG_THREADS, VgSmem<64>::BYTES, s>>>(tm_in, tm_w, e, flag);
  } else {
    if (pool) k_vgg_conv<128, true><<<(unsigned)grid, VG_THREADS, VgSmem<128>::BYTES, s>>>(tm_in, tm_w, e, flag);
    else k_vgg_conv<128, false><<<(unsigned)grid, VG_THREADS, VgSmem<128>::BYTES, s>>>(tm_in, tm_w, e, flag);
  }
}

}  // namespace ds

extern "C" int ds_vgg_create(const ds_vgg_config* cfg, ds_vgg** out) {
  if (!cfg || !out) return fail(DS_ERR_INVALID, "null argument");
  *out = nullptr;
  if (cfg->precision != DS_PREC_FP32 && cfg->precision != DS_PREC_BF16)
    return fail(DS_ERR_INVALID, "vgg16: precision %d unknown", cfg->precision);
  if (cfg->capacity < 1 || cfg->capacity > 256)
    return fail(DS_ERR_INVALID, "vgg16: capacity %d outside [1, 256]", cfg->capacity);
  int ndev = 0;
  if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) {
    cudaGetLastError();
    return fail(DS_ERR_NO_DEVICE, "no CUDA device: diffuscene_b200 has no CPU fallback");
  }
  if (cfg->device < 0 || cfg->device >= ndev) return fail(DS_ERR_INVALID, "device %d out of range", cfg->device);
  CK(cudaSetDevice(cfg->device));
  cudaDeviceProp prop;
  CK(cudaGetDeviceProperties(&prop, cfg->device));
  if (prop.major != 9)
    return fail(DS_ERR_NO_DEVICE, "device %d is sm_%d%d; this library is built for sm_90a only", cfg->device, prop.major,
                prop.minor);
  if (cfg->precision == DS_PREC_BF16) {
    const int rc = vg_set_attrs();
    if (rc) return rc;
  }
  ds_vgg* h = new ds_vgg();
  h->cfg = *cfg;
  h->bf16 = cfg->precision == DS_PREC_BF16;
  h->esz = h->bf16 ? 2 : 4;
  int H = VG_IMG;
  size_t b_total = 0;
  for (int l = 0; l < VG_NCONV; ++l) {
    VgConv& c = h->conv[l];
    conv_geom(c, kCin[l], kCout[l], H, H, kPool[l]);
    c.wp_off = h->wp_total;
    h->wp_total += (size_t)c.cout * c.g.Kp;
    c.b_off = b_total;
    b_total += c.cout;
    c.w_idx = int(h->names.size());
    const std::string pre = "features." + std::to_string(kFeatIdx[l]);
    add_name(h, pre + ".weight", (int64_t)c.cout * c.cin * 9);
    add_name(h, pre + ".bias", c.cout);
    if (c.pool) H /= 2;
  }
  h->fc1_idx = int(h->names.size());
  add_name(h, "classifier.0.weight", (int64_t)DS_VGG_FEATURES * VG_FC1_K);
  add_name(h, "classifier.0.bias", DS_VGG_FEATURES);
  h->fc2_idx = int(h->names.size());
  add_name(h, "classifier.3.weight", (int64_t)DS_VGG_FEATURES * DS_VGG_FEATURES);
  add_name(h, "classifier.3.bias", DS_VGG_FEATURES);
  h->fc1_off = h->wp_total;
  h->wp_total += (size_t)DS_VGG_FEATURES * VG_FC1_K;
  h->fc2_off = h->wp_total;
  h->wp_total += (size_t)DS_VGG_FEATURES * DS_VGG_FEATURES;
  h->fc1_b = b_total;
  h->fc2_b = b_total + DS_VGG_FEATURES;
  b_total += 2 * DS_VGG_FEATURES;

  const int64_t cap = cfg->capacity, px = (int64_t)VG_IMG * VG_IMG;
  const size_t e = h->esz;
  // largest activation: 224 x 224 x 64; fp32 im2col of conv 2: 224 x 224 x 576; bf16: conv 1's 64 columns only
  const size_t act_n = (size_t)cap * px * 64;
  const size_t cols_n = (size_t)cap * px * (h->bf16 ? 64 : 576);
  cudaError_t ce = cudaSuccess;
  auto alloc = [&](void** p, size_t bytes) { if (ce == cudaSuccess) ce = cudaMalloc(p, bytes); };
  alloc(&h->wp, h->wp_total * e);
  alloc((void**)&h->bias, b_total * 4);
  alloc(&h->x0, (size_t)cap * px * 3 * e);
  alloc(&h->cols, cols_n * e);
  alloc(&h->act[0], act_n * e);
  alloc(&h->act[1], act_n * e);
  if (!h->bf16) alloc(&h->z, act_n * e);
  alloc(&h->h1, (size_t)cap * DS_VGG_FEATURES * e);
  if (ce != cudaSuccess) {
    vg_free(h);
    delete h;
    return fail(DS_ERR_CUDA, "vgg16: buffers for %d images: %s", cfg->capacity, cudaGetErrorString(ce));
  }
  if (h->bf16) {
    const int rc = vg_plan_bf16(h);
    if (rc) {
      vg_free(h);
      delete h;
      return rc;
    }
  }
  *out = h;
  return 0;
}

extern "C" int ds_vgg_destroy(ds_vgg* h) {
  if (!h) return 0;
  cudaSetDevice(h->cfg.device);
  vg_free(h);
  delete h;
  return 0;
}

extern "C" int ds_vgg_expected_weight_count(ds_vgg* h) {
  if (!h) return fail(DS_ERR_INVALID, "null handle");
  return int(h->names.size());
}

extern "C" int ds_vgg_expected_weight(ds_vgg* h, int index, const char** name, int64_t* numel) {
  if (!h || !name || !numel) return fail(DS_ERR_INVALID, "null argument");
  if (index < 0 || index >= (int)h->names.size()) return fail(DS_ERR_INVALID, "weight index %d out of range", index);
  *name = h->names[index].c_str();
  *numel = h->numel[index];
  return 0;
}

extern "C" int ds_vgg_set_weights(ds_vgg* h, const float* flat_params_dev, int64_t count, void* stream) {
  if (!h || !flat_params_dev) return fail(DS_ERR_INVALID, "null argument");
  if (count != h->n_params)
    return fail(DS_ERR_INVALID, "vgg16: %lld parameters given, %lld expected", (long long)count, (long long)h->n_params);
  CK(cudaSetDevice(h->cfg.device));
  cudaStream_t s = (cudaStream_t)stream;
  const float* p = flat_params_dev;
  for (int l = 0; l < VG_NCONV; ++l) {
    const VgConv& c = h->conv[l];
    if (h->bf16) k_vgg_pack_conv<bf16><<<c.cout, 256, 0, s>>>(p + h->off[c.w_idx], c.cin, c.g.Kp, (bf16*)h->wp + c.wp_off);
    else k_vgg_pack_conv<float><<<c.cout, 256, 0, s>>>(p + h->off[c.w_idx], c.cin, c.g.Kp, (float*)h->wp + c.wp_off);
    CK(cudaMemcpyAsync(h->bias + c.b_off, p + h->off[c.w_idx + 1], c.cout * 4, cudaMemcpyDeviceToDevice, s));
  }
  if (h->bf16) {
    k_vgg_pack_fc<bf16><<<DS_VGG_FEATURES, 256, 0, s>>>(p + h->off[h->fc1_idx], VG_FC1_K, 1, (bf16*)h->wp + h->fc1_off);
    k_vgg_pack_fc<bf16><<<DS_VGG_FEATURES, 256, 0, s>>>(p + h->off[h->fc2_idx], DS_VGG_FEATURES, 0, (bf16*)h->wp + h->fc2_off);
  } else {
    k_vgg_pack_fc<float><<<DS_VGG_FEATURES, 256, 0, s>>>(p + h->off[h->fc1_idx], VG_FC1_K, 1, (float*)h->wp + h->fc1_off);
    k_vgg_pack_fc<float><<<DS_VGG_FEATURES, 256, 0, s>>>(p + h->off[h->fc2_idx], DS_VGG_FEATURES, 0,
                                                         (float*)h->wp + h->fc2_off);
  }
  CK(cudaMemcpyAsync(h->bias + h->fc1_b, p + h->off[h->fc1_idx + 1], DS_VGG_FEATURES * 4, cudaMemcpyDeviceToDevice, s));
  CK(cudaMemcpyAsync(h->bias + h->fc2_b, p + h->off[h->fc2_idx + 1], DS_VGG_FEATURES * 4, cudaMemcpyDeviceToDevice, s));
  CK(cudaGetLastError());
  h->weights_set = true;
  return 0;
}

extern "C" int ds_vgg_features(ds_vgg* h, const float* images_dev, int32_t batch, int32_t height, int32_t width,
                               float* features_dev, void* stream) {
  if (!h || !images_dev || !features_dev) return fail(DS_ERR_INVALID, "null argument");
  if (batch < 0) return fail(DS_ERR_INVALID, "vgg16: batch %d < 0", batch);
  if (height < 1 || width < 1 || height > 4096 || width > 4096)
    return fail(DS_ERR_INVALID, "vgg16: image %d x %d outside [1, 4096]", height, width);
  if (!h->weights_set) return fail(DS_ERR_STATE, "vgg16: ds_vgg_set_weights first");
  CK(cudaSetDevice(h->cfg.device));
  cudaStream_t s = (cudaStream_t)stream;
  const int64_t img_n = (int64_t)3 * height * width;
  for (int b0 = 0; b0 < batch; b0 += h->cfg.capacity) {
    const int B = std::min(h->cfg.capacity, batch - b0);
    const int64_t n = (int64_t)B * VG_IMG * VG_IMG * 3;
    if (h->bf16) k_vgg_pack<bf16><<<blocks(n, 256), 256, 0, s>>>(images_dev + b0 * img_n, height, width, (bf16*)h->x0, n);
    else k_vgg_pack<float><<<blocks(n, 256), 256, 0, s>>>(images_dev + b0 * img_n, height, width, (float*)h->x0, n);
    float* feat = features_dev + (int64_t)b0 * DS_VGG_FEATURES;
    const int rc = h->bf16 ? vg_pass_bf16(h, B, feat, s) : vg_pass_fp32(h, B, feat, s);
    if (rc) return rc;
  }
  CK(cudaGetLastError());
  return 0;
}

extern "C" int ds_vgg_test_conv(const float* in_dev, int32_t batch, int32_t height, int32_t width, int32_t cin,
                                int32_t cout, int32_t pool, const float* weight_dev, const float* bias_dev,
                                float* out_dev, void* stream) {
  if (!in_dev || !weight_dev || !bias_dev || !out_dev) return fail(DS_ERR_INVALID, "null argument");
  if (batch < 1 || height < 1 || width < 1 || height > 4096 || width > 4096)
    return fail(DS_ERR_INVALID, "vgg16 conv: batch %d, image %d x %d", batch, height, width);
  if (!(cin == 3 || (cin >= 64 && cin % 64 == 0 && cin <= 4096)) || !(cout == 64 || (cout % 128 == 0 && cout <= 4096)))
    return fail(DS_ERR_INVALID, "vgg16 conv: cin %d must be 3 or a multiple of 64, cout %d 64 or a multiple of 128",
                cin, cout);
  if (pool && (height % 2 || width % 2)) return fail(DS_ERR_INVALID, "vgg16 conv: pooled sides must be even");
  int ndev = 0;
  if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) {
    cudaGetLastError();
    return fail(DS_ERR_NO_DEVICE, "no CUDA device: diffuscene_b200 has no CPU fallback");
  }
  int rc = vg_set_attrs();
  if (rc) return rc;
  cudaStream_t s = (cudaStream_t)stream;
  VgConv c;
  conv_geom(c, cin, cout, height, width, pool != 0);
  c.wp_off = 0;
  const int64_t px = (int64_t)batch * height * width;
  const int64_t n_out = (int64_t)batch * (pool ? height / 2 : height) * (pool ? width / 2 : width) * cout;
  bf16 *x = nullptr, *cols = nullptr, *wp = nullptr, *y = nullptr;
  CK(cudaMallocAsync((void**)&x, px * cin * 2, s));
  CK(cudaMallocAsync((void**)&wp, (size_t)cout * c.g.Kp * 2, s));
  CK(cudaMallocAsync((void**)&y, n_out * 2, s));
  if (cin == 3) CK(cudaMallocAsync((void**)&cols, px * 64 * 2, s));
  launch_te_convert<bf16>(in_dev, x, px * cin, s);
  k_vgg_pack_conv<bf16><<<cout, 256, 0, s>>>(weight_dev, cin, c.g.Kp, wp);
  if (cin == 3) launch_re_im2col<bf16>(x, c.g, batch, cols, s);
  rc = conv_maps(c, cin == 3 ? (const void*)cols : (const void*)x, wp, batch, 0);
  if (!rc) {
    conv_fwd_bf16(c, y, bias_dev, batch, s);
    k_vgg_bf16_to_f32<<<blocks(n_out, 256), 256, 0, s>>>(y, out_dev, n_out);
  }
  cudaFreeAsync(x, s);
  cudaFreeAsync(wp, s);
  cudaFreeAsync(y, s);
  if (cols) cudaFreeAsync(cols, s);
  if (rc) return rc;
  CK(cudaGetLastError());
  CK(cudaStreamSynchronize(s));
  return 0;
}
