// k_gemm_ln: the tail of the reference's attention wrappers as ONE kernel,
//     out = LayerNorm_g( A[M, K] * W[C, K]^T + bias ) + residual
// i.e. `to_out = Sequential(Conv1d(hidden, dim, 1), LayerNorm(dim))` of LinearAttention / LinearAttentionCross
// (scene_synthesis/networks/denoise_net.py:214-217,234-235 and :268-271,296-297; LayerNorm :93-102: biased variance,
// eps 1e-5, gain only) followed by the `Residual` add of the un-normalised input (:39-45).  Unfused this is a GEMM
// launch plus a LayerNorm launch with the projection written to HBM and re-read between them; fused, it never leaves
// the accumulator registers.
//
// Shape: K = heads * dim_head <= 128, C = 512.  That makes the WHOLE weight matrix <= 128 KB of bf16: every CTA loads
// it once into shared memory (TMA, 128B swizzle) and keeps it for all of its tiles, so the only streamed operand is the
// 64 x K activation tile, double-buffered.  One persistent CTA per SM, 256 threads = two warpgroups; warpgroup g owns
// output columns 256 g .. 256 g + 255 of the tile's 64 rows (two wgmma m64n128k16 accumulators, 128 registers).  A row's
// LayerNorm statistics are sums over the thread's 64 columns, the quad of threads sharing the row, and the two
// warpgroups (through shared memory).
#include <stdio.h>
#include <string.h>

#include "kernels.cuh"
#include "tc_common.cuh"

namespace ds {

bool tc_encode_2d(CUtensorMap* map, const void* base, uint64_t inner, uint64_t rows, uint64_t pitch_elems,
                  uint32_t box_rows, char* err, int err_len);      // gemm_tc.cu
int* tc_error_flag_dev();
int tc_num_sms();

namespace {

constexpr int LN_C = 512;                 // output channels = LayerNorm width
constexpr int LN_KMAX = 128;              // weights stay resident: C x K x 2 B <= 128 KB
constexpr int LN_ROWS = 64;               // token rows per tile
constexpr int LN_THREADS = 256;
constexpr int LN_WKB_BYTES = LN_C * BK * 2;                  // one k-block of the weights: 64 KB
constexpr int LN_AKB_BYTES = LN_ROWS * BK * 2;               // one k-block of an activation tile: 8 KB
constexpr int LN_A_OFF = (LN_KMAX / BK) * LN_WKB_BYTES;      // 131072
constexpr int LN_A_BUF = (LN_KMAX / BK) * LN_AKB_BYTES;      // 16 KB per activation buffer
constexpr int LN_BAR_OFF = LN_A_OFF + 2 * LN_A_BUF;
constexpr int LN_CHAN_OFF = LN_BAR_OFF + 64;                 // bias[512], gain[512]
constexpr int LN_PART_OFF = LN_CHAN_OFF + 2 * LN_C * 4;      // (sum, sum of squares)[64 rows][2 warpgroups]
constexpr int LN_SMEM = 1024 + LN_PART_OFF + LN_ROWS * 2 * 8;
static_assert(LN_SMEM <= 232448, "shared memory budget exceeded");

struct LnEpi {
  const float* bias;
  const float* gain;
  bf16* d; int ldd;
  const bf16* res; int ldres;
  int M, kblocks;
};

__global__ void __launch_bounds__(LN_THREADS, 1)
k_gemm_ln(const __grid_constant__ CUtensorMap tm_a, const __grid_constant__ CUtensorMap tm_w, LnEpi epi, int* err_flag) {
  extern __shared__ uint8_t smem_raw[];
  const uint32_t raw = smem_u32(smem_raw);
  const uint32_t base = (raw + 1023u) & ~1023u;
  uint8_t* const base_ptr = smem_raw + (base - raw);
  const uint32_t wbar = base + LN_BAR_OFF;
  auto afull = [&](int b) { return base + LN_BAR_OFF + 8u * (1 + b); };
  float* const bias_s = reinterpret_cast<float*>(base_ptr + LN_CHAN_OFF);
  float* const gain_s = bias_s + LN_C;
  float2* const part = reinterpret_cast<float2*>(base_ptr + LN_PART_OFF);

  const int tid = threadIdx.x, wg = tid >> 7, wq = (tid >> 5) & 3, lane = tid & 31;
  const int num_tiles = (epi.M + LN_ROWS - 1) / LN_ROWS;
  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
  if (tid == 0) {
    tma_prefetch_desc(&tm_a);
    tma_prefetch_desc(&tm_w);
    mbar_init(wbar, 1);
    mbar_init(afull(0), 1);
    mbar_init(afull(1), 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
  }
  asm volatile("griddepcontrol.wait;" ::: "memory");
  for (int c = tid; c < LN_C; c += LN_THREADS) {
    bias_s[c] = epi.bias ? __ldg(epi.bias + c) : 0.f;
    gain_s[c] = __ldg(epi.gain + c);
  }
  __syncthreads();
  auto load_a = [&](int tile, int b) {
    mbar_expect_tx(afull(b), uint32_t(epi.kblocks * LN_AKB_BYTES));
    for (int kb = 0; kb < epi.kblocks; ++kb)
      tma_load_2d(base + uint32_t(LN_A_OFF + b * LN_A_BUF + kb * LN_AKB_BYTES), &tm_a, kb * BK, tile * LN_ROWS, afull(b));
  };
  if (tid == 0 && int(blockIdx.x) < num_tiles) {
    mbar_expect_tx(wbar, uint32_t(epi.kblocks * LN_WKB_BYTES));
    for (int kb = 0; kb < epi.kblocks; ++kb)
      for (int h = 0; h < 2; ++h)      // TMA boxes have at most 256 rows
        tma_load_2d(base + uint32_t(kb * LN_WKB_BYTES + h * (LN_WKB_BYTES / 2)), &tm_w, kb * BK, h * 256, wbar);
    load_a(blockIdx.x, 0);
  }

  const int r0 = wq * 16 + (lane >> 2);          // rows r0 and r0 + 8 of the tile
  const int cq = 2 * (lane & 3);
  int it = 0;
  for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x, ++it) {
    const int b = it & 1;
    // the other buffer was read by the previous tile's MMAs, which completed before the barrier that ended it
    if (tid == 0 && tile + int(gridDim.x) < num_tiles) load_a(tile + gridDim.x, b ^ 1);
    __syncwarp();
    mbar_wait(wbar, 0, err_flag, 31);
    mbar_wait(afull(b), uint32_t(it >> 1) & 1u, err_flag, 32);
    float acc[2][64];
#pragma unroll
    for (int nb = 0; nb < 2; ++nb)
#pragma unroll
      for (int j = 0; j < 64; ++j) acc[nb][j] = 0.f;
    wgmma_fence();
    for (int kb = 0; kb < epi.kblocks; ++kb) {
      const uint32_t sa = base + uint32_t(LN_A_OFF + b * LN_A_BUF + kb * LN_AKB_BYTES);
      const uint32_t sw = base + uint32_t(kb * LN_WKB_BYTES + wg * 256 * 128);
#pragma unroll
      for (int k = 0; k < BK / 16; ++k)
#pragma unroll
        for (int nb = 0; nb < 2; ++nb)
          wgmma_m64n128k16(acc[nb], wgmma_desc_sw128(sa + uint32_t(k * 32)),
                           wgmma_desc_sw128(sw + uint32_t(nb * 128 * 128 + k * 32)), uint32_t(kb | k));
    }
    wgmma_commit();
    wgmma_wait0();

    // row statistics of (acc + bias): this thread's 64 columns of each of its two rows, then the quad, then the two
    // warpgroups.  Column of acc[nb][4 j + 2 h + e] = 256 wg + 128 nb + 8 j + cq + e, row r0 + 8 h.
    float2 st[2];
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      float s = 0.f, ss = 0.f;
#pragma unroll
      for (int nb = 0; nb < 2; ++nb)
#pragma unroll
        for (int j = 0; j < 16; ++j)
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            const float v = acc[nb][4 * j + 2 * h + e] + bias_s[wg * 256 + nb * 128 + 8 * j + cq + e];
            s += v;
            ss = fmaf(v, v, ss);
          }
      s += __shfl_xor_sync(0xffffffffu, s, 1);
      ss += __shfl_xor_sync(0xffffffffu, ss, 1);
      s += __shfl_xor_sync(0xffffffffu, s, 2);
      ss += __shfl_xor_sync(0xffffffffu, ss, 2);
      if ((lane & 3) == 0) part[(r0 + 8 * h) * 2 + wg] = make_float2(s, ss);
    }
    __syncthreads();
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const float2 p0 = part[(r0 + 8 * h) * 2], p1 = part[(r0 + 8 * h) * 2 + 1];
      const float mean = (p0.x + p1.x) * (1.0f / LN_C);
      const float var = fmaxf((p0.y + p1.y) * (1.0f / LN_C) - mean * mean, 0.f);
      st[h] = make_float2(mean, rsqrtf(var + 1e-5f));
    }
    // normalise, gain, residual
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int m = tile * LN_ROWS + r0 + 8 * h;
      if (m >= epi.M) continue;
      const float rstd = st[h].y, nmr = -st[h].x * st[h].y;
#pragma unroll
      for (int nb = 0; nb < 2; ++nb)
#pragma unroll
        for (int j = 0; j < 16; ++j) {
          const int c = wg * 256 + nb * 128 + 8 * j + cq;
          // ((acc + b) - mean) * rstd * g  =  fma(acc + b, rstd, -mean * rstd) * g
          float v0 = fmaf(acc[nb][4 * j + 2 * h] + bias_s[c], rstd, nmr) * gain_s[c];
          float v1 = fmaf(acc[nb][4 * j + 2 * h + 1] + bias_s[c + 1], rstd, nmr) * gain_s[c + 1];
          if (epi.res) {
            const float2 r2 = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(epi.res + (int64_t)m * epi.ldres + c));
            v0 += r2.x;
            v1 += r2.y;
          }
          *reinterpret_cast<__nv_bfloat162*>(epi.d + (int64_t)m * epi.ldd + c) = __floats2bfloat162_rn(v0, v1);
        }
    }
    __syncthreads();      // `part` and the activation buffer are free for the next tile
  }
}

}  // namespace

struct LnGemmPlan {
  CUtensorMap tm_a, tm_w;
  LnEpi epi;
};

bool ln_gemm_supported(int N, int K) { return N == LN_C && K % BK == 0 && K > 0 && K <= LN_KMAX; }

LnGemmPlan* ln_plan_create(const GemmArgs& g, int rows_capacity, char* err, int err_len) {
  if (!tc_runtime_available(err, err_len)) return nullptr;
  if (!ln_gemm_supported(g.N, g.k0) || g.a1 || !g.gamma || (g.lda0 % 8) || (g.ldw % 8) || (g.ldd % 2) ||
      (g.res && (g.ldres % 2))) {
    if (err) snprintf(err, err_len, "fused GEMM + LayerNorm needs N = %d, K %% 64 == 0, K <= %d, one operand, a gain",
                      LN_C, LN_KMAX);
    return nullptr;
  }
  static bool attr_set = false;
  if (!attr_set) {
    cudaFuncSetAttribute(k_gemm_ln, cudaFuncAttributeMaxDynamicSharedMemorySize, LN_SMEM);
    attr_set = true;
  }
  LnGemmPlan* p = new LnGemmPlan();
  memset(p, 0, sizeof(*p));
  bool ok = tc_encode_2d(&p->tm_a, g.a0, g.k0, rows_capacity, g.lda0, LN_ROWS, err, err_len);
  if (ok) ok = tc_encode_2d(&p->tm_w, g.w, g.k0, LN_C, g.ldw, 256, err, err_len);
  if (!ok) {
    delete p;
    return nullptr;
  }
  p->epi.bias = g.bias;
  p->epi.gain = g.gamma;
  p->epi.d = (bf16*)g.d;
  p->epi.ldd = g.ldd;
  p->epi.res = (const bf16*)g.res;
  p->epi.ldres = g.ldres;
  p->epi.kblocks = g.k0 / BK;
  return p;
}
void ln_plan_destroy(LnGemmPlan* p) { delete p; }

int launch_gemm_ln(const LnGemmPlan* p, int M, cudaStream_t s) {
  LnEpi epi = p->epi;
  epi.M = M;
  const int tiles = (M + LN_ROWS - 1) / LN_ROWS;
  if (tiles == 0) return 0;
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3(tiles < tc_num_sms() ? tiles : tc_num_sms());
  cfg.blockDim = dim3(LN_THREADS);
  cfg.dynamicSmemBytes = LN_SMEM;
  cfg.stream = s;
  cudaLaunchAttribute attr[1];
  if (pdl_enabled(0, M)) {
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = attr;
    cfg.numAttrs = 1;
  }
  return (int)cudaLaunchKernelEx(&cfg, k_gemm_ln, p->tm_a, p->tm_w, epi, tc_error_flag_dev());
}

}  // namespace ds
