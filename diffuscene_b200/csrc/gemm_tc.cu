// Hopper tensor-core GEMM (sm_90a):  D[M,N] = act([A0|A1][M,K] * W[N,K]^T + bias) (+ residual)
// bf16 operands, fp32 accumulation in registers (wgmma), bf16 output.
//
// This kernel carries every 1x1-conv / linear layer of the denoiser in throughput mode (reference:
// F.conv1d / nn.Linear calls of scene_synthesis/networks/denoise_net.py:91,183,214-217,244-245,487-502).
//
// Structure (one CTA per 128 x 128 output tile and K split, 256 threads = two warpgroups, two CTAs per SM):
//   TMA         thread 0 keeps a STAGES-deep shared-memory ring of A (128 x 64) and W (128 x 64) tiles
//               (cp.async.bulk.tensor, 128B swizzle) filled ahead of the MMAs; completion on mbarriers, every
//               thread of the CTA arrives on the slot's `empty` barrier once its MMAs have read it.
//   wgmma       warpgroup g multiplies rows 64 g .. 64 g + 63 of the A tile with the whole W tile:
//               wgmma.mma_async m64n128k16 x 4 per k-block, accumulator in 64 registers per thread.
//               Two resident CTAs per SM let one CTA's epilogue overlap the other's MMAs.
//   epilogue    from the accumulator registers; results are staged in the drained ring (bf16, or fp32 when a
//               residual follows) and written out as whole 256-byte rows, the residual added in that row pass
//               from 16-byte loads of whole rows.  Three forms:
//                 plain  bias / GELU|SiLU / residual -> bf16
//                 d32    split-K partial sums added to an fp32 output with atomics (weight-gradient GEMMs)
//                 GN     the whole `Block` of the reference (denoise_net.py:160-176) after the conv:
//                        bias -> GroupNorm(8) statistics per (scene, group) reduced across the rows of a
//                        scene through shared memory -> affine -> FiLM -> SiLU (-> + residual).  M tiles
//                        are whole scenes (120 of 128 rows for N=12, 126 for N=21), N tiles are 2 whole
//                        groups of 64 channels, so the statistics never leave the CTA.  The affine
//                        coefficients per (scene, column) and the tile's FiLM rows are tabled in the ring
//                        once, so the element loop reads two 16-byte entries per column pair.
// Both operands are K-major (activations [rows, K], weights [N, K] exactly as PyTorch stores them), so no
// transposes exist anywhere in the data path.  A "virtual concat" [A0|A1] (the U-Net skip connections,
// denoise_net.py:562,566,573) is served by switching tensor maps inside the k loop.
#include <cuda.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include "kernels.cuh"
#include "tc_common.cuh"

namespace ds {

static constexpr int BN = 128;
static constexpr int STAGES = 3;
static constexpr int TC_THREADS = 256;
static constexpr int STAGE_BYTES = A_BYTES + BN * BK * 2;      // 32 KB
static constexpr int GN_GROUP = 64;                            // channels per GroupNorm group (C = 512, 8 groups)
// ring | 2 x STAGES mbarriers (256 B reserved) | bias, gamma, beta [BN] | GN partials [BM][2] | GN statistics [BM][2]
static constexpr int CHAN_OFF = STAGES * STAGE_BYTES + 256;
static constexpr int PART_OFF = CHAN_OFF + 3 * BN * 4;
static constexpr int STAT_OFF = PART_OFF + BM * 2 * 8;
static constexpr int SMEM_BYTES = 1024 /*align slack*/ + STAT_OFF + BM * 2 * 8;
static_assert(2 * (SMEM_BYTES + 1024) <= 233472, "two CTAs per SM");
// output tile staged in the drained ring before it is written out, bf16 or (launches with a residual) fp32.  The row
// pitch of 136 elements puts the 8 rows one fragment store touches on distinct banks: 68 words for bf16 (one
// wavefront), 136 words for fp32 (rows 4 apart share banks: two wavefronts, the least for 256 bytes)
static constexpr int STG_PITCH = BN + 8;
static constexpr int STG16_BYTES = BM * STG_PITCH * 2;
static constexpr int STG32_BYTES = BM * STG_PITCH * 4;
// GN epilogue tables behind the staging tile, one row of BN / 2 float4 per scene of the tile (GroupNorm affine) and
// per FiLM row.  At most GN_MAX_SPT scenes per tile (>= 12 objects per scene), so the affine table always fits; the
// FiLM table is used where it fits as well and read from global memory otherwise
static constexpr int TBL_ROW_BYTES = BN / 2 * 16;
static constexpr int GN_MAX_SPT = 10;
static_assert(STG32_BYTES + 2 * GN_MAX_SPT * TBL_ROW_BYTES <= STAGES * STAGE_BYTES, "tables fit in the ring");

struct TcEpi {
  const float* bias;
  bf16* d; int ldd;
  const bf16* res; int ldres;
  int act;
  int M, N;
  int kb0, kb1;          // k-blocks taken from A0 and from A1
  int tile_rows;         // rows advanced per M tile (128, or whole scenes for the GN epilogue)
  // GroupNorm epilogue
  int n_obj;             // rows per scene
  int C;                 // channel count of the FiLM table rows ([scale(C) | shift(C)])
  const float* gamma;
  const float* beta;
  FilmRef film;
  float* d32;            // fp32 output accumulated with atomics (split-K weight-gradient GEMMs), else nullptr
  int ksplit;            // ... number of K splits (work units = tiles x ksplit)
};

template <bool GN>
__global__ void __launch_bounds__(TC_THREADS, 2)
k_gemm_wg(const __grid_constant__ CUtensorMap tm_a0, const __grid_constant__ CUtensorMap tm_a1,
          const __grid_constant__ CUtensorMap tm_w, TcEpi epi, int* err_flag) {
  extern __shared__ uint8_t smem_raw[];
  const uint32_t raw = smem_u32(smem_raw);
  const uint32_t base = (raw + 1023u) & ~1023u;
  uint8_t* const base_ptr = smem_raw + (base - raw);
  const uint32_t bar_base = base + STAGES * STAGE_BYTES;
  auto full_bar = [&](int s) { return bar_base + 8u * s; };
  auto empty_bar = [&](int s) { return bar_base + 8u * (STAGES + s); };
  float* const chan = reinterpret_cast<float*>(base_ptr + CHAN_OFF);       // [0, BN) bias, [BN, 2BN) gamma, then beta
  float2* const part = reinterpret_cast<float2*>(base_ptr + PART_OFF);     // [row][group] (sum, sum of squares)
  float2* const stat = reinterpret_cast<float2*>(base_ptr + STAT_OFF);     // [scene][group] (mean, rstd)

  const int tid = threadIdx.x, wg = tid >> 7, wq = (tid >> 5) & 3, lane = tid & 31;
  const int num_n = epi.N / BN;
  const int num_m = (epi.M + epi.tile_rows - 1) / epi.tile_rows;
  const int tiles = num_m * num_n;
  const int tile = blockIdx.x % tiles, split = blockIdx.x / tiles;
  const int n_idx = tile % num_n, m_idx = tile / num_n;          // N fastest: neighbouring CTAs share A in L2
  const int m0 = m_idx * epi.tile_rows, n0 = n_idx * BN;
  const int kblocks = epi.kb0 + epi.kb1;
  const int kb_per = (kblocks + epi.ksplit - 1) / epi.ksplit;
  const int kb_lo = split * kb_per, kb_hi = min(kblocks, kb_lo + kb_per);
  const int nk = kb_hi - kb_lo;

  // programmatic dependent launch: the next kernel's CTAs may be scheduled as SMs drain (its prologue overlaps our
  // tail); it still waits for this grid's completion at its own griddepcontrol.wait
  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
  if (tid == 0) {
    tma_prefetch_desc(&tm_a0);
    tma_prefetch_desc(&tm_a1);
    tma_prefetch_desc(&tm_w);
    for (int s = 0; s < STAGES; ++s) {
      mbar_init(full_bar(s), 1);
      mbar_init(empty_bar(s), TC_THREADS);
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
  }
  // everything above touched no global memory; from here on we read buffers written by earlier kernels
  asm volatile("griddepcontrol.wait;" ::: "memory");
  for (int c = tid; c < BN; c += TC_THREADS) {
    chan[c] = epi.bias ? __ldg(epi.bias + n0 + c) : 0.f;
    if constexpr (GN) {
      chan[BN + c] = __ldg(epi.gamma + n0 + c);
      chan[2 * BN + c] = __ldg(epi.beta + n0 + c);
    }
  }
  __syncthreads();
  if (nk <= 0) return;      // an empty K split (more splits than k-blocks): contributes nothing

  auto issue = [&](int i) {
    const int s = i % STAGES, kb = kb_lo + i;
    const uint32_t sa = base + uint32_t(s * STAGE_BYTES);
    mbar_expect_tx(full_bar(s), STAGE_BYTES);
    if (kb < epi.kb0) tma_load_2d(sa, &tm_a0, kb * BK, m0, full_bar(s));
    else tma_load_2d(sa, &tm_a1, (kb - epi.kb0) * BK, m0, full_bar(s));
    tma_load_2d(sa + A_BYTES, &tm_w, kb * BK, n0, full_bar(s));
  };
  if (tid == 0)
    for (int i = 0; i < STAGES && i < nk; ++i) issue(i);

  float acc[64];
#pragma unroll
  for (int j = 0; j < 64; ++j) acc[j] = 0.f;
  for (int i = 0; i < nk; ++i) {
    const int s = i % STAGES;
    const uint32_t ph = uint32_t(i / STAGES) & 1u;
    mbar_wait(full_bar(s), ph, err_flag, 1);
    const uint32_t sa = base + uint32_t(s * STAGE_BYTES);
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < BK / 16; ++k)      // advance 16 elements (32 bytes) along K inside the 128-byte swizzle row
      wgmma_m64n128k16(acc, wgmma_desc_sw128(sa + uint32_t(wg * 64 * 128 + k * 32)),
                       wgmma_desc_sw128(sa + uint32_t(A_BYTES + k * 32)), uint32_t(i | k));
    wgmma_commit();
    wgmma_wait0();
    mbar_arrive(empty_bar(s));             // this thread's MMAs have read the slot
    if (tid == 0 && i + STAGES < nk) {
      mbar_wait(empty_bar(s), ph, err_flag, 2);
      issue(i + STAGES);
    }
    __syncwarp();
  }

  // accumulator layout of wgmma m64nN: this thread holds rows r0 and r0 + 8 of its warpgroup's 64 rows, columns
  // 8 j + cq + {0, 1} (j = 0 .. 15) in acc[4 j + 2 h + {0, 1}] for row r0 + 8 h
  const int r0 = wg * 64 + wq * 16 + (lane >> 2);
  const int cq = 2 * (lane & 3);
  if (epi.d32) {
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int rt = r0 + 8 * h, m = m0 + rt;
      if (rt >= epi.tile_rows || m >= epi.M) continue;
      float* op = epi.d32 + (int64_t)m * epi.ldd + n0 + cq;
#pragma unroll
      for (int j = 0; j < 16; ++j)      // vector reduction: both floats of the column pair in one L2 atomic
        asm volatile("red.global.add.v2.f32 [%0], {%1, %2};" ::"l"(op + 8 * j), "f"(acc[4 * j + 2 * h]),
                     "f"(acc[4 * j + 2 * h + 1]) : "memory");
    }
    return;
  }

  // the output tile is staged in the drained ring: fp32 when a residual is added in the row pass, else bf16
  const bool stage32 = epi.res != nullptr;
  const int tbl_off = stage32 ? STG32_BYTES : STG16_BYTES;
  // GN: per (scene of the tile, column pair) float4 (a0, a1, b0, b1) of y = a x + b (GroupNorm affine with the conv
  // bias folded in), then the FiLM rows of the tile as float4 (scale0 + 1, scale1 + 1, shift0, shift1) per column
  // pair: one row per scene (time) or per object (shared context).  Both tables sit behind the staging tile.
  float4* const ab_tab = reinterpret_cast<float4*>(base_ptr + tbl_off);
  float4* film_tab = nullptr;
  const float* film_row0 = nullptr;        // FiLM table rows are read from here on (column n0)
  int film_rows = 0, film_items = 0;
  int spt = 0;
  if constexpr (GN) {
    spt = epi.tile_rows / epi.n_obj;
    const int mode = epi.film.mode;
    film_rows = mode == FILM_TIME ? min(spt, (epi.M - m0) / epi.n_obj) : mode == FILM_OBJECT ? epi.n_obj : 0;
    if (film_rows && tbl_off + (spt + film_rows) * TBL_ROW_BYTES <= STAGES * STAGE_BYTES) {
      film_tab = ab_tab + spt * (BN / 2);
      film_row0 = epi.film.base + n0;
      film_items = film_rows * (BN / 4);
    }
    // item i = (table row i / 32, columns 4 (i % 32) .. + 3): one float4 of scales and one of shifts
    auto film_src = [&](int i) {
      const int row = i / (BN / 4);
      const int64_t r = mode == FILM_TIME ? (int64_t)__ldg(epi.film.t + m0 / epi.n_obj + row) : row;
      return film_row0 + r * epi.film.row_stride + 4 * (i % (BN / 4));
    };
    float4 fs[2], fh[2];                   // the first two items of each thread, loaded before the barrier
#pragma unroll
    for (int k = 0; k < 2; ++k) {
      const int i = tid + k * TC_THREADS;
      if (i < film_items) {
        const float* src = film_src(i);
        fs[k] = __ldg(reinterpret_cast<const float4*>(src));
        fh[k] = __ldg(reinterpret_cast<const float4*>(src + epi.C));
      }
    }
    auto film_put = [&](int i, float4 s, float4 h) {
      float4* dst = film_tab + (i / (BN / 4)) * (BN / 2) + 2 * (i % (BN / 4));
      dst[0] = make_float4(s.x + 1.0f, s.y + 1.0f, h.x, h.y);
      dst[1] = make_float4(s.z + 1.0f, s.w + 1.0f, h.z, h.w);
    };

    // per-row partial (sum, sum of squares) of the two 64-channel groups of the tile: 16 values per thread,
    // then across the 4 threads of a quad that share the row
#pragma unroll
    for (int h = 0; h < 2; ++h) {
#pragma unroll
      for (int g = 0; g < 2; ++g) {
        float s = 0.f, ss = 0.f;
#pragma unroll
        for (int j = 8 * g; j < 8 * g + 8; ++j) {
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            const float v = acc[4 * j + 2 * h + e] + chan[8 * j + cq + e];
            s += v;
            ss = fmaf(v, v, ss);
          }
        }
        s += __shfl_xor_sync(0xffffffffu, s, 1);
        ss += __shfl_xor_sync(0xffffffffu, ss, 1);
        s += __shfl_xor_sync(0xffffffffu, s, 2);
        ss += __shfl_xor_sync(0xffffffffu, ss, 2);
        if ((lane & 3) == 0) part[(r0 + 8 * h) * 2 + g] = make_float2(s, ss);
      }
    }
    __syncthreads();        // partials complete; every MMA of the CTA is done, so the ring is free
#pragma unroll
    for (int k = 0; k < 2; ++k)
      if (tid + k * TC_THREADS < film_items) film_put(tid + k * TC_THREADS, fs[k], fh[k]);
    for (int i = tid + 2 * TC_THREADS; i < film_items; i += TC_THREADS) {
      const float* src = film_src(i);
      film_put(i, __ldg(reinterpret_cast<const float4*>(src)), __ldg(reinterpret_cast<const float4*>(src + epi.C)));
    }
    if (tid < spt * 2) {
      const int sc = tid >> 1, g = tid & 1;
      float s = 0.f, ss = 0.f;
      for (int r = 0; r < epi.n_obj; ++r) {
        const float2 p2 = part[(sc * epi.n_obj + r) * 2 + g];
        s += p2.x;
        ss += p2.y;
      }
      const float inv = 1.0f / float(epi.n_obj * GN_GROUP);
      const float mean = s * inv;
      const float var = fmaxf(ss * inv - mean * mean, 0.f);
      stat[tid] = make_float2(mean, rsqrtf(var + 1e-5f));
    }
    __syncthreads();
    for (int i = tid; i < spt * (BN / 2); i += TC_THREADS) {
      const int sc = i / (BN / 2), c = 2 * (i % (BN / 2));
      const float2 st = stat[sc * 2 + c / GN_GROUP];
      const float a0 = st.y * chan[BN + c], a1 = st.y * chan[BN + c + 1];
      ab_tab[i] = make_float4(a0, a1, fmaf(chan[c] - st.x, a0, chan[2 * BN + c]),
                              fmaf(chan[c + 1] - st.x, a1, chan[2 * BN + c + 1]));
    }
  }
  __syncthreads();        // GN: tables complete; plain: the other warpgroup's MMAs may still read the ring

  float* const stg32 = reinterpret_cast<float*>(base_ptr);   // [BM][STG_PITCH] fp32 (launches with a residual)
  bf16* const stg = reinterpret_cast<bf16*>(base_ptr);       // [BM][STG_PITCH] bf16
  bool live[2];
  int sc[2] = {0, 0}, fkey[2] = {0, 0};
  const float* frow[2] = {nullptr, nullptr};   // GN without a FiLM table: this token's row [scale(C) | shift(C)] at n0
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int rt = r0 + 8 * h, m = m0 + rt;
    live[h] = rt < epi.tile_rows && m < epi.M;
    if constexpr (GN) {
      sc[h] = rt / epi.n_obj;
      fkey[h] = epi.film.mode == FILM_TIME ? sc[h] : rt % epi.n_obj;
      if (!film_tab && live[h]) {
        if (epi.film.mode == FILM_TIME)
          frow[h] = epi.film.base + (int64_t)__ldg(epi.film.t + m / epi.n_obj) * epi.film.row_stride + n0;
        else if (epi.film.mode == FILM_OBJECT)
          frow[h] = epi.film.base + (int64_t)(m % epi.n_obj) * epi.film.row_stride + n0;
        else if (epi.film.mode == FILM_TOKEN)
          frow[h] = epi.film.base + (int64_t)m * epi.film.row_stride + n0;
      }
    }
  }
#pragma unroll
  for (int j = 0; j < 16; ++j) {
    const int c = 8 * j + cq, cp = 4 * j + (lane & 3);      // column, column pair
    const float2 bias = *reinterpret_cast<const float2*>(chan + c);
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      if (!live[h]) continue;
      float y0 = acc[4 * j + 2 * h], y1 = acc[4 * j + 2 * h + 1];
      if constexpr (GN) {
        const float4 ab = ab_tab[sc[h] * (BN / 2) + cp];
        y0 = fmaf(y0, ab.x, ab.z);
        y1 = fmaf(y1, ab.y, ab.w);
        if (film_tab) {
          const float4 f = film_tab[fkey[h] * (BN / 2) + cp];
          y0 = fmaf(y0, f.x, f.z);
          y1 = fmaf(y1, f.y, f.w);
        } else if (frow[h]) {
          const float2 s = __ldg(reinterpret_cast<const float2*>(frow[h] + c));
          const float2 t = __ldg(reinterpret_cast<const float2*>(frow[h] + epi.C + c));
          y0 = fmaf(y0, s.x + 1.0f, t.x);
          y1 = fmaf(y1, s.y + 1.0f, t.y);
        }
        y0 = silu_tanh(y0);
        y1 = silu_tanh(y1);
      } else {
        y0 += bias.x;
        y1 += bias.y;
        if (epi.act == ACT_GELU) { y0 = gelu_tanh(y0); y1 = gelu_tanh(y1); }
        else if (epi.act == ACT_SILU) { y0 = silu_tanh(y0); y1 = silu_tanh(y1); }
        else if (epi.act == ACT_RELU) { y0 = y0 < 0.f ? 0.f : y0; y1 = y1 < 0.f ? 0.f : y1; }
      }
      const int rt = r0 + 8 * h;
      if (stage32) *reinterpret_cast<float2*>(stg32 + rt * STG_PITCH + c) = make_float2(y0, y1);
      else *reinterpret_cast<__nv_bfloat162*>(stg + rt * STG_PITCH + c) = __floats2bfloat162_rn(y0, y1);
    }
  }

  // whole output rows: 16 threads x 16 bytes per 256-byte row, instead of the fragment layout's 16 bytes per row and
  // store instruction
  constexpr int ROW_ITERS = BM * (BN / 8) / TC_THREADS;
  if (stage32) {
    // the residual is added here, read as whole rows: every load is issued before the first store (a thread reads
    // its 16 bytes before it writes them, so accumulating in place, res == d, stays correct) and overlaps the barrier
    uint4 rv[ROW_ITERS];
#pragma unroll
    for (int it = 0; it < ROW_ITERS; ++it) {
      const int idx = tid + it * TC_THREADS, rt = idx / (BN / 8), m = m0 + rt;
      if (rt < epi.tile_rows && m < epi.M)       // plain (coherent) load, not __ldg: res may be d
        rv[it] = *reinterpret_cast<const uint4*>(epi.res + (int64_t)m * epi.ldres + n0 + (idx % (BN / 8)) * 8);
    }
    __syncthreads();
#pragma unroll
    for (int it = 0; it < ROW_ITERS; ++it) {
      const int idx = tid + it * TC_THREADS, rt = idx / (BN / 8), q = idx % (BN / 8), m = m0 + rt;
      if (rt >= epi.tile_rows || m >= epi.M) continue;
      // the two halves in an order that gives the 8 threads of a quarter warp 8 distinct 16-byte bank groups
      const float* sp = stg32 + rt * STG_PITCH + 8 * q;
      const int sw = 4 * ((q >> 2) & 1);
      const float4 u = *reinterpret_cast<const float4*>(sp + sw), w = *reinterpret_cast<const float4*>(sp + (4 - sw));
      const float4 lo = sw ? w : u, hi = sw ? u : w;
      const __nv_bfloat162* r2 = reinterpret_cast<const __nv_bfloat162*>(&rv[it]);
      const float2 ra = __bfloat1622float2(r2[0]), rb = __bfloat1622float2(r2[1]);
      const float2 rc = __bfloat1622float2(r2[2]), rd = __bfloat1622float2(r2[3]);
      uint4 o;
      __nv_bfloat162* o2 = reinterpret_cast<__nv_bfloat162*>(&o);
      o2[0] = __floats2bfloat162_rn(lo.x + ra.x, lo.y + ra.y);
      o2[1] = __floats2bfloat162_rn(lo.z + rb.x, lo.w + rb.y);
      o2[2] = __floats2bfloat162_rn(hi.x + rc.x, hi.y + rc.y);
      o2[3] = __floats2bfloat162_rn(hi.z + rd.x, hi.w + rd.y);
      *reinterpret_cast<uint4*>(epi.d + (int64_t)m * epi.ldd + n0 + 8 * q) = o;
    }
  } else {
    __syncthreads();
#pragma unroll
    for (int it = 0; it < ROW_ITERS; ++it) {
      const int idx = tid + it * TC_THREADS, rt = idx / (BN / 8), c = (idx % (BN / 8)) * 8, m = m0 + rt;
      if (rt < epi.tile_rows && m < epi.M)
        *reinterpret_cast<uint4*>(epi.d + (int64_t)m * epi.ldd + n0 + c) =
            *reinterpret_cast<const uint4*>(stg + rt * STG_PITCH + c);
    }
  }
}

// ------------------------------------------------------------------------------------------------
// host side: tensor maps + launch
// ------------------------------------------------------------------------------------------------
struct TcGemmPlan {
  CUtensorMap tm_a0, tm_a1, tm_w;
  TcEpi epi;
  bool gn;
};

typedef CUresult (*PFN_encodeTiled)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                    const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                    CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
static PFN_encodeTiled g_encode = nullptr;
static int* g_err_flag = nullptr;       // pinned host memory, device-visible
static int g_num_sms = 0;

bool tc_runtime_available(char* err, int err_len) {
  if (g_encode) return true;
  void* fn = nullptr;
  cudaDriverEntryPointQueryResult qres;
  cudaError_t e = cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &qres);
  if (e != cudaSuccess || qres != cudaDriverEntryPointSuccess || !fn) {
    if (err) snprintf(err, err_len, "cuTensorMapEncodeTiled unavailable (%s)", cudaGetErrorString(e));
    return false;
  }
  int dev = 0;
  cudaGetDevice(&dev);
  cudaDeviceProp prop;
  cudaGetDeviceProperties(&prop, dev);
  if (prop.major != 9) {
    if (err) snprintf(err, err_len, "wgmma GEMM needs sm_90 (found sm_%d%d)", prop.major, prop.minor);
    return false;
  }
  g_num_sms = prop.multiProcessorCount;
  if (!g_err_flag) {
    cudaHostAlloc((void**)&g_err_flag, sizeof(int), cudaHostAllocMapped);
    *g_err_flag = 0;
  }
  cudaFuncSetAttribute(k_gemm_wg<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM_BYTES);
  cudaFuncSetAttribute(k_gemm_wg<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM_BYTES);
  g_encode = (PFN_encodeTiled)fn;
  return true;
}

PFN_encodeTiled tc_encode_tiled() { return g_encode; }

static bool encode_2d(CUtensorMap* map, const void* base, uint64_t inner, uint64_t rows, uint64_t pitch_elems,
                      uint32_t box_rows, char* err, int err_len) {
  cuuint64_t dims[2] = {inner, rows};
  cuuint64_t strides[1] = {pitch_elems * 2};
  cuuint32_t box[2] = {uint32_t(BK), box_rows};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = g_encode(map, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<void*>(base), dims, strides, box, estr,
                        CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                        CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    if (err) snprintf(err, err_len, "cuTensorMapEncodeTiled failed (%d): inner=%llu rows=%llu pitch=%llu box=%u",
                      (int)r, (unsigned long long)inner, (unsigned long long)rows, (unsigned long long)pitch_elems,
                      box_rows);
    return false;
  }
  return true;
}

TcGemmPlan* tc_plan_create(const GemmArgs& g, int rows_capacity, char* err, int err_len) {
  if (!tc_runtime_available(err, err_len)) return nullptr;
  const int K = g.k0 + g.k1;
  if (g.k0 % BK || g.k1 % BK || g.N % BN || K == 0) {
    if (err) snprintf(err, err_len, "wgmma GEMM needs K%%64==0 and N%%128==0 (k0=%d k1=%d N=%d)", g.k0, g.k1, g.N);
    return nullptr;
  }
  if ((g.lda0 % 8) || (g.a1 && (g.lda1 % 8)) || (g.ldw % 8) || (g.ldd % 8) || (g.res && (g.ldres % 8)) ||
      ((uintptr_t)g.a0 % 16) || ((uintptr_t)g.w % 16) || ((uintptr_t)g.d % 16) || (g.a1 && ((uintptr_t)g.a1 % 16)) ||
      (g.res && ((uintptr_t)g.res % 16))) {
    if (err) snprintf(err, err_len, "wgmma GEMM needs 16-byte aligned operands and pitches");
    return nullptr;
  }
  const bool gn = g.gn != 0;
  if (gn && (g.N != 8 * GN_GROUP || g.n_obj < 1 || g.n_obj > BM || BM / g.n_obj > GN_MAX_SPT || !g.gamma || !g.beta)) {
    if (err) snprintf(err, err_len, "fused GroupNorm epilogue needs N == %d (8 groups of %d), %d <= n_obj <= %d, gamma/beta",
                      8 * GN_GROUP, GN_GROUP, BM / (GN_MAX_SPT + 1) + 1, BM);
    return nullptr;
  }
  TcGemmPlan* p = new TcGemmPlan();
  memset(p, 0, sizeof(*p));
  p->gn = gn;
  bool ok = encode_2d(&p->tm_a0, g.a0, g.k0, rows_capacity, g.lda0, BM, err, err_len);
  if (ok && g.a1) ok = encode_2d(&p->tm_a1, g.a1, g.k1, rows_capacity, g.lda1, BM, err, err_len);
  if (ok && !g.a1) p->tm_a1 = p->tm_a0;
  if (ok) ok = encode_2d(&p->tm_w, g.w, K, g.N, g.ldw, BN, err, err_len);
  if (!ok) {
    delete p;
    return nullptr;
  }
  p->epi.bias = g.bias;
  p->epi.d = (bf16*)g.d;
  p->epi.ldd = g.ldd;
  p->epi.res = (const bf16*)g.res;
  p->epi.ldres = g.ldres;
  p->epi.act = g.act;
  p->epi.M = g.M;
  p->epi.N = g.N;
  p->epi.kb0 = g.k0 / BK;
  p->epi.kb1 = g.k1 / BK;
  p->epi.tile_rows = gn ? (BM / g.n_obj) * g.n_obj : BM;
  p->epi.n_obj = g.n_obj;
  p->epi.C = g.film_C;
  p->epi.gamma = g.gamma;
  p->epi.beta = g.beta;
  p->epi.film = g.film;
  p->epi.d32 = nullptr;
  p->epi.ksplit = 1;
  return p;
}
void tc_plan_destroy(TcGemmPlan* p) { delete p; }
void tc_plan_set_film(TcGemmPlan* p, const FilmRef& f) { p->epi.film = f; }
// split-K mode: D (fp32, pitch ldd floats) += A W^T, partial sums added with atomics
void tc_plan_set_atomic_out(TcGemmPlan* p, float* d32, int ldd, int ksplit) {
  p->epi.d32 = d32;
  p->epi.ldd = ldd;
  p->epi.ksplit = ksplit < 1 ? 1 : ksplit;
}
void tc_plan_set_residual(TcGemmPlan* p, const void* res) { p->epi.res = (const bf16*)res; }
int tc_plan_tiles(const TcGemmPlan* p, int M) {
  return ((M + p->epi.tile_rows - 1) / p->epi.tile_rows) * (p->epi.N / BN);
}

int launch_gemm_tc(const TcGemmPlan* p, int M, cudaStream_t s) {
  TcEpi epi = p->epi;
  epi.M = M;
  const int units = tc_plan_tiles(p, M) * epi.ksplit;
  if (units == 0) return 0;
  int* flag_dev = nullptr;
  cudaHostGetDevicePointer((void**)&flag_dev, g_err_flag, 0);
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3(units);
  cfg.blockDim = dim3(TC_THREADS);
  cfg.dynamicSmemBytes = SMEM_BYTES;
  cfg.stream = s;
  cudaLaunchAttribute attr[1];
  if (pdl_enabled(0, M)) {      // may start while the previous kernel in the stream drains
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = attr;
    cfg.numAttrs = 1;
  }
  if (p->gn) return (int)cudaLaunchKernelEx(&cfg, k_gemm_wg<true>, p->tm_a0, p->tm_a1, p->tm_w, epi, flag_dev);
  return (int)cudaLaunchKernelEx(&cfg, k_gemm_wg<false>, p->tm_a0, p->tm_a1, p->tm_w, epi, flag_dev);
}

int tc_error_flag() { return g_err_flag ? *g_err_flag : 0; }
// shared with the fused LayerNorm / attention kernels (gemm_ln.cu, gemm_attn.cu)
bool tc_encode_2d(CUtensorMap* map, const void* base, uint64_t inner, uint64_t rows, uint64_t pitch_elems,
                  uint32_t box_rows, char* err, int err_len) {
  return encode_2d(map, base, inner, rows, pitch_elems, box_rows, err, err_len);
}
int* tc_error_flag_dev() {
  int* fd = nullptr;
  cudaHostGetDevicePointer((void**)&fd, g_err_flag, 0);
  return fd;
}
int tc_num_sms() { return g_num_sms; }

}  // namespace ds
