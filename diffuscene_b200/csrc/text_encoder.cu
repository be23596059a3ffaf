// Frozen BERT text encoder: the forward pass of Hugging Face `BertModel` up to `last_hidden_state` (no pooler, no
// backward pass), for the text-conditioned networks (the reference runs `bert-base-cased` on every description,
// scene_synthesis/networks/diffusion_scene_layout_ddpm.py:217-218, 285-287).  A handle of its own (ds_text_enc_*).
//
// Activations are token rows [B * L, width] like the rest of the library.  Per layer (post-LN):
//   qkv   = x [Wq | Wk | Wv]^T + [bq | bk | bv]            one GEMM, N = 3 hidden
//   ctx   = softmax(q k^T / 8, keys >= length[b] masked) v  k_te_attn_* (one CTA per sequence, head, 64 queries)
//   y     = ctx Wo^T + bo + x                              GEMM with residual
//   h1    = LayerNorm(y)                                   k_te_layernorm (weight, bias, eps 1e-12)
//   inter = GELU(h1 W1^T + b1)                             GEMM with activation
//   y     = inter W2^T + b2 + h1                           GEMM with residual
//   x     = LayerNorm(y)                                   (fp32 into the caller's output after the last layer)
// The GEMMs are k_gemm_wg through TcGemmPlans in bf16 (its epilogue's GELU is the tanh form) and the SIMT GEMM with
// the erf GELU in the fp32 parity mode.  Padded query positions are computed like any other query (HF returns them and
// the text projection consumes all L positions); padded keys get exactly zero weight, and key tiles past length[b]
// are skipped.  LayerNorm statistics and the softmax are fp32 in both modes.
#include "engine_internal.h"

namespace ds {

// LayerNorm of one row of H values produced by `val(c)`, one warp per row: mean, then the centred variance (both
// passes recompute the values, which come from L1), y = (v - mean) / sqrt(var + eps) * g + b.  `valid == false`
// writes NaN.
template <typename TO, typename F>
__device__ __forceinline__ void te_ln_row(F val, const float* __restrict__ g, const float* __restrict__ b,
                                          TO* __restrict__ out, int H, float eps, bool valid) {
  const int lane = threadIdx.x & 31;
  float s = 0.f;
  for (int c = lane; c < H; c += 32) s += val(c);
  const float mean = warp_sum(s) / float(H);
  float ss = 0.f;
  for (int c = lane; c < H; c += 32) {
    const float d = val(c) - mean;
    ss = fmaf(d, d, ss);
  }
  const float rstd = 1.0f / sqrtf(warp_sum(ss) / float(H) + eps);
  for (int c = lane; c < H; c += 32) stf(out + c, valid ? (val(c) - mean) * rstd * g[c] + b[c] : NAN);
}

// embeddings: LayerNorm((word[id] + token_type[0]) + position[r % L]), HF's order of the two additions.  An id outside
// [0, vocab) reads nothing and gives a NaN row.
template <typename TO>
__global__ void __launch_bounds__(256) k_te_embed_ln(const int* __restrict__ ids, const float* __restrict__ word,
                                                     const float* __restrict__ pos, const float* __restrict__ type0,
                                                     const float* __restrict__ g, const float* __restrict__ b,
                                                     TO* __restrict__ out, int M, int L, int H, int vocab, float eps) {
  const int64_t r = (int64_t)blockIdx.x * 8 + (threadIdx.x >> 5);
  if (r >= M) return;
  const int id = ids[r];
  const bool ok = id >= 0 && id < vocab;
  const float* wr = word + (int64_t)(ok ? id : 0) * H;
  const float* pr = pos + (int64_t)(r % L) * H;
  te_ln_row([&](int c) { return (wr[c] + type0[c]) + pr[c]; }, g, b, out + r * H, H, eps, ok);
}

template <typename TI, typename TO>
__global__ void __launch_bounds__(256) k_te_layernorm(const TI* __restrict__ in, const float* __restrict__ g,
                                                      const float* __restrict__ b, TO* __restrict__ out, int M, int H,
                                                      float eps) {
  const int64_t r = (int64_t)blockIdx.x * 8 + (threadIdx.x >> 5);
  if (r >= M) return;
  const TI* x = in + r * H;
  te_ln_row([&](int c) { return ldf(x + c); }, g, b, out + r * H, H, eps, true);
}

template <typename TO>
void launch_te_embed_ln(const int* ids, const float* word, const float* pos, const float* type0, const float* g,
                        const float* b, TO* out, int M, int L, int H, int vocab, float eps, cudaStream_t s) {
  k_te_embed_ln<TO><<<ceil_div(M, 8), 256, 0, s>>>(ids, word, pos, type0, g, b, out, M, L, H, vocab, eps);
}
template <typename TI, typename TO>
void launch_te_layernorm(const TI* in, const float* g, const float* b, TO* out, int M, int H, float eps,
                         cudaStream_t s) {
  k_te_layernorm<TI, TO><<<ceil_div(M, 8), 256, 0, s>>>(in, g, b, out, M, H, eps);
}

// ---- masked self-attention, head dim 64 -------------------------------------------------------------------------
// qkv [B * L, 3 H] (q | k | v, head h in columns 64 h .. 64 h + 63 of each third) -> out [B * L, H].  One CTA per
// (sequence, 64-query block) in blockIdx.x and head in blockIdx.y; keys in tiles of the sequence's first length[b]
// rows only (length clamped to [1, L]), online softmax in fp32.

// fp32: one thread per query, q and the output accumulator in registers, keys in chunks of 16 per softmax rescale
constexpr int TE_F32_KT = 32;
__global__ void __launch_bounds__(64) k_te_attn_f32(const float* __restrict__ qkv, const int* __restrict__ lengths,
                                                    float* __restrict__ out, int L, int H, int qblocks) {
  __shared__ __align__(16) float Ks[TE_F32_KT][64];
  __shared__ __align__(16) float Vs[TE_F32_KT][64];
  const int b = blockIdx.x / qblocks, qb = blockIdx.x % qblocks, head = blockIdx.y;
  const int len = min(max(lengths[b], 1), L);
  const int64_t ld = 3 * (int64_t)H;
  const float* base = qkv + (int64_t)b * L * ld + head * 64;
  const int qi = qb * 64 + threadIdx.x;
  float q[64], acc[64];
#pragma unroll
  for (int d = 0; d < 64; ++d) {
    q[d] = qi < L ? base[qi * ld + d] * 0.125f : 0.f;      // the 1/8 scale is a power of two: exact
    acc[d] = 0.f;
  }
  float m = -INFINITY, l = 0.f;
  for (int k0 = 0; k0 < len; k0 += TE_F32_KT) {
    __syncthreads();
    for (int i = threadIdx.x; i < TE_F32_KT * 64; i += 64) {
      const int r = i >> 6, d = i & 63, key = k0 + r;
      Ks[r][d] = key < len ? base[key * ld + H + d] : 0.f;
      Vs[r][d] = key < len ? base[key * ld + 2 * H + d] : 0.f;
    }
    __syncthreads();
    const int nk = min(TE_F32_KT, len - k0);
    for (int c = 0; c < nk; c += 16) {
      float s[16];
      float mx = m;
#pragma unroll
      for (int j = 0; j < 16; ++j) {
        float v = -INFINITY;
        if (c + j < nk) {
          v = 0.f;
#pragma unroll
          for (int d = 0; d < 64; d += 4) {
            const float4 k4 = *reinterpret_cast<const float4*>(&Ks[c + j][d]);
            v = fmaf(q[d], k4.x, v);
            v = fmaf(q[d + 1], k4.y, v);
            v = fmaf(q[d + 2], k4.z, v);
            v = fmaf(q[d + 3], k4.w, v);
          }
        }
        s[j] = v;
        mx = fmaxf(mx, v);
      }
      const float corr = expf(m - mx);      // 0 on the first chunk (m = -inf); mx is finite: key c is valid
      l *= corr;
#pragma unroll
      for (int d = 0; d < 64; ++d) acc[d] *= corr;
#pragma unroll
      for (int j = 0; j < 16; ++j) {
        if (c + j < nk) {
          const float p = expf(s[j] - mx);
          l += p;
#pragma unroll
          for (int d = 0; d < 64; d += 4) {
            const float4 v4 = *reinterpret_cast<const float4*>(&Vs[c + j][d]);
            acc[d] = fmaf(p, v4.x, acc[d]);
            acc[d + 1] = fmaf(p, v4.y, acc[d + 1]);
            acc[d + 2] = fmaf(p, v4.z, acc[d + 2]);
            acc[d + 3] = fmaf(p, v4.w, acc[d + 3]);
          }
        }
      }
      m = mx;
    }
  }
  if (qi >= L) return;
  float* o = out + ((int64_t)b * L + qi) * H + head * 64;
  const float inv = 1.0f / l;
#pragma unroll
  for (int d = 0; d < 64; d += 4)
    *reinterpret_cast<float4*>(o + d) = make_float4(acc[d] * inv, acc[d + 1] * inv, acc[d + 2] * inv, acc[d + 3] * inv);
}

// bf16: 4 warps, 16 queries each; S = Q K^T and O += P V on mma.sync m16n8k16 (bf16 in, fp32 accumulate), P rounded
// to bf16 for the second product.  Fragment layouts (PTX ISA, mma.m16n8k16 .bf16), g = lane / 4, t = lane % 4:
//   A 16x16 row-major: {a0,a1} (g, 2t..2t+1), {a2,a3} (g+8, 2t..), {a4,a5} (g, 2t+8..), {a6,a7} (g+8, 2t+8..)
//   B 16x8:            {b0,b1} (k = 2t..2t+1, n = g), {b2,b3} (k = 2t+8.., n = g)
//   C 16x8 fp32:       c0,c1 (g, 2t..2t+1), c2,c3 (g+8, 2t..2t+1)
// so the C fragments of two adjacent 8-key tiles of S are the A fragment of P for one 16-key step.
constexpr int TE_PITCH = 72;      // bf16 per shared-memory row: 144 bytes, the 8 rows of a fragment load on distinct banks
__device__ __forceinline__ void te_mma(float (&c)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
  asm volatile(
      "mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0, %1, %2, %3}, {%4, %5, %6, %7}, {%8, %9}, "
      "{%0, %1, %2, %3};"
      : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}
__device__ __forceinline__ uint32_t te_ld32(const bf16* p) { return *reinterpret_cast<const uint32_t*>(p); }
__device__ __forceinline__ uint32_t te_pack(float lo, float hi) {
  const __nv_bfloat162 v = __floats2bfloat162_rn(lo, hi);
  return *reinterpret_cast<const uint32_t*>(&v);
}
__device__ __forceinline__ uint32_t te_pack(bf16 lo, bf16 hi) {
  return (uint32_t)__bfloat16_as_ushort(lo) | ((uint32_t)__bfloat16_as_ushort(hi) << 16);
}

// rows [row0, row0 + 64) of one 64-column head slice into shared memory, zero past `rows`
__device__ __forceinline__ void te_load_tile(bf16* dst, const bf16* src, int64_t ld, int row0, int rows) {
  for (int i = threadIdx.x; i < 64 * 8; i += 128) {
    const int r = i >> 3, ch = i & 7;
    uint4 v = make_uint4(0, 0, 0, 0);
    if (row0 + r < rows) v = *reinterpret_cast<const uint4*>(src + (int64_t)(row0 + r) * ld + ch * 8);
    *reinterpret_cast<uint4*>(dst + r * TE_PITCH + ch * 8) = v;
  }
}

__global__ void __launch_bounds__(128) k_te_attn_bf16(const bf16* __restrict__ qkv, const int* __restrict__ lengths,
                                                      bf16* __restrict__ out, int L, int H, int qblocks) {
  __shared__ __align__(16) bf16 Qs[64 * TE_PITCH];
  __shared__ __align__(16) bf16 Ks[64 * TE_PITCH];
  __shared__ __align__(16) bf16 Vs[64 * TE_PITCH];
  const int b = blockIdx.x / qblocks, qb = blockIdx.x % qblocks, head = blockIdx.y;
  const int len = min(max(lengths[b], 1), L);
  const int64_t ld = 3 * (int64_t)H;
  const bf16* base = qkv + (int64_t)b * L * ld + head * 64;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, g = lane >> 2, t = lane & 3;
  const int qr = warp * 16;

  te_load_tile(Qs, base + (int64_t)qb * 64 * ld, ld, 0, L - qb * 64);
  __syncthreads();
  uint32_t qa[4][4];
#pragma unroll
  for (int kk = 0; kk < 4; ++kk) {
    const bf16* p = Qs + (qr + g) * TE_PITCH + 16 * kk + 2 * t;
    qa[kk][0] = te_ld32(p);
    qa[kk][1] = te_ld32(p + 8 * TE_PITCH);
    qa[kk][2] = te_ld32(p + 8);
    qa[kk][3] = te_ld32(p + 8 * TE_PITCH + 8);
  }
  float o[8][4];
#pragma unroll
  for (int j = 0; j < 8; ++j) o[j][0] = o[j][1] = o[j][2] = o[j][3] = 0.f;
  float m[2] = {-INFINITY, -INFINITY}, l[2] = {0.f, 0.f};
  const float sl2 = 0.125f * 1.4426950408889634f;      // 1/8 and log2(e): softmax through exp2

  for (int k0 = 0; k0 < len; k0 += 64) {
    __syncthreads();      // the previous tile has been read by every warp
    te_load_tile(Ks, base + H, ld, k0, len);
    te_load_tile(Vs, base + 2 * H, ld, k0, len);
    __syncthreads();
    float s[8][4];
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      s[j][0] = s[j][1] = s[j][2] = s[j][3] = 0.f;
#pragma unroll
      for (int kk = 0; kk < 4; ++kk) {
        const bf16* p = Ks + (8 * j + g) * TE_PITCH + 16 * kk + 2 * t;
        te_mma(s[j], qa[kk], te_ld32(p), te_ld32(p + 8));
      }
    }
    float mx[2] = {m[0], m[1]};
#pragma unroll
    for (int j = 0; j < 8; ++j)
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const float v = k0 + 8 * j + 2 * t + (e & 1) < len ? s[j][e] * sl2 : -INFINITY;
        s[j][e] = v;
        mx[e >> 1] = fmaxf(mx[e >> 1], v);
      }
    float corr[2];
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      mx[h] = fmaxf(mx[h], __shfl_xor_sync(0xffffffffu, mx[h], 1));
      mx[h] = fmaxf(mx[h], __shfl_xor_sync(0xffffffffu, mx[h], 2));
      corr[h] = exp2f(m[h] - mx[h]);      // 0 on the first tile; key 0 is valid, so mx is finite
      m[h] = mx[h];
      l[h] *= corr[h];
    }
#pragma unroll
    for (int j = 0; j < 8; ++j)
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const float p = exp2f(s[j][e] - m[e >> 1]);
        s[j][e] = p;
        l[e >> 1] += p;
        o[j][e] *= corr[e >> 1];
      }
#pragma unroll
    for (int kk = 0; kk < 4; ++kk) {
      const uint32_t pa[4] = {te_pack(s[2 * kk][0], s[2 * kk][1]), te_pack(s[2 * kk][2], s[2 * kk][3]),
                              te_pack(s[2 * kk + 1][0], s[2 * kk + 1][1]), te_pack(s[2 * kk + 1][2], s[2 * kk + 1][3])};
      const bf16* v0 = Vs + (16 * kk + 2 * t) * TE_PITCH + g;
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const bf16* v = v0 + 8 * j;
        te_mma(o[j], pa, te_pack(v[0], v[TE_PITCH]), te_pack(v[8 * TE_PITCH], v[9 * TE_PITCH]));
      }
    }
  }
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    l[h] += __shfl_xor_sync(0xffffffffu, l[h], 1);
    l[h] += __shfl_xor_sync(0xffffffffu, l[h], 2);
    const int qi = qb * 64 + qr + g + 8 * h;
    if (qi >= L) continue;
    const float inv = 1.0f / l[h];
    bf16* op = out + ((int64_t)b * L + qi) * H + head * 64 + 2 * t;
#pragma unroll
    for (int j = 0; j < 8; ++j)
      *reinterpret_cast<__nv_bfloat162*>(op + 8 * j) = __floats2bfloat162_rn(o[j][2 * h] * inv, o[j][2 * h + 1] * inv);
  }
}

template <typename T>
void launch_te_attention(const T* qkv, const int* lengths, T* out, int B, int L, int H, cudaStream_t s) {
  const int qblocks = (L + 63) / 64;
  const dim3 grid((unsigned)B * qblocks, H / 64);
  if constexpr (sizeof(T) == 2) k_te_attn_bf16<<<grid, 128, 0, s>>>(qkv, lengths, out, L, H, qblocks);
  else k_te_attn_f32<<<grid, 64, 0, s>>>(qkv, lengths, out, L, H, qblocks);
}

template <typename T>
__global__ void k_te_convert(const float* __restrict__ in, T* __restrict__ out, int64_t n) {
  const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (i < n) stf(out + i, in[i]);
}
template <typename T>
void launch_te_convert(const float* in, T* out, int64_t n, cudaStream_t s) {
  if (n > 0) k_te_convert<T><<<ceil_div(n, 256), 256, 0, s>>>(in, out, n);
}
__global__ void k_widen_bf16(const bf16* __restrict__ in, float* __restrict__ out, int64_t n) {
  const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (i < n) out[i] = __bfloat162float(in[i]);
}
void launch_widen_bf16(const bf16* in, float* out, int64_t n, cudaStream_t s) {
  if (n > 0) k_widen_bf16<<<ceil_div(n, 256), 256, 0, s>>>(in, out, n);
}

#define INST_TE(T)                                                                                                   \
  template void launch_te_embed_ln<T>(const int*, const float*, const float*, const float*, const float*,            \
                                      const float*, T*, int, int, int, int, float, cudaStream_t);                    \
  template void launch_te_attention<T>(const T*, const int*, T*, int, int, int, cudaStream_t);                       \
  template void launch_te_convert<T>(const float*, T*, int64_t, cudaStream_t);
INST_TE(float)
INST_TE(bf16)
template void launch_te_layernorm<float, float>(const float*, const float*, const float*, float*, int, int, float, cudaStream_t);
template void launch_te_layernorm<bf16, bf16>(const bf16*, const float*, const float*, bf16*, int, int, float, cudaStream_t);
template void launch_te_layernorm<bf16, float>(const bf16*, const float*, const float*, float*, int, int, float, cudaStream_t);
}  // namespace ds

// ------------------------------------------------------------------------------------------------
// handle and C ABI
// ------------------------------------------------------------------------------------------------
namespace {
constexpr float TE_LN_EPS = 1e-12f;                 // BertConfig.layer_norm_eps
constexpr int64_t TE_MAX_TOKENS = 65535LL * 64;     // the SIMT GEMM's gridDim.y (64 rows per CTA row)
constexpr int TE_PER_LAYER = 16;                    // state-dict tensors per encoder layer
enum { G_QKV = 0, G_OUT, G_INTER, G_FFN_OUT };
constexpr int TE_TAPS = DS_TE_OUT + 1;
}  // namespace

struct ds_text_enc {
  ds_text_enc_config cfg;
  bool bf16 = false;
  size_t esz = 4;
  WeightTable w;
  bool weights_set = false;
  float* params = nullptr;        // copy of the flat parameters: embeddings, biases and LayerNorm read from here
  void* wmat = nullptr;           // per layer, storage type: [Wq | Wk | Wv] [3H, H], Wo [H, H], W1 [I, H], W2 [H, I]
  float* bqkv = nullptr;          // per layer [bq | bk | bv]
  std::vector<size_t> w_off;      // element offset of each layer's four matrices in wmat, 4 per layer
  void *x = nullptr, *qkv = nullptr, *ctx = nullptr, *y = nullptr, *h1 = nullptr, *inter = nullptr;
  std::vector<GemmArgs> gemm;     // 4 per layer, M = capacity
  std::vector<TcGemmPlan*> tc;    // bf16: one plan per GEMM
  // per-layer tap (ds_text_enc_set_tap): the tapped layer's arrays, storage type, one region per DS_TE_* kind
  int tap_layer = -1;             // -1: off
  void* tap = nullptr;            // allocated by the first ds_text_enc_set_tap, `capacity` tokens
  int64_t tap_width[TE_TAPS] = {}, tap_off[TE_TAPS] = {};
  int tapped_layer = -1, tapped_M = 0;      // layer and tokens of the last forward that ran with a tap set
};

namespace {
template <typename T> T* P(void* v, size_t off = 0) { return (T*)v + off; }

void te_release(ds_text_enc* h) {
  for (auto* p : h->tc) if (p) tc_plan_destroy(p);
  h->tc.clear();
  void* bufs[] = {h->params, h->wmat, h->bqkv, h->x, h->qkv, h->ctx, h->y, h->h1, h->inter, h->tap};
  for (void* b : bufs) cudaFree(b);
  delete h;
}

// flat offset of tensor `k` (0 .. 15, state-dict order) of layer `l`
const float* layer_param(const ds_text_enc* h, const float* base, int l, int k) { return base + h->w.off[5 + TE_PER_LAYER * l + k]; }

// copy `src` [M, width] of the tapped layer into the tap store (storage type)
int te_tap(ds_text_enc* h, int l, int kind, const void* src, int M, cudaStream_t s) {
  if (l != h->tap_layer) return 0;
  const size_t n = (size_t)M * h->tap_width[kind] * h->esz;
  const cudaError_t e = cudaMemcpyAsync((char*)h->tap + (size_t)h->tap_off[kind] * h->esz, src, n,
                                        cudaMemcpyDeviceToDevice, s);
  return e == cudaSuccess ? 0 : fail(DS_ERR_CUDA, "text encoder: tap copy failed: %s", cudaGetErrorString(e));
}

template <typename T>
int te_forward(ds_text_enc* h, const int* ids, const int* lengths, int B, int L, float* out, cudaStream_t s) {
  const ds_text_enc_config& c = h->cfg;
  const int H = c.hidden, M = B * L;
  const float* pr = h->params;
  h->tapped_layer = -1;
  launch_te_embed_ln<T>(ids, pr + h->w.off[0], pr + h->w.off[1], pr + h->w.off[2], pr + h->w.off[3], pr + h->w.off[4],
                        P<T>(h->x), M, L, H, c.vocab, TE_LN_EPS, s);
  for (int l = 0; l < c.layers; ++l) {
    if (const int rc = te_tap(h, l, DS_TE_X, h->x, M, s)) return rc;
    for (int k = 0; k < 4; ++k) {
      const int gi = 4 * l + k;
      if (h->bf16) {
        const int e = launch_gemm_tc(h->tc[gi], M, s);
        if (e) return fail(DS_ERR_CUDA, "text encoder: GEMM %d of layer %d failed: %s", k, l, cudaGetErrorString((cudaError_t)e));
      } else {
        GemmArgs g = h->gemm[gi];
        g.M = M;
        launch_gemm_simt<float>(g, true, s);
      }
      int rc = 0;
      if (k == G_QKV) {
        rc = te_tap(h, l, DS_TE_QKV, h->qkv, M, s);
        launch_te_attention<T>(P<T>(h->qkv), lengths, P<T>(h->ctx), B, L, H, s);
        if (!rc) rc = te_tap(h, l, DS_TE_CTX, h->ctx, M, s);
      } else if (k == G_OUT) {
        rc = te_tap(h, l, DS_TE_Y1, h->y, M, s);
        launch_te_layernorm<T, T>(P<T>(h->y), layer_param(h, pr, l, 8), layer_param(h, pr, l, 9), P<T>(h->h1), M, H,
                                  TE_LN_EPS, s);
        if (!rc) rc = te_tap(h, l, DS_TE_H1, h->h1, M, s);
      } else if (k == G_INTER) {
        rc = te_tap(h, l, DS_TE_INTER, h->inter, M, s);
      } else {
        rc = te_tap(h, l, DS_TE_Y2, h->y, M, s);
        const float* g = layer_param(h, pr, l, 14);
        const float* b = layer_param(h, pr, l, 15);
        if (l + 1 < c.layers) {
          launch_te_layernorm<T, T>(P<T>(h->y), g, b, P<T>(h->x), M, H, TE_LN_EPS, s);
          if (!rc) rc = te_tap(h, l, DS_TE_OUT, h->x, M, s);
        } else {
          launch_te_layernorm<T, float>(P<T>(h->y), g, b, out, M, H, TE_LN_EPS, s);
        }
      }
      if (rc) return rc;
    }
  }
  h->tapped_layer = h->tap_layer;
  h->tapped_M = h->tap_layer >= 0 ? M : 0;
  return 0;
}

template <typename T>
void te_pack(ds_text_enc* h, cudaStream_t s) {
  const int H = h->cfg.hidden, I = h->cfg.intermediate;
  const float* pr = h->params;
  for (int l = 0; l < h->cfg.layers; ++l) {
    T* w = P<T>(h->wmat, h->w_off[4 * l]);
    for (int k = 0; k < 3; ++k) {      // query, key, value: rows k H .. (k + 1) H of the fused matrix
      launch_te_convert<T>(layer_param(h, pr, l, 2 * k), w + (size_t)k * H * H, (int64_t)H * H, s);
      cudaMemcpyAsync(h->bqkv + (size_t)l * 3 * H + (size_t)k * H, layer_param(h, pr, l, 2 * k + 1), H * 4,
                      cudaMemcpyDeviceToDevice, s);
    }
    launch_te_convert<T>(layer_param(h, pr, l, 6), P<T>(h->wmat, h->w_off[4 * l + 1]), (int64_t)H * H, s);
    launch_te_convert<T>(layer_param(h, pr, l, 10), P<T>(h->wmat, h->w_off[4 * l + 2]), (int64_t)I * H, s);
    launch_te_convert<T>(layer_param(h, pr, l, 12), P<T>(h->wmat, h->w_off[4 * l + 3]), (int64_t)H * I, s);
  }
}
}  // namespace

extern "C" int ds_text_enc_create(const ds_text_enc_config* cfg, ds_text_enc** out) {
  if (!cfg || !out) return fail(DS_ERR_INVALID, "null argument");
  *out = nullptr;
  if (cfg->precision != DS_PREC_FP32 && cfg->precision != DS_PREC_BF16)
    return fail(DS_ERR_INVALID, "text encoder: precision %d unknown", cfg->precision);
  if (cfg->layers < 1 || cfg->heads < 1 || cfg->hidden != 64 * cfg->heads || cfg->hidden % 128 || cfg->hidden > 16384)
    return fail(DS_ERR_INVALID, "text encoder: needs layers >= 1 and hidden = 64 x heads, a multiple of 128 up to 16384 "
                "(layers %d, hidden %d, heads %d)", cfg->layers, cfg->hidden, cfg->heads);
  if (cfg->intermediate < 128 || cfg->intermediate % 128 || cfg->intermediate > 65536)
    return fail(DS_ERR_INVALID, "text encoder: intermediate %d is not a multiple of 128 in [128, 65536]", cfg->intermediate);
  if (cfg->vocab < 1 || cfg->max_positions < 1 || cfg->type_vocab < 1)
    return fail(DS_ERR_INVALID, "text encoder: vocab %d, max_positions %d and type_vocab %d must be positive", cfg->vocab,
                cfg->max_positions, cfg->type_vocab);
  if (cfg->capacity < 1 || cfg->capacity > TE_MAX_TOKENS)
    return fail(DS_ERR_INVALID, "text encoder: token capacity %d outside [1, %lld]", cfg->capacity, (long long)TE_MAX_TOKENS);
  if (const int rc = open_device(cfg->device)) return rc;
  if (cfg->precision == DS_PREC_BF16) {
    char err[256] = "";
    if (!tc_runtime_available(err, sizeof err)) return fail(DS_ERR_CUDA, "%s", err);
  }
  ds_text_enc* h = new ds_text_enc();
  h->cfg = *cfg;
  h->bf16 = cfg->precision == DS_PREC_BF16;
  h->esz = h->bf16 ? 2 : 4;
  const int64_t H = cfg->hidden, I = cfg->intermediate;
  h->w.add("embeddings.word_embeddings.weight", (int64_t)cfg->vocab * H);
  h->w.add("embeddings.position_embeddings.weight", (int64_t)cfg->max_positions * H);
  h->w.add("embeddings.token_type_embeddings.weight", (int64_t)cfg->type_vocab * H);
  h->w.add("embeddings.LayerNorm.weight", H);
  h->w.add("embeddings.LayerNorm.bias", H);
  size_t wtotal = 0;
  for (int l = 0; l < cfg->layers; ++l) {
    const std::string pre = "encoder.layer." + std::to_string(l) + ".";
    for (const char* n : {"query", "key", "value"}) {
      h->w.add(pre + "attention.self." + n + ".weight", H * H);
      h->w.add(pre + "attention.self." + n + ".bias", H);
    }
    h->w.add(pre + "attention.output.dense.weight", H * H);
    h->w.add(pre + "attention.output.dense.bias", H);
    h->w.add(pre + "attention.output.LayerNorm.weight", H);
    h->w.add(pre + "attention.output.LayerNorm.bias", H);
    h->w.add(pre + "intermediate.dense.weight", I * H);
    h->w.add(pre + "intermediate.dense.bias", I);
    h->w.add(pre + "output.dense.weight", H * I);
    h->w.add(pre + "output.dense.bias", H);
    h->w.add(pre + "output.LayerNorm.weight", H);
    h->w.add(pre + "output.LayerNorm.bias", H);
    for (int64_t n : {3 * H * H, H * H, I * H, H * I}) {
      h->w_off.push_back(wtotal);
      wtotal += (size_t)n;
    }
  }
  const size_t cap = (size_t)cfg->capacity, e = h->esz;
  cudaError_t err = cudaMalloc(&h->params, (size_t)h->w.total * 4);
  if (err == cudaSuccess) err = cudaMalloc(&h->wmat, wtotal * e);
  if (err == cudaSuccess) err = cudaMalloc(&h->bqkv, (size_t)cfg->layers * 3 * H * 4);
  if (err == cudaSuccess) err = cudaMalloc(&h->x, cap * H * e);
  if (err == cudaSuccess) err = cudaMalloc(&h->qkv, cap * 3 * H * e);
  if (err == cudaSuccess) err = cudaMalloc(&h->ctx, cap * H * e);
  if (err == cudaSuccess) err = cudaMalloc(&h->y, cap * H * e);
  if (err == cudaSuccess) err = cudaMalloc(&h->h1, cap * H * e);
  if (err == cudaSuccess) err = cudaMalloc(&h->inter, cap * I * e);
  if (err != cudaSuccess) {
    cudaGetLastError();
    te_release(h);
    return fail(DS_ERR_CUDA, "text encoder: allocation for %d tokens failed: %s", cfg->capacity, cudaGetErrorString(err));
  }
  // the four GEMMs of every layer: A, W, bias, output, residual, activation
  for (int l = 0; l < cfg->layers; ++l) {
    const float* pr = h->params;
    struct { void* a; int k; int wi; const float* bias; void* d; int n; void* res; int act; } spec[4] = {
        {h->x, (int)H, 4 * l + 0, h->bqkv + (size_t)l * 3 * H, h->qkv, (int)(3 * H), nullptr, ACT_NONE},
        {h->ctx, (int)H, 4 * l + 1, layer_param(h, pr, l, 7), h->y, (int)H, h->x, ACT_NONE},
        {h->h1, (int)H, 4 * l + 2, layer_param(h, pr, l, 11), h->inter, (int)I, nullptr, ACT_GELU},
        {h->inter, (int)I, 4 * l + 3, layer_param(h, pr, l, 13), h->y, (int)H, h->h1, ACT_NONE}};
    for (const auto& sp : spec) {
      GemmArgs g;
      memset(&g, 0, sizeof g);
      g.a0 = sp.a; g.lda0 = sp.k; g.k0 = sp.k;
      g.w = (const char*)h->wmat + h->w_off[sp.wi] * e; g.ldw = sp.k;
      g.bias = sp.bias;
      g.d = sp.d; g.ldd = sp.n;
      g.res = sp.res; g.ldres = sp.n;
      g.M = cfg->capacity; g.N = sp.n; g.act = sp.act;
      h->gemm.push_back(g);
      if (h->bf16) {
        char msg[256] = "";
        TcGemmPlan* p = tc_plan_create(g, cfg->capacity, msg, sizeof msg);
        if (!p) {
          te_release(h);
          return fail(DS_ERR_CUDA, "text encoder: tensor-core GEMM plan failed: %s", msg);
        }
        h->tc.push_back(p);
      }
    }
  }
  *out = h;
  return 0;
}

extern "C" int ds_text_enc_destroy(ds_text_enc* h) {
  if (!h) return 0;
  cudaSetDevice(h->cfg.device);
  te_release(h);
  return 0;
}

extern "C" int ds_text_enc_expected_weight_count(ds_text_enc* h) {
  if (!h) return fail(DS_ERR_INVALID, "null handle");
  return h->w.count();
}

extern "C" int ds_text_enc_expected_weight(ds_text_enc* h, int index, const char** name, int64_t* numel) {
  if (!h) return fail(DS_ERR_INVALID, "null argument");
  return h->w.get(index, name, numel);
}

extern "C" int ds_text_enc_set_weights(ds_text_enc* h, const float* flat_params_dev, void* stream) {
  if (!h || !flat_params_dev) return fail(DS_ERR_INVALID, "null argument");
  CK(cudaSetDevice(h->cfg.device));
  cudaStream_t s = (cudaStream_t)stream;
  CK(cudaMemcpyAsync(h->params, flat_params_dev, (size_t)h->w.total * 4, cudaMemcpyDeviceToDevice, s));
  if (h->bf16) te_pack<bf16>(h, s);
  else te_pack<float>(h, s);
  CK(cudaGetLastError());
  h->weights_set = true;
  return 0;
}

extern "C" int ds_text_enc_forward(ds_text_enc* h, const int32_t* ids_dev, const int32_t* lengths_dev, int32_t batch,
                                   int32_t seq_len, float* out_dev, void* stream) {
  if (!h || !ids_dev || !lengths_dev || !out_dev) return fail(DS_ERR_INVALID, "null argument");
  if (!h->weights_set) return fail(DS_ERR_STATE, "text encoder: ds_text_enc_set_weights has not been called");
  if (batch < 1 || seq_len < 1) return fail(DS_ERR_INVALID, "text encoder: batch %d and length %d must be positive", batch, seq_len);
  if (seq_len > h->cfg.max_positions)
    return fail(DS_ERR_INVALID, "text encoder: length %d exceeds max_positions %d", seq_len, h->cfg.max_positions);
  if ((int64_t)batch * seq_len > h->cfg.capacity)
    return fail(DS_ERR_INVALID, "text encoder: %lld tokens exceed the handle's capacity %d", (long long)batch * seq_len,
                h->cfg.capacity);
  CK(cudaSetDevice(h->cfg.device));
  cudaStream_t s = (cudaStream_t)stream;
  const int rc = h->bf16 ? te_forward<bf16>(h, ids_dev, lengths_dev, batch, seq_len, out_dev, s)
                         : te_forward<float>(h, ids_dev, lengths_dev, batch, seq_len, out_dev, s);
  if (rc) return rc;
  CK(cudaGetLastError());
  return 0;
}

extern "C" int ds_text_enc_set_tap(ds_text_enc* h, int32_t layer) {
  if (!h) return fail(DS_ERR_INVALID, "null handle");
  if (layer < -1 || layer >= h->cfg.layers)
    return fail(DS_ERR_INVALID, "text encoder: tap layer %d outside [-1, %d)", layer, h->cfg.layers);
  if (layer >= 0 && !h->tap) {
    const int64_t H = h->cfg.hidden, w[TE_TAPS] = {H, 3 * H, H, H, H, h->cfg.intermediate, H, H};
    int64_t total = 0;
    for (int k = 0; k < TE_TAPS; ++k) {
      h->tap_width[k] = w[k];
      h->tap_off[k] = total * h->cfg.capacity;
      total += w[k];
    }
    CK(cudaSetDevice(h->cfg.device));
    const cudaError_t e = cudaMalloc(&h->tap, (size_t)total * h->cfg.capacity * h->esz);
    if (e != cudaSuccess) {
      cudaGetLastError();
      h->tap = nullptr;
      return fail(DS_ERR_CUDA, "text encoder: tap store for %d tokens failed: %s", h->cfg.capacity, cudaGetErrorString(e));
    }
  }
  h->tap_layer = layer;
  return 0;
}

extern "C" int ds_text_enc_read(ds_text_enc* h, int32_t kind, float* dev_out, int64_t capacity, int32_t* rows,
                                int32_t* width, void* stream) {
  if (!h) return fail(DS_ERR_INVALID, "null handle");
  if (h->tapped_layer < 0) return fail(DS_ERR_STATE, "text encoder: the last forward ran without a tap");
  if (kind < 0 || kind >= TE_TAPS) return fail(DS_ERR_INVALID, "text encoder: bad tap kind %d", kind);
  if (kind == DS_TE_OUT && h->tapped_layer == h->cfg.layers - 1)
    return fail(DS_ERR_INVALID, "text encoder: the last layer's output is the forward's own output");
  const int64_t r = h->tapped_M, w = h->tap_width[kind], n = r * w;
  if (rows) *rows = int32_t(r);
  if (width) *width = int32_t(w);
  if (!dev_out) return 0;      // size query
  if (n > capacity) return fail(DS_ERR_INVALID, "output capacity %lld < %lld", (long long)capacity, (long long)n);
  CK(cudaSetDevice(h->cfg.device));
  cudaStream_t s = (cudaStream_t)stream;
  const void* src = (const char*)h->tap + (size_t)h->tap_off[kind] * h->esz;
  if (h->bf16) launch_widen_bf16((const bf16*)src, dev_out, n, s);
  else CK(cudaMemcpyAsync(dev_out, src, (size_t)n * 4, cudaMemcpyDeviceToDevice, s));
  CK(cudaGetLastError());
  return 0;
}
