// Host-side launchers of every kernel in the library (definitions in pointwise.cu, gemm_simt.cu,
// gemm_tc.cu).  All pointers are device pointers; `ld*` are row pitches in elements.
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include "common.cuh"

namespace ds {

// FiLM (scale, shift) source for the GroupNorm op.  Row `r` of the activation matrix belongs to scene
// r / n_obj and object r % n_obj.  The table row holds [scale(C) | shift(C)] (chunk(2, dim=1),
// reference denoise_net.py:200).
enum FilmMode { FILM_NONE = 0, FILM_TIME = 1, FILM_OBJECT = 2, FILM_TOKEN = 3 };
struct FilmRef {
  const float* base;      // already offset to this block's [2C] slice
  int mode;
  int64_t row_stride;     // floats between consecutive table rows
  const int* t;           // FILM_TIME: per-scene timestep index (device)
};

template <typename T>
void launch_pack_input(const float* x, T* out, int ld_out, int M, int d, cudaStream_t s);
template <typename T>
void launch_unpack_output(const T* in, int ld_in, float* out, int M, int d, cudaStream_t s);
template <typename T>
void launch_groupnorm(const T* in, int ld_in, T* out, int ld_out, const float* gamma, const float* beta,
                      FilmRef film, const T* res, int ld_res, int n_scenes, int n_obj, int C, int groups,
                      cudaStream_t s);
template <typename T>
void launch_layernorm(const T* in, int ld_in, T* out, int ld_out, const float* g, const T* res, int ld_res,
                      int M, int C, cudaStream_t s);
template <typename T>
void launch_linattn(const T* qkv, int ld, T* out, int ld_out, int n_scenes, int n_obj, cudaStream_t s);
template <typename T>
void launch_softattn(const T* qkv, int ld, T* out, int ld_out, int n_scenes, int n_obj, cudaStream_t s);
// cross linear attention: ctx [n_scenes][4][32(d)][32(e)] fp32 precomputed from the text
template <typename T>
void launch_xattn_apply(const T* q, int ldq, const float* ctx, T* out, int ld_out, int n_scenes, int n_obj,
                        cudaStream_t s);
void launch_xattn_prepare(const float* kv, int ld_kv, float* ctx, int n_scenes, int L, cudaStream_t s);
// adjoints of the two (training step, backward.cu / pointwise.cu): dq (= | += by `accumulate`) and dctx
// [n_scenes][4][32][32] fp32 from the kept pre-softmax q; dkv [n_scenes * L, 256] fp32 from kv and dctx
template <typename T>
void launch_xattn_apply_bwd(const T* q, int ldq, const T* dout, int ldo, const float* ctx, T* dq, int lddq,
                            int accumulate, float* dctx, int n_scenes, int n_obj, cudaStream_t s);
void launch_xattn_prepare_bwd(const float* kv, int ld_kv, const float* dctx, float* dkv, int ld_dkv, int n_scenes,
                              int L, cudaStream_t s);
// text tokens the prepare kernels hold in shared memory: 1 KB per token (k and v, 4 heads x 32 channels, fp32)
// within the 200 KB dynamic shared-memory limit init_pointwise_attrs() raises them to
constexpr int XATTN_SMEM_LIMIT = 200 * 1024;
constexpr int XATTN_MAX_L = XATTN_SMEM_LIMIT / (4 * 2 * 32 * 4);

void sinusoid_freqs_host(int dim, float* hf /*[dim / 2]*/);
void launch_sinusoid(float* out, const float* freq_dev, int T, int dim, cudaStream_t s);
void launch_sinusoid_t(float* out, const float* freq_dev, const int* t_dev, int B, int dim, cudaStream_t s);
void launch_silu_f32(const float* in, float* out, int64_t n, cudaStream_t s);
void launch_t_convert(const int64_t* t, int* out, int B, cudaStream_t s);

// ---- sampling-step kernels --------------------------------------------------------------------
// Per-step coefficients, one row per loop iteration (device table).
struct StepCoef {
  float a_x, a_o;         // x0 = a_x * x_t + a_o * model_out
  float c_0, c_x, c_z;    // x_next = c_0 * x0 + c_x * x_t + c_z * noise
  float q_a, q_b;         // completion re-noising: x[:P] = q_a * partial + q_b * noise2
  int   t;                // timestep fed to the denoiser
};
struct StepState {        // device-resident loop state (advanced by the kernels themselves), one per handle
  int step;               // loop iteration index (0 .. n_steps-1)
  unsigned int done;      // blocks of the running step_update kernel that have finished (last one advances `step`)
  // Philox key / global index of scene 0 of this call: read from HERE by the step kernels (not passed as kernel
  // parameters), so that a captured step graph is reusable across calls with different seeds / shards
  unsigned long long seed;
  unsigned long long scene_offset;
};
// start of a step: t_dev[b] = coef[step].t ; optional completion re-noise of the first P objects
void launch_begin_step(const StepCoef* coef, const StepState* st, int* t_dev, float* x, const float* partial,
                       const float* partial_noise, int B, int n_obj, int d, int P, cudaStream_t s);
// end of a step: x <- update(x, model_out, noise) ; advances st->step
template <typename T>
void launch_step_update(const StepCoef* coef, StepState* st, float* x, const T* model_out, int ld_out,
                        const float* noise, int B, int n_obj, int d, int clip, cudaStream_t s);
void launch_randn(float* out, int B, int per_scene, uint64_t seed, uint64_t scene_offset, uint32_t stream_id,
                  cudaStream_t s);
// single explicit reverse step with per-sample t (p_sample)
template <typename T>
void launch_p_sample(const float* x, const T* model_out, int ld_out, const int* t, const float* noise, float* out,
                     const float* a_x, const float* a_o, const float* c1, const float* c2, const float* sigma,
                     int B, int n_obj, int d, int clip, cudaStream_t s);
void launch_q_sample(const float* x0, const int64_t* t, const float* noise, float* out, const float* sqrt_ac,
                     const float* sqrt_1mac, int B, int per_scene, cudaStream_t s);

// variational bound (diffusion_ddpm.py:511-518, 679-717), one CTA per scene, fixed-order reductions (no atomics).
// End of a VLB step: x = x_t of the step (k_begin_step with P = n_obj, partial = x0), coef[step] holds the x0
// conversion (a_x, a_o), the posterior-mean coefficients (c_0, c_x) and t.  vb[b][t] = mean KL(true posterior ||
// model) / ln 2 with logvar1 = post_logvar[t], logvar2 = model_logvar[t]; mse[b][t] = mean (x0_hat - x0)^2.
// Advances st->step.
template <typename T>
void launch_vlb_terms(const StepCoef* coef, StepState* st, const float* x, const T* model_out, int ld_out,
                      const float* x0, const float* post_logvar, const float* model_logvar, float* vb /*[B][n_t]*/,
                      float* mse /*[B][n_t]*/, int B, int n_obj, int d, int n_t, int clip, cudaStream_t s);
// prior[b] = mean KL(N(sqrt_ac[t_last] x0, exp(log_1mac[t_last])) || N(0, 1)) / ln 2
void launch_prior_bpd(const float* x0, const float* sqrt_ac, const float* log_1mac, int t_last, int B, int per_scene,
                      float* prior, cudaStream_t s);

// p_losses value (reference diffusion_ddpm.py:520-652): one CTA per scene
struct LossArgs {
  int n_obj, d, trans, size, angle, cls, objn, feat;
  int mean_type, loss_separate, loss_iou, arrange;
  float bounds[12];     // trans_min[3], trans_max[3], size_min[3], size_max[3]
};
template <typename T>
void launch_p_losses(const float* x0, const float* noise, const float* x_t, const T* model_out, int ld_out,
                     const int64_t* t, const float* sqrt_ac, const float* sqrt_1mac, const float* sqrt_recip_ac,
                     const float* sqrt_recipm1_ac, const float* loss_weight, const float* alphas_cumprod,
                     LossArgs a, float* losses, float* parts /*[B][9]*/, int B, cudaStream_t s);
void launch_loss_dict_mean(const float* parts, float* dict9, int B, cudaStream_t s);

// nearest catalogue model per query object (threed_future_dataset.py:28-77); see k_retrieve
void launch_retrieve(const int* class_start, int n_classes, const float* cat_feat, const float* cat_size, int feat_dim,
                     int size_dim, const int64_t* q_label, const float* q_feat, const float* q_size, int Q, int mode,
                     int64_t* out, cudaStream_t s);

// ---- floor-plan encoder (room_encoder.cu): NHWC activation rows (scene, y, x) x channels ---------------------
// One convolution: input [B * hin * win, cin] -> output [B * hout * wout, cout]; im2col columns (ky, kx, cin),
// zero-padded to Kp (a multiple of 64).
struct RoomConvGeom { int cin, cout, k, stride, pad, hin, win, hout, wout, Kp; };
template <typename T> void launch_re_pack_mask(const float* mask, T* out, int B, int C, int H, int W, cudaStream_t s);
template <typename T> void launch_re_im2col(const T* in, const RoomConvGeom& g, int B, T* cols, cudaStream_t s);
// gather adjoint of im2col: out (= | +=) col2im(dcols) (+ add), zeroed where mask <= 0 (add / mask optional)
template <typename T>
void launch_re_col2im(const T* dcols, const RoomConvGeom& g, int B, T* out, int accumulate, const T* add, const T* mask,
                      cudaStream_t s);
template <typename T> void launch_re_add_relu(const T* z, const T* res, T* out, int64_t n, cudaStream_t s);
// 3x3 / stride 2 / pad 1 max pool (torch's first-maximum argmax) and its gather adjoint (zeroed where in <= 0)
template <typename T> void launch_re_maxpool(const T* in, T* out, int B, int C, int hin, int win, int hout, int wout, cudaStream_t s);
template <typename T>
void launch_re_maxpool_bwd(const T* in, const T* dout, T* din, int B, int C, int hin, int win, int hout, int wout,
                           cudaStream_t s);
template <typename T> void launch_re_avgpool(const T* in, float* feat, int B, int C, int hw, cudaStream_t s);
template <typename T> void launch_re_avgpool_bwd(const float* dfeat, const T* out, T* d, int B, int C, int hw, cudaStream_t s);
// FrozenBatchNorm fold (bn = weight, bias, running_mean, running_var of cout floats each) and its adjoint:
// dW [cout, cin, k, k], dbn = [d weight | d bias]
template <typename T>
void launch_re_fold(const float* W, const float* bn, const RoomConvGeom& g, T* wp, float* bias, cudaStream_t s);
void launch_re_fold_bwd(const float* dwp, const float* dbias, const float* W, const float* bn, const RoomConvGeom& g,
                        float* dW, float* dbn, cudaStream_t s);

// ---- frozen BERT text encoder (text_encoder.cu): token rows [B * L, width] -------------------------------------
// out = LayerNorm(word[ids[r]] + token_type[0] + position[r % L]) with weight g, bias b; NaN rows for ids outside
// [0, vocab)
template <typename TO>
void launch_te_embed_ln(const int* ids, const float* word, const float* pos, const float* type0, const float* g,
                        const float* b, TO* out, int M, int L, int H, int vocab, float eps, cudaStream_t s);
template <typename TI, typename TO>
void launch_te_layernorm(const TI* in, const float* g, const float* b, TO* out, int M, int H, float eps, cudaStream_t s);
// masked self-attention, head dim 64, scale 1/8: qkv [B * L, 3H] -> out [B * L, H]; keys at or past lengths[b]
// (clamped to [1, L]) get zero weight
template <typename T>
void launch_te_attention(const T* qkv, const int* lengths, T* out, int B, int L, int H, cudaStream_t s);
template <typename T> void launch_te_convert(const float* in, T* out, int64_t n, cudaStream_t s);
void launch_widen_bf16(const bf16* in, float* out, int64_t n, cudaStream_t s);

// ---- GEMMs: D[M,N] = act([A0 | A1][M, K0+K1] * W[N, K0+K1]^T + bias) (+ residual) -----------------
struct GemmArgs {
  const void* a0; int lda0; int k0;
  const void* a1; int lda1; int k1;      // a1 == nullptr when there is no second operand
  const void* w;  int ldw;               // [N, K] row-major, same element type as A
  const float* bias;                     // [N] or nullptr
  void* d; int ldd;
  const void* res; int ldres;            // optional residual added after the activation
  int M, N, act;
  // fused GroupNorm(8 groups) + affine + FiLM + SiLU epilogue (tensor-core backend only)
  int gn;
  int n_obj;
  int film_C;
  const float* gamma;
  const float* beta;
  FilmRef film;
};
template <typename T> void launch_gemm_simt(const GemmArgs& g, bool exact, cudaStream_t s);
// fp32 D[M, N] (row pitch ldd) = act(A[M, K] W[N, K]^T + bias) on the exact SIMT GEMM, launched in row chunks that
// keep gridDim.y (64 rows per CTA row) below 65535
void launch_gemm_simt_chunked(const float* a, int K, const float* w, const float* bias, float* d, int ldd, int M, int N,
                              int act, cudaStream_t s);
// fp32 A/W in, fp32 out (time / context FiLM tables; always fp32)
void launch_gemm_f32(const GemmArgs& g, cudaStream_t s);

// tensor-core (wgmma) path: operands described by TMA tensor maps built by the engine (gemm_tc.cu)
struct TcGemmPlan;   // opaque, owns tensor maps
TcGemmPlan* tc_plan_create(const GemmArgs& g, int rows_capacity, char* err, int err_len);
void tc_plan_destroy(TcGemmPlan* p);
void tc_plan_set_film(TcGemmPlan* p, const FilmRef& f);     // FiLM tables may be (re)allocated after planning
// Programmatic-dependent-launch policy shared by every launcher of the library (pointwise.cu).  kind 0: tensor-core
// GEMM kernels (DS_TC_PDL), kind 1: pointwise kernels (DS_PW_PDL); values 0 off, 1 on, 2 (default) automatic: on when
// `rows` (tokens of the launch) <= DS_PDL_ROWS (default 32768), where the kernel prologue is a large share of a launch.
bool pdl_enabled(int kind, int64_t rows);
void tc_plan_set_atomic_out(TcGemmPlan* p, float* d32, int ldd, int ksplit);      // split-K, fp32 atomics (dW GEMMs)
int tc_plan_tiles(const TcGemmPlan* p, int M);
void tc_plan_set_residual(TcGemmPlan* p, const void* res);      // nullptr: plain store; == output: accumulate in place
int launch_gemm_tc(const TcGemmPlan* p, int M, cudaStream_t s);   // returns 0 or cudaError
bool tc_runtime_available(char* err, int err_len);
// the driver's cuTensorMapEncodeTiled as tc_runtime_available() resolved it (nullptr until that succeeds)
decltype(&cuTensorMapEncodeTiled) tc_encode_tiled();
int tc_num_sms();      // SMs of the device tc_runtime_available() checked
// fused GEMM + channel LayerNorm (+ residual) for K <= 128, N = 512 (gemm_ln.cu): GemmArgs.gamma = LayerNorm gain
struct LnGemmPlan;
bool ln_gemm_supported(int N, int K);
LnGemmPlan* ln_plan_create(const GemmArgs& g, int rows_capacity, char* err, int err_len);
void ln_plan_destroy(LnGemmPlan* p);
int launch_gemm_ln(const LnGemmPlan* p, int M, cudaStream_t s);
// fused channel LayerNorm + to_qkv + linear-attention core (gemm_attn.cu)
struct AttnQkvPlan;
bool attn_qkv_supported(int n_obj, int C);
AttnQkvPlan* attn_qkv_plan_create(const void* x, int ldx, const void* w, int ldw, const float* cs, void* o, int ldo,
                                  int n_obj, int K, int rows_capacity, char* err, int err_len);
void attn_qkv_plan_destroy(AttnQkvPlan* p);
int launch_ln_qkv_attn(const AttnQkvPlan* p, int M, cudaStream_t s);

}  // namespace ds
