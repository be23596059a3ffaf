/*
 * diffuscene_b200 -- C ABI of the H100-native (sm_90a) DiffuScene denoising hot path.
 *
 * The reference (tangjiapeng/DiffuScene) is pure Python/PyTorch and has no FFI of its own; this
 * header is the boundary a maintainer binds with ctypes (see INTEGRATION.md).  Each entry point
 * names the reference interface it replaces (paths relative to the reference repository root).
 *
 * Conventions
 *   - plain C types only; no torch / CUDA types in signatures (streams travel as void*).
 *   - "dev" pointers are device (HBM) pointers borrowed from the caller; "host" pointers are host
 *     memory.  Nothing is allocated inside the hot calls once a batch size has been seen.
 *   - every function returns 0 on success or a negative ds_status; ds_last_error() gives the text.
 *   - a handle is bound to one device and is not thread-safe; distinct handles are independent.
 *   - there is NO CPU fallback: without a CUDA device ds_create() fails with DS_ERR_NO_DEVICE
 *     (ds_plan_describe() is the only compute-free introspection call that works without one).
 */
#ifndef DIFFUSCENE_B200_H_
#define DIFFUSCENE_B200_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#if defined(__GNUC__)
#define DS_API __attribute__((visibility("default")))
#else
#define DS_API
#endif

typedef struct ds_handle ds_handle;

enum ds_status {
  DS_OK = 0,
  DS_ERR_INVALID = -1,      /* bad argument / unsupported configuration            */
  DS_ERR_NO_DEVICE = -2,    /* no CUDA device or not sm_90                         */
  DS_ERR_CUDA = -3,         /* a CUDA runtime / driver call failed                 */
  DS_ERR_STATE = -4,        /* call order violated (weights / schedule / context)  */
  DS_ERR_MISSING_WEIGHT = -5
};

enum ds_precision {
  DS_PREC_FP32 = 0,   /* parity mode: fp32 storage + fp32 FMA GEMMs (rtol 1e-3 / atol 1e-4 vs reference) */
  DS_PREC_BF16 = 1    /* throughput mode: bf16 storage, wgmma tensor-core GEMMs, fp32 accumulate/norms */
};

enum ds_gemm_backend {
  DS_GEMM_AUTO = 0,   /* tensor cores (wgmma) for bf16, SIMT for fp32 */
  DS_GEMM_SIMT = 1,   /* CUDA-core GEMM for either precision (debug / cross-check) */
  DS_GEMM_TCGEN05 = 2 /* the tensor-core (wgmma) backend; the name is kept for ABI compatibility */
};

enum ds_mean_type { DS_MEAN_EPS = 0, DS_MEAN_X0 = 1, DS_MEAN_V = 2 };

/* Mirrors the reference's `net_kwargs` for Unet1D (scene_synthesis/networks/denoise_net.py:336-362)
 * plus the engine knobs.  dim_mults must be all ones (every shipped config). */
typedef struct ds_config {
  int32_t dim;              /* hidden width C (512)                                   */
  int32_t channels;         /* point_dim when seperate_all == 0                        */
  int32_t seperate_all;     /* 1: per-attribute encoder / decoder MLPs                 */
  int32_t objectness_dim, class_dim, translation_dim, size_dim, angle_dim, objfeat_dim;
  int32_t cond_dim;         /* context_dim + instanclass_dim: width of `context`       */
  int32_t text_condition;   /* 1: LinearAttentionCross layers present                  */
  int32_t text_dim;
  int32_t n_stages;         /* len(dim_mults), 4                                       */
  int32_t num_objects;      /* N: objects per scene (12 bedroom / 21 living)           */
  int32_t num_timesteps;    /* T of the diffusion schedule (time FiLM table rows)      */
  int32_t precision;        /* ds_precision                                            */
  int32_t gemm_backend;     /* ds_gemm_backend                                         */
  int32_t device;           /* CUDA device ordinal                                     */
  int32_t fuse_level;       /* 0: one kernel per op; 1: conv + GroupNorm + FiLM + SiLU blocks
                                  as one GEMM with a GroupNorm epilogue;
                               2, 3: the channels-on-tensor-memory-lanes GEMM variants of the
                                  sm_100a build; sm_90a has no tensor memory, so these levels
                                  run the level-1 program;
                               4: level 1 + to_out + LayerNorm + residual of the attention
                                  wrappers as one GEMM with a LayerNorm epilogue;
                               5: level 4 + LayerNorm + to_qkv + linear-attention core as one
                                  kernel (N = 12 or 21) */
  int32_t train;            /* 1: training step program -- one op per reference layer (no fused epilogues, activations
                               as their own ops), every intermediate kept for the backward pass (ds_train_*)   */
  int32_t reserved[6];
} ds_config;

/* ---- lifetime ----------------------------------------------------------------------------- */
/* Replaces Unet1D.__init__ + DiffusionPoint.__init__ (denoise_net.py:336-482, diffusion_ddpm.py:721-731). */
DS_API int ds_create(const ds_config* cfg, ds_handle** out);
DS_API int ds_destroy(ds_handle* h);
DS_API const char* ds_last_error(void);
DS_API const char* ds_version(void);

/* ---- weights ------------------------------------------------------------------------------
 * Replaces nn.Module.load_state_dict (scene_synthesis/networks/__init__.py:62-66).  Names are the
 * reference state-dict keys with the "diffusion.model." prefix removed ("downs.0.1.block1.proj.weight").
 * Data is fp32, host memory, C-contiguous, `numel` elements.  ds_commit_weights() folds the weight
 * standardisation (denoise_net.py:78-91), packs for the selected precision, uploads, and rebuilds the
 * time-FiLM table (time_mlp + the per-block Linear of denoise_net.py:181-200 for every t in [0, T)). */
DS_API int ds_load_weight(ds_handle* h, const char* name, const float* host_data, int64_t numel);
DS_API int ds_commit_weights(ds_handle* h);
/* Number of parameter tensors the configuration expects and the i-th expected name / numel. */
DS_API int ds_expected_weight_count(ds_handle* h);
DS_API int ds_expected_weight(ds_handle* h, int index, const char** name, int64_t* numel);

/* ---- diffusion schedule -------------------------------------------------------------------
 * Replaces the table set of GaussianDiffusion.__init__ (diffusion_ddpm.py:168-203).  Each array has T
 * fp32 entries (host).  sigma[t] = (t != 0) * exp(0.5 * model_log_variance[t]) (:314-323, :348-350). */
typedef struct ds_schedule {
  int32_t T;
  int32_t mean_type;                 /* ds_mean_type */
  const float* sqrt_ac;              /* sqrt_alphas_cumprod              */
  const float* sqrt_1mac;            /* sqrt_one_minus_alphas_cumprod    */
  const float* sqrt_recip_ac;        /* sqrt_recip_alphas_cumprod        */
  const float* sqrt_recipm1_ac;      /* sqrt_recipm1_alphas_cumprod      */
  const float* coef1;                /* posterior_mean_coef1             */
  const float* coef2;                /* posterior_mean_coef2             */
  const float* sigma;                /* see above                        */
  const float* alphas_cumprod;
  const float* loss_weight;          /* p_losses weight per t (:194-203) */
} ds_schedule;
DS_API int ds_set_schedule(ds_handle* h, const ds_schedule* s);
/* The extra tables of the variational bound (ds_vlb_loop), T fp32 host entries each, of the same schedule:
 * post_logvar = posterior_log_variance_clipped (:190), model_logvar = the model log-variance of model_var_type
 * (:314-323; fixedsmall: the same table, fixedlarge: log(cat(posterior_variance[1:2], betas[1:]))) and
 * log_1mac = log_one_minus_alphas_cumprod (:179).  Kept apart from ds_schedule, whose layout is ABI. */
DS_API int ds_set_vlb_schedule(ds_handle* h, int32_t T, const float* post_logvar, const float* model_logvar,
                               const float* log_1mac);

/* ---- conditioning -------------------------------------------------------------------------
 * `context` is the [B, N, cond_dim] tensor handed to Unet1D.forward (denoise_net.py:507, built at
 * diffusion_scene_layout_ddpm.py:172-207).  shared != 0: one [N, cond_dim] block used for every scene
 * (the unconditional configs, where it is positional_embedding broadcast over the batch).
 * Device pointers, fp32.  Precomputes the 9 context-FiLM projections (they do not depend on x_t or t). */
DS_API int ds_set_context(ds_handle* h, const float* context_dev, int32_t batch, int32_t shared, void* stream);
/* `context_cross` [B, L, text_dim] fp32 device (diffusion_scene_layout_ddpm.py:210-221); precomputes the
 * k/v side of every LinearAttentionCross (denoise_net.py:284-293). Pass NULL to clear. */
DS_API int ds_set_context_cross(ds_handle* h, const float* cross_dev, int32_t batch, int32_t L, void* stream);

/* ---- denoiser forward ---------------------------------------------------------------------
 * Replaces DiffusionPoint._denoise / Unet1D.forward (diffusion_ddpm.py:748-756, denoise_net.py:507-593).
 * x_t [B, N, d] fp32, t [B] int64, out [B, N, d] fp32 -- all device pointers. */
DS_API int ds_denoise_forward(ds_handle* h, const float* x_t_dev, const int64_t* t_dev, float* out_dev,
                       int32_t batch, void* stream);
/* Same call with HOST buffers: copies in, runs, copies out, synchronises. */
DS_API int ds_denoise_forward_host(ds_handle* h, const float* x_t, const int64_t* t, float* out, int32_t batch);

/* ---- sampling -----------------------------------------------------------------------------
 * Replaces GaussianDiffusion.p_sample_loop / _trajectory / _complete / ddim (diffusion_ddpm.py:355-476)
 * and p_sample (:339-352).  One CUDA graph per step, replayed T times; t lives on the device. */
typedef struct ds_sample_args {
  int32_t batch;
  int32_t clip_denoised;        /* clamp x0 estimate to [-1, 1] (:310-311)                          */
  int32_t num_steps;            /* 0: full schedule T;  DDIM: number of sampling steps              */
  int32_t ddim;                 /* 0: ancestral DDPM (:355-371); 1: DDIM (:401-444 formula)         */
  float   ddim_eta;
  uint64_t seed;                /* Philox seed when no noise is injected                             */
  uint64_t scene_offset;        /* global index of scene 0 (keeps RNG streams independent of sharding) */
  const float* x_init_dev;      /* optional [B,N,d] x_T; NULL: drawn from Philox                     */
  const float* noise_dev;       /* optional injected noise [num_steps, B, N, d], step order T-1..0   */
  const float* partial_dev;     /* completion: clean [B, P, d] (p_sample_loop_complete :447-476)     */
  int32_t num_partial;          /* P                                                                 */
  const float* partial_noise_dev;/* optional injected q_sample noise [num_steps, B, P, d]            */
  int32_t traj_freq;            /* >0: snapshot when t % freq == 0 or t == T-1 (:394)                */
  float* traj_dev;              /* [n_snap, B, N, d] (excluding x_T); n_snap from ds_traj_count      */
  int32_t use_graph;            /* 1: CUDA-graph the step (default); 0: plain launches               */
  const int32_t* ddim_times;    /* optional host array [num_steps+1], descending, last = -1 (:407-409) */
  int32_t chunk_scenes;         /* >0: run the whole loop for sub-batches of this many scenes, one after the other,
                                   so that a sub-batch's activations stay L2-resident (Philox noise path only) */
  int32_t reserved[5];
} ds_sample_args;
DS_API int ds_sample_loop(ds_handle* h, const ds_sample_args* a, float* out_dev, void* stream);
DS_API int ds_sample_loop_host(ds_handle* h, const ds_sample_args* a, float* out_host);
DS_API int ds_traj_count(int32_t T, int32_t freq);
/* One reverse step with explicit per-sample t (p_sample, diffusion_ddpm.py:339-352). */
DS_API int ds_p_sample_step(ds_handle* h, const float* x_t_dev, const int64_t* t_dev, const float* noise_dev,
                     int32_t clip_denoised, float* out_dev, int32_t batch, void* stream);

/* ---- variational bound --------------------------------------------------------------------
 * Replaces GaussianDiffusion.calc_bpd_loop and _prior_bpd (diffusion_ddpm.py:679-717, behind DiffusionPoint.all_kl /
 * prior_kl :734-745): for t = T-1 .. 0, x_t = q_sample(x0, t) -> denoiser -> vb[b][t] = mean over N*d of
 * normal_kl(true posterior, model posterior) / ln 2 (:511-518) and mse[b][t] = mean (x0_hat - x0)^2, with x0_hat
 * clamped when clip_denoised; prior[b] = _prior_bpd.  Like ds_sample_loop: one CUDA graph per step replayed T times
 * (its own cached graph: a VLB call does not evict the sampling graph), t and the Philox state on the device, each
 * scene's numbers independent of the batch it runs in.  Conditioning comes from ds_set_context /
 * ds_set_context_cross with the same batch rules as sampling.  vb_dev and mse_dev ([batch, T] fp32 device) may both be
 * NULL: then only prior_dev ([batch]) is computed, with no denoiser pass.  At t = 0 the reference compares against a
 * posterior variance clipped to 1e-20, so for fixedsmall vb[b][0] ~ 0.5e20 * mean (x0 - x0_hat)^2 / ln 2. */
typedef struct ds_vlb_args {
  int32_t batch;
  int32_t clip_denoised;        /* clamp the x0 estimate to [-1, 1] (:310-311)                                   */
  const float* x0_dev;          /* [B, N, d] clean scenes                                                        */
  uint64_t seed;                /* Philox seed of the q_sample draws when no noise is injected                   */
  uint64_t scene_offset;        /* global index of scene 0 (RNG streams independent of sharding)                  */
  const float* noise_dev;       /* optional injected q_sample noise [T, B, N, d], loop order T-1 .. 0             */
  int32_t use_graph;            /* 1: CUDA-graph the step (default); 0: plain launches                            */
  int32_t reserved[7];
} ds_vlb_args;
DS_API int ds_vlb_loop(ds_handle* h, const ds_vlb_args* a, float* vb_dev, float* mse_dev, float* prior_dev,
                       void* stream);

/* ---- training-side forward pieces ---------------------------------------------------------
 * q_sample (diffusion_ddpm.py:276-286) and the p_losses value (:520-652, loss.py:7-102): per-sample
 * losses [B] and the 9 means of the reference loss dict (order: bbox, trans, size, angle, class, object,
 * objfeat, liou, bbox_iou).  bounds = {trans_min[3], trans_max[3], size_min[3], size_max[3]} or NULL. */
DS_API int ds_q_sample(ds_handle* h, const float* x0_dev, const int64_t* t_dev, const float* noise_dev,
                float* out_dev, int32_t batch, void* stream);
DS_API int ds_p_losses(ds_handle* h, const float* x0_dev, const int64_t* t_dev, const float* noise_dev,
                int32_t loss_separate, int32_t loss_iou, const float* bounds_host,
                float* losses_dev, float* loss_dict_dev, int32_t batch, void* stream);

/* ---- native training step ---------------------------------------------------------------------
 * Replaces what `loss.backward()` + `optimizer.step()` do in train_on_batch
 * (scene_synthesis/networks/diffusion_scene_layout_ddpm.py:456-473) for the denoiser: forward of p_losses
 * (diffusion_ddpm.py:520-652) with every intermediate kept, then the hand-written backward pass of every layer of
 * Unet1D (denoise_net.py:78-593: weight-standardised convs, GroupNorm + FiLM + SiLU blocks, LayerNorms, linear /
 * softmax attention, text cross-attention, the time-embedding MLP and all FiLM projections) and of the loss (MSE terms
 * + IoU regulariser).
 * Parameters and gradients are ONE flat fp32 device buffer each, laid out in ds_expected_weight() order
 * (ds_train_param_count() floats).  grad_scale multiplies d(mean-over-batch loss); pass 1 / world_size to get the
 * data-parallel mean after a sum all-reduce.  context [ctx_shared ? N : B*N, cond_dim] is the conditioning input of
 * Unet1D.forward; dcontext_dev (optional, same shape) receives its gradient (it continues into
 * positional_embedding / the condition MLPs on the caller's side).  flat_grads_dev == NULL: forward + loss only.
 * Uses the handle's schedule (ds_set_schedule) and precision.  Networks with text cross-attention
 * (text_condition != 0) train through ds_train_step_cross; ds_train_step returns DS_ERR_INVALID for them. */
DS_API int64_t ds_train_param_count(ds_handle* h);
DS_API int ds_train_step(ds_handle* h, const float* flat_params_dev, const float* x0_dev, const int64_t* t_dev,
                         const float* noise_dev, const float* context_dev, int32_t ctx_batch, int32_t ctx_shared,
                         int32_t loss_separate, int32_t loss_iou, const float* bounds_host, float grad_scale,
                         float* losses_dev, float* loss_dict_dev, float* flat_grads_dev, float* dcontext_dev,
                         int32_t batch, void* stream);
/* Longest text ds_train_step_cross accepts: the text-side kernels keep k and v of every token in shared memory,
 * 1 KB per token within a 200 KB limit.  BERT descriptions of the reference are far shorter. */
#define DS_TRAIN_CROSS_MAX_L 200
/* ds_train_step for the text-conditioned networks (LinearAttentionCross layers, denoise_net.py:261-297): the same
 * arguments, plus cross_dev = context_cross [batch, cross_L, text_dim] fp32 on the device (the projected text, as in
 * ds_set_context_cross).  The gradients of every to_kv weight land in flat_grads_dev like all others; dcross_dev
 * (optional, same shape as cross_dev, overwritten) receives d(loss)/d(cross), which continues into the text
 * projection (fc_text_f) on the caller's side.  DS_ERR_INVALID for a network without text condition, a NULL cross_dev
 * or cross_L outside [1, DS_TRAIN_CROSS_MAX_L]. */
DS_API int ds_train_step_cross(ds_handle* h, const float* flat_params_dev, const float* x0_dev, const int64_t* t_dev,
                               const float* noise_dev, const float* context_dev, int32_t ctx_batch, int32_t ctx_shared,
                               int32_t loss_separate, int32_t loss_iou, const float* bounds_host, float grad_scale,
                               float* losses_dev, float* loss_dict_dev, float* flat_grads_dev, float* dcontext_dev,
                               const float* cross_dev, int32_t cross_L, float* dcross_dev, int32_t batch, void* stream);
/* Overlap of the data-parallel gradient all-reduce with the backward pass: bucket k is the flat range
 * [bounds[k], bounds[k + 1]) (bounds[0] = 0, bounds[n] = ds_train_param_count()); ds_train_step records events[k] (a
 * cudaEvent_t owned by the caller) on its stream as soon as every gradient inside the bucket is final -- the backward
 * pass finalises the buffer from its end towards its start -- so the caller's communication stream can wait on the
 * event and all-reduce that bucket while the rest of the backward pass still runs.  n_buckets = 0 clears. */
DS_API int ds_train_set_buckets(ds_handle* h, const int64_t* bounds, int32_t n_buckets, void* const* events);
/* Device time of the phases of the last ds_train_step with gradients, milliseconds (profiling aid; synchronises):
 * weight packing, forward, loss + d(loss)/d(output), backward through the step program, conditioning paths,
 * gradient unpacking (weight-standardisation adjoint). */
DS_API int ds_train_phase_ms(ds_handle* h, float* out6);
/* Arrays of the training state ds_train_read copies (`kind`), and what `index` selects for each:
 *   DS_TRAIN_ACT   activation buffer `index` of the train step program (ds_plan_export_json with train = 1,
 *                  no_reuse = 1: every op output has its own buffer), [B*N, width]
 *   DS_TRAIN_GRAD  the gradient buffer of the same activation after the backward pass, [B*N, width]
 *   DS_TRAIN_DW    packed gradient of weight matrix `index` (the plan's wmats), [N, K], before the
 *                  weight-standardisation adjoint
 *   DS_TRAIN_DVEC  gradient of fp32 vector `index` (the plan's vecs), [1, n]
 *   DS_TRAIN_COND  one array of the fp32 conditioning paths, `index` from the DS_TRAIN_COND_* list below */
enum { DS_TRAIN_ACT = 0, DS_TRAIN_GRAD = 1, DS_TRAIN_DW = 2, DS_TRAIN_DVEC = 3, DS_TRAIN_COND = 4 };
/* [B, C] sinusoidal time embedding; [B, 4C] time_mlp.1 output z1, its GELU h1, time_mlp.3 output temb and SiLU(temb)
 * st; [B, time blocks x 2C] time-FiLM rows film and their gradient dfilm; [B, 4C] d(temb), d(h1) and dst -- after the
 * step dst holds d(z1), not d(st); [context rows, cond_dim] SiLU(context) and its gradient; [context rows, context
 * blocks x 2C] context-FiLM rows and their gradient; text networks: [layers x B x L, 256] text-side kv and
 * [layers x B, 4096] per-head contexts; [B*N, d] the noisy input x_t the step computed (q_sample, fp32). */
enum {
  DS_TRAIN_EMB = 0, DS_TRAIN_Z1, DS_TRAIN_H1, DS_TRAIN_TEMB, DS_TRAIN_ST, DS_TRAIN_FILM, DS_TRAIN_DFILM, DS_TRAIN_DTEMB,
  DS_TRAIN_DH1, DS_TRAIN_DST, DS_TRAIN_CTX_ACT, DS_TRAIN_CTX_FILM, DS_TRAIN_DCTX_FILM, DS_TRAIN_DCTX_ACT, DS_TRAIN_XKV,
  DS_TRAIN_XCTX, DS_TRAIN_XT
};
/* After a ds_train_step[_cross] with gradients: copy one array of the training state, widened to fp32, into
 * dev_out [rows, width] on `stream` (profiling / test aid; the step itself is unchanged).  Rows are those of the last
 * step (B, its context rows, its text length).  DS_ERR_STATE before any step with gradients; DS_ERR_INVALID for a bad
 * kind or index, an array the network does not have, or capacity < rows * width floats.  dev_out == NULL: a
 * size query, only rows and width are set. */
DS_API int ds_train_read(ds_handle* h, int32_t kind, int32_t index, float* dev_out, int64_t capacity,
                         int32_t* rows, int32_t* width, void* stream);
/* out[0] += sum(g^2) (device scalar; the caller zeroes it) -- the global gradient norm of clip_grad_norm_. */
DS_API int ds_sumsq(const float* g_dev, int64_t n, float* out_dev, void* stream);
/* torch.optim.Adam (weight decay 0, networks/__init__.py:15-34) on flat buffers.  sumsq_dev (optional): device
 * scalar holding the squared L2 norm of ALL gradients; with max_norm > 0 the clip coefficient
 * min(1, max_norm / (norm + 1e-6)) of clip_grad_norm_ is applied to the gradient on the fly. */
DS_API int ds_adam_step(float* params_dev, const float* grads_dev, float* exp_avg_dev, float* exp_avg_sq_dev, int64_t n,
                        float lr, float beta1, float beta2, float eps, int32_t step, const float* sumsq_dev,
                        float max_norm, void* stream);

/* ---- post-processing: object retrieval -----------------------------------------------------
 * Replaces ThreedFutureDataset.get_closest_furniture_to_objfeats_and_size (mode 0), _to_objfeats (mode 1) and
 * _to_box (mode 2) (scene_synthesis/datasets/threed_future_dataset.py:28-77) for a whole batch of generated objects:
 * out[q] = index of the catalogue entry of class q_label[q] minimising (size mse, feature mse) lexicographically
 * (mode 0; np.lexsort((mses_feat, mses_size))), the feature mse (1) or the size mse (2); ties -> lowest index;
 * -1 when the class has no entry.  The catalogue is grouped by class (stable order inside a class):
 * class_start[c] .. class_start[c + 1] is the entry range of class c (n_classes + 1 ints).  cat_feat
 * [n_entries, feat_dim], cat_size [n_entries, size_dim], q_feat [Q, feat_dim], q_size [Q, size_dim] fp32; all
 * device pointers.  Distances are accumulated in numpy's float32 order, so indices are bit-exact.  Stateless. */
DS_API int ds_retrieve_objects(const int32_t* class_start_dev, int32_t n_classes, const float* cat_feat_dev,
                               const float* cat_size_dev, int32_t feat_dim, int32_t size_dim,
                               const int64_t* q_label_dev, const float* q_feat_dev, const float* q_size_dev,
                               int32_t num_queries, int32_t mode, int64_t* out_index_dev, void* stream);

/* ---- post-processing: scene evaluation -------------------------------------------------------
 * The statistics the reference writes with --compute_intersec (scripts/utils.py:560-745) for a whole batch of
 * generated scenes.  Both calls are stateless; all pointers are device pointers.
 *
 * ds_scene_boxes: per object q of num_objects, the world-space axis-aligned bounds [x1, y1, z1, x2, y2, z2] (fp64)
 * of its retrieved model placed as scene_synthesis/utils.py:114-163 places it: scaled by size / raw_half, centred on
 * the scaled raw AABB, rotated about y by angle and translated.  translation [Q, 3], size [Q, 3] (half extents) and
 * angle [Q] are fp32 world-space attributes.  model_index [Q] indexes the footprint table; -1 (or a NULL
 * model_index, or a model whose hull row is empty) makes the object its own box: half sizes = size, centred.
 * The footprint table of num_models models: hull_offsets [num_models + 1] int32 (row m of hull_xz is hull_offsets[m]
 * .. hull_offsets[m + 1]), hull_xz [num_hull_vertices, 2] the raw xz convex-hull vertices, raw_half [num_models, 3]
 * and raw_aabb [num_models, 6] (min xyz, max xyz of the raw vertices), fp64.  The x / z bounds are exact over the
 * hull, y over the raw range.  DS_ERR_INVALID for NULL pointers, negative counts, hull offsets that are negative,
 * decrease or pass num_hull_vertices, and a model index outside [-1, num_models); the last two are found on the
 * device, so this call waits for `stream`.
 *
 * ds_scene_stats: one scene per row b of batch, over its kept objects (keep [batch, num_objects] uint8, NULL = all),
 * num_objects <= 64: bounds [batch, num_objects, 6] fp64 as ds_scene_boxes writes them, class [batch, num_objects]
 * int64, model_id [batch, num_objects] int64 (NULL: the symmetry test does not compare models).  Outputs per scene:
 * the kept objects, the pairs n (n - 1) / 2, the fp32 IoU sum over pairs i < j in lexicographic order (the bounds
 * rounded to fp32, each pair bit-equal to the reference's), the pairs with IoU > 0, the overlap ratio (fp32 from overlap and
 * volume sums taken in fp64; 0 / 0 gives NaN) and the symmetric pairs (judge_if_symmetry on the fp64 bounds, equal class and model).  Scenes with 0 or
 * 1 kept objects give (n, 1, 0, 0, 0) and 0, as the reference does.  pair_iou [batch, num_objects, num_objects]
 * (optional) receives the IoU matrix by slot, 0 where a slot is not kept.  No atomics: a scene's outputs do not depend
 * on the batch.  DS_ERR_INVALID for NULL required pointers, batch < 0 or num_objects outside [0, 64]. */
DS_API int ds_scene_boxes(const float* translation_dev, const float* size_dev, const float* angle_dev,
                          const int64_t* model_index_dev, int32_t num_objects, const int32_t* hull_offsets_dev,
                          const double* hull_xz_dev, int32_t num_hull_vertices, const double* raw_half_dev,
                          const double* raw_aabb_dev, int32_t num_models, double* bounds_dev, void* stream);
DS_API int ds_scene_stats(const double* bounds_dev, const uint8_t* keep_dev, const int64_t* class_dev,
                          const int64_t* model_id_dev, int32_t batch, int32_t num_objects, int32_t* num_objects_dev,
                          int32_t* num_pairs_dev, float* iou_sum_dev, int32_t* insec_count_dev,
                          float* overlap_ratio_dev, int32_t* num_symmetry_dev, float* pair_iou_dev, void* stream);

/* ---- rendering: top-down images of placed scenes ------------------------------------------------
 * The reference renders every scene top-down with simple-3dviz (scripts/utils.py:220-254); these calls draw the
 * placed catalogue meshes of a whole batch of scenes straight into device memory (DESIGN.md, "Rendering").
 *
 * ds_mesh_catalog_create copies a mesh catalogue from HOST arrays to `device` and returns its handle:
 * vertex_offsets / face_offsets [num_models + 1] int32 (both start at 0), vertices [V, 3] fp32 raw vertices, faces
 * [F, 3] int32 model-local vertex indices, uvs [F, 3, 2] fp32 per-corner texture coordinates (NaN: the face has none),
 * raw_half [num_models, 3] and raw_aabb [num_models, 6] fp64 as ds_scene_boxes takes them, kd [num_models, 3] fp32
 * and textures [num_models, texture_size, texture_size, 3] uint8 (row 0 is the image's top row).  DS_ERR_INVALID for
 * a NULL handle pointer or array, offsets that do not start at 0 or decrease, a face index outside its model, a model
 * with 2^25 faces or more, a half size <= 0 or a texture size outside [1, 4096].  ds_mesh_catalog_destroy frees it;
 * any pointer that is not a live catalogue handle gives DS_ERR_INVALID. */
typedef struct ds_render_camera {
  float eye[3], target[3], up[3];       /* pyrr create_look_at(eye, target, up) */
  float left, right, bottom, top;       /* orthographic: pyrr orthogonal_projection(left, right, bottom, top, near,
                                           far); perspective: the frustum bounds on the near plane, pyrr
                                           create_perspective_projection_from_bounds(left, right, bottom, top, near,
                                           far).  Array row r counts from y_ndc = -1 in both: bottom > top gives an
                                           upright image */
  float near_plane, far_plane;          /* view depth (-z_view) range kept per pixel: 0 <= near < far, and near > 0
                                           for perspective */
  int32_t width, height;                /* image size, each in [1, 4096] */
  int32_t projection;                   /* DS_RENDER_ORTHOGRAPHIC (0, a zeroed struct) or DS_RENDER_PERSPECTIVE */
  int32_t reserved[3];
} ds_render_camera;

enum { DS_RENDER_ORTHOGRAPHIC = 0, DS_RENDER_PERSPECTIVE = 1 };
enum { DS_RENDER_NO_TEXTURE = 1, DS_RENDER_WHITE_BACKGROUND = 2 };

/* Per-call inputs of ds_render_scenes; every pointer is a device pointer.  Scene b holds num_objects slots
 * (<= 64): translation / size [batch, num_objects, 3] and angle [batch, num_objects] fp32 in world space (after
 * post_process_batch), model_index [batch, num_objects] int64 into the catalogue (-1: empty slot), class_index
 * [batch, num_objects] int64 into palette [num_colors, 3] fp32 (needed with DS_RENDER_NO_TEXTURE only).  The optional
 * floor of scene b is triangles floor_offsets[b] .. floor_offsets[b + 1] of floor_tris [num_floor_tris, 3, 3] fp32,
 * already centred; floor_offsets NULL draws no floor.  floor_texture_index [batch] int32 (optional) picks one of
 * floor_textures [num_floor_textures, S, S, 3] uint8 per scene (-1 or NULL: white).  Outputs: image [batch, height,
 * width, 3] uint8 and, when id is not NULL, id [batch, height, width] int64 = slot << 32 | face of the visible
 * triangle (slot num_objects: the floor), -1 for background. */
typedef struct ds_render_args {
  int32_t batch, num_objects;
  const float* translation_dev;
  const float* size_dev;
  const float* angle_dev;
  const int64_t* model_index_dev;
  const int64_t* class_index_dev;
  const int32_t* floor_offsets_dev;
  const float* floor_tris_dev;
  int32_t num_floor_tris;
  int32_t num_colors;
  const float* palette_dev;
  const uint8_t* floor_textures_dev;
  int32_t num_floor_textures, floor_texture_size;
  const int32_t* floor_texture_index_dev;
  int32_t flags;                        /* DS_RENDER_* */
  int32_t reserved0;
  uint8_t* image_dev;
  int64_t* id_dev;
  int32_t reserved[8];
} ds_render_args;

DS_API int ds_mesh_catalog_create(int32_t num_models, const int32_t* vertex_offsets, const float* vertices,
                                  const int32_t* face_offsets, const int32_t* faces, const float* uvs,
                                  const double* raw_half, const double* raw_aabb, const float* kd,
                                  const uint8_t* textures, int32_t texture_size, int32_t device, void** handle);
DS_API int ds_mesh_catalog_destroy(void* handle);
/* Sample at pixel centres with a top-left fill rule and no culling; the nearest view depth in [near, far] wins, ties
 * go to the lower (slot, face).  A perspective face that crosses the near plane draws exactly its part with depth >=
 * near; depth, world position and UVs are interpolated perspective-correctly.  DS_ERR_INVALID for a handle that is
 * not a live catalogue or lives on another device, NULL required pointers, batch < 0, num_objects outside [0, 64], an
 * unsupported image size, projection or view volume (left == right, bottom == top, perspective near <= 0), and
 * (found on the device, so the call waits for `stream`) a model index outside [-1, M), a class index outside the
 * palette, bad floor offsets or a floor texture index outside [-1, num_floor_textures). */
DS_API int ds_render_scenes(void* handle, const ds_render_camera* camera, const ds_render_args* args, void* stream);

/* Pillow's separable resize on the device, bit-exact with PIL given Pillow's coefficient tables (computed on the
 * host by diffuscene_b200.render): horizontal pass, then vertical, with Pillow's intermediate rounding.  in [batch,
 * in_h, in_w, 3] uint8.  Horizontal table: h_bounds [out_w, 2] int32 (first input column, count), h_coeffs
 * [out_w, h_ksize]; vertical table likewise over rows.  Tables are device arrays.
 * ds_resize_f32: each channel as a float32 'F' image, fp64 coefficients (clean-fid's clean resize), output
 * [batch, 3, out_h, out_w] fp32 clipped to [0, 255].
 * ds_resize_u8: 8-bit with int32 fixed-point coefficients (22 fraction bits), then (x / 255 - mean[c]) / std[c] in
 * fp32 (ToTensor + Normalize; mean_std is a HOST array of 6 floats), output [batch, 3, out_h, out_w] fp32.
 * DS_ERR_INVALID for NULL pointers, batch < 0, sizes outside [1, 4096], a kernel size outside [1, 1024] or a bound
 * outside the input (found on the device, so these calls wait for `stream`). */
DS_API int ds_resize_f32(const uint8_t* in_dev, int32_t batch, int32_t in_h, int32_t in_w, int32_t out_h,
                         int32_t out_w, const int32_t* h_bounds_dev, const double* h_coeffs_dev, int32_t h_ksize,
                         const int32_t* v_bounds_dev, const double* v_coeffs_dev, int32_t v_ksize, float* out_dev,
                         void* stream);
DS_API int ds_resize_u8(const uint8_t* in_dev, int32_t batch, int32_t in_h, int32_t in_w, int32_t out_h,
                        int32_t out_w, const int32_t* h_bounds_dev, const int32_t* h_coeffs_dev, int32_t h_ksize,
                        const int32_t* v_bounds_dev, const int32_t* v_coeffs_dev, int32_t v_ksize,
                        const float* mean_std, float* out_dev, void* stream);

/* ---- floor-plan encoder --------------------------------------------------------------------
 * Replaces the ResNet-18 trunk of the reference's room-mask feature extractor (scene_synthesis/networks/
 * feature_extractors.py:19-47 with FrozenBatchNorm2d, frozen_batchnorm.py): conv1 -> bn1 -> ReLU -> maxpool ->
 * layer1 .. layer4 -> global average pool, giving the [B, 512] input of its fc head.  The fc head and fc_room_f stay
 * on the caller's side.  A handle of its own, independent of ds_handle.
 * Parameters are ONE flat fp32 device buffer in ds_room_enc_expected_weight() order: the reference names under
 * `feature_extractor._feature_extractor.` (conv1.weight, bn1.weight, bn1.bias, bn1.running_mean, bn1.running_var,
 * layer1.0.conv1.weight, ...), the BatchNorm running statistics included.  The running variance already holds the
 * eps (FrozenBatchNorm2d.from_batch_norm folds it in).  Buffers grow on the first call at a larger batch; after that
 * nothing is allocated inside a call.  `stream` is used as given: NULL is the default stream, not a stream of the
 * handle's own. */
typedef struct ds_room_enc ds_room_enc;
typedef struct ds_room_enc_config {
  int32_t precision;        /* ds_precision: fp32 parity mode or bf16 tensor-core mode                      */
  int32_t input_channels;   /* channels of the mask, 1 .. 8                                                  */
  int32_t height, width;    /* mask size, each a multiple of 32 and at least 32 (64 x 64 in the reference)   */
  int32_t device;           /* CUDA device ordinal                                                           */
  int32_t reserved[3];
} ds_room_enc_config;
/* DS_ERR_INVALID for input_channels outside [1, 8] or a height / width below 32 or not a multiple of 32. */
DS_API int ds_room_enc_create(const ds_room_enc_config* cfg, ds_room_enc** out);
DS_API int ds_room_enc_destroy(ds_room_enc* h);
DS_API int ds_room_enc_expected_weight_count(ds_room_enc* h);
DS_API int ds_room_enc_expected_weight(ds_room_enc* h, int index, const char** name, int64_t* numel);
/* mask [batch, input_channels, height, width] fp32 -> feat [batch, 512] fp32, device pointers.  A scene's features do
 * not depend on the batch it runs in.  keep_for_backward != 0 keeps the activations, and the flat_params_dev pointer
 * (which must stay valid and unchanged), for ds_room_enc_backward. */
DS_API int ds_room_enc_forward(ds_room_enc* h, const float* flat_params_dev, const float* mask_dev, int32_t batch,
                               float* feat_dev, int32_t keep_for_backward, void* stream);
/* d(loss)/d(feat) [batch, 512] of the kept forward -> flat_grads_dev (same layout as the parameters, overwritten;
 * the running statistics get 0).  DS_ERR_INVALID when no forward was kept. */
DS_API int ds_room_enc_backward(ds_room_enc* h, const float* dfeat_dev, float* flat_grads_dev, void* stream);
/* Arrays of the encoder's state ds_room_enc_read copies (`kind`), and what `index` selects.  Rows are those of the
 * last forward (B scenes; an H x W mask, H2 = H / 2, H4 = H / 4); activations are NHWC rows (scene, y, x) x channels.
 * Convs are numbered in ds_room_enc_expected_weight order: 0 the stem, then per block conv1, conv2 (, downsample).
 *   after a forward:
 *   DS_RE_X0     the packed mask, [B H W, input_channels]
 *   DS_RE_A1     the stem output after its ReLU, [B H2 W2, 64]
 *   DS_RE_P      the max-pool output, [B H4 W4, 64]
 *   DS_RE_H      block `index` (0 .. 7): conv1's output after its ReLU, [block rows, block width]
 *   DS_RE_O      block `index`: the block output relu(conv2 + residual)
 *   DS_RE_WP     conv `index`: the folded weight W' the kernels read, [cout, Kp] (columns (ky, kx, cin), zero past
 *                k k cin up to Kp, a multiple of 64)
 *   DS_RE_BIAS   conv `index`: the folded fp32 bias, [1, cout]
 *   after a backward (and no forward since):
 *   DS_RE_DWP    conv `index`: dW' [cout, Kp], before the adjoint of the fold
 *   DS_RE_DBIAS  conv `index`: d(bias) [1, cout]
 *   DS_RE_DZ     block `index`: the gradient of the block's pre-ReLU sum conv2 + residual
 *   DS_RE_DH     block `index`: the gradient of conv1's pre-ReLU output
 *   DS_RE_DP     the gradient of the max-pool output
 *   DS_RE_DA1    the gradient of the stem's pre-ReLU output (the max-pool adjoint, masked by the stem's ReLU) */
enum {
  DS_RE_X0 = 0, DS_RE_A1, DS_RE_P, DS_RE_H, DS_RE_O, DS_RE_WP, DS_RE_BIAS, DS_RE_DWP, DS_RE_DBIAS, DS_RE_DZ, DS_RE_DH,
  DS_RE_DP, DS_RE_DA1
};
/* Copy one array of the encoder's state, widened to fp32, into dev_out [rows, width] on `stream` (test / profiling
 * aid; forward and backward are unchanged by it).  DS_ERR_STATE before any forward, and for the gradient kinds when no
 * backward ran after the last forward; DS_ERR_INVALID for a bad kind or index, or capacity < rows * width floats.
 * dev_out == NULL: a size query, only rows and width are set. */
DS_API int ds_room_enc_read(ds_room_enc* h, int32_t kind, int32_t index, float* dev_out, int64_t capacity,
                            int32_t* rows, int32_t* width, void* stream);

/* ---- object shape auto-encoder ---------------------------------------------------------------
 * The reference's KLAutoEncoder (scene_synthesis/networks/foldingnet_autoencoder.py:131-390): a FoldingNet encoder
 * (kNN covariances, three 1x1 convs, two kNN graph layers, conv4, max over the points), a KL latent head and a
 * two-stage folding decoder onto a fixed 45 x 45 grid, trained with the Chamfer distance.  fp32 throughout.  A handle
 * of its own, independent of ds_handle.
 * Parameters are ONE flat fp32 device buffer in ds_shape_ae_expected_weight() order: the reference's state-dict names
 * (encoder.conv1.weight, ..., decoder.fold2.layers.6.bias) with the BatchNorm running statistics included and
 * num_batches_tracked left out.  Points are [batch, num_points, 3], the latent and eps [batch, latent_dim], kl
 * [batch], the reconstruction [batch, 2025, 3]; all device pointers.  Buffers grow on the first call at a larger
 * batch; `stream` is used as given. */
typedef struct ds_shape_ae ds_shape_ae;
typedef struct ds_shape_ae_config {
  int32_t latent_dim;       /* objfeat_dim of the reference config, 1 .. 512 (32 or 64 in the shipped configs)      */
  int32_t num_points;       /* points per object, at least 16 (2048 in the reference's dataset)                   */
  int32_t device;           /* CUDA device ordinal                                                                */
  int32_t reserved[5];
} ds_shape_ae_config;
/* DS_ERR_INVALID for latent_dim outside [1, 512] or num_points < 16. */
DS_API int ds_shape_ae_create(const ds_shape_ae_config* cfg, ds_shape_ae** out);
DS_API int ds_shape_ae_destroy(ds_shape_ae* h);
DS_API int ds_shape_ae_expected_weight_count(ds_shape_ae* h);
DS_API int ds_shape_ae_expected_weight(ds_shape_ae* h, int index, const char** name, int64_t* numel);
/* kl, latent = mean + exp(logvar / 2) eps and the reconstruction of `points` (each output optional).  eps is the
 * caller's N(0, 1) draw.  train != 0: BatchNorm uses batch statistics and updates the running statistics inside
 * flat_params_dev; train == 0: running statistics, and an object's outputs do not depend on the batch it runs in.
 * keep != 0 keeps this pass readable through ds_shape_ae_get_knn. */
DS_API int ds_shape_ae_forward(ds_shape_ae* h, float* flat_params_dev, const float* points_dev, int32_t batch,
                               const float* eps_dev, int32_t train, int32_t keep, float* latent_dev, float* kl_dev,
                               float* recon_dev, void* stream);
/* One training step of get_loss (:374-390): a train-mode forward, the Chamfer distance, losses_dev[3] = {loss,
 * loss.cd, loss.kl} with loss = cd + kl_weight * sum(kl) / batch, and the backward pass into flat_grads_dev (same
 * layout as the parameters, overwritten; the running statistics get 0).  The pass is kept for ds_shape_ae_get_knn. */
DS_API int ds_shape_ae_train_step(ds_shape_ae* h, float* flat_params_dev, const float* points_dev, int32_t batch,
                                  const float* eps_dev, float kl_weight, float* flat_grads_dev, float* losses_dev,
                                  void* stream);
/* The reference's chamfer_3DDist as a standalone op: for a [batch, n, 3] and b [batch, m, 3], dist1 [batch, n] is the
 * squared distance from each point of a to its nearest point of b, idx1 its index (the first minimum in index order),
 * and dist2 / idx2 the same from b to a.  The backward pass takes d(dist1), d(dist2) and writes grad_a [batch, n, 3]
 * and / or grad_b [batch, m, 3] (either may be NULL) as gathers in a fixed order: bit-identical from run to run. */
DS_API int ds_chamfer_forward(const float* a_dev, int32_t n, const float* b_dev, int32_t m, int32_t batch,
                              float* dist1_dev, float* dist2_dev, int32_t* idx1_dev, int32_t* idx2_dev, void* stream);
DS_API int ds_chamfer_backward(const float* a_dev, int32_t n, const float* b_dev, int32_t m, int32_t batch,
                               const int32_t* idx1_dev, const int32_t* idx2_dev, const float* g1_dev,
                               const float* g2_dev, float* grad_a_dev, float* grad_b_dev, void* stream);

/* ---- frozen BERT text encoder ------------------------------------------------------------------
 * The forward pass of Hugging Face `BertModel` up to `last_hidden_state` (no pooler, no backward pass), which the
 * text-conditioned networks run on each tokenized description: embeddings + LayerNorm, then `layers` post-LN blocks
 * of masked self-attention (head dim 64, scale 1/8) and an erf-GELU feed-forward, LayerNorm eps 1e-12.  In bf16 mode
 * the feed-forward GELU is the tanh form of the tensor-core GEMM epilogue.  A handle of its own, independent of
 * ds_handle.
 * Parameters are ONE flat fp32 device buffer in ds_text_enc_expected_weight() order: the `BertModel` state-dict names
 * and sizes in state-dict order (embeddings.word_embeddings.weight, ..., encoder.layer.{i}.output.LayerNorm.bias),
 * `pooler.*` left out.  ds_text_enc_set_weights copies and packs them, so the buffer may be released afterwards.
 * Buffers for `capacity` tokens are allocated at creation; nothing is allocated inside a call.  `stream` is used as
 * given. */
typedef struct ds_text_enc ds_text_enc;
typedef struct ds_text_enc_config {
  int32_t layers;           /* num_hidden_layers, >= 1 (12 for bert-base-cased)                                  */
  int32_t hidden;           /* hidden_size = 64 x heads, a multiple of 128 (768)                                */
  int32_t heads;            /* num_attention_heads (12)                                                          */
  int32_t intermediate;     /* intermediate_size, a multiple of 128 (3072)                                       */
  int32_t vocab;            /* vocab_size (28996)                                                                */
  int32_t max_positions;    /* max_position_embeddings: the longest sequence accepted (512)                     */
  int32_t type_vocab;       /* type_vocab_size (2); only token type 0 is used                                    */
  int32_t precision;        /* ds_precision: fp32 parity mode or bf16 tensor-core mode                          */
  int32_t capacity;         /* tokens (batch x padded length) one forward may hold, 1 .. 4194240                 */
  int32_t device;           /* CUDA device ordinal                                                               */
  int32_t reserved[6];
} ds_text_enc_config;
/* DS_ERR_INVALID for any other geometry or capacity. */
DS_API int ds_text_enc_create(const ds_text_enc_config* cfg, ds_text_enc** out);
DS_API int ds_text_enc_destroy(ds_text_enc* h);
DS_API int ds_text_enc_expected_weight_count(ds_text_enc* h);
DS_API int ds_text_enc_expected_weight(ds_text_enc* h, int index, const char** name, int64_t* numel);
/* Copies the flat parameters and packs the weight matrices (bf16 and a fused query/key/value matrix in bf16 mode),
 * ordered on `stream`. */
DS_API int ds_text_enc_set_weights(ds_text_enc* h, const float* flat_params_dev, void* stream);
/* ids [batch, seq_len] int32 right-padded token ids, lengths [batch] int32 valid tokens per sequence -> out [batch,
 * seq_len, hidden] fp32, device pointers.  Every position is computed, padding included: a padded query attends to
 * its sequence's first lengths[b] keys like any other query.  Token type 0 throughout.  An id outside [0, vocab) gives
 * a NaN row and reads nothing; lengths are clamped to [1, seq_len].  A sequence's output does not depend on the other
 * sequences of the batch.  DS_ERR_STATE before ds_text_enc_set_weights; DS_ERR_INVALID for NULL pointers, seq_len
 * above max_positions or batch x seq_len above the capacity. */
DS_API int ds_text_enc_forward(ds_text_enc* h, const int32_t* ids_dev, const int32_t* lengths_dev, int32_t batch,
                               int32_t seq_len, float* out_dev, void* stream);

/* ---- improved precision and recall of rendered scenes ------------------------------------------
 * Feature extractor: torchvision `vgg16` as scripts/improved_precision_recall.py:159-163 (reference) uses it,
 * `classifier[:4](features(x).view(-1, 7 * 7 * 512))`, i.e. the fc2 output before its ReLU, for images already
 * normalised with the ImageNet mean / std.  No avgpool (the identity at 224 x 224).  bf16 mode runs the 13 3x3
 * convolutions as implicit GEMMs on wgmma (NHWC bf16 activations, fp32 accumulation, bias + ReLU (+ 2x2 max-pool) in
 * the epilogue) and fc1 / fc2 on the tensor-core GEMM; fp32 mode runs im2col and the exact SIMT GEMM.  The features
 * are fp32 in both modes.
 * Parameters are ONE flat fp32 device buffer in ds_vgg_expected_weight() order: the torchvision state-dict names and
 * sizes in state-dict order, features.{0,2,5,7,10,12,14,17,19,21,24,26,28}.{weight,bias}, classifier.0.{weight,bias},
 * classifier.3.{weight,bias} (classifier.6, which the feature never reaches, left out).  ds_vgg_set_weights packs them,
 * so the buffer may be released afterwards.  A handle of its own, independent of ds_handle. */
typedef struct ds_vgg ds_vgg;
typedef struct ds_vgg_config {
  int32_t precision;        /* ds_precision: fp32 parity mode or bf16 tensor-core mode                          */
  int32_t capacity;         /* images one internal pass holds, 1 .. 256; larger batches run in passes of this size */
  int32_t device;           /* CUDA device ordinal                                                               */
  int32_t reserved[5];
} ds_vgg_config;
#define DS_VGG_FEATURES 4096
DS_API int ds_vgg_create(const ds_vgg_config* cfg, ds_vgg** out);
DS_API int ds_vgg_destroy(ds_vgg* h);
DS_API int ds_vgg_expected_weight_count(ds_vgg* h);
DS_API int ds_vgg_expected_weight(ds_vgg* h, int index, const char** name, int64_t* numel);
/* DS_ERR_INVALID for NULL pointers or a parameter count other than the sum of the expected sizes. */
DS_API int ds_vgg_set_weights(ds_vgg* h, const float* flat_params_dev, int64_t count, void* stream);
/* images [batch, 3, height, width] fp32 NCHW, normalised -> features [batch, 4096] fp32, device pointers.  Images
 * that are not 224 x 224 are resized with the pixel choice of F.interpolate(size=(224, 224)) in its default nearest
 * mode (src = min(floor(dst * (float)in / 224), in - 1), the scale in fp32), as extract_features does
 * (improved_precision_recall.py:152-156).  An image's features do not depend on the other images of the batch.
 * DS_ERR_STATE before ds_vgg_set_weights; DS_ERR_INVALID for NULL pointers, batch < 0 or a side outside [1, 4096]. */
DS_API int ds_vgg_features(ds_vgg* h, const float* images_dev, int32_t batch, int32_t height, int32_t width,
                           float* features_dev, void* stream);

/* ---- FID and KID of rendered scenes ------------------------------------------------------------
 * Feature extractor: the FID Inception-v3 (clean-fid's `clean` mode as pytorch-fid restates its blocks), the 2048-d
 * pool3 output of torchvision's Inception3 layout with aux_logits off, where the branch_pool average pools of
 * Mixed_5b-d, 6b-e and 7b exclude the padding and Mixed_7c's branch_pool is a 3 x 3 / stride 1 / pad 1 max pool.
 * Every BasicConv2d's BatchNorm (eps 1e-3, running statistics) is folded into its weights when they are set.  fp32
 * mode runs im2col and the exact SIMT GEMM; bf16 mode runs the convolutions as implicit GEMMs on wgmma (the stride-2
 * ones and the first over an im2col).  Features are fp32 in both modes.
 * Parameters are ONE flat fp32 device buffer in ds_inception_expected_weight() order: torchvision
 * Inception3(aux_logits=False) state-dict names and sizes in state-dict order, without fc.* and
 * num_batches_tracked (94 x {conv.weight, bn.weight, bn.bias, bn.running_mean, bn.running_var}). */
typedef struct ds_inception ds_inception;
typedef struct ds_inception_config {
  int32_t precision;        /* ds_precision: fp32 parity mode or bf16 tensor-core mode                          */
  int32_t capacity;         /* images one internal pass holds, 1 .. 256; larger batches run in passes of this size */
  int32_t device;           /* CUDA device ordinal                                                               */
  int32_t reserved[5];
} ds_inception_config;
#define DS_INCEPTION_FEATURES 2048
DS_API int ds_inception_create(const ds_inception_config* cfg, ds_inception** out);
DS_API int ds_inception_destroy(ds_inception* h);
DS_API int ds_inception_expected_weight_count(ds_inception* h);
DS_API int ds_inception_expected_weight(ds_inception* h, int index, const char** name, int64_t* numel);
/* DS_ERR_INVALID for NULL pointers or a parameter count other than the sum of the expected sizes. */
DS_API int ds_inception_set_weights(ds_inception* h, const float* flat_params_dev, int64_t count, void* stream);
/* images [batch, 3, 299, 299] fp32 NCHW in [0, 255] (already resized) -> features [batch, 2048] fp32, device
 * pointers; the detector's input is (x - 128) / 128.  An image's features do not depend on the other images of the
 * batch.  DS_ERR_STATE before ds_inception_set_weights; DS_ERR_INVALID for NULL pointers, batch < 0 or a size other
 * than 299 x 299. */
DS_API int ds_inception_features(ds_inception* h, const float* images_dev, int32_t batch, int32_t height, int32_t width,
                                 float* features_dev, void* stream);
/* One convolution alone, for unit tests, through the kernels, tensor maps and packing ds_inception_features runs in
 * `precision`: x [batch, height, width, cin] fp32 NHWC (rounded to bf16 in bf16 mode) -> relu(conv(x, W, b)) with
 * kernel kh x kw, stride 1 or 2 and padding (pad_h, pad_w), W [cout, cin, kh, kw] and b [cout] fp32, written to
 * channels [out_offset, out_offset + cout) of out [batch, Ho, Wo, out_pitch] fp32; the other channels keep their values
 * (rounded to bf16 in bf16 mode).  cout, out_pitch and out_offset are multiples of 8.  Synchronises `stream`. */
DS_API int ds_inception_test_conv(int32_t precision, const float* in_dev, int32_t batch, int32_t height, int32_t width,
                                  int32_t cin, int32_t cout, int32_t kh, int32_t kw, int32_t stride, int32_t pad_h,
                                  int32_t pad_w, const float* weight_dev, const float* bias_dev, float* out_dev,
                                  int32_t out_pitch, int32_t out_offset, void* stream);

/* FID statistics of fp32 features [n, d]: mean [d] and cov [d, d] = (X - mean)^T (X - mean) / (n - 1), fp64, as
 * np.mean / np.cov on float64-promoted features, in a fixed summation order.  DS_ERR_INVALID for NULL pointers,
 * n < 2 or d < 1.  Stateless. */
DS_API int ds_feature_stats(const float* feats_dev, int32_t n, int32_t d, double* mean_dev, double* cov_dev,
                            void* stream);
/* KID terms of `subsets` subsets of m rows (clean-fid's kernel_distance): for subset s, x = fake[idx_fake[s * m ..]],
 * y = real[idx_real[s * m ..]] (int64 indices), a = (x x^T / d + 1)^3 + (y y^T / d + 1)^3, b = (x y^T / d + 1)^3 and
 * terms[s] = (sum a - sum diag a) / (m - 1) - 2 sum b / m, fp64 (KID = sum of terms / subsets / m).  Each term is
 * deterministic and independent of the other subsets of the call.  The indices are checked on the device first (the
 * call synchronises `stream` for that); DS_ERR_INVALID for one outside its set, NULL pointers, m < 2, m above either
 * set's size, subsets < 1 or d < 1.  Scratch is allocated on `stream`. */
DS_API int ds_kid_terms(const float* real_dev, int32_t n_real, const float* fake_dev, int32_t n_fake, int32_t d,
                        const int64_t* idx_fake_dev, const int64_t* idx_real_dev, int32_t subsets, int32_t m,
                        double* terms_dev, void* stream);

/* Manifold metrics (improved_precision_recall.py:196-256) on fp64 features [rows, d] (row-major, any d >= 1), without
 * an N x N matrix: distances are sqrt(max(0, (|x|^2 - 2 x.y) + |y|^2)) in fp64 on the fp64 tensor cores, and
 * `clamped_dev` (int64 on the device, may be NULL) receives how many squared distances were negative and set to 0,
 * as the reference prints.  Stateless; scratch is allocated on `stream`. */
#define DS_MANIFOLD_MAX_K 16
/* out [n, m] = distances of x [n, d] to y [m, d] (for small inputs and tests). */
DS_API int ds_manifold_distances(const double* x_dev, int32_t n, const double* y_dev, int32_t m, int32_t d,
                                 double* out_dev, int64_t* clamped_dev, void* stream);
/* radii [n]: radius i is the (k+1)-th smallest distance of row i of x's self-distance matrix, the ~0 distance to
 * itself counted (distances2radii).  DS_ERR_INVALID for NULL pointers, k outside [1, DS_MANIFOLD_MAX_K], n <= k or
 * d < 1. */
DS_API int ds_manifold_radii(const double* x_dev, int32_t n, int32_t d, int32_t k, double* radii_dev,
                             int64_t* clamped_dev, void* stream);
/* One pass over reference x subject pairs (compute_metric and realism, strict <):
 *   subj_covered [n_subj] uint8: 1 when some reference i has dist(ref_i, subj_j) < ref_radii[i] (precision flags)
 *   ref_covered  [n_ref]  uint8: 1 when some subject j has dist(ref_i, subj_j) < subj_radii[j] (recall flags)
 *   realism      [n_subj] fp64:  max_i ref_radii[i] / (dist(ref_i, subj_j) + 1e-6)
 * Each output may be NULL; ref_covered needs subj_radii.  DS_ERR_INVALID for NULL required pointers or a count < 1. */
DS_API int ds_manifold_cover(const double* ref_dev, const double* ref_radii_dev, int32_t n_ref, const double* subj_dev,
                             const double* subj_radii_dev, int32_t n_subj, int32_t d, uint8_t* subj_covered_dev,
                             uint8_t* ref_covered_dev, double* realism_dev, int64_t* clamped_dev, void* stream);

/* ---- introspection / debugging ------------------------------------------------------------ */
/* The encoder's kNN (k = 16, the point itself included): x [batch, num_points, channels] fp32 -> idx [batch,
 * num_points, 16] int32, ascending squared distance sum_c (x_i - x_j)^2 in fp32, ties broken by the lower index.
 * channels in {3, 64, 128}, num_points >= 16. */
DS_API int ds_knn(const float* x_dev, int32_t batch, int32_t num_points, int32_t channels, int32_t* idx_dev,
                  void* stream);
/* Parity aid: idx_dev [3, batch, num_points, 16] int32 (the xyz, 64-d and 128-d stages) replaces the shape
 * auto-encoder's own kNN in every following forward / training step until it is set to NULL.  The pointer must stay
 * valid and hold indices for the batch size of each call. */
DS_API int ds_shape_ae_set_knn(ds_shape_ae* h, const int32_t* idx_dev);
/* The three stages' kNN indices [3, batch, num_points, 16] of the last kept pass.  DS_ERR_INVALID when there is none. */
DS_API int ds_shape_ae_get_knn(ds_shape_ae* h, int32_t* idx_dev, void* stream);
/* Human-readable op list of the step program (works without a device when h == NULL: builds the plan
 * for `cfg` on the host only).  Returns bytes written (excluding NUL) or a negative status. */
DS_API int ds_plan_describe(const ds_config* cfg, char* buf, int64_t buf_len);
/* The same plan (ops, buffer table, weight-packing recipes) as JSON, for host-side verification of the
 * program against the oracle without a GPU.  no_reuse != 0: one buffer per op output. */
DS_API int ds_plan_export_json(const ds_config* cfg, int32_t no_reuse, char* buf, int64_t buf_len);
/* After a forward with taps enabled, copy the named intermediate [B*N, width] to host as fp32. */
DS_API int ds_enable_taps(ds_handle* h, int32_t on);
DS_API int ds_read_tap(ds_handle* h, const char* name, float* host_out, int64_t capacity, int32_t* rows, int32_t* width);
/* Kernel launches issued by this handle since creation (ours only; no library kernels exist). */
DS_API int64_t ds_launch_count(ds_handle* h);
/* How many times ds_sample_loop had to capture + instantiate its step graph (it is cached across calls whose
 * batch / flags / injected-buffer pointers agree; seeds and shard offsets live in device memory). */
DS_API int64_t ds_graph_build_count(ds_handle* h);
/* Per-op device time of one forward (CUDA events around each op; profiling aid, not a bench number).
 * Writes up to `cap` entries of (name, microseconds). Returns op count. */
DS_API int ds_profile_ops(ds_handle* h, int32_t batch, char* names_buf, int64_t names_len, float* usec, int32_t cap);
/* One bf16 VGG16 convolution alone, for unit tests: x [batch, height, width, cin] fp32 NHWC, rounded to bf16 ->
 * relu(conv3x3(x, W, b), pad 1) (-> 2 x 2 max-pool when pool != 0) [batch, height (/ 2), width (/ 2), cout] fp32,
 * computed by the kernel ds_vgg_features runs (W [cout, cin, 3, 3] fp32, rounded to bf16 when packed; b [cout] fp32).
 * cin is 3 (the first layer's im2col path) or a multiple of 64; cout is 64 or a multiple of 128; pooled sides are
 * even.  Synchronises `stream`. */
DS_API int ds_vgg_test_conv(const float* in_dev, int32_t batch, int32_t height, int32_t width, int32_t cin,
                            int32_t cout, int32_t pool, const float* weight_dev, const float* bias_dev, float* out_dev,
                            void* stream);
/* Standalone GEMM for unit tests: D[M,N] = A[M,K] * W[N,K]^T (+bias), bf16 in / bf16 out via the selected
 * backend. Device pointers. */
DS_API int ds_test_gemm_bf16(int backend, const void* a_dev, const void* w_dev, const float* bias_dev, void* d_dev,
                      int32_t M, int32_t N, int32_t K, int32_t act, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* DIFFUSCENE_B200_H_ */
