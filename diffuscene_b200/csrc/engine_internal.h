// Internal definitions shared by the engine translation units (engine.cu: handle, sampling, inference-side C ABI;
// train.cu: the training step).  Not part of the public interface.
#pragma once
#include <math.h>
#include <stdarg.h>
#include <stdio.h>
#include <string.h>

#include <algorithm>
#include <map>
#include <string>
#include <vector>

#include "kernels.cuh"
#include "plan.h"

namespace ds {
int tc_error_flag();
void init_pointwise_attrs();
}
using namespace ds;

int fail(int code, const char* fmt, ...);      // engine.cu: records the message for ds_last_error()
#define CK(call)                                                                                         \
  do {                                                                                                   \
    cudaError_t e_ = (call);                                                                             \
    if (e_ != cudaSuccess)                                                                               \
      return fail(DS_ERR_CUDA, "%s failed: %s (%s:%d)", #call, cudaGetErrorString(e_), __FILE__, __LINE__); \
  } while (0)

// engine.cu.  require_device(): DS_ERR_NO_DEVICE unless a CUDA device exists.  open_device(): that, then the index is
// in range, the device is made current and is an sm_90 part.  Both return 0 or the fail() code.
int require_device();
int open_device(int device);

// Parameter inventory of a model handle in state-dict order: each tensor's name, size and offset into the flat fp32
// parameter buffer the handle takes.
struct WeightTable {
  std::vector<std::string> names;
  std::vector<int64_t> numel, off;
  int64_t total = 0;

  int add(const std::string& name, int64_t n) {
    names.push_back(name);
    numel.push_back(n);
    off.push_back(total);
    total += n;
    return int(names.size()) - 1;
  }
  int count() const { return int(names.size()); }
  int get(int index, const char** name, int64_t* n) const {
    if (!name || !n) return fail(DS_ERR_INVALID, "null argument");
    if (index < 0 || index >= count()) return fail(DS_ERR_INVALID, "weight index %d out of range", index);
    *name = names[index].c_str();
    *n = numel[index];
    return 0;
  }
};

// S_POST_LOGVAR .. S_LOG_1MAC are the variational-bound tables of ds_set_vlb_schedule; ds_set_schedule fills the rest
enum { S_SQRT_AC = 0, S_SQRT_1MAC, S_SQRT_RECIP, S_SQRT_RECIPM1, S_COEF1, S_COEF2, S_SIGMA, S_AC, S_LW, S_NEG_1MAC,
       S_NEG_RECIPM1, S_ZERO, S_ONE, S_POST_LOGVAR, S_MODEL_LOGVAR, S_LOG_1MAC, S_COUNT };
constexpr int S_VLB_FIRST = S_POST_LOGVAR;

struct TrainState;
void train_state_destroy(TrainState* t);      // train.cu

struct ds_handle {
  ds_config cfg;
  Plan plan;
  bool taps = false;
  bool bf16_mode = false, use_tc = false;
  size_t esz = 4;
  cudaStream_t own_stream = nullptr;
  std::map<std::string, std::vector<float>> host_w;
  bool committed = false;
  // packed weights
  char* warena = nullptr;
  std::vector<size_t> w_off;
  float* varena = nullptr;
  std::vector<size_t> v_off;
  // fp32 conditioning path
  float *time_w1 = nullptr, *time_b1 = nullptr, *time_w3 = nullptr, *time_b3 = nullptr, *time_wall = nullptr,
        *time_ball = nullptr, *time_table = nullptr, *sin_freq = nullptr;
  float *ctx_wall = nullptr, *ctx_ball = nullptr, *ctx_table = nullptr;
  int ctx_rows = 0, ctx_batch = 0;
  bool ctx_shared = false, ctx_set = false;
  std::vector<float*> kv_w;
  float* xctx = nullptr;
  int xctx_batch = 0, xctx_cap = 0;
  // activations
  int cap_scenes = 0, rows_cap = 0;
  std::vector<void*> bufs;
  std::vector<TcGemmPlan*> tc;
  std::vector<LnGemmPlan*> lnp;      // fused GEMM + LayerNorm ops
  std::vector<AttnQkvPlan*> atp;     // fused LayerNorm + to_qkv + linear-attention ops
  float* attn_cs = nullptr;          // [n wmats][384] column sums of the gain-folded to_qkv weights (rows of unused matrices are 0)
  int* t_dev = nullptr;
  float* x_state = nullptr;      // [cap, N, d] running sample
  float* x_tmp = nullptr;        // [cap, N, d] scratch (q_sample / host staging)
  int64_t* t64_tmp = nullptr;
  float* loss_parts = nullptr;
  // schedule
  int T = 0, mean_type = DS_MEAN_V;
  std::vector<float> sched_host[S_COUNT];
  float* sched_dev[S_COUNT] = {nullptr};
  StepCoef* coef_dev = nullptr;
  int coef_cap = 0;
  StepState* state_dev = nullptr;
  int64_t launches = 0;
  // instantiated step graph, reused across ds_sample_loop calls whose captured parameters agree (batch, flags,
  // injected-buffer pointers); seed / scene offset / coefficients live in device memory and are not captured
  struct GraphKey {
    int batch = -1, clip = 0, num_partial = 0, plan_gen = 0;
    const void *noise = nullptr, *partial = nullptr, *partial_noise = nullptr;
    cudaStream_t stream = nullptr;
    bool operator==(const GraphKey& o) const {
      return batch == o.batch && clip == o.clip && num_partial == o.num_partial && plan_gen == o.plan_gen &&
             noise == o.noise && partial == o.partial && partial_noise == o.partial_noise && stream == o.stream;
    }
  } gkey;
  cudaGraphExec_t gexec = nullptr;
  int64_t g_launches = 0;     // kernel launches inside one replay
  int plan_gen = 0;           // bumped whenever buffers / tensor maps / tables are rebuilt
  int64_t graph_builds = 0;
  // variational bound (ds_vlb_loop): its own step graph, coefficient table and staging buffers, so that a VLB call
  // neither evicts nor rebuilds the sampling graph above.  The key holds every pointer the capture bakes in that
  // plan_gen does not cover.
  bool vlb_set = false;                 // ds_set_vlb_schedule() has been called
  struct VlbKey {
    int batch = -1, clip = 0, plan_gen = 0;
    const void *noise = nullptr, *x0 = nullptr, *vb = nullptr, *mse = nullptr, *coef = nullptr, *lv1 = nullptr,
               *lv2 = nullptr;
    cudaStream_t stream = nullptr;
    bool operator==(const VlbKey& o) const {
      return batch == o.batch && clip == o.clip && plan_gen == o.plan_gen && noise == o.noise && x0 == o.x0 &&
             vb == o.vb && mse == o.mse && coef == o.coef && lv1 == o.lv1 && lv2 == o.lv2 && stream == o.stream;
    }
  } vkey;
  cudaGraphExec_t vexec = nullptr;
  int64_t v_launches = 0;
  StepCoef* vlb_coef = nullptr;         // [T] per-step coefficients of the VLB loop (step i <-> t = T-1-i)
  float *vlb_x0 = nullptr, *vlb_vb = nullptr, *vlb_mse = nullptr;      // [cap, N, d], [cap, T], [cap, T]
  int vlb_cap = 0;
  TrainState* train = nullptr;      // lazily created by ds_train_* (train.cu)
};
void drop_graph(ds_handle* h);

