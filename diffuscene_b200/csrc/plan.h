// Host-side step program ("plan") of the denoiser: an ordered op list over token-major activation
// buffers, plus the recipes that assemble packed weight matrices from reference state-dict tensors.
//
// The op order restates Unet1D.forward (reference scene_synthesis/networks/denoise_net.py:507-593) with
// the legal hoists of SURVEY.md A.5 applied: weight standardisation folded at load time, time- and
// context-FiLM projections looked up from precomputed tables, the three encoder / decoder MLPs batched
// into block-structured GEMMs, and U-Net skip concatenations served as two-operand GEMMs.
// Pure C++ (no CUDA): also used by ds_plan_describe() on machines without a GPU.
#pragma once
#include <stdint.h>

#include <map>
#include <string>
#include <vector>

#include "../../include/diffuscene_b200.h"

namespace ds {

enum OpKind {
  OP_PACK = 0,      // x_t fp32 [M, d] -> zero-padded activation [M, kin_pad]
  OP_GEMM,          // out = act([in0|in1] W^T + b) (+res)
  OP_GN,            // GroupNorm + affine (+FiLM) + SiLU (+res)
  OP_LN,            // channel LayerNorm * g (+res)
  OP_LINATTN,       // linear-attention core on qkv [M, 384] -> [M, 128]
  OP_ATTN,          // softmax-attention core
  OP_XATTN,         // cross linear-attention apply (q [M,128] x precomputed text context)
  OP_GEMM_GN,       // GEMM with the GroupNorm + affine (+FiLM) + SiLU (+res) epilogue fused (tensor-core backend only)
  OP_GEMM_LN,       // GEMM with the channel LayerNorm (gain `gamma`) (+res) epilogue fused (fuse_level >= 4; no sm_90a kernel, the engine runs level 1)
  OP_LN_QKV_ATTN,   // channel LayerNorm + to_qkv + linear-attention core in one kernel (fuse_level >= 4, N = 12): the
                    // weight matrix carries the LayerNorm gain (WRecipe::scale_k), out = o [M, 128]
  OP_ACT,           // train mode only: out[:, out_col : out_col + N] = act(in0) (GELU / SiLU as their own op, pre-activation kept)
};

struct Slice { int buf = -1; int col = 0; int k = 0; };

struct Op {
  int kind = 0;
  std::string name;
  Slice in0, in1;          // GEMM operands / the input of pointwise ops (in0)
  int out = -1, out_col = 0;
  int res = -1;            // residual buffer (full width C) or -1
  int w = -1, b = -1;      // weight matrix id / fp32 vector id (bias, or LN g)
  int gamma = -1, beta = -1;
  int N = 0;               // GEMM output width / pointwise width
  int act = 0;
  int film = 0;            // FilmMode: 0 none, 1 time, 2 context
  int film_blk = 0;        // index into the time / context FiLM block list
  int xlayer = 0;          // cross-attention layer index
};

struct WPiece { std::string name; int row_off, col_off, rows, cols; };
struct WRecipe {           // packed matrix [N, K] in the activation dtype
  int N = 0, K = 0;
  bool ws = false;         // weight-standardise each piece (denoise_net.py:83-89)
  std::string scale_k;     // optional [K] vector multiplied into the columns (a LayerNorm gain folded into the next conv)
  std::vector<WPiece> pieces;
};
struct VPiece { std::string name; int off, n; };
struct VRecipe {           // fp32 vector of length n; pieces landing on the same offsets are summed
  int n = 0;
  std::vector<VPiece> pieces;
};

struct Plan {
  ds_config cfg;
  int C = 0, G = 0, d = 0, kin_pad = 0, dpad = 0;
  std::vector<Op> ops;
  std::vector<int> buf_width;
  std::vector<WRecipe> wmats;
  std::vector<VRecipe> vecs;
  std::vector<std::string> time_blocks;      // resblock names whose FiLM comes from the time table
  std::vector<std::string> ctx_blocks;       // ... from the context table
  std::vector<std::string> xattn_layers;     // cross-attention layer names (to_kv recipes)
  int out_buf = -1;                          // decoder output [M, dpad]
  std::map<std::string, int64_t> expected;   // weight name -> numel
  std::vector<std::string> expected_order;
  std::string error;
};

bool build_plan(const ds_config& cfg, bool no_reuse, Plan* plan);
std::string describe_plan(const Plan& p);
std::string export_plan_json(const Plan& p);

}  // namespace ds
