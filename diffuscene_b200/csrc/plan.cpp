// Plan construction: see plan.h.  Reference for the op order: denoise_net.py:507-593.
#include "plan.h"

#include <stdio.h>

#include <sstream>

namespace ds {
namespace {

struct Builder {
  Plan* p;
  bool no_reuse;
  bool fuse = false;
  bool fuse_ln = false;     // to_out + LayerNorm + residual of the attention wrappers as one op
  bool fuse_attn = false;   // LayerNorm + to_qkv + linear-attention core as one op
  bool train = false;       // activations as separate ops (the backward pass needs the pre-activation)
  std::map<int, int> zbuf;  // train: output buffer -> buffer of the same width holding the pre-activations
  std::vector<int> refs;
  std::map<int, std::vector<int>> free_by_width;
  int C;

  int new_buf(int width) {
    auto& fl = free_by_width[width];
    if (!no_reuse && !fl.empty()) {
      int id = fl.back();
      fl.pop_back();
      refs[id] = 1;
      return id;
    }
    p->buf_width.push_back(width);
    refs.push_back(1);
    return int(p->buf_width.size()) - 1;
  }
  void retain(int id) { refs[id]++; }
  void release(int id) {
    if (--refs[id] == 0) free_by_width[p->buf_width[id]].push_back(id);
  }

  void expect(const std::string& name, int64_t numel) {
    if (!p->expected.count(name)) {
      p->expected[name] = numel;
      p->expected_order.push_back(name);
    }
  }
  int wmat(const WRecipe& r) {
    for (auto& pc : r.pieces) expect(pc.name, int64_t(pc.rows) * pc.cols);
    p->wmats.push_back(r);
    return int(p->wmats.size()) - 1;
  }
  int wsingle(const std::string& name, int N, int K, bool ws = false) {
    WRecipe r;
    r.N = N; r.K = K; r.ws = ws;
    r.pieces.push_back({name, 0, 0, N, K});
    return wmat(r);
  }
  int vec(const VRecipe& r) {
    for (auto& pc : r.pieces) expect(pc.name, pc.n);
    p->vecs.push_back(r);
    return int(p->vecs.size()) - 1;
  }
  int vsingle(const std::string& name, int n) {
    VRecipe r;
    r.n = n;
    r.pieces.push_back({name, 0, n});
    return vec(r);
  }

  void gemm(const std::string& name, Slice a0, Slice a1, int w, int b, int N, int act, int res, int out, int out_col) {
    if (train && act != 0) {
      if (!zbuf.count(out)) zbuf[out] = new_buf(p->buf_width[out]);
      const int zb = zbuf[out];
      gemm(name + ".pre", a0, a1, w, b, N, 0, -1, zb, out_col);
      Op o;
      o.kind = OP_ACT; o.name = name; o.in0 = Slice{zb, out_col, N}; o.out = out; o.out_col = out_col; o.N = N; o.act = act;
      o.res = res;
      p->ops.push_back(o);
      return;
    }
    Op o;
    o.kind = OP_GEMM; o.name = name; o.in0 = a0; o.in1 = a1; o.w = w; o.b = b; o.N = N; o.act = act; o.res = res;
    o.out = out; o.out_col = out_col;
    p->ops.push_back(o);
  }
  Slice full(int buf) { return Slice{buf, 0, p->buf_width[buf]}; }

  // ResnetBlock (denoise_net.py:178-206). `a0`(+`a1`) is the (possibly concatenated) input; the caller keeps
  // ownership of the inputs.  film: 1 time, 2 context.
  int resblock(const std::string& name, Slice a0, Slice a1, int film) {
    const int cin = a0.k + a1.k;
    int film_blk;
    if (film == 1) {
      film_blk = int(p->time_blocks.size());
      p->time_blocks.push_back(name);
      expect(name + ".mlp.1.weight", int64_t(2 * C) * (4 * C));
      expect(name + ".mlp.1.bias", 2 * C);
    } else {
      film_blk = int(p->ctx_blocks.size());
      p->ctx_blocks.push_back(name);
      expect(name + ".mlp.1.weight", int64_t(2 * C) * p->cfg.cond_dim);
      expect(name + ".mlp.1.bias", 2 * C);
    }
    if (fuse) {
      // Block = conv -> GroupNorm -> FiLM -> SiLU as ONE kernel (GEMM with the GroupNorm epilogue)
      int h1 = new_buf(C);
      {
        Op o;
        o.kind = OP_GEMM_GN; o.name = name + ".block1"; o.in0 = a0; o.in1 = a1; o.out = h1; o.N = C;
        o.w = wsingle(name + ".block1.proj.weight", C, cin, true);
        o.b = vsingle(name + ".block1.proj.bias", C);
        o.gamma = vsingle(name + ".block1.norm.weight", C);
        o.beta = vsingle(name + ".block1.norm.bias", C);
        o.film = film; o.film_blk = film_blk;
        p->ops.push_back(o);
      }
      int rs;
      if (cin != C) {
        rs = new_buf(C);
        gemm(name + ".res_conv", a0, a1, wsingle(name + ".res_conv.weight", C, cin),
             vsingle(name + ".res_conv.bias", C), C, 0, -1, rs, 0);
      } else {
        rs = a0.buf;
        retain(rs);
      }
      int out = new_buf(C);
      {
        Op o;
        o.kind = OP_GEMM_GN; o.name = name; o.in0 = full(h1); o.out = out; o.N = C; o.res = rs;
        o.w = wsingle(name + ".block2.proj.weight", C, C, true);
        o.b = vsingle(name + ".block2.proj.bias", C);
        o.gamma = vsingle(name + ".block2.norm.weight", C);
        o.beta = vsingle(name + ".block2.norm.bias", C);
        p->ops.push_back(o);
      }
      release(h1);
      release(rs);
      return out;
    }
    int t1 = new_buf(C);
    gemm(name + ".block1.proj", a0, a1, wsingle(name + ".block1.proj.weight", C, cin, true),
         vsingle(name + ".block1.proj.bias", C), C, 0, -1, t1, 0);
    int h1 = new_buf(C);
    {
      Op o;
      o.kind = OP_GN; o.name = name + ".block1"; o.in0 = full(t1); o.out = h1; o.N = C;
      o.gamma = vsingle(name + ".block1.norm.weight", C);
      o.beta = vsingle(name + ".block1.norm.bias", C);
      o.film = film; o.film_blk = film_blk;
      p->ops.push_back(o);
    }
    release(t1);
    int t2 = new_buf(C);
    gemm(name + ".block2.proj", full(h1), Slice(), wsingle(name + ".block2.proj.weight", C, C, true),
         vsingle(name + ".block2.proj.bias", C), C, 0, -1, t2, 0);
    release(h1);
    int rs;
    if (cin != C) {
      rs = new_buf(C);
      gemm(name + ".res_conv", a0, a1, wsingle(name + ".res_conv.weight", C, cin), vsingle(name + ".res_conv.bias", C),
           C, 0, -1, rs, 0);
    } else {
      rs = a0.buf;
      retain(rs);
    }
    int out = new_buf(C);
    {
      Op o;
      o.kind = OP_GN; o.name = name; o.in0 = full(t2); o.out = out; o.N = C; o.res = rs;
      o.gamma = vsingle(name + ".block2.norm.weight", C);
      o.beta = vsingle(name + ".block2.norm.bias", C);
      p->ops.push_back(o);
    }
    release(t2);
    release(rs);
    return out;
  }

  void ln(const std::string& name, int in, int out, int g, int res) {
    Op o;
    o.kind = OP_LN; o.name = name; o.in0 = full(in); o.out = out; o.N = C; o.b = g; o.res = res;
    p->ops.push_back(o);
  }

  // to_out = Sequential(Conv1d(hidden, dim, 1), LayerNorm(dim)) followed by the Residual add (denoise_net.py:214-217,
  // 234-235, 39-45): one GEMM with the LayerNorm epilogue at fuse_level >= 4, a GEMM and a LayerNorm op otherwise
  int to_out_ln(const std::string& name, int o, int x, int H) {
    int out = new_buf(C);
    if (fuse_ln) {
      Op op;
      op.kind = OP_GEMM_LN; op.name = name; op.in0 = full(o); op.out = out; op.N = C; op.res = x;
      op.w = wsingle(name + ".fn.fn.to_out.0.weight", C, H);
      op.b = vsingle(name + ".fn.fn.to_out.0.bias", C);
      op.gamma = vsingle(name + ".fn.fn.to_out.1.g", C);
      p->ops.push_back(op);
      return out;
    }
    int y = new_buf(C);
    gemm(name + ".to_out", full(o), Slice(), wsingle(name + ".fn.fn.to_out.0.weight", C, H),
         vsingle(name + ".fn.fn.to_out.0.bias", C), C, 0, -1, y, 0);
    ln(name, y, out, vsingle(name + ".fn.fn.to_out.1.g", C), x);
    release(y);
    return out;
  }

  // Residual(PreNorm(LinearAttention)) (denoise_net.py:208-235) / Attention for the mid block (:237-259)
  int self_attn(const std::string& name, int x, bool softmax_kind) {
    const int H = 128;
    int o;
    if (fuse_attn && !softmax_kind) {
      o = new_buf(H);
      Op op;
      op.kind = OP_LN_QKV_ATTN; op.name = name + ".core"; op.in0 = full(x); op.out = o; op.N = H;
      WRecipe r;
      r.N = 3 * H; r.K = C; r.scale_k = name + ".fn.norm.g";
      r.pieces.push_back({name + ".fn.fn.to_qkv.weight", 0, 0, 3 * H, C});
      expect(r.scale_k, C);
      op.w = wmat(r);
      p->ops.push_back(op);
    } else {
      int n1 = new_buf(C);
      ln(name + ".prenorm", x, n1, vsingle(name + ".fn.norm.g", C), -1);
      int qkv = new_buf(3 * H);
      gemm(name + ".to_qkv", full(n1), Slice(), wsingle(name + ".fn.fn.to_qkv.weight", 3 * H, C), -1, 3 * H, 0, -1, qkv,
           0);
      release(n1);
      o = new_buf(H);
      {
        Op op;
        op.kind = softmax_kind ? OP_ATTN : OP_LINATTN;
        op.name = name + ".core"; op.in0 = full(qkv); op.out = o; op.N = H;
        p->ops.push_back(op);
      }
      release(qkv);
    }
    int out;
    if (softmax_kind) {
      out = new_buf(C);
      gemm(name, full(o), Slice(), wsingle(name + ".fn.fn.to_out.weight", C, H), vsingle(name + ".fn.fn.to_out.bias", C),
           C, 0, x, out, 0);
    } else {
      out = to_out_ln(name, o, x, H);
    }
    release(o);
    return out;
  }

  // ResidualCross(PreNormCross(LinearAttentionCross)) (denoise_net.py:261-297)
  int cross_attn(const std::string& name, int x) {
    const int H = 128;
    const int layer = int(p->xattn_layers.size());
    p->xattn_layers.push_back(name);
    expect(name + ".fn.fn.to_kv.weight", int64_t(2 * H) * p->cfg.text_dim);
    int n1 = new_buf(C);
    ln(name + ".prenorm", x, n1, vsingle(name + ".fn.norm.g", C), -1);
    int q = new_buf(H);
    gemm(name + ".to_q", full(n1), Slice(), wsingle(name + ".fn.fn.to_q.weight", H, C), -1, H, 0, -1, q, 0);
    release(n1);
    int o = new_buf(H);
    {
      Op op;
      op.kind = OP_XATTN; op.name = name + ".core"; op.in0 = full(q); op.out = o; op.N = H; op.xlayer = layer;
      p->ops.push_back(op);
    }
    release(q);
    int out = to_out_ln(name, o, x, H);
    release(o);
    return out;
  }
};

int round_up(int a, int b) { return (a + b - 1) / b * b; }

}  // namespace

bool build_plan(const ds_config& cfg, bool no_reuse, Plan* plan) {
  Plan& P = *plan;
  P = Plan();
  P.cfg = cfg;
  const int C = cfg.dim;
  P.C = C;
  char msg[256];
  if (C <= 0 || C % 128 != 0 || C > 1024) {
    snprintf(msg, sizeof msg, "dim must be a multiple of 128 in (0, 1024], got %d", C);
    P.error = msg;
    return false;
  }
  if (cfg.n_stages < 1 || cfg.n_stages > 8 || cfg.num_objects < 1 || cfg.num_objects > 64 || cfg.cond_dim < 1 ||
      cfg.num_timesteps < 1) {
    P.error = "invalid n_stages / num_objects (1..64) / cond_dim / num_timesteps";
    return false;
  }
  struct Attr { const char* enc; const char* dec; int k; };
  std::vector<Attr> attrs;
  const int bbox = cfg.translation_dim + cfg.size_dim + cfg.angle_dim;
  if (cfg.seperate_all) {
    if (bbox <= 0 || cfg.class_dim <= 0) {
      P.error = "seperate_all needs positive bbox and class dims";
      return false;
    }
    attrs.push_back({"bbox_embedf", "bbox_hidden2output", bbox});
    attrs.push_back({"class_embedf", "class_hidden2output", cfg.class_dim});
    if (cfg.objectness_dim > 0) attrs.push_back({"objectness_embedf", "objectness_hidden2output", cfg.objectness_dim});
    if (cfg.objfeat_dim > 0) attrs.push_back({"objfeat_embedf", "objfeat_hidden2output", cfg.objfeat_dim});
    P.d = bbox + cfg.class_dim + cfg.objectness_dim + cfg.objfeat_dim;
  } else {
    if (cfg.channels <= 0) {
      P.error = "channels must be positive";
      return false;
    }
    P.d = cfg.channels;
  }
  const int G = int(attrs.size());
  P.G = G;
  P.kin_pad = round_up(P.d, 64);
  P.dpad = round_up(P.d, 128);

  Builder b;
  b.p = &P;
  b.no_reuse = no_reuse;
  b.C = C;
  b.train = cfg.train != 0;
  b.fuse = !b.train && cfg.fuse_level >= 1 && cfg.precision == DS_PREC_BF16 && cfg.gemm_backend != DS_GEMM_SIMT && C == 512 &&
           128 / cfg.num_objects <= 10;   // GroupNorm groups of 64 channels (k_gemm_wg); >= 12 objects per scene

  b.fuse_ln = b.fuse && cfg.fuse_level >= 4 && C == 512;
  b.fuse_attn = b.fuse && cfg.fuse_level >= 5 && C == 512 && (cfg.num_objects == 12 || cfg.num_objects == 21);

  // ---- input + encoder ----
  int xin = b.new_buf(P.kin_pad);
  {
    Op o;
    o.kind = OP_PACK; o.name = "pack"; o.out = xin; o.N = P.kin_pad;
    P.ops.push_back(o);
  }
  int x;
  if (cfg.seperate_all) {
    // layer 0 of the G attribute MLPs as one block-structured GEMM over the raw attribute columns
    WRecipe w0; w0.N = G * C; w0.K = P.kin_pad;
    VRecipe b0; b0.n = G * C;
    int col = 0;
    for (int g = 0; g < G; ++g) {
      w0.pieces.push_back({std::string(attrs[g].enc) + ".0.weight", g * C, col, C, attrs[g].k});
      b0.pieces.push_back({std::string(attrs[g].enc) + ".0.bias", g * C, C});
      col += attrs[g].k;
    }
    int e1 = b.new_buf(G * C);
    b.gemm("enc.l0", b.full(xin), Slice(), b.wmat(w0), b.vec(b0), G * C, 1, -1, e1, 0);
    b.release(xin);
    int e2 = b.new_buf(G * 2 * C);
    for (int g = 0; g < G; ++g) {
      std::string n = attrs[g].enc;
      b.gemm("enc.l1." + n, Slice{e1, g * C, C}, Slice(), b.wsingle(n + ".2.weight", 2 * C, C),
             b.vsingle(n + ".2.bias", 2 * C), 2 * C, 1, -1, e2, g * 2 * C);
    }
    b.release(e1);
    // layer 2 of all branches + the sum over branches (denoise_net.py:525) as one K-concatenated GEMM
    WRecipe w2; w2.N = C; w2.K = G * 2 * C;
    VRecipe b2; b2.n = C;
    for (int g = 0; g < G; ++g) {
      w2.pieces.push_back({std::string(attrs[g].enc) + ".4.weight", 0, g * 2 * C, C, 2 * C});
      b2.pieces.push_back({std::string(attrs[g].enc) + ".4.bias", 0, C});
    }
    int enc = b.new_buf(C);
    b.gemm("encoder", b.full(e2), Slice(), b.wmat(w2), b.vec(b2), C, 0, -1, enc, 0);
    b.release(e2);
    x = b.new_buf(C);
    b.gemm("init_conv", b.full(enc), Slice(), b.wsingle("init_conv.weight", C, C), b.vsingle("init_conv.bias", C), C, 0,
           -1, x, 0);
    b.release(enc);
  } else {
    WRecipe w0; w0.N = C; w0.K = P.kin_pad;
    w0.pieces.push_back({"init_conv.weight", 0, 0, C, P.d});
    x = b.new_buf(C);
    b.gemm("init_conv", b.full(xin), Slice(), b.wmat(w0), b.vsingle("init_conv.bias", C), C, 0, -1, x, 0);
    b.release(xin);
  }
  const int r = x;
  b.retain(r);      // kept for the final concat (denoise_net.py:534,573)

  b.expect("time_mlp.1.weight", int64_t(4 * C) * C);
  b.expect("time_mlp.1.bias", 4 * C);
  b.expect("time_mlp.3.weight", int64_t(4 * C) * (4 * C));
  b.expect("time_mlp.3.bias", 4 * C);

  auto step = [&](int& cur, int next) {   // replace the running activation
    b.release(cur);
    cur = next;
  };

  std::vector<int> skips;
  for (int i = 0; i < cfg.n_stages; ++i) {
    std::string d = "downs." + std::to_string(i);
    step(x, b.resblock(d + ".0", b.full(x), Slice(), 2));
    step(x, b.resblock(d + ".1", b.full(x), Slice(), 1));
    b.retain(x);
    skips.push_back(x);
    if (cfg.text_condition) step(x, b.cross_attn(d + ".2", x));
    step(x, b.resblock(d + ".3", b.full(x), Slice(), 1));
    step(x, b.self_attn(d + ".4", x, false));
    b.retain(x);
    skips.push_back(x);
    if (i == cfg.n_stages - 1) {
      int y = b.new_buf(C);
      b.gemm(d + ".5", b.full(x), Slice(), b.wsingle(d + ".5.weight", C, C), b.vsingle(d + ".5.bias", C), C, 0, -1, y, 0);
      step(x, y);
    }
  }
  step(x, b.resblock("mid_block0", b.full(x), Slice(), 2));
  step(x, b.resblock("mid_block1", b.full(x), Slice(), 1));
  if (cfg.text_condition) step(x, b.cross_attn("mid_attn_cross", x));
  step(x, b.self_attn("mid_attn", x, true));
  step(x, b.resblock("mid_block2", b.full(x), Slice(), 1));
  for (int i = 0; i < cfg.n_stages; ++i) {
    std::string u = "ups." + std::to_string(i);
    step(x, b.resblock(u + ".0", b.full(x), Slice(), 2));
    int s1 = skips.back();
    skips.pop_back();
    step(x, b.resblock(u + ".1", b.full(x), b.full(s1), 1));
    b.release(s1);
    if (cfg.text_condition) step(x, b.cross_attn(u + ".2", x));
    int s2 = skips.back();
    skips.pop_back();
    step(x, b.resblock(u + ".3", b.full(x), b.full(s2), 1));
    b.release(s2);
    step(x, b.self_attn(u + ".4", x, false));
    if (i == cfg.n_stages - 1) {
      int y = b.new_buf(C);
      b.gemm(u + ".5", b.full(x), Slice(), b.wsingle(u + ".5.weight", C, C), b.vsingle(u + ".5.bias", C), C, 0, -1, y, 0);
      step(x, y);
    }
  }
  step(x, b.resblock("final_res_block", b.full(x), b.full(r), 1));
  b.release(r);

  // ---- decoder ----
  int dec = b.new_buf(P.dpad);
  if (cfg.seperate_all) {
    WRecipe w0; w0.N = G * 2 * C; w0.K = C;
    VRecipe b0; b0.n = G * 2 * C;
    for (int g = 0; g < G; ++g) {
      w0.pieces.push_back({std::string(attrs[g].dec) + ".0.weight", g * 2 * C, 0, 2 * C, C});
      b0.pieces.push_back({std::string(attrs[g].dec) + ".0.bias", g * 2 * C, 2 * C});
    }
    int d1 = b.new_buf(G * 2 * C);
    b.gemm("dec.l0", b.full(x), Slice(), b.wmat(w0), b.vec(b0), G * 2 * C, 1, -1, d1, 0);
    b.release(x);
    int d2 = b.new_buf(G * C);
    for (int g = 0; g < G; ++g) {
      std::string n = attrs[g].dec;
      b.gemm("dec.l1." + n, Slice{d1, g * 2 * C, 2 * C}, Slice(), b.wsingle(n + ".2.weight", C, 2 * C),
             b.vsingle(n + ".2.bias", C), C, 1, -1, d2, g * C);
    }
    b.release(d1);
    WRecipe w2; w2.N = P.dpad; w2.K = G * C;
    VRecipe b2; b2.n = P.dpad;
    int row = 0;
    for (int g = 0; g < G; ++g) {
      w2.pieces.push_back({std::string(attrs[g].dec) + ".4.weight", row, g * C, attrs[g].k, C});
      b2.pieces.push_back({std::string(attrs[g].dec) + ".4.bias", row, attrs[g].k});
      row += attrs[g].k;
    }
    b.gemm("out", b.full(d2), Slice(), b.wmat(w2), b.vec(b2), P.dpad, 0, -1, dec, 0);
    b.release(d2);
  } else {
    WRecipe w0; w0.N = P.dpad; w0.K = C;
    w0.pieces.push_back({"final_conv.weight", 0, 0, P.d, C});
    VRecipe b0; b0.n = P.dpad;
    b0.pieces.push_back({"final_conv.bias", 0, P.d});
    b.gemm("out", b.full(x), Slice(), b.wmat(w0), b.vec(b0), P.dpad, 0, -1, dec, 0);
    b.release(x);
  }
  P.out_buf = dec;
  return true;
}

std::string describe_plan(const Plan& p) {
  static const char* kinds[] = {"PACK", "GEMM", "GN", "LN", "LINATTN", "ATTN", "XATTN", "GEMM_GN", "GEMM_LN", "LN_QKV_ATTN", "ACT"};
  std::ostringstream os;
  os << "plan: C=" << p.C << " d=" << p.d << " kin_pad=" << p.kin_pad << " dpad=" << p.dpad << " buffers="
     << p.buf_width.size() << " ops=" << p.ops.size() << " time_blocks=" << p.time_blocks.size()
     << " ctx_blocks=" << p.ctx_blocks.size() << " xattn_layers=" << p.xattn_layers.size() << "\n";
  for (size_t i = 0; i < p.ops.size(); ++i) {
    const Op& o = p.ops[i];
    os << i << " " << kinds[o.kind] << " " << o.name;
    if (o.kind == OP_GEMM || o.kind == OP_GEMM_GN || o.kind == OP_GEMM_LN) {
      os << " K=" << (o.in0.k + o.in1.k) << " N=" << o.N << " a0=b" << o.in0.buf << "[" << o.in0.col << ":" << o.in0.k
         << "]";
      if (o.in1.buf >= 0) os << " a1=b" << o.in1.buf;
      os << " act=" << o.act;
      if (o.film) os << " film=" << o.film << ":" << o.film_blk;
    } else {
      os << " in=b" << o.in0.buf;
      if (o.film) os << " film=" << o.film << ":" << o.film_blk;
    }
    if (o.res >= 0) os << " res=b" << o.res;
    os << " -> b" << o.out;
    if (o.out_col) os << "[" << o.out_col << "]";
    os << "\n";
  }
  return os.str();
}

std::string export_plan_json(const Plan& p) {
  std::ostringstream os;
  auto slice = [&](const Slice& s) {
    os << "{\"buf\":" << s.buf << ",\"col\":" << s.col << ",\"k\":" << s.k << "}";
  };
  os << "{\"C\":" << p.C << ",\"d\":" << p.d << ",\"kin_pad\":" << p.kin_pad << ",\"dpad\":" << p.dpad
     << ",\"out_buf\":" << p.out_buf << ",\"buf_width\":[";
  for (size_t i = 0; i < p.buf_width.size(); ++i) os << (i ? "," : "") << p.buf_width[i];
  os << "],\"ops\":[";
  for (size_t i = 0; i < p.ops.size(); ++i) {
    const Op& o = p.ops[i];
    os << (i ? "," : "") << "{\"kind\":" << o.kind << ",\"name\":\"" << o.name << "\",\"in0\":";
    slice(o.in0);
    os << ",\"in1\":";
    slice(o.in1);
    os << ",\"out\":" << o.out << ",\"out_col\":" << o.out_col << ",\"res\":" << o.res << ",\"w\":" << o.w
       << ",\"b\":" << o.b << ",\"gamma\":" << o.gamma << ",\"beta\":" << o.beta << ",\"N\":" << o.N
       << ",\"act\":" << o.act << ",\"film\":" << o.film << ",\"film_blk\":" << o.film_blk << ",\"xlayer\":"
       << o.xlayer << "}";
  }
  os << "],\"wmats\":[";
  for (size_t i = 0; i < p.wmats.size(); ++i) {
    const WRecipe& r = p.wmats[i];
    os << (i ? "," : "") << "{\"N\":" << r.N << ",\"K\":" << r.K << ",\"ws\":" << (r.ws ? 1 : 0) << ",\"scale_k\":\""
       << r.scale_k << "\",\"pieces\":[";
    for (size_t j = 0; j < r.pieces.size(); ++j) {
      const WPiece& pc = r.pieces[j];
      os << (j ? "," : "") << "{\"name\":\"" << pc.name << "\",\"row_off\":" << pc.row_off << ",\"col_off\":"
         << pc.col_off << ",\"rows\":" << pc.rows << ",\"cols\":" << pc.cols << "}";
    }
    os << "]}";
  }
  os << "],\"vecs\":[";
  for (size_t i = 0; i < p.vecs.size(); ++i) {
    const VRecipe& r = p.vecs[i];
    os << (i ? "," : "") << "{\"n\":" << r.n << ",\"pieces\":[";
    for (size_t j = 0; j < r.pieces.size(); ++j)
      os << (j ? "," : "") << "{\"name\":\"" << r.pieces[j].name << "\",\"off\":" << r.pieces[j].off << ",\"n\":"
         << r.pieces[j].n << "}";
    os << "]}";
  }
  auto strs = [&](const char* key, const std::vector<std::string>& v) {
    os << ",\"" << key << "\":[";
    for (size_t i = 0; i < v.size(); ++i) os << (i ? "," : "") << "\"" << v[i] << "\"";
    os << "]";
  };
  os << "]";
  strs("time_blocks", p.time_blocks);
  strs("ctx_blocks", p.ctx_blocks);
  strs("xattn_layers", p.xattn_layers);
  os << "}";
  return os.str();
}

}  // namespace ds
