"""ORACLE (test infrastructure): CPU interpreter of the engine's step program.

Executes the op list exported by `ds_plan_export_json` (diffuscene_b200/csrc/plan.cpp) with plain torch
ops, assembling the packed weight matrices from the same recipes the CUDA engine uses.  Comparing its
output with the golden vectors verifies -- without a GPU -- that the engine's *program* (op order, buffer
wiring, hoisted FiLM tables, block-structured encoder / decoder GEMMs, folded weight standardisation) is
a faithful restatement of Unet1D.forward (reference denoise_net.py:507-593).  With emulate_bf16=True,
weights and every op output are rounded to bf16, predicting the error of the throughput mode.
"""
from __future__ import annotations

import math
from typing import Dict, Optional

import torch
import torch.nn.functional as F

from .unet1d_ref import sinusoidal_embedding

OP_PACK, OP_GEMM, OP_GN, OP_LN, OP_LINATTN, OP_ATTN, OP_XATTN, OP_GEMM_GN, OP_GEMM_LN, OP_LN_QKV_ATTN, OP_ACT = range(11)


def _r(x, on):
    return x.to(torch.bfloat16).to(torch.float32) if on else x


def assemble_wmat(r, sd):
    W = torch.zeros(r["N"], r["K"], dtype=torch.float32)
    for pc in r["pieces"]:
        src = sd[pc["name"]].reshape(pc["rows"], pc["cols"]).to(torch.float32)
        if r["ws"]:
            mean = src.mean(dim=1, keepdim=True)
            var = src.var(dim=1, unbiased=False, keepdim=True)
            src = (src - mean) * torch.rsqrt(var + 1e-5)
        W[pc["row_off"]:pc["row_off"] + pc["rows"], pc["col_off"]:pc["col_off"] + pc["cols"]] = src
    if r.get("scale_k"):       # a LayerNorm gain folded into the columns (fused LN + to_qkv op)
        W = W * sd[r["scale_k"]].reshape(1, -1).to(torch.float32)
    return W


def assemble_vec(r, sd):
    v = torch.zeros(r["n"], dtype=torch.float32)
    for pc in r["pieces"]:
        v[pc["off"]:pc["off"] + pc["n"]] += sd[pc["name"]].reshape(-1).to(torch.float32)
    return v


class PlanTables:
    """Everything an op reads besides its input buffers: packed weight matrices, vectors, the hoisted FiLM tables
    and the cross-attention contexts, for one batch of B scenes of N objects."""

    def __init__(self, plan, B, N, wm, vecs, film_t, film_c, xctx, x=None):
        self.plan, self.B, self.N, self.C = plan, B, N, plan["C"]
        self.wm, self.vecs, self.film_t, self.film_c, self.xctx, self.x = wm, vecs, film_t, film_c, xctx, x


def film_tables(plan, sd, t, context, M, dtype=torch.float32):
    """The hoisted time (per scene) and context (per row) FiLM tables of every ResnetBlock, in `dtype`."""
    sdt = lambda n: sd[n].to(dtype)
    e = sinusoidal_embedding(t, plan["C"]).to(dtype)
    e = F.gelu(F.linear(e, sdt("time_mlp.1.weight"), sdt("time_mlp.1.bias")))
    e = F.silu(F.linear(e, sdt("time_mlp.3.weight"), sdt("time_mlp.3.bias")))
    film_t = [F.linear(e, sdt(n + ".mlp.1.weight"), sdt(n + ".mlp.1.bias")) for n in plan["time_blocks"]]   # [B, 2C]
    cs = F.silu(context.to(dtype).reshape(M, -1))
    film_c = [F.linear(cs, sdt(n + ".mlp.1.weight"), sdt(n + ".mlp.1.bias")) for n in plan["ctx_blocks"]]  # [M, 2C]
    return film_t, film_c


def xattn_contexts(plan, sd, context_cross, dtype=torch.float32):
    """ctx[b, h] = softmax_L(k)^T v of every cross-attention layer (the text prefix is fixed over the sampling loop)."""
    out = []
    for n in plan["xattn_layers"]:
        kv = F.linear(context_cross.to(dtype), sd[n + ".fn.fn.to_kv.weight"].to(dtype).reshape(256, -1))   # [B, L, 256]
        k, v = kv[..., :128], kv[..., 128:]
        B, L = kv.shape[0], kv.shape[1]
        k = k.reshape(B, L, 4, 32).softmax(dim=1)
        v = v.reshape(B, L, 4, 32)
        out.append(torch.einsum("blhd,blhe->bhde", k, v))
    return out


def _gn_film_silu(op, y, tb):
    B, N, C = tb.B, tb.N, tb.C
    h = y.reshape(B, N, 8, C // 8)
    mean = h.mean(dim=(1, 3), keepdim=True)
    var = h.var(dim=(1, 3), unbiased=False, keepdim=True)
    y = ((h - mean) * torch.rsqrt(var + 1e-5)).reshape(B, N, C) * tb.vecs[op["gamma"]] + tb.vecs[op["beta"]]
    if op["film"] == 1:
        f = tb.film_t[op["film_blk"]][:, None, :]
        y = y * (f[..., :C] + 1) + f[..., C:]
    elif op["film"] == 2:
        f = tb.film_c[op["film_blk"]].reshape(B, N, 2 * C)
        y = y * (f[..., :C] + 1) + f[..., C:]
    return F.silu(y).reshape(B * N, C)


def _ln(h, eps=1e-5):
    mean = h.mean(dim=1, keepdim=True)
    var = h.var(dim=1, unbiased=False, keepdim=True)
    return (h - mean) * torch.rsqrt(var + eps)


def _linattn_core(qkv, tb, inner):
    """LinearAttention core (denoise_net.py:208-233); `inner` rounds at the points where the kernel stores bf16."""
    B, N = tb.B, tb.N
    heads = lambda z: z.reshape(B, N, 4, 32)
    q, kk, v = heads(qkv[:, :128]), heads(qkv[:, 128:256]), heads(qkv[:, 256:384])
    q = inner(q.softmax(dim=-1) * (32 ** -0.5))
    kk = inner(kk.softmax(dim=1))
    ctx = inner(torch.einsum("bnhd,bnhe->bhde", kk, v))
    return torch.einsum("bhde,bnhd->bnhe", ctx, q).reshape(B * N, 128)


def eval_op(op: dict, bufs, tb: PlanTables, emulate_bf16: bool = False, inner=None):
    """One op of the step program on the buffers `bufs` (a list indexed by buffer id, each [M, width]); returns
    the new contents of the op's output buffer and changes nothing.  Arithmetic runs in the dtype of `bufs` and
    `tb`.  With emulate_bf16 the result is rounded to bf16; `inner` (identity by default) is applied where the
    attention kernels round their intermediates (q | k | v, softmaxed k and q, the context)."""
    k = op["kind"]
    bf = emulate_bf16
    inner = inner or (lambda z: z)
    M = tb.B * tb.N
    if k == OP_PACK:
        d = tb.x.shape[-1]
        out = torch.zeros(M, tb.plan["kin_pad"], dtype=tb.x.dtype, device=tb.x.device)
        out[:, :d] = tb.x.reshape(M, d)
        return _r(out, bf)
    i0 = op["in0"]
    if k == OP_GEMM or k == OP_GEMM_GN or k == OP_GEMM_LN:
        a = bufs[i0["buf"]][:, i0["col"]:i0["col"] + i0["k"]]
        if op["in1"]["buf"] >= 0:
            i1 = op["in1"]
            a = torch.cat([a, bufs[i1["buf"]][:, i1["col"]:i1["col"] + i1["k"]]], dim=1)
        y = a @ tb.wm[op["w"]].t()
        if op["b"] >= 0:
            y = y + tb.vecs[op["b"]]
    if k == OP_GEMM_GN:      # the GEMM result stays in fp32 (registers) through the GroupNorm epilogue
        y = _gn_film_silu(op, y, tb)
        if op["res"] >= 0:
            y = y + bufs[op["res"]]
        return _r(y, bf)
    if k == OP_GEMM_LN:      # the projection stays in fp32 (registers) through the LayerNorm epilogue
        y = _ln(y) * tb.vecs[op["gamma"]]
        if op["res"] >= 0:
            y = y + bufs[op["res"]]
        return _r(y, bf)
    if k == OP_GEMM:
        if op["act"] == 1:
            y = F.gelu(y)
        elif op["act"] == 2:
            y = F.silu(y)
        if op["res"] >= 0:
            y = y + bufs[op["res"]]
        out = bufs[op["out"]].clone()
        out[:, op["out_col"]:op["out_col"] + op["N"]] = _r(y, bf)
        return out
    if k == OP_ACT:      # train program: the activation of a `<name>.pre` GEMM's column slice, other columns kept
        c0, c1 = op["out_col"], op["out_col"] + op["N"]
        z = bufs[i0["buf"]][:, i0["col"]:i0["col"] + i0["k"]]
        y = F.gelu(z) if op["act"] == 1 else F.silu(z)
        if op["res"] >= 0:
            y = y + bufs[op["res"]][:, c0:c1]
        out = bufs[op["out"]].clone()
        out[:, c0:c1] = _r(y, bf)
        return out
    if k == OP_GN:
        y = _gn_film_silu(op, bufs[i0["buf"]], tb)
        if op["res"] >= 0:
            y = y + bufs[op["res"]]
        return _r(y, bf)
    if k == OP_LN:
        y = _ln(bufs[i0["buf"]]) * tb.vecs[op["b"]]
        if op["res"] >= 0:
            y = y + bufs[op["res"]]
        return _r(y, bf)
    if k == OP_LN_QKV_ATTN:      # LayerNorm (gain folded into the packed weights) + to_qkv + linear-attention core
        qkv = inner(_ln(bufs[i0["buf"]]) @ tb.wm[op["w"]].t())
        return _r(_linattn_core(qkv, tb, inner), bf)
    if k == OP_LINATTN:
        return _r(_linattn_core(bufs[i0["buf"]], tb, inner), bf)
    if k == OP_ATTN:
        qkv = bufs[i0["buf"]]
        heads = lambda z: z.reshape(tb.B, tb.N, 4, 32)
        q, kk, v = heads(qkv[:, :128]), heads(qkv[:, 128:256]), heads(qkv[:, 256:384])
        sim = torch.einsum("bihd,bjhd->bhij", q * (32 ** -0.5), kk)
        o = torch.einsum("bhij,bjhd->bihd", sim.softmax(dim=-1), v)
        return _r(o.reshape(M, 128), bf)
    if k == OP_XATTN:
        q = bufs[i0["buf"]].reshape(tb.B, tb.N, 4, 32).softmax(dim=-1) * (32 ** -0.5)
        o = torch.einsum("bhde,bnhd->bnhe", tb.xctx[op["xlayer"]], q)
        return _r(o.reshape(M, 128), bf)
    raise ValueError("op kind %d has no interpreter" % k)


def run_plan(plan: dict, sd: Dict[str, torch.Tensor], x: torch.Tensor, t: torch.Tensor, context: torch.Tensor,
             context_cross: Optional[torch.Tensor] = None, emulate_bf16: bool = False, taps: Optional[dict] = None):
    """sd keys are reference names without the 'diffusion.model.' prefix."""
    B, N, d = x.shape
    M = B * N
    bf = emulate_bf16
    bufs = [torch.zeros(M, w) for w in plan["buf_width"]]
    wm = [_r(assemble_wmat(r, sd), bf) for r in plan["wmats"]]
    vecs = [assemble_vec(r, sd) for r in plan["vecs"]]
    film_t, film_c = film_tables(plan, sd, t, context, M)      # hoisted FiLM tables (always fp32 in the engine)
    xctx = xattn_contexts(plan, sd, context_cross)
    tb = PlanTables(plan, B, N, wm, vecs, film_t, film_c, xctx, x)
    for op in plan["ops"]:
        bufs[op["out"]] = eval_op(op, bufs, tb, emulate_bf16=bf)
        if taps is not None:
            taps[op["name"]] = bufs[op["out"]].clone()
    return bufs[plan["out_buf"]][:, :d].reshape(B, N, d)
