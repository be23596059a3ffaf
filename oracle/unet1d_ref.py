"""ORACLE (test infrastructure, not product code): CPU restatement of the reference denoiser.

A functional, token-major ([B, N, C], `F.linear`) restatement of `Unet1D.forward`
(reference scene_synthesis/networks/denoise_net.py:507-593) operating directly on a
reference-format state dict.  The reference itself is channel-major Conv1d modules; this file
shares no code with it and is pinned against the live reference by tests/golden/make_golden.py
(the reference ships no golden vectors of its own: SURVEY.md section 8c).

Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs may
import this module.  Everything runs in fp32 on the CPU (eps 1e-5, denoise_net.py:84,99).
"""
from __future__ import annotations

import math
from typing import Callable, Dict, Optional

import torch
import torch.nn.functional as F

Tensor = torch.Tensor
P = "diffusion.model."


def _w2(sd, key):
    """Conv1d(k=1) weight [Cout, Cin, 1] or Linear weight [Cout, Cin] -> [Cout, Cin]."""
    w = sd[key]
    return w.reshape(w.shape[0], -1)


def sinusoidal_embedding(t: Tensor, dim: int) -> Tensor:
    """denoise_net.py:127-139: [sin(t*f_k) | cos(t*f_k)], f_k = exp(-k*ln(1e4)/(dim/2-1))."""
    half = dim // 2
    freq = torch.exp(torch.arange(half, dtype=torch.float32, device=t.device) * -(math.log(10000) / (half - 1)))
    ang = t.to(torch.float32)[:, None] * freq[None, :]
    return torch.cat([ang.sin(), ang.cos()], dim=-1)


def standardize_weight(w: Tensor, eps: float = 1e-5) -> Tensor:
    """denoise_net.py:83-89: per-output-channel (w - mean) * rsqrt(biased var + eps)."""
    w2 = w.reshape(w.shape[0], -1)
    mean = w2.mean(dim=1, keepdim=True)
    var = w2.var(dim=1, unbiased=False, keepdim=True)
    return (w2 - mean) * torch.rsqrt(var + eps)


def channel_layer_norm(x: Tensor, g: Tensor, eps: float = 1e-5) -> Tensor:
    """denoise_net.py:93-102 on token-major x [B, N, C]: no bias, biased variance."""
    mean = x.mean(dim=-1, keepdim=True)
    var = x.var(dim=-1, unbiased=False, keepdim=True)
    return (x - mean) * torch.rsqrt(var + eps) * g.reshape(1, 1, -1)


def group_norm_tokens(x: Tensor, gamma: Tensor, beta: Tensor, groups: int = 8, eps: float = 1e-5) -> Tensor:
    """nn.GroupNorm(groups, C) of denoise_net.py:164 on [B, N, C]: stats over (C/groups channels x N tokens)."""
    B, N, C = x.shape
    xg = x.reshape(B, N, groups, C // groups)
    mean = xg.mean(dim=(1, 3), keepdim=True)
    var = xg.var(dim=(1, 3), unbiased=False, keepdim=True)
    y = ((xg - mean) * torch.rsqrt(var + eps)).reshape(B, N, C)
    return y * gamma + beta


def ws_block(sd, name: str, x: Tensor, scale_shift=None) -> Tensor:
    """`Block` (denoise_net.py:160-176): WS-conv -> GroupNorm -> FiLM -> SiLU."""
    w = standardize_weight(sd[name + ".proj.weight"])
    h = F.linear(x, w, sd[name + ".proj.bias"])
    h = group_norm_tokens(h, sd[name + ".norm.weight"], sd[name + ".norm.bias"])
    if scale_shift is not None:
        scale, shift = scale_shift
        h = h * (scale + 1) + shift
    return F.silu(h)


def resnet_block(sd, name: str, x: Tensor, cond: Optional[Tensor], tap=None) -> Tensor:
    """`ResnetBlock` (denoise_net.py:178-206). cond is [B, E] (time) or [B, N, E] (per object)."""
    scale_shift = None
    if cond is not None:
        e = F.linear(F.silu(cond), sd[name + ".mlp.1.weight"], sd[name + ".mlp.1.bias"])
        if e.dim() == 2:
            e = e[:, None, :]
        scale_shift = e.chunk(2, dim=-1)
    h = ws_block(sd, name + ".block1", x, scale_shift)
    if tap:
        tap(name + ".block1", h)
    h = ws_block(sd, name + ".block2", h)
    if (name + ".res_conv.weight") in sd:
        res = F.linear(x, _w2(sd, name + ".res_conv.weight"), sd[name + ".res_conv.bias"])
    else:
        res = x
    out = h + res
    if tap:
        tap(name, out)
    return out


def _heads(t: Tensor, h: int) -> Tensor:
    B, N, HC = t.shape
    return t.reshape(B, N, h, HC // h).permute(0, 2, 1, 3)      # [B, h, N, c]


def linear_attention(sd, name: str, x: Tensor, heads: int = 4, tap=None) -> Tensor:
    """`Residual(PreNorm(LinearAttention))` (denoise_net.py:208-235, wrappers 39-45, 104-112)."""
    xn = channel_layer_norm(x, sd[name + ".fn.norm.g"])
    qkv = F.linear(xn, _w2(sd, name + ".fn.fn.to_qkv.weight"))
    q, k, v = (_heads(t, heads) for t in qkv.chunk(3, dim=-1))        # [B, h, N, 32]
    q = q.softmax(dim=-1) * (q.shape[-1] ** -0.5)                     # over head channels, then scale
    k = k.softmax(dim=-2)                                             # over tokens
    ctx = torch.einsum("bhnd,bhne->bhde", k, v)
    o = torch.einsum("bhde,bhnd->bhne", ctx, q)
    o = o.permute(0, 2, 1, 3).reshape(x.shape[0], x.shape[1], -1)
    if tap:
        tap(name + ".core", o)
    y = F.linear(o, _w2(sd, name + ".fn.fn.to_out.0.weight"), sd[name + ".fn.fn.to_out.0.bias"])
    y = channel_layer_norm(y, sd[name + ".fn.fn.to_out.1.g"])
    out = y + x
    if tap:
        tap(name, out)
    return out


def softmax_attention(sd, name: str, x: Tensor, heads: int = 4, tap=None) -> Tensor:
    """`Residual(PreNorm(Attention))` (denoise_net.py:237-259): no LayerNorm on the output."""
    xn = channel_layer_norm(x, sd[name + ".fn.norm.g"])
    qkv = F.linear(xn, _w2(sd, name + ".fn.fn.to_qkv.weight"))
    q, k, v = (_heads(t, heads) for t in qkv.chunk(3, dim=-1))
    q = q * (q.shape[-1] ** -0.5)
    sim = torch.einsum("bhid,bhjd->bhij", q, k)
    attn = sim.softmax(dim=-1)
    o = torch.einsum("bhij,bhjd->bhid", attn, v)
    o = o.permute(0, 2, 1, 3).reshape(x.shape[0], x.shape[1], -1)
    if tap:
        tap(name + ".core", o)
    out = F.linear(o, _w2(sd, name + ".fn.fn.to_out.weight"), sd[name + ".fn.fn.to_out.bias"]) + x
    if tap:
        tap(name, out)
    return out


def cross_linear_attention(sd, name: str, x: Tensor, text: Tensor, heads: int = 4, tap=None) -> Tensor:
    """`ResidualCross(PreNormCross(LinearAttentionCross))` (denoise_net.py:261-297, 47-53, 115-123).

    text is [B, L, text_dim]; only x is pre-normalised (PreNormCross.forward normalises x alone).
    """
    xn = channel_layer_norm(x, sd[name + ".fn.norm.g"])
    q = _heads(F.linear(xn, _w2(sd, name + ".fn.fn.to_q.weight")), heads)          # [B,h,N,32]
    kv = F.linear(text, _w2(sd, name + ".fn.fn.to_kv.weight"))
    k, v = (_heads(t, heads) for t in kv.chunk(2, dim=-1))                          # [B,h,L,32]
    q = q.softmax(dim=-1) * (q.shape[-1] ** -0.5)
    k = k.softmax(dim=-2)
    ctx = torch.einsum("bhld,bhle->bhde", k, v)
    o = torch.einsum("bhde,bhnd->bhne", ctx, q)
    o = o.permute(0, 2, 1, 3).reshape(x.shape[0], x.shape[1], -1)
    y = F.linear(o, _w2(sd, name + ".fn.fn.to_out.0.weight"), sd[name + ".fn.fn.to_out.0.bias"])
    y = channel_layer_norm(y, sd[name + ".fn.fn.to_out.1.g"])
    out = y + x
    if tap:
        tap(name, out)
    return out


def mlp3(sd, name: str, x: Tensor) -> Tensor:
    """`_encoder_mlp` / `_decoder_mlp` (denoise_net.py:484-504): conv, GELU(erf), conv, GELU, conv."""
    h = F.gelu(F.linear(x, _w2(sd, name + ".0.weight"), sd[name + ".0.bias"]))
    h = F.gelu(F.linear(h, _w2(sd, name + ".2.weight"), sd[name + ".2.bias"]))
    return F.linear(h, _w2(sd, name + ".4.weight"), sd[name + ".4.bias"])


def time_embedding(sd, t: Tensor, dim: int, prefix: str = P) -> Tensor:
    """`time_mlp` (denoise_net.py:417-422): sinusoid -> Linear -> GELU -> Linear."""
    w1 = sd[prefix + "time_mlp.1.weight"]
    e = sinusoidal_embedding(t, dim).to(w1.dtype)      # fp32 as in the reference; widened for an fp64 evaluation
    e = F.gelu(F.linear(e, sd[prefix + "time_mlp.1.weight"], sd[prefix + "time_mlp.1.bias"]))
    return F.linear(e, sd[prefix + "time_mlp.3.weight"], sd[prefix + "time_mlp.3.bias"])


def unet1d_forward(sd: Dict[str, Tensor], spec, x: Tensor, t: Tensor, context: Optional[Tensor],
                   context_cross: Optional[Tensor] = None,
                   tap: Optional[Callable[[str, Tensor], None]] = None, prefix: str = P) -> Tensor:
    """Restatement of Unet1D.forward (denoise_net.py:507-593).

    x [B, N, d] fp32, t [B] int64, context [B, N, cond_dim], context_cross [B, L, text_dim] | None.
    `spec` is a diffuscene_b200.weights.NetSpec.  `tap(name, tensor)` receives intermediates.
    """
    sdp = {k[len(prefix):]: v for k, v in sd.items() if k.startswith(prefix)}
    s = spec
    x = x if x.dtype == torch.float64 else x.to(torch.float32)      # fp64 for a high-precision evaluation
    b0 = s.bbox_dim
    if s.seperate_all:
        c0 = b0 + s.class_dim
        h = mlp3(sdp, "class_embedf", x[..., b0:c0]) + mlp3(sdp, "bbox_embedf", x[..., :b0])
        if s.objectness_dim > 0:
            h = h + mlp3(sdp, "objectness_embedf", x[..., c0:c0 + s.objectness_dim])
        if s.objfeat_dim > 0:
            o0 = c0 + s.objectness_dim
            h = h + mlp3(sdp, "objfeat_embedf", x[..., o0:o0 + s.objfeat_dim])
    else:
        h = x
    if tap:
        tap("encoder", h)
    h = F.linear(h, _w2(sdp, "init_conv.weight"), sdp["init_conv.bias"])
    r = h
    if tap:
        tap("init_conv", h)
    temb = time_embedding(sdp, t, s.dim, prefix="")
    if tap:
        tap("temb", temb)

    text = context_cross if s.text_condition else None
    skips = []
    for i in range(s.n_stages):
        d = "downs.%d" % i
        h = resnet_block(sdp, d + ".0", h, context, tap)
        h = resnet_block(sdp, d + ".1", h, temb, tap)
        skips.append(h)
        if text is not None:
            h = cross_linear_attention(sdp, d + ".2", h, text, s.heads, tap)
        h = resnet_block(sdp, d + ".3", h, temb, tap)
        h = linear_attention(sdp, d + ".4", h, s.heads, tap)
        skips.append(h)
        if i == s.n_stages - 1:
            h = F.linear(h, _w2(sdp, d + ".5.weight"), sdp[d + ".5.bias"])
            if tap:
                tap(d + ".5", h)

    h = resnet_block(sdp, "mid_block0", h, context, tap)
    h = resnet_block(sdp, "mid_block1", h, temb, tap)
    if text is not None:
        h = cross_linear_attention(sdp, "mid_attn_cross", h, text, s.heads, tap)
    h = softmax_attention(sdp, "mid_attn", h, s.heads, tap)
    h = resnet_block(sdp, "mid_block2", h, temb, tap)

    for i in range(s.n_stages):
        u = "ups.%d" % i
        h = resnet_block(sdp, u + ".0", h, context, tap)
        h = resnet_block(sdp, u + ".1", torch.cat([h, skips.pop()], dim=-1), temb, tap)
        if text is not None:
            h = cross_linear_attention(sdp, u + ".2", h, text, s.heads, tap)
        h = resnet_block(sdp, u + ".3", torch.cat([h, skips.pop()], dim=-1), temb, tap)
        h = linear_attention(sdp, u + ".4", h, s.heads, tap)
        if i == s.n_stages - 1:
            h = F.linear(h, _w2(sdp, u + ".5.weight"), sdp[u + ".5.bias"])
            if tap:
                tap(u + ".5", h)

    h = resnet_block(sdp, "final_res_block", torch.cat([h, r], dim=-1), temb, tap)
    if s.seperate_all:
        outs = [mlp3(sdp, "bbox_hidden2output", h), mlp3(sdp, "class_hidden2output", h)]
        if s.objectness_dim > 0:
            outs.append(mlp3(sdp, "objectness_hidden2output", h))
        if s.objfeat_dim > 0:
            outs.append(mlp3(sdp, "objfeat_hidden2output", h))
        out = torch.cat(outs, dim=-1)
    else:
        out = F.linear(h, _w2(sdp, "final_conv.weight"), sdp["final_conv.bias"])
    if tap:
        tap("out", out)
    return out
