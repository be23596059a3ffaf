"""GPU, op by op: every op of the step program against a float64 evaluation of the same op from the kernel's own
input buffers, at multi-tile batches, ragged last tiles and object counts other than 12 and 21; and scene isolation
(a NaN, Inf or changed scene never changes another scene's output, within a call or across calls).

The end-to-end bf16 gates (test_gpu_bf16.py) are set to the ~5e-3 rounding noise of a whole forward, where a kernel
that is off by 1 % in one epilogue term can hide.  Here errors do not compound: each op is evaluated in fp64 from the
bf16 values its kernel actually read (the taps of the no_reuse program, whose buffers are never overwritten after
they are read: tests/test_plan_cpu.py::test_no_reuse_plan_taps_are_op_inputs), with the packed weights restated
exactly as ds_commit_weights builds them.

Bounds (bf16 mode).  ulp(v) is the bf16 spacing at |v|: 2^(e - 8) for |v| in [2^(e-1), 2^e).
- One final bf16 rounding (GEMM, GEMM_GN, GEMM_LN, GN, LN): the kernel rounds a pre-value p to nearest, |p - ref| = d,
  so |out - ref| <= ulp(p) / 2 + d <= ulp(ref) + d (ulp(p) <= 2 ulp(ref) at a binade edge).  d collects fp32
  accumulation (K <= 1536 products: < 2^-13 of the row RMS), rsqrtf (2^-22 relative), one-pass fp32 statistics at
  the offsets the shipped networks reach (printed), and SiLU as h + h tanh.approx(h), h = x / 2, whose absolute error is
  |h| 2^-11 <= |x| 2^-12; with |x| within 8 RMS of the row this is 2^-9 RMS.  Bound: ulp(ref) + 2^-9 RMS(row).
- GELU GEMMs: the kernel uses the tanh form (tc_common.cuh gelu_tanh) with tanh.approx; the reference is the erf
  form.  Extra allowance per element: |gelu_tanh(x) - gelu_erf(x)| (computed in fp64) + |x| 2^-12.
- Tensor-core linear-attention cores (LINATTN and LN_QKV_ATTN, N <= 32): the reference rounds to bf16 where the
  kernel does (q | k | v when the kernel computes them, k~, q~, ctx).  Their pre-rounding values differ by fp32
  error only (ex2.approx, the mean * cs cancellation of the folded LayerNorm), so an intermediate can land one ulp
  away when it sits near a bf16 midpoint.  Bound: ulp(ref) + the first-order effect of one ulp in every rounded
  intermediate (_linattn_flip_bound, elementwise in fp64) + 2^-12 RMS(row).
- Softmax attention, the cross-attention core and the SIMT linear-attention core (N > 32) have no intermediate bf16
  rounding: 2 ulp(ref) + 2^-9 RMS(row).
- fp32 mode (SIMT kernels, no intermediate rounding): 2^-15 (|ref| + RMS(row)).
No bound is on a mean: every element must hold its own bound.
"""
import math

import pytest
import torch
import torch.nn.functional as F

from diffuscene_b200 import capi
from diffuscene_b200.engine import DenoiserEngine
from diffuscene_b200.weights import NetSpec, seeded_state_dict, unet1d_param_specs
from oracle.plan_interp import (OP_ATTN, OP_GEMM, OP_GEMM_GN, OP_GEMM_LN, OP_GN, OP_LINATTN, OP_LN, OP_LN_QKV_ATTN,
                                OP_PACK, OP_XATTN, PlanTables, _ln, assemble_vec, eval_op, film_tables,
                                xattn_contexts)
from tests.cases import CASES, make_inputs
from tests.gpu_common import case_tables

pytestmark = pytest.mark.gpu

KIND = {OP_GEMM: "GEMM", OP_GN: "GN", OP_LN: "LN", OP_LINATTN: "LINATTN", OP_ATTN: "ATTN", OP_XATTN: "XATTN",
        OP_GEMM_GN: "GEMM_GN", OP_GEMM_LN: "GEMM_LN", OP_LN_QKV_ATTN: "LN_QKV_ATTN"}
NORM_KINDS = (OP_GN, OP_LN, OP_GEMM_GN, OP_GEMM_LN, OP_LN_QKV_ATTN)
_ENG = {}


def _engine(name, prec, fuse, n_obj=None, edit=None, cache=True):
    """Seeded engine of case `name`'s network at `n_obj` objects per scene (a private cache: two alive at most).
    edit: (tag, fn) with fn changing the seeded state dict in place before it is loaded."""
    case = CASES[name]
    n = n_obj or case["N"]
    key = (name, prec, fuse, n, edit[0] if edit else None)
    if key not in _ENG or not cache:
        while len(_ENG) >= 2:
            _ENG.pop(next(iter(_ENG)))[0].close()
        spec = NetSpec.from_net_kwargs(case["net_kwargs"])
        eng = DenoiserEngine(spec, n, case["diffusion_kwargs"]["time_num"], precision=prec, fuse_level=fuse)
        sd = seeded_state_dict(unet1d_param_specs(spec), seed=case["seed"])
        if edit:
            edit[1](sd)
        eng.load_state_dict(sd)
        eng.set_schedule(case_tables(case))
        g = torch.Generator().manual_seed(case["seed"] + n)
        ctx = torch.randn(n, spec.cond_dim, generator=g)
        eng.set_context(ctx, shared=True)
        _ENG[key] = (eng, spec, {k[len("diffusion.model."):]: v for k, v in sd.items()}, ctx)
    return _ENG[key]


def _inputs(spec, B, N, T, seed):
    g = torch.Generator().manual_seed(seed)
    return torch.randn(B, N, spec.point_dim, generator=g), torch.randint(0, T, (B,), generator=g)


def packed_wmat(r, sd, bf16):
    """A packed weight matrix as ds_commit_weights builds it: fp32 weight standardisation with double-precision
    statistics, the folded LayerNorm gain, then round-to-nearest-even to bf16 (bf16 mode)."""
    W = torch.zeros(r["N"], r["K"], dtype=torch.float32)
    for pc in r["pieces"]:
        src = sd[pc["name"]].reshape(pc["rows"], pc["cols"]).to(torch.float32)
        if r["ws"]:
            m64 = src.double().mean(dim=1, keepdim=True)
            var = ((src.double() - m64) ** 2).mean(dim=1, keepdim=True)
            rs = 1.0 / torch.sqrt(var.float() + 1e-5)
            src = (src - m64.float()) * rs
        W[pc["row_off"]:pc["row_off"] + pc["rows"], pc["col_off"]:pc["col_off"] + pc["cols"]] = src
    if r.get("scale_k"):
        W = W * sd[r["scale_k"]].reshape(1, -1).to(torch.float32)
    return (W.to(torch.bfloat16) if bf16 else W).double()


def bf16_ulp(v):
    _, e = torch.frexp(v.abs())
    u = torch.ldexp(torch.ones_like(v), e - 8)
    return torch.where(v == 0, torch.zeros_like(v), u)


def _rnd_bf16(z):
    return z.to(torch.bfloat16).to(torch.float64)


def _gelu_tanh(x):
    return 0.5 * x * (1 + torch.tanh(math.sqrt(2 / math.pi) * (x + 0.044715 * x ** 3)))


def _linattn_flip_bound(qkv, B, N, own_qkv):
    """First-order bound on what a rounding on the other side of a bf16 midpoint, in every intermediate the
    tensor-core linear-attention kernels round (q | k | v when the kernel computes them, k~, q~, ctx), can change in
    the output.  A softmax whose logits move by at most u moves each probability by a factor within e^(+-2u)."""
    heads = lambda z: z.reshape(B, N, 4, 32)
    q, k, v = heads(qkv[:, :128]), heads(qkv[:, 128:256]), heads(qkv[:, 256:384])
    qs = _rnd_bf16(q.softmax(dim=-1) * (32 ** -0.5))
    ks = _rnd_bf16(k.softmax(dim=1))
    ctx = _rnd_bf16(torch.einsum("bnhd,bnhe->bhde", ks, v))
    uq = bf16_ulp(q).amax(dim=-1, keepdim=True) if own_qkv else 0.0      # over the channels a q-softmax spans
    uk = bf16_ulp(k).amax(dim=1, keepdim=True) if own_qkv else 0.0       # over the tokens a k-softmax spans
    uv = bf16_ulp(v) if own_qkv else torch.zeros_like(v)
    dqs = bf16_ulp(qs) + qs * torch.expm1(2 * torch.as_tensor(uq, dtype=qs.dtype, device=qs.device))
    dks = bf16_ulp(ks) + ks * torch.expm1(2 * torch.as_tensor(uk, dtype=ks.dtype, device=ks.device))
    dctx = bf16_ulp(ctx) + torch.einsum("bnhd,bnhe->bhde", dks, v.abs()) + torch.einsum("bnhd,bnhe->bhde", ks, uv)
    do = torch.einsum("bhde,bnhd->bnhe", ctx.abs(), dqs) + torch.einsum("bhde,bnhd->bnhe", dctx, qs)
    return do.reshape(B * N, 128)


WORST = {}      # (precision, op kind) -> worst |err| / bound seen in this session
OFFSET = {}     # op kind -> largest |mean| / std of a normalised row or group seen in this session


def _offset_ratio(z, op, B, N):
    if op["kind"] in (OP_GN, OP_GEMM_GN):
        z = z.reshape(B, N, 8, -1).permute(0, 2, 1, 3).reshape(B * 8, -1)
    var = z.var(dim=1, unbiased=False)
    return (z.mean(dim=1).abs() / var.sqrt().clamp_min(1e-30)).max().item(), var.min().item()


def check_ops(eng, spec, sd, ctx, x, t, context_cross=None):
    """One forward with taps on; every op except PACK evaluated in fp64 from its input taps against its output tap."""
    bf = eng.precision == "bf16"
    B, N = x.shape[0], x.shape[1]
    M = B * N
    dev = torch.device("cuda")
    plan = capi.plan_export(eng.cfg, no_reuse=True)
    eng.enable_taps(True)      # rebuilds the buffers and recommits the weights: the context tables go with them
    try:
        eng.set_context(ctx, shared=True)
        if context_cross is not None:
            eng.set_context_cross(context_cross)
        eng.forward(x.cuda(), t.cuda())
        torch.cuda.synchronize()
        writer = {}
        for op in plan["ops"]:
            writer.setdefault(op["out"], op["name"])
        bufs = [eng.read_tap(writer[b], M).to(dev, torch.float64) if b in writer else None
                for b in range(len(plan["buf_width"]))]
    finally:
        eng.enable_taps(False)
        eng.set_context(ctx, shared=True)
    sd64 = {k: v.double() for k, v in sd.items()}
    ctx_b = ctx[None].expand(B, N, ctx.shape[-1]).double()
    film_t, film_c = film_tables(plan, sd64, t, ctx_b, M, dtype=torch.float64)
    xctx = xattn_contexts(plan, sd64, context_cross, dtype=torch.float64) if context_cross is not None else []
    tb = PlanTables(plan, B, N, [packed_wmat(r, sd, bf).to(dev) for r in plan["wmats"]],
                    [assemble_vec(r, sd).double().to(dev) for r in plan["vecs"]],
                    [f.to(dev) for f in film_t], [f.to(dev) for f in film_c], [c.to(dev) for c in xctx])
    fails = []
    seen = {}       # op kind -> (largest |mean| / std, smallest variance) of a normalised row or group in this call
    for op in plan["ops"]:
        k = op["kind"]
        if k == OP_PACK:
            continue
        attn = k in (OP_LINATTN, OP_LN_QKV_ATTN, OP_ATTN, OP_XATTN)
        # the tensor-core linear-attention cores (N <= 32) round q | k | v, k~, q~ and ctx to bf16
        inner = _rnd_bf16 if (bf and k in (OP_LINATTN, OP_LN_QKV_ATTN) and N <= 32) else None
        ref = eval_op(op, bufs, tb, inner=inner)
        got = bufs[op["out"]]
        c0 = op["out_col"] if k == OP_GEMM else 0
        c1 = c0 + op["N"] if k == OP_GEMM else got.shape[1]
        ref, got = ref[:, c0:c1], got[:, c0:c1]
        assert torch.isfinite(got).all(), op["name"]
        rms = ref.pow(2).mean(dim=1, keepdim=True).sqrt()
        if bf and inner is not None:
            if k == OP_LN_QKV_ATTN:
                qkv = _rnd_bf16(_ln(bufs[op["in0"]["buf"]]) @ tb.wm[op["w"]].t())
            else:
                qkv = bufs[op["in0"]["buf"]]
            bound = bf16_ulp(ref) + _linattn_flip_bound(qkv, B, N, k == OP_LN_QKV_ATTN) + 2.0 ** -12 * rms
        elif bf:
            bound = (2 if attn else 1) * bf16_ulp(ref) + 2.0 ** -9 * rms
            if k == OP_GEMM and op["act"] in (1, 2):
                pre = eval_op(dict(op, act=0, res=-1), bufs, tb)[:, c0:c1]
                bound = bound + pre.abs() * 2.0 ** -12
                if op["act"] == 1:
                    bound = bound + (_gelu_tanh(pre) - F.gelu(pre)).abs()
        else:
            bound = 2.0 ** -15 * (ref.abs() + rms)
        ratio = ((got - ref).abs() / bound).max().item()
        key = (eng.precision, KIND[k])
        WORST[key] = max(WORST.get(key, 0.0), ratio)
        if k in NORM_KINDS:
            if k == OP_GEMM_GN or k == OP_GEMM_LN:
                z = eval_op(dict(op, kind=OP_GEMM, act=0, res=-1, out_col=0), bufs, tb)[:, :op["N"]]
            else:
                z = bufs[op["in0"]["buf"]]
            r, mv = _offset_ratio(z, op, B, N)
            OFFSET[KIND[k]] = max(OFFSET.get(KIND[k], 0.0), r)
            seen[KIND[k]] = (max(seen.get(KIND[k], (0.0, 1e30))[0], r), min(seen.get(KIND[k], (0.0, 1e30))[1], mv))
        if ratio > 1.0:
            fails.append((op["name"], KIND[k], ratio))
    print("worst error / bound:", {"%s/%s" % kk: round(v, 3) for kk, v in sorted(WORST.items())})
    print("largest |mean| / std into a normalisation:", {kk: round(v, 3) for kk, v in sorted(OFFSET.items())})
    assert not fails, fails[:10]
    return seen


@pytest.mark.parametrize("name", list(CASES))
def test_ops_case_fuse5(name):
    """Every golden case at the default fuse level (B = 2 or 3 scenes: one tile)."""
    case = CASES[name]
    eng, spec, sd, ctx = _engine(name, "bf16", 5)
    inp = make_inputs(case, spec)
    check_ops(eng, spec, sd, ctx, inp["x"], inp["t"], inp["context_cross"])


@pytest.mark.parametrize("fuse", [0, 1, 4])
@pytest.mark.parametrize("name", ["bed62", "liv65", "text62"])
def test_ops_case_lower_fuse(name, fuse):
    case = CASES[name]
    eng, spec, sd, ctx = _engine(name, "bf16", fuse)
    inp = make_inputs(case, spec)
    check_ops(eng, spec, sd, ctx, inp["x"], inp["t"], inp["context_cross"])


@pytest.mark.parametrize("prec,fuse", [("bf16", 5), ("bf16", 1), ("fp32", 0)])
@pytest.mark.parametrize("name", ["bed62", "liv65"])
def test_ops_multi_tile(name, prec, fuse):
    """B = 1003 scenes: ragged last tiles of 128-row, 64-row, 10-, 6- and 5-scene tiles; at N = 12, 12036 rows are
    more than 132 x 64, so k_gemm_ln's persistent loop runs past one tile per CTA."""
    case = CASES[name]
    eng, spec, sd, ctx = _engine(name, prec, fuse)
    x, t = _inputs(spec, 1003, case["N"], case["diffusion_kwargs"]["time_num"], 1003)
    check_ops(eng, spec, sd, ctx, x, t)


@pytest.mark.parametrize("n_obj", [1, 7, 13, 16, 17, 25, 32, 33, 64])
def test_ops_object_count_sweep(n_obj):
    """The bed62 network at other object counts: GroupNorm epilogue tiles of floor(128 / N) N rows (N >= 12), the
    <16,0> / <32,0> tensor-core attention cores and the SIMT core above 32; >= 3 tiles and a ragged last tile."""
    case = CASES["bed62"]
    eng, spec, sd, ctx = _engine("bed62", "bf16", 5, n_obj)
    spt = max(1, 128 // n_obj)
    x, t = _inputs(spec, 3 * spt + max(1, spt // 2), n_obj, case["diffusion_kwargs"]["time_num"], n_obj)
    check_ops(eng, spec, sd, ctx, x, t)


# ---------------------------------------------------------------------------------------------------------------
# scene isolation
# ---------------------------------------------------------------------------------------------------------------
ISO = {12: 33, 21: 23, 17: 22}      # batch: attention / GroupNorm tiles of 10 | 5, 6 | 7 scenes, ragged last tile


def _positions(B):
    # first, middle and last scene of a tile (10-scene attention tiles at N = 12, 5 / 6-scene tiles at N = 21), the
    # first of the next, and the last two scenes (the ragged tile)
    return sorted({0, 2, 4, 5, 6, 9, 10, 11, 12, B - 2, B - 1})


@pytest.mark.parametrize("fuse", [0, 1, 4, 5])
@pytest.mark.parametrize("name,n_obj", [("bed62", 12), ("liv65", 21), ("bed62", 17)])
def test_scene_isolation(name, n_obj, fuse):
    """Replacing scene j by other finite values, NaN or +Inf changes no other scene's output by a single bit."""
    if n_obj == 17 and fuse != 5:
        pytest.skip("one fuse level for the sweep object count")
    case = CASES[name]
    eng, spec, sd, ctx = _engine(name, "bf16", fuse, n_obj)
    B = ISO[n_obj]
    x, t = _inputs(spec, B, n_obj, case["diffusion_kwargs"]["time_num"], 77)
    x, t = x.cuda(), t.cuda()
    base = eng.forward(x, t).clone()
    assert torch.isfinite(base).all()
    bad = []
    for j in _positions(B):
        for what, val in (("finite", None), ("nan", float("nan")), ("inf", float("inf"))):
            xj = x.clone()
            xj[j] = 3.0 * torch.randn_like(xj[j]) if val is None else val
            out = eng.forward(xj, t)
            keep = torch.ones(B, dtype=torch.bool, device=out.device)
            keep[j] = False
            if not torch.equal(out[keep], base[keep]):
                diff = (out != base).flatten(1).any(dim=1).nonzero().flatten().tolist()
                bad.append((j, what, [s for s in diff if s != j]))
    assert not bad, bad


@pytest.mark.parametrize("fuse", [0, 1, 4, 5])
@pytest.mark.parametrize("name,n_obj", [("bed62", 12), ("liv65", 21)])
def test_stale_rows_of_a_larger_batch_do_not_leak(name, n_obj, fuse):
    """A batch of B1 scenes leaves its rows past the next, ragged B2-scene batch's last row in the activation
    buffers.  Whether those stale rows are NaN or other finite values, the B2 batch must equal the same batch run on
    its own by a freshly created engine that has never seen a larger batch."""
    case = CASES[name]
    B2 = ISO[n_obj]
    B1 = B2 + 7
    fresh, spec, _, _ = _engine(name, "bf16", fuse, n_obj, cache=False)
    x, t = _inputs(spec, B1, n_obj, case["diffusion_kwargs"]["time_num"], 78)
    x, t = x.cuda(), t.cuda()
    ref = fresh.forward(x[:B2].contiguous(), t[:B2].contiguous()).clone()
    assert torch.isfinite(ref).all()
    eng, _, _, _ = _engine(name, "bf16", fuse, n_obj, cache=False)
    for tail in (None, float("nan"), 5.0):
        xn = x.clone()
        if tail is None:
            xn[B2:] = 3.0 * torch.randn_like(xn[B2:])
        else:
            xn[B2:] = tail
        eng.forward(xn, t)
        out = eng.forward(x[:B2].contiguous(), t[:B2].contiguous())
        assert torch.equal(out, ref), (tail, (out != ref).flatten(1).any(dim=1).nonzero().flatten().tolist())


# ---------------------------------------------------------------------------------------------------------------
# normalisation statistics: offset and small-variance inputs
# ---------------------------------------------------------------------------------------------------------------
SHIPPED_OFFSET = 1.5        # largest |mean| / std into any normalisation of the shipped networks (printed above: 1.45)


def _shift_biases(edit_sd):
    """Shifts every normalisation input far from zero while the exact results stay O(1): +30 on every conv bias in
    front of a GroupNorm (block1 / block2 proj; those outputs have std ~1.3), +1 on every to_out bias in front of a
    LayerNorm (std ~0.06), and +20 on the first ResnetBlock's last GroupNorm shift, which offsets the residual stream
    that every later LayerNorm (+ to_qkv) reads.  Each lands at |mean| / std of 15 to 120, 10x and more the 1.45
    the shipped networks reach."""
    for key in edit_sd:
        if key.endswith((".block1.proj.bias", ".block2.proj.bias")):
            edit_sd[key] = edit_sd[key] + 30.0
        elif key.endswith(".to_out.0.bias"):
            edit_sd[key] = edit_sd[key] + 1.0
    k = "diffusion.model.downs.0.0.block2.norm.bias"
    edit_sd[k] = edit_sd[k] + 20.0


@pytest.mark.parametrize("name,fuse", [("bed62", 5), ("liv65", 5), ("bed62", 0)])
def test_ops_hold_bound_at_offset_inputs(name, fuse):
    """The fused epilogues compute var = E[x^2] - mean^2 in one fp32 pass (k_gemm_wg GroupNorm, k_gemm_ln,
    k_ln_qkv_attn); the unfused k_groupnorm / k_layernorm use two passes.  With every normalisation input at 10x or
    more the shipped |mean| / std, each op still holds its bound.  (A one-pass variance loses ~ratio^2 2^-24 of
    itself per term: near a ratio of 100 k_gemm_ln exceeds the bound, 70x beyond anything the networks produce.)"""
    case = CASES[name]
    eng, spec, sd, ctx = _engine(name, "bf16", fuse, edit=("shift", _shift_biases))
    x, t = _inputs(spec, 37, case["N"], case["diffusion_kwargs"]["time_num"], 5)
    seen = check_ops(eng, spec, sd, ctx, x, t)
    print("offset inputs, fuse %d:" % fuse, {k: round(v[0], 1) for k, v in sorted(seen.items())})
    kinds = (("GEMM_GN", "GEMM_LN") + (("LN_QKV_ATTN",) if fuse == 5 else ())) if fuse else ("GN", "LN")
    for kind in kinds:
        assert seen[kind][0] >= 10 * SHIPPED_OFFSET, (kind, seen[kind])


def _quiet_first_block(s):
    """Scales the encoder output by s and zeroes the first block conv's bias, so the first GroupNorm of the network
    sees groups whose variance is comparable to its eps (1e-5): the eps then changes the output by a large factor."""
    def edit(sd):
        sd["diffusion.model.init_conv.weight"] = sd["diffusion.model.init_conv.weight"] * s
        sd["diffusion.model.init_conv.bias"] = sd["diffusion.model.init_conv.bias"] * 0
        sd["diffusion.model.downs.0.0.block1.proj.bias"] = sd["diffusion.model.downs.0.0.block1.proj.bias"] * 0
    return ("quiet%g" % s, edit)


@pytest.mark.parametrize("fuse", [5, 0])
def test_ops_hold_bound_at_small_group_variance(fuse):
    """A normalisation whose input variance is near eps: the eps of every GroupNorm / LayerNorm kernel must be the
    reference's 1e-5 (denoise_net.py GroupNorm / LayerNorm defaults)."""
    case = CASES["bed62"]
    lo = 1e30
    for s in (3e-2, 1e-2, 3e-3):
        eng, spec, sd, ctx = _engine("bed62", "bf16", fuse, edit=_quiet_first_block(s))
        x, t = _inputs(spec, 37, case["N"], case["diffusion_kwargs"]["time_num"], 6)
        seen = check_ops(eng, spec, sd, ctx, x, t)
        lo = min(lo, seen["GEMM_GN" if fuse else "GN"][1])
        print("scale %g: smallest group variance %.3g" % (s, seen["GEMM_GN" if fuse else "GN"][1]))
    assert lo <= 1e-4, lo      # some group had a variance where eps matters at the percent level
