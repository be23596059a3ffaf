"""GPU, op by op: the backward pass of the native training step (ds_train_step[_cross]) against float64, at the batch
`bench.py --config train` runs (1024 scenes of 21 objects) and at the shapes where its kernels change behaviour.

One native step runs with gradients; then every op of the train program is re-evaluated on the GPU in float64 with
torch.func.vjp of oracle.plan_interp.eval_op, from the exact values its kernels read (ds_train_read: activations,
final gradient buffers, packed dW, vector gradients, FiLM rows; tests/test_plan_cpu.py::
test_train_plan_state_after_the_step_is_what_each_backward_read shows that the post-step buffers are those values).
Primals: the widened input activations, the packed weights restated as ds_train_step packs them (packed_wmat of
test_gpu_bf16_ops, bf16 in bf16 mode), the vectors and the FiLM rows; cotangent: the op's final output-gradient
slice.  Checked: packed dW, bias / gamma / beta / LayerNorm-gain gradients, d(FiLM rows), and every input gradient
buffer against the SUM of its consumers' input cotangents (a dropped or doubled consumer, or a wrong first-writer
flag, fails).  Then the named flat gradients: the weight-standardisation adjoint applied to the native packed dW,
and the conditioning paths (time MLP, FiLM projections, context MLPs, d(context)) each stage from the native values
of the stage before.  Errors do not compound.  No CPU reference runs at these sizes.

Bounds, per element (never on a mean).  u = 2^-24; ulp(v) is the bf16 spacing at |v| (test_gpu_bf16_ops.bf16_ulp).
- fp32-accumulated reductions (dW on the tensor cores or the SIMT kernel, bias / gamma / beta / FiLM sums, the
  conditioning GEMMs): D * 2u * sum|terms|, sum|terms| in fp64 (|dY|^T |X| for a GEMM), D the longest chain of fp32
  additions any result sees, from the launch geometry:
    tensor-core split-K dW: K_split / 16 + ksplit + 2 (k16 products per split, then the fp32 atomics);
    SIMT dW (k_gemm_tn): m_chunk + splits + 2;  SIMT dX / conditioning GEMMs (k_gemm_nn): K + 2;
    bias from the dY transpose: M / 32 + 12;  k_colsum: 256 + M / 256 + 2;
    GroupNorm gamma / beta: N + B + 2;  time FiLM: N + 2;  shared-context FiLM: N + B + 2;  LayerNorm gain:
    64 + M / 64 + 2.
  The data is random-signed, so a missing 64-row k-block moves a dW element by ~sqrt(64) / K_split of sum|terms|,
  far above this bound at the bench shape; the margin reached is printed.  Normalisation gradients add 2^-18 *
  sum|terms| for the fp32 statistics the kernels recompute.
- Outputs stored in bf16 (input-gradient buffers, d(model output)): ulp(S) per rounding in the accumulation chain
  (one per consumer writing the slice), S = sum over consumers of |contribution|, plus the fp32 term of each
  consumer: the GEMM term above for dX, 2^-12 * RMS(row) of the contribution for the elementwise / normalisation /
  attention backward kernels (fp32 arithmetic with exact erf-GELU and SiLU, backward.cu act_grad: no approximation
  allowance is needed).
- fp32 mode: the same fp32 terms, with 2^-15 * (|ref| + RMS(row)) for the elementwise kernels and no rounding term.
- The loss gradient: fp64 autograd of oracle.diffusion_ref.p_losses on the device, from the model output and the fp32
  x_t the kernels read: ulp(ref) (bf16 mode) + 2^-16 * (|ref| + max |ref| of the scene), and on the box channels the
  derived fp32 bound of the IoU regulariser (iou_grad_bound).
- Named gradients of standardised weights: the fp64 adjoint of the native packed dW, 2^-16 (|ref| + RMS(row)).
WORST collects (precision, op kind, gradient kind) -> worst err / bound and is printed.
"""
import dataclasses
import math
import time

import pytest
import torch
import torch.nn.functional as F

from diffuscene_b200 import capi
from diffuscene_b200.engine import DenoiserEngine
from diffuscene_b200.weights import NetSpec, seeded_state_dict, unet1d_param_specs
from oracle import diffusion_ref as D
from oracle.plan_interp import (OP_ACT, OP_ATTN, OP_GEMM, OP_GN, OP_LINATTN, OP_LN, OP_PACK, OP_XATTN, PlanTables,
                                assemble_vec, eval_op, xattn_contexts)
from tests.cases import CASES, STATS, _clean_scene, _dk
from tests.gpu_common import case_tables
from tests.test_gpu_bf16_ops import bf16_ulp, packed_wmat

pytestmark = pytest.mark.gpu

KIND = {OP_GEMM: "GEMM", OP_ACT: "ACT", OP_GN: "GN", OP_LN: "LN", OP_LINATTN: "LINATTN", OP_ATTN: "ATTN",
        OP_XATTN: "XATTN"}
U = 2.0 ** -24
GRAD_SCALE = 0.125      # the data-parallel mean over 8 ranks
WORST = {}              # (precision, op kind, gradient kind) -> worst |err| / bound
MARGIN = {}             # case -> smallest (k-block effect / bound) of a tensor-core split-K dW
LIVE = []               # at most two engines alive

# case: network, objects, batch, precision, text length, shared context
NETS = {
    # the living-room network of `bench.py --config train`: v-prediction, fixedsmall, loss_separate + loss_iou, d = 65
    "liv": (CASES["liv65"]["net_kwargs"], CASES["liv65"]["net_cfg"], _dk(mean="v", var="fixedsmall", iou=True), 21),
    "bed": (CASES["bed62"]["net_kwargs"], CASES["bed62"]["net_cfg"], CASES["bed62"]["diffusion_kwargs"], 12),
    "text": (CASES["text62"]["net_kwargs"], CASES["text62"]["net_cfg"], CASES["text62"]["diffusion_kwargs"], 12),
    "arr": (CASES["arr5"]["net_kwargs"], CASES["arr5"]["net_cfg"], dict(CASES["arr5"]["diffusion_kwargs"], loss_separate=False), 12),
    "obj": (CASES["obj29"]["net_kwargs"], CASES["obj29"]["net_cfg"], CASES["obj29"]["diffusion_kwargs"], 12),
}
TABLE = {
    "bench": ("liv", 1024, "bf16", 0, True),
    "bench32": ("liv", 512, "fp32", 0, True),
    "ragged": ("bed", 1003, "bf16", 0, True),
    "text": ("text", 256, "bf16", 33, True),
    "token_ctx": ("arr", 512, "bf16", 0, False),
    "objectness": ("obj", 256, "bf16", 0, True),
}


def _release(keep=1):
    while len(LIVE) > keep:
        LIVE.pop(0).close()
    torch.cuda.empty_cache()


class Net:
    """A seeded network, its train plan and one handle."""

    def __init__(self, net, prec, seed=29):
        kw, self.ncfg, self.dk, self.N = NETS[net]
        self.spec = NetSpec.from_net_kwargs(kw)
        self.prec = prec
        _release(1)
        self.eng = DenoiserEngine(self.spec, self.N, self.dk["time_num"], precision=prec)
        LIVE.append(self.eng)
        self.eng.set_schedule(case_tables(dict(diffusion_kwargs=self.dk)))
        sd = seeded_state_dict(unet1d_param_specs(self.spec), seed=seed)
        self.sd = {k[len("diffusion.model."):]: v for k, v in sd.items()}
        self.layout = {k[len("diffusion.model."):]: v for k, v in self.eng.flat_layout().items()}
        total = sum(n for _, n in self.layout.values())
        self.flat = torch.empty(total, device="cuda")
        for k, (off, n) in self.layout.items():
            self.flat[off:off + n] = self.sd[k].reshape(-1).cuda()
        cfg = capi.make_config(self.spec, self.N, self.dk["time_num"], train=True,
                               precision=capi.DS_PREC_BF16 if prec == "bf16" else capi.DS_PREC_FP32)
        self.plan = capi.plan_export(cfg, no_reuse=True)
        self.max_B = 0

    def batch(self, B, seed, L=0, shared=True):
        g = torch.Generator().manual_seed(seed)
        s, N = self.spec, self.N
        if self.ncfg.get("room_arrange_condition"):
            tr = torch.rand(B, N, s.translation_dim, generator=g) * 2 - 1
            an = F.normalize(torch.randn(B, N, s.point_dim - s.translation_dim, generator=g), dim=-1)
            x0 = torch.cat([tr, an], dim=-1)
        else:
            x0 = _clean_scene(g, B, N, s)
        t = torch.randint(0, self.dk["time_num"], (B,), generator=g)
        noise = torch.randn(x0.shape, generator=g)
        ctx = torch.randn(*((N,) if shared else (B, N)), s.cond_dim, generator=g)
        cross = torch.randn(B, L, s.text_dim, generator=g) if L else None
        return dict(x0=x0, t=t, noise=noise, ctx=ctx, shared=shared, cross=cross, B=B)

    def step(self, b):
        self.max_B = max(self.max_B, b["B"])
        grads = torch.full_like(self.flat, float("nan"))
        out = self.eng.train_step(self.flat, b["x0"].cuda(), b["t"].cuda(), b["noise"].cuda(), b["ctx"].cuda(),
                                  b["shared"], self.dk["loss_separate"], self.dk["loss_iou"],
                                  STATS["bounds_translations"] + STATS["bounds_sizes"], flat_grads=grads,
                                  grad_scale=GRAD_SCALE, cross=None if b["cross"] is None else b["cross"].cuda())
        torch.cuda.synchronize()
        return dict(losses=out[0], dctx=out[2], dcross=out[3] if len(out) > 3 else None, grads=grads)


# ---------------------------------------------------------------------------------------------------------------------
# launch geometry -> length of the longest fp32 accumulation chain (train.cu / backward.cu)
# ---------------------------------------------------------------------------------------------------------------------
def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _cdiv(a, b):
    return (a + b - 1) // b


def tc_dw_depth(N_out, k_in, rows_cap):
    """train_capacity: ksplit of the split-K dW plan, and its chain length K_split / 16 + ksplit + 2."""
    tiles = _cdiv(N_out, 128) * (k_in // 128)
    kblocks = rows_cap // 64
    ksplit = min(max(1, 2 * _sms() // max(1, tiles)), kblocks)
    kb_per = _cdiv(kblocks, ksplit)
    ksplit = _cdiv(kblocks, kb_per)
    return kb_per * 4 + ksplit + 2, ksplit, kb_per


def simt_dw_depth(M, Ka, Kb):
    """launch_gemm_tn: m_chunk sequential rows per thread, then one atomic per split."""
    tiles = _cdiv(Ka, 64) * _cdiv(Kb, 64)
    splits = _cdiv(4 * _sms(), tiles)
    m_chunk = max(64, _cdiv(_cdiv(M, splits), 16) * 16)
    return m_chunk + _cdiv(M, m_chunk) + 2


def last_split_block(gout, M, N_out, k_in, rows_cap):
    """First row of the 64-row k-block of the last split whose dY has the largest norm."""
    _, ksplit, kb_per = tc_dw_depth(N_out, k_in, rows_cap)
    first = min((ksplit - 1) * kb_per * 64, (M - 1) // (kb_per * 64) * kb_per * 64)      # the last with real rows
    rows = list(range(first, M, 64))
    norms = [gout[r:r + 64].norm().item() for r in rows]
    return rows[max(range(len(rows)), key=norms.__getitem__)]


def _rms(z):
    return z.pow(2).mean(dim=-1, keepdim=True).sqrt()


def _ratio(key, got, ref, bound):
    err = (got - ref).abs()
    r = (err / bound.clamp_min(1e-300)).max().item() if err.numel() else 0.0
    if not math.isfinite(r):
        r = float("inf")
    WORST[key] = max(WORST.get(key, 0.0), r)
    return r


# ---------------------------------------------------------------------------------------------------------------------
# the loss: oracle.diffusion_ref on the device, and what fp32 evaluation of the IoU regulariser may change
# ---------------------------------------------------------------------------------------------------------------------
def loss_schedule(dk, dev="cuda"):
    s = D.make_schedule(D.make_betas(dk["schedule_type"], dk["beta_start"], dk["beta_end"], dk["time_num"]),
                        dk["model_mean_type"], dk["model_var_type"])
    return dataclasses.replace(s, **{f.name: getattr(s, f.name).to(dev) for f in dataclasses.fields(s)
                                      if isinstance(getattr(s, f.name), torch.Tensor)})


def loss_spec(net):
    return D.LossSpec(class_dim=net.ncfg["class_dim"], angle_dim=net.ncfg["angle_dim"],
                      objfeat_dim=net.ncfg["objfeat_dim"], objectness_dim=net.ncfg["objectness_dim"],
                      loss_separate=net.dk["loss_separate"], loss_iou=net.dk["loss_iou"],
                      bounds_translations=STATS["bounds_translations"], bounds_sizes=STATS["bounds_sizes"],
                      room_arrange_condition=net.ncfg.get("room_arrange_condition", False))


def iou_grad_bound(net, sched, out, xt, t, B):
    """Per-element bound [B, N, d] on what k_p_losses_bwd's fp32 evaluation of the IoU regulariser may differ from
    its fp64 gradient, from the same out and x_t.  The kernel forms raw = a_x x_t + a_o out (error e_raw <= 4u (|a_x x_t|
    + |a_o out|)), the clamped reconstruction, box corners (error e_c), and per ordered pair (i, j) the IoU terms,
    summed per corner by fp32 shared-memory atomics (4N + 8 additions).  Each pair term is a product / quotient of
    sides, overlaps wh and the union un, so to first order its relative error is
    r = 2 e_un / un + 2 sum_m e_wh / wh_m + sum of side errors / sides + 16u.  Besides r |term|, three predicates can
    flip between fp32 and fp64, and only where they are within that error of flipping is more allowed:
    - a min / max of two corners within 2 e_c of a tie, or an overlap width raww within 2 e_c of 0: the whole
      overlap term |gwh| of that pair and axis, on both boxes;
    - a clamp within e_raw of +-1: the element's whole would-be gradient;
    - a valid flag within e_raw of its threshold: every box channel of the scene (with the flag either way).
    Each term is added to both boxes' lo and hi corners, an upper bound of what any assignment gives them."""
    s, ncfg = net.spec, net.ncfg
    N, dv = out.shape[1], out.dtype
    per_scene = GRAD_SCALE / B
    sa, s1 = sched.sqrt_ac.double()[t], sched.sqrt_1mac.double()[t]
    mt = net.dk["model_mean_type"]
    if mt == "v":
        ax, ao = sa, -s1
    elif mt == "eps":
        ax, ao = sched.sqrt_recip_ac.double()[t], -sched.sqrt_recipm1_ac.double()[t]
    else:
        ax, ao = torch.zeros_like(sa), torch.ones_like(sa)
    ax, ao = ax[:, None, None], ao[:, None, None]
    raw = ax * xt + ao * out
    e_raw = 4 * U * ((ax * xt).abs() + (ao * out).abs())
    xr = raw.clamp(-1, 1)
    td = s.translation_dim
    bb = td + s.size_dim + s.angle_dim
    vch = bb + ncfg["class_dim"] if ncfg["objectness_dim"] > 0 else bb + ncfg["class_dim"] - 1
    rv, ev = raw[..., vch], e_raw[..., vch]
    valid = (rv >= 0) if ncfg["objectness_dim"] > 0 else (rv <= 0)
    v_amb = rv.abs() <= ev
    valid_any = valid | v_amb
    bt = torch.tensor(STATS["bounds_translations"], dtype=torch.float32).double().to(out.device)
    bs = torch.tensor(STATS["bounds_sizes"], dtype=torch.float32).double().to(out.device)
    rt, rs = bt[3:] - bt[:3], bs[3:] - bs[:3]
    tr = (xr[..., :3] + 1) / 2 * rt + bt[:3]
    sz = (xr[..., td:td + 3] + 1) / 2 * rs + bs[:3]
    e_c = (e_raw[..., :3] * rt / 2 + e_raw[..., td:td + 3] * rs / 2
           + 8 * U * (tr.abs() + sz.abs() + rt + rs + bt[:3].abs() + bs[:3].abs()))
    lo, hi = tr - sz, tr + sz
    side = hi - lo
    assert side.prod(-1).min().item() > 1e-5      # unions stay far above the kernel's 1e-6 floor
    area = side.prod(-1)
    li, lj, hi_i, hj = lo[:, :, None], lo[:, None], hi[:, :, None], hi[:, None]
    eij = e_c[:, :, None] + e_c[:, None]
    raww = torch.minimum(hi_i, hj) - torch.maximum(li, lj)       # [B, N, N, 3]
    wh = raww.clamp_min(0)
    ov = wh.prod(-1)
    un = (area[:, :, None] + area[:, None] - ov).clamp_min(1e-6)
    nv_min = (valid & ~v_amb).sum(1).to(dv)
    wpair = (sched.alphas_cumprod.double()[t] * 0.1 / (nv_min ** 2 + 1e-6) * per_scene)[:, None, None]
    vv = (valid_any[:, :, None] & valid_any[:, None]).to(dv)
    d_ov = wpair * (1 / un + ov / un ** 2) * vv
    d_area = wpair * ov / un ** 2 * vv
    other = torch.stack([wh[..., 1] * wh[..., 2], wh[..., 0] * wh[..., 2], wh[..., 0] * wh[..., 1]], -1)
    gwh = d_ov[..., None] * other
    act = (raww >= 0).to(dv)
    prod_i = area[:, :, None, None] / side[:, :, None, :]
    e_wh = eij / wh.clamp_min(1e-300)
    e_wh = torch.where(wh > eij, e_wh, torch.ones_like(e_wh))
    e_side = (2 * e_c / side).sum(-1)
    e_un = (area[:, :, None] * e_side[:, :, None] + area[:, None] * e_side[:, None] + ov * e_wh.sum(-1)
            + 3 * U * (area[:, :, None] + area[:, None] + ov))
    r = (2 * e_un / un + 2 * e_wh.sum(-1) + e_side[:, :, None] + e_side[:, None] + 16 * U)[..., None]
    term = d_area[..., None] * prod_i + act * gwh                  # magnitude, per ordered pair, axis
    flip = ((hi_i - hj).abs() <= 2 * eij) | ((li - lj).abs() <= 2 * eij) | (raww.abs() <= 2 * eij)
    excuse = gwh * flip.to(dv)
    # i gets each pair term as first and as second box of an ordered pair; lo and hi alike
    T = 2 * term.sum(2)
    err = 2 * (r * term + excuse).sum(2) + (4 * N + 8) * 2 * U * T
    res = torch.zeros_like(out)
    amb_pass = ((raw.abs() - 1).abs() <= e_raw)
    for k in range(3):
        for ch, rng in ((k, rt[k]), (td + k, rs[k])):
            mag = T[..., k] * rng * ao[..., 0].abs()                 # would-be gradient magnitude of the channel
            e = err[..., k] * rng * ao[..., 0].abs()
            passes = (raw[..., ch].abs() <= 1).to(dv)
            res[..., ch] = e * passes + mag * amb_pass[..., ch].to(dv) + mag * v_amb.any(1, keepdim=True).to(dv)
    return res


# ---------------------------------------------------------------------------------------------------------------------
# the checker
# ---------------------------------------------------------------------------------------------------------------------
def check_backward(net, b, mutate=None, case=None):
    """Everything of the last step against fp64; returns the list of (what, ratio) over 1.  `mutate(kind, index, t)`
    may replace a native array before it is compared (the perturbation tests)."""
    eng, plan, prec = net.eng, net.plan, net.prec
    bf = prec == "bf16"
    use_tc = bf
    B, N = b["B"], net.N
    M, C = B * N, plan["C"]
    rows_cap = _cdiv(net.max_B * N, 128) * 128
    dev = torch.device("cuda")
    fails = []

    def rd(kind, idx):
        t = eng.train_read(kind, idx)
        if mutate is not None:
            t = mutate(kind, idx, t)
        return t.double()

    def note(what, key, got, ref, bound):
        r = _ratio((prec,) + key, got, ref, bound)
        if r > 1.0:
            fails.append((what, round(r, 3)))
        return r

    ops = plan["ops"]
    pack_buf = next(op["out"] for op in ops if op["kind"] == OP_PACK)
    wm = {}
    vecs = [assemble_vec(r, net.sd).double().to(dev) for r in plan["vecs"]]
    film = rd(capi.DS_TRAIN_COND, "film") if plan["time_blocks"] else None
    ctx_film = rd(capi.DS_TRAIN_COND, "ctx_film") if plan["ctx_blocks"] else None
    dfilm = rd(capi.DS_TRAIN_COND, "dfilm") if plan["time_blocks"] else None
    dctx_film = rd(capi.DS_TRAIN_COND, "dctx_film") if plan["ctx_blocks"] else None
    xctx = None
    if plan["xattn_layers"]:
        xctx = rd(capi.DS_TRAIN_COND, "xctx").reshape(len(plan["xattn_layers"]), B, 4, 32, 32)
    dxctx_ref = {}
    shared = b["shared"]

    # ---- 1. loss backward: fp64 autograd of p_losses on the model output the kernel read
    d = net.spec.point_dim
    out_w = rd(capi.DS_TRAIN_ACT, plan["out_buf"])
    o = out_w[:, :d].reshape(B, N, d).requires_grad_(True)
    sched = loss_schedule(net.dk)
    ls = loss_spec(net)
    xt = rd(capi.DS_TRAIN_COND, "x_t").reshape(B, N, d)      # the noisy input the loss kernels read (fp32 q_sample)
    x0, tt, nz = b["x0"].to(dev, torch.float64), b["t"].to(dev), b["noise"].to(dev, torch.float64)
    with torch.enable_grad():
        losses, _ = D.p_losses(sched, ls, lambda xx, t_: o, x0, tt, nz, x_t=xt)
        (losses.mean() * GRAD_SCALE).backward()
    ref = o.grad.reshape(M, d)
    got_full = rd(capi.DS_TRAIN_GRAD, plan["out_buf"])
    got = got_full[:, :d]
    smax = ref.reshape(B, N * d).abs().amax(dim=1, keepdim=True).expand(B, N * d).reshape(M, d)
    bound = 2.0 ** -16 * (ref.abs() + smax) + (bf16_ulp(ref) if bf else 0)
    if ls.loss_iou and not ls.room_arrange_condition:
        bound = bound + iou_grad_bound(net, sched, o.detach(), xt, tt, B).reshape(M, d)
    note("d(model output)", ("LOSS", "dX"), got, ref, bound)
    if got_full.shape[1] > d and got_full[:, d:].abs().max().item() != 0:
        fails.append(("d(model output) padding is not zero", float("inf")))

    # ---- 2. every op in reverse
    acc, mag, bnd, cnt = {}, {}, {}, {}      # per input-gradient buffer: sum of consumer cotangents and their bounds
    first_writer = {}
    for i, op in enumerate(ops):
        first_writer.setdefault(op["out"], i)

    def add_in(buf, c0, c1, val, bound_c):
        w = plan["buf_width"][buf]
        if buf not in acc:
            acc[buf] = torch.zeros(M, w, dtype=torch.float64, device=dev)
            mag[buf] = torch.zeros_like(acc[buf])
            bnd[buf] = torch.zeros_like(acc[buf])
            cnt[buf] = torch.zeros(w, dtype=torch.float64, device=dev)
        acc[buf][:, c0:c1] += val
        mag[buf][:, c0:c1] += val.abs()
        bnd[buf][:, c0:c1] += bound_c
        cnt[buf][c0:c1] += 1

    def close_buf(buf, opname):
        if buf not in acc:
            return
        ref, m, bd, n = acc.pop(buf), mag.pop(buf), bnd.pop(buf), cnt.pop(buf)
        live = n > 0
        got = rd(capi.DS_TRAIN_GRAD, buf)[:, live]
        bound = bd[:, live] + (n[live] * bf16_ulp(m[:, live]) if bf else 0)
        note("d(%s)" % opname, ("BUF", "dX"), got, ref[:, live], bound)

    for i in range(len(ops) - 1, -1, -1):
        op = ops[i]
        k = op["kind"]
        if k == OP_PACK:
            continue
        c0, c1 = op["out_col"], op["out_col"] + op["N"]
        gout = rd(capi.DS_TRAIN_GRAD, op["out"])[:, c0:c1]
        ct = torch.zeros(M, plan["buf_width"][op["out"]], dtype=torch.float64, device=dev)
        ct[:, c0:c1] = gout
        p = {}
        ins = [s for s in (op["in0"], op.get("in1", {"buf": -1})) if s["buf"] >= 0]
        for s in ins:
            p["b%d" % s["buf"]] = rd(capi.DS_TRAIN_ACT, s["buf"])
        if op.get("res", -1) >= 0:
            p["b%d" % op["res"]] = rd(capi.DS_TRAIN_ACT, op["res"])
        if k == OP_GEMM:
            if op["w"] not in wm:
                wm[op["w"]] = packed_wmat(plan["wmats"][op["w"]], net.sd, bf).to(dev)
            p["w"] = wm.pop(op["w"])
            if op["b"] >= 0:
                p["v%d" % op["b"]] = vecs[op["b"]]
        elif k == OP_GN:
            p["v%d" % op["gamma"]] = vecs[op["gamma"]]
            p["v%d" % op["beta"]] = vecs[op["beta"]]
            if op["film"] == 1:
                p["film"] = film[:, op["film_blk"] * 2 * C:(op["film_blk"] + 1) * 2 * C]
            elif op["film"] == 2:
                p["film"] = ctx_film[:, op["film_blk"] * 2 * C:(op["film_blk"] + 1) * 2 * C]
        elif k == OP_LN:
            p["v%d" % op["b"]] = vecs[op["b"]]
        elif k == OP_XATTN:
            p["xctx"] = xctx[op["xlayer"]]
        placeholder = torch.zeros(M, plan["buf_width"][op["out"]], dtype=torch.float64, device=dev)

        def f(pp, op=op, placeholder=placeholder):
            bufs = {int(key[1:]): v for key, v in pp.items() if key[0] == "b"}
            bufs.setdefault(op["out"], placeholder)
            vv = {int(key[1:]): v for key, v in pp.items() if key[0] == "v"}
            ft, fc = {}, {}
            if "film" in pp:
                if op["film"] == 1:
                    ft[op["film_blk"]] = pp["film"]
                elif shared:
                    fc[op["film_blk"]] = pp["film"][None].expand(B, N, 2 * C).reshape(M, 2 * C)
                else:
                    fc[op["film_blk"]] = pp["film"]
            tb = PlanTables(plan, B, N, {op.get("w", -1): pp.get("w")}, vv, ft, fc,
                            {op.get("xlayer", 0): pp.get("xctx")})
            return eval_op(op, bufs, tb)

        _, vjp = torch.func.vjp(f, p)
        (g,) = vjp(ct)
        name = op["name"]
        kk = KIND[k]
        if k == OP_GEMM:
            X = torch.cat([p["b%d" % s["buf"]][:, s["col"]:s["col"] + s["k"]] for s in ins], dim=1)
            K = op["N"]
            ref_dw, got_dw = g["w"], rd(capi.DS_TRAIN_DW, op["w"])
            absdw = gout.abs().t() @ X.abs()
            koff = 0
            tc_bias = False
            for s in ins:
                sl = slice(koff, koff + s["k"])
                tc = use_tc and s["k"] % 128 == 0 and op["N"] % 128 == 0
                if tc:
                    depth, ksplit, kb_per = tc_dw_depth(op["N"], s["k"], rows_cap)
                    tc_bias = True
                else:
                    depth = simt_dw_depth(M, op["N"], s["k"])
                bound = depth * 2 * U * absdw[:, sl]
                note("dW %s" % name, (kk, "dW"), got_dw[:, sl], ref_dw[:, sl], bound)
                if tc and case is not None:
                    # what one 64-row k-block of the last split contributes, against the bound
                    r0 = last_split_block(gout, M, op["N"], s["k"], rows_cap)
                    blk = gout[r0:r0 + 64].t() @ X[r0:r0 + 64, sl]
                    eff = (blk.abs() / bound.clamp_min(1e-300)).max().item()
                    MARGIN[case] = min(MARGIN.get(case, float("inf")), eff)
                koff += s["k"]
            if op["b"] >= 0:
                depth = M / 32 + 12 if tc_bias else 256 + M / 256 + 2
                note("db %s" % name, (kk, "dvec"), rd(capi.DS_TRAIN_DVEC, op["b"])[0], g["v%d" % op["b"]],
                     depth * 2 * U * gout.abs().sum(dim=0))
            koff = 0
            for s in ins:
                Wsl = p["w"][:, koff:koff + s["k"]]
                koff += s["k"]
                if s["buf"] == pack_buf:
                    continue
                tcx = use_tc and s["k"] % 128 == 0 and op["N"] % 64 == 0
                depth = K / 16 + 2 if tcx else K + 2
                val = g["b%d" % s["buf"]][:, s["col"]:s["col"] + s["k"]]
                add_in(s["buf"], s["col"], s["col"] + s["k"], val, depth * 2 * U * (gout.abs() @ Wsl.abs()))
            if op.get("res", -1) >= 0:
                add_in(op["res"], 0, plan["buf_width"][op["res"]], g["b%d" % op["res"]], torch.zeros_like(gout))
        else:
            for s in ins:
                val = g["b%d" % s["buf"]][:, s["col"]:s["col"] + s["k"]]
                ew = (2.0 ** -12 * _rms(val)) if bf else 2.0 ** -15 * (val.abs() + _rms(val))
                add_in(s["buf"], s["col"], s["col"] + s["k"], val, ew.expand_as(val))
            if op.get("res", -1) >= 0:
                add_in(op["res"], 0, plan["buf_width"][op["res"]], g["b%d" % op["res"]], torch.zeros_like(gout))
            if k in (OP_GN, OP_LN):
                nv = _norm_vec_terms(op, p, gout, B, N, C, shared)
                for key, (vid, depth) in nv["vecs"].items():
                    note("d%s %s" % (key, name), (kk, "dvec"), rd(capi.DS_TRAIN_DVEC, vid)[0], g["v%d" % vid],
                         (depth * 2 * U + 2.0 ** -18) * nv["abs"][key])
                if "film" in p:
                    blk = op["film_blk"]
                    got_f = (dfilm if op["film"] == 1 else dctx_film)[:, blk * 2 * C:(blk + 1) * 2 * C]
                    depth = N + 2 if op["film"] == 1 else (N + B + 2 if shared else 1)
                    note("dfilm %s" % name, (kk, "dfilm"), got_f, g["film"],
                         (depth * 2 * U + 2.0 ** -18) * nv["abs"]["film"] + 2.0 ** -40)
            if k == OP_XATTN:
                dxctx_ref[op["xlayer"]] = g["xctx"]
        del g, p, ct
        # a buffer is complete once the backward pass has gone past its first writer
        for buf in [bb for bb in acc if first_writer.get(bb, -1) >= i]:
            close_buf(buf, name)
    for buf in list(acc):
        close_buf(buf, "end")

    # ---- 3. weight-standardisation adjoint and vector copies: named flat gradients from the native packed ones
    grads = b["grads"]
    G = lambda n: grads[net.layout[n][0]:net.layout[n][0] + net.layout[n][1]].double()
    for w, r in enumerate(plan["wmats"]):
        dwp = rd(capi.DS_TRAIN_DW, w)
        for pc in r["pieces"]:
            dp = dwp[pc["row_off"]:pc["row_off"] + pc["rows"], pc["col_off"]:pc["col_off"] + pc["cols"]]
            if r["ws"]:
                src = net.sd[pc["name"]].reshape(pc["rows"], pc["cols"]).double().to(dev)
                std = lambda z: (z - z.mean(dim=1, keepdim=True)) / torch.sqrt(z.var(dim=1, unbiased=False, keepdim=True) + 1e-5)
                _, vj = torch.func.vjp(std, src)
                (ref,) = vj(dp)
                note("ws adjoint %s" % pc["name"], ("UNPACK", "dW"), G(pc["name"]).reshape(ref.shape), ref,
                     2.0 ** -16 * (ref.abs() + _rms(ref)))
            elif not torch.equal(G(pc["name"]).reshape(dp.shape), dp):
                fails.append(("copy of %s" % pc["name"], float("inf")))
    for v, r in enumerate(plan["vecs"]):
        dv = rd(capi.DS_TRAIN_DVEC, v)[0]
        for pc in r["pieces"]:
            if not torch.equal(G(pc["name"]), dv[pc["off"]:pc["off"] + pc["n"]]):
                fails.append(("copy of %s" % pc["name"], float("inf")))

    # ---- 4. conditioning paths, each stage from the native values of the stage before
    cond = lambda n: rd(capi.DS_TRAIN_COND, n)
    W = lambda n: net.sd[n].double().to(dev)
    silu_d = lambda x: torch.sigmoid(x) * (1 + x * (1 - torch.sigmoid(x)))
    gelu_d = lambda x: 0.5 * (1 + torch.erf(x / math.sqrt(2))) + x * torch.exp(-0.5 * x * x) / math.sqrt(2 * math.pi)
    rnd = (lambda z: z.to(torch.bfloat16).double()) if bf else (lambda z: z)
    ntb = len(plan["time_blocks"])
    st = cond("st")
    film_tc = bf
    dst_ref = torch.zeros_like(st)
    dst_abs = torch.zeros_like(st)
    for i, n in enumerate(plan["time_blocks"]):
        df = dfilm[:, i * 2 * C:(i + 1) * 2 * C]
        if film_tc:      # k_dfilm_prepare rounds d(FiLM); the packers round the weights and SiLU(temb)
            a, x, w_ = rnd(df), rnd(st), rnd(W(n + ".mlp.1.weight"))
            depth, _, _ = tc_dw_depth(2 * C, 4 * C, _cdiv(B, 128) * 128)
            dbd = B / 32 + 12
        else:
            a, x, w_ = df, st, W(n + ".mlp.1.weight")
            depth, dbd = simt_dw_depth(B, 2 * C, 4 * C), 256 + B / 256 + 2
        note("%s.mlp.1.weight" % n, ("TIME_FILM", "dW"), G(n + ".mlp.1.weight").reshape(2 * C, 4 * C), a.t() @ x,
             depth * 2 * U * (a.abs().t() @ x.abs()))
        note("%s.mlp.1.bias" % n, ("TIME_FILM", "dvec"), G(n + ".mlp.1.bias"), df.sum(dim=0),
             dbd * 2 * U * df.abs().sum(dim=0))
        dst_ref += a @ w_
        dst_abs += a.abs() @ w_.abs()
    temb, h1, z1, emb = cond("temb"), cond("h1"), cond("z1"), cond("emb")
    # d(st) is a [B, 19 x 2C] x [19 x 2C, 4C] product, rounded to bf16 once in bf16 mode (first order through SiLU')
    kd = ntb * 2 * C
    e_dst = ((kd / 16 + 2) if film_tc else (2 * C + ntb + 2)) * 2 * U * dst_abs + (bf16_ulp(dst_ref) if bf else 0)
    dtemb = cond("dtemb")
    note("d(temb)", ("TIME_MLP", "dX"), dtemb, dst_ref * silu_d(temb), e_dst * silu_d(temb).abs() + 2.0 ** -20 * _rms(dtemb))
    w3 = W("time_mlp.3.weight")
    dd = simt_dw_depth(B, 4 * C, 4 * C)
    note("time_mlp.3.weight", ("TIME_MLP", "dW"), G("time_mlp.3.weight").reshape(4 * C, 4 * C), dtemb.t() @ h1,
         dd * 2 * U * (dtemb.abs().t() @ h1.abs()))
    note("time_mlp.3.bias", ("TIME_MLP", "dvec"), G("time_mlp.3.bias"), dtemb.sum(0), (258 + B / 256) * 2 * U * dtemb.abs().sum(0))
    dh1 = cond("dh1")
    note("d(h1)", ("TIME_MLP", "dX"), dh1, dtemb @ w3, (4 * C + 2) * 2 * U * (dtemb.abs() @ w3.abs()))
    dz1 = cond("dst")      # after the step dst holds d(z1)
    note("d(z1)", ("TIME_MLP", "dX"), dz1, dh1 * gelu_d(z1), 2.0 ** -20 * (dz1.abs() + _rms(dz1)))
    dd = simt_dw_depth(B, 4 * C, C)
    note("time_mlp.1.weight", ("TIME_MLP", "dW"), G("time_mlp.1.weight").reshape(4 * C, C), dz1.t() @ emb,
         dd * 2 * U * (dz1.abs().t() @ emb.abs()))
    note("time_mlp.1.bias", ("TIME_MLP", "dvec"), G("time_mlp.1.bias"), dz1.sum(0), (258 + B / 256) * 2 * U * dz1.abs().sum(0))
    if plan["ctx_blocks"]:
        ca = cond("ctx_act")
        rows = ca.shape[0]
        E = ca.shape[1]
        dca_ref = torch.zeros_like(ca)
        dca_abs = torch.zeros_like(ca)
        for i, n in enumerate(plan["ctx_blocks"]):
            df = dctx_film[:, i * 2 * C:(i + 1) * 2 * C]
            dd = simt_dw_depth(rows, 2 * C, E)
            note("%s.mlp.1.weight" % n, ("CTX_FILM", "dW"), G(n + ".mlp.1.weight").reshape(2 * C, E), df.t() @ ca,
                 dd * 2 * U * (df.abs().t() @ ca.abs()))
            note("%s.mlp.1.bias" % n, ("CTX_FILM", "dvec"), G(n + ".mlp.1.bias"), df.sum(0),
                 (258 + rows / 256) * 2 * U * df.abs().sum(0))
            dca_ref += df @ W(n + ".mlp.1.weight")
            dca_abs += df.abs() @ W(n + ".mlp.1.weight").abs()
        dca = cond("dctx_act")
        note("d(SiLU(context))", ("CTX_FILM", "dX"), dca, dca_ref, (2 * C + len(plan["ctx_blocks"]) + 2) * 2 * U * dca_abs)
        c = b["ctx"].reshape(rows, E).double().to(dev)
        dc_ref = dca * silu_d(c)
        note("d(context)", ("CTX_FILM", "dcontext"), res_dctx(b), dc_ref, 2.0 ** -20 * (dc_ref.abs() + _rms(dc_ref)))
    if plan["xattn_layers"]:
        cross = b["cross"].double().to(dev)
        dcross_ref = torch.zeros_like(cross)
        for l, n in enumerate(plan["xattn_layers"]):
            kn = n + ".fn.fn.to_kv.weight"
            wkv = W(kn)

            def ctxf(wk, x, n=n, kn=kn):
                return xattn_contexts({"xattn_layers": [n]}, {kn: wk}, x, dtype=torch.float64)[0]
            _, vj = torch.func.vjp(ctxf, wkv, cross)
            dw_ref, dx_ref = vj(dxctx_ref[l])
            dcross_ref += dx_ref
            dw_ref = dw_ref.reshape(256, -1)
            note("%s.to_kv" % n, ("XATTN_TEXT", "dW"), G(kn).reshape(256, -1), dw_ref,
                 2.0 ** -12 * (dw_ref.abs() + _rms(dw_ref)))
        got = b["dcross"].double()
        note("d(cross)", ("XATTN_TEXT", "dcross"), got, dcross_ref, 2.0 ** -12 * (dcross_ref.abs() + _rms(dcross_ref)))
    return fails


def res_dctx(b):
    return b["dctx"].double().reshape(-1, b["dctx"].shape[-1])


def _norm_vec_terms(op, p, gout, B, N, C, shared):
    """|terms| summed by the GroupNorm / LayerNorm backward reductions, from the op's own inputs in fp64."""
    x = p["b%d" % op["in0"]["buf"]]
    if op["kind"] == OP_LN:
        z = x
        xh = (z - z.mean(1, keepdim=True)) / torch.sqrt(z.var(1, unbiased=False, keepdim=True) + 1e-5)
        return {"vecs": {"g": (op["b"], 64 + B * N / 64 + 2)}, "abs": {"g": (gout * xh).abs().sum(0)}}
    h = x.reshape(B, N, 8, C // 8)
    xh = ((h - h.mean(dim=(1, 3), keepdim=True)) / torch.sqrt(h.var(dim=(1, 3), unbiased=False, keepdim=True) + 1e-5))
    xh = xh.reshape(B, N, C)
    u = xh * p["v%d" % op["gamma"]] + p["v%d" % op["beta"]]
    sc, sh = torch.ones_like(u), torch.zeros_like(u)
    if op["film"] == 1:
        sc, sh = p["film"][:, None, :C] + 1, p["film"][:, None, C:]
    elif op["film"] == 2:
        f = p["film"][None].expand(B, N, 2 * C) if shared else p["film"].reshape(B, N, 2 * C)
        sc, sh = f[..., :C] + 1, f[..., C:]
    w = u * sc + sh
    s = torch.sigmoid(w)
    dw = gout.reshape(B, N, C) * s * (1 + w * (1 - s))
    du = dw * sc
    out = {"vecs": {"gamma": (op["gamma"], N + B + 2), "beta": (op["beta"], N + B + 2)},
           "abs": {"gamma": (du * xh).abs().sum(dim=(0, 1)), "beta": du.abs().sum(dim=(0, 1))}}
    if op["film"]:
        fa = torch.cat([(dw * u).abs(), dw.abs()], dim=-1)      # [B, N, 2C]
        if op["film"] == 1:
            out["abs"]["film"] = fa.sum(dim=1)
        elif shared:
            out["abs"]["film"] = fa.sum(dim=0)
        else:
            out["abs"]["film"] = fa.reshape(B * N, 2 * C)
    return out


def _report(label, t0):
    torch.cuda.synchronize()
    print("%s: %.1f s, peak device memory %.2f GB" % (label, time.time() - t0, torch.cuda.max_memory_allocated() / 2 ** 30))
    print("worst error / bound:", {"/".join(k): round(v, 3) for k, v in sorted(WORST.items())})
    if MARGIN:
        print("one 64-row k-block of the last split / dW bound (smallest):", {k: round(v, 1) for k, v in MARGIN.items()})


@pytest.mark.parametrize("case", list(TABLE))
def test_train_backward_op_by_op(case):
    net_name, B, prec, L, shared = TABLE[case]
    t0 = time.time()
    torch.cuda.reset_peak_memory_stats()
    net = Net(net_name, prec)
    b = net.batch(B, seed=B + L, L=L, shared=shared)
    b.update(net.step(b))
    fails = check_backward(net, b, case=case)
    _report(case, t0)
    if case == "bench":
        assert MARGIN["bench"] > 10, MARGIN      # a dropped k-block would be far outside the bound
    assert not fails, fails[:10]


def test_train_backward_after_shrink_and_grow():
    """One handle: the bench batch, then B = 37 (rows past M and the padded FiLM rows hold the larger batch's values;
    per-sample losses equal a fresh handle's), then B = 1100 (every tensor-core plan rebuilt)."""
    t0 = time.time()
    torch.cuda.reset_peak_memory_stats()
    net = Net("liv", "bf16")
    net.step(net.batch(1024, seed=5))
    small = net.batch(37, seed=6)
    small.update(net.step(small))
    fails = check_backward(net, small, case="shrink")
    fresh = Net("liv", "bf16")
    ref = fresh.step(small)
    # stale rows do not leak: equal to fp32 summation-order noise (measured: 2.4e-7 at most)
    torch.testing.assert_close(small["losses"], ref["losses"], rtol=1e-6, atol=1e-6)
    LIVE.remove(fresh.eng)
    fresh.eng.close()
    grow = net.batch(1100, seed=7)
    grow.update(net.step(grow))
    fails += check_backward(net, grow, case="grow")
    _report("shrink / grow", t0)
    assert not fails, fails[:10]


# ---------------------------------------------------------------------------------------------------------------------
# the checker rejects wrong results
# ---------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def pert_net():
    """A bed network at B = 128 (24 k-blocks: the last of 12 splits owns two), its handle kept out of LIVE's
    eviction for the perturbation tests and closed after them."""
    _release(0)
    net = Net("bed", "bf16")
    LIVE.remove(net.eng)
    b = net.batch(128, seed=64)
    b.update(net.step(b))
    assert not check_backward(net, b)
    yield net, b
    net.eng.close()


@pytest.mark.parametrize("what", ["kblock", "consumer", "film_shift", "dgamma_group"])
def test_checker_rejects_perturbed_results(what, pert_net):
    net, b = pert_net
    plan, ops = net.plan, net.plan["ops"]
    M = b["B"] * net.N
    if what == "kblock":
        op = next(o for o in ops if o["kind"] == OP_GEMM and o["name"].endswith("to_qkv"))
        dy = net.eng.train_read(capi.DS_TRAIN_GRAD, op["out"])
        r0 = last_split_block(dy, M, op["N"], op["in0"]["k"], _cdiv(M, 128) * 128)
        dy = dy[r0:r0 + 64]
        x = net.eng.train_read(capi.DS_TRAIN_ACT, op["in0"]["buf"])[r0:r0 + 64]
        blk = dy.t() @ x

        def mutate(kind, idx, t):
            return t - blk if (kind == capi.DS_TRAIN_DW and idx == op["w"]) else t
    elif what == "consumer":
        op = next(o for o in ops if o["kind"] == OP_GN and o.get("res", -1) >= 0)
        g = net.eng.train_read(capi.DS_TRAIN_GRAD, op["out"])

        def mutate(kind, idx, t):
            return (t - g).to(torch.bfloat16).float() if (kind == capi.DS_TRAIN_GRAD and idx == op["res"]) else t
    elif what == "film_shift":
        def mutate(kind, idx, t):
            return t.roll(1, dims=0) if (kind == capi.DS_TRAIN_COND and idx == "film") else t
    else:
        op = next(o for o in ops if o["kind"] == OP_GN)

        def mutate(kind, idx, t):
            if kind == capi.DS_TRAIN_DVEC and idx == op["gamma"]:
                t = t.clone()
                t[:, 64:128] = 0
            return t
    saved = dict(WORST)
    fails = check_backward(net, b, mutate=mutate)
    WORST.clear()
    WORST.update(saved)
    print(what, "rejected by:", fails[:4])
    assert fails


# ---------------------------------------------------------------------------------------------------------------------
# the whole step against fp64 autograd of the oracle network
# ---------------------------------------------------------------------------------------------------------------------
E2E_TOL = 1e-4      # max |native - fp64| / max |fp64| per named gradient and for d(context)


def test_whole_step_fp32_against_fp64_oracle_autograd():
    """bench32's network at B = 128 in fp32: every named gradient and d(context) of ds_train_step against fp64
    autograd of oracle.unet1d_ref + oracle.diffusion_ref.p_losses on the GPU, from the same x_t.  Covers the wiring
    between stages that the op-by-op checks, which start every stage from native values, cannot see."""
    from oracle.unet1d_ref import unet1d_forward
    t0 = time.time()
    net = Net("liv", "fp32")
    b = net.batch(128, seed=128)
    b.update(net.step(b))
    B, N, d = 128, net.N, net.spec.point_dim
    dev = torch.device("cuda")
    xt = net.eng.train_read(capi.DS_TRAIN_COND, "x_t").double().reshape(B, N, d)
    sd = {"diffusion.model." + k: v.to(dev, torch.float64).requires_grad_(True) for k, v in net.sd.items()}
    ctx = b["ctx"].to(dev, torch.float64).requires_grad_(True)
    x0, t, nz = b["x0"].to(dev, torch.float64), b["t"].to(dev), b["noise"].to(dev, torch.float64)
    with torch.enable_grad():
        den = lambda xx, tt: unet1d_forward(sd, net.spec, xx, tt, ctx[None].expand(B, N, -1), None)
        losses, _ = D.p_losses(loss_schedule(net.dk), loss_spec(net), den, x0, t, nz, x_t=xt)
        (losses.mean() * GRAD_SCALE).backward()
    grads = b["grads"]
    worst = []
    for k, (off, n) in net.layout.items():
        ref = sd["diffusion.model." + k].grad.reshape(-1)
        got = grads[off:off + n].double()
        worst.append(((got - ref).abs().max().item() / max(ref.abs().max().item(), 1e-30), k))
    ref = ctx.grad
    worst.append(((b["dctx"].double() - ref).abs().max().item() / ref.abs().max().item(), "d(context)"))
    worst.sort(reverse=True)
    torch.cuda.synchronize()
    print("whole step, fp32 vs fp64 oracle: worst max-relative errors", [(round(e, 8), k) for e, k in worst[:5]],
          "%.1f s, peak %.2f GB" % (time.time() - t0, torch.cuda.max_memory_allocated() / 2 ** 30))
    assert worst[0][0] < E2E_TOL, worst[:8]


def test_train_read_errors():
    """The error paths of ds_train_read: no step with gradients yet (none, or a loss-only step), a bad kind or index,
    an array the network does not have, too small a capacity; a size query (NULL output) sets the shape only."""
    import ctypes as C
    net = Net("bed", "bf16")
    lib, h = net.eng.lib, net.eng.h
    r, w = C.c_int32(), C.c_int32()
    out = torch.empty(1 << 20, device="cuda")
    call = lambda kind, idx, cap, ptr=C.c_void_p(out.data_ptr()): lib.ds_train_read(h, kind, idx, ptr, cap, C.byref(r),
                                                                                   C.byref(w), None)
    assert call(capi.DS_TRAIN_ACT, 0, out.numel()) == -4                 # DS_ERR_STATE: no step yet
    b = net.batch(4, seed=4)
    net.eng.train_step(net.flat, b["x0"].cuda(), b["t"].cuda(), b["noise"].cuda(), b["ctx"].cuda(), True,
                       net.dk["loss_separate"], net.dk["loss_iou"], STATS["bounds_translations"] + STATS["bounds_sizes"])
    torch.cuda.synchronize()
    assert call(capi.DS_TRAIN_ACT, 0, out.numel()) == -4                 # a loss-only step has no gradients
    net.step(b)
    assert call(capi.DS_TRAIN_ACT, 0, out.numel()) == 0
    assert (r.value, w.value) == (4 * net.N, net.plan["buf_width"][0])
    r.value = w.value = 0
    assert call(capi.DS_TRAIN_DW, 0, 0, None) == 0                       # size query
    assert (r.value, w.value) == (net.plan["wmats"][0]["N"], net.plan["wmats"][0]["K"])
    assert call(capi.DS_TRAIN_DW, 0, r.value * w.value - 1) == -1        # capacity too small
    assert call(7, 0, out.numel()) == -1                                  # bad kind
    for kind, n in ((capi.DS_TRAIN_ACT, len(net.plan["buf_width"])), (capi.DS_TRAIN_DW, len(net.plan["wmats"])),
                    (capi.DS_TRAIN_DVEC, len(net.plan["vecs"])), (capi.DS_TRAIN_COND, len(capi.TRAIN_COND))):
        assert call(kind, n, out.numel()) == -1 and call(kind, -1, out.numel()) == -1
    assert call(capi.DS_TRAIN_COND, capi.TRAIN_COND["xkv"], out.numel()) == -1    # no text cross-attention here
    with pytest.raises(capi.DsError):
        net.eng.train_read(capi.DS_TRAIN_COND, "xctx")
    assert net.eng.train_read(capi.DS_TRAIN_COND, "x_t").shape == (4 * net.N, net.spec.point_dim)
