"""GPU, op by op: the floor-plan encoder (ds_room_enc_*, csrc/room_encoder.cu) forward and backward against float64,
at the batches scripts/bench_floorplan.py runs (training at 1024 scenes, sample() at 4096 on the same handle), across
the row split of the SIMT GEMMs and k_colsum (RE_ROW_CHUNK rows), and on non-square, multi-channel, continuous masks.

One native forward (and backward, where the case has one) runs; then every op is re-evaluated on the GPU in float64
from the exact values its kernels read, taken with ds_room_enc_read (activations, the folded weights and biases,
dW', d(bias) and every input-gradient buffer).  Errors do not compound.  The float64 reference is torch's own: unfold
and fold for im2col / col2im (columns reordered to the kernels' (ky, kx, cin)), max_pool2d and its autograd adjoint
(first maximum of the window in row-major order).

Bounds, per element (never on a mean).  u = 2^-24; ulp(v) is the bf16 spacing at |v| (test_gpu_bf16_ops.bf16_ulp).
D is the longest chain of fp32 additions a result sees, from the launch geometry, times 2u sum|terms| (fp64):
- SIMT forward GEMM k_gemm_simt (fp32 mode; bf16 mode where cout = 64: the stem and layer1): one fmaf per column of
  Kp, then the bias: D = Kp + 2.  k_gemm_wg (bf16, cout a multiple of 128, ksplit = 1): k16 products per MMA
  step, D = Kp / 16 + 2, as test_gpu_train_ops derives it for the tensor-core dX.
- A value the kernel rounds to bf16 once from a pre-value p with |p - ref| <= D' is within ulp(ref) + D' (1 + 2^-7)
  (|round(p) - p| <= 2^-8 |p|).  So conv + bias + ReLU (a1, h[b]): ulp(pre) + D (1 + 2^-7); the block tail
  o = relu(round(round(conv2 + b2) + round(downsample + b_ds) or x)): one such term for z, for dsb and for o.
  fp32 mode: D, and 2u |operand| per addition.
- BatchNorm fold: s = weight / sqrt(running_var) and W s in fp32 (8u |ref|), then one bf16 rounding; the Kp padding
  columns are exactly 0.  The packed mask is exactly the (bf16-rounded) mask.  Max pool: bit-exact.
- Average pool: fp32 sum of hw terms then a division: (hw + 2) 2u mean |o|.
- dW' = dY^T cols (k_gemm_tn): m_chunk + splits + 2 (test_gpu_train_ops.simt_dw_depth), over the whole batch.
  d(bias) (k_colsum: 256 rows per thread, then one fp32 atomic per 256-row block into the same sum, whichever of the
  RE_ROW_CHUNK launches it comes from): 256 + M / 256 + 2.
- Input gradients: dcols = dY W' (k_gemm_nn, D = cout + 2, stored in bf16: + ulp(dcols)), then a col2im gather of at
  most k^2 taps in fp32 (k^2 2u sum|taps|) and one final rounding.  The block's dx sums both consumers: conv1's
  col2im and either the identity residual (added before the one rounding) or the downsample col2im, which runs after
  conv1's col2im was stored (accumulate = 1: one more rounding).  A dropped or doubled consumer is off by a whole
  term.  d(a1): at most 4 addends per pixel, (4 * 2u) sum|terms| and one rounding.
- Fold adjoint, from the native dW' and d(bias): dW = dW' s (8u |ref|); d weight = (sum dW' W - rm dbias) /
  sqrt(rv): per thread ceil(kin / 256) fmaf, a 5-level warp sum, 8 partials, then 4 more operations; d bias is
  exactly d(bias); the running statistics get exactly 0.
WORST[(precision, op, kind)] collects the worst |err| / bound and is printed with the module's wall time.
"""
import math
import time

import pytest
import torch
import torch.nn.functional as F

from diffuscene_b200.room_encoder import BN_KEYS, RoomMaskEncoder, trunk_specs
from tests.cases_floorplan import trunk_value
from tests.test_gpu_bf16_ops import bf16_ulp
from tests.test_gpu_train_ops import simt_dw_depth

pytestmark = pytest.mark.gpu

U = 2.0 ** -24
ROW_CHUNK = 32768 * 64      # RE_ROW_CHUNK of room_encoder.cu
SLACK = 1 + 2.0 ** -7       # one bf16 rounding of a pre-value that carries an fp32 error (docstring)
WORST = {}                  # (precision, op, kind) -> worst |err| / bound


@pytest.fixture(scope="module", autouse=True)
def _wall_time():
    t0 = time.time()
    yield
    print("\ntest_gpu_room_encoder_ops: wall time %.1f s" % (time.time() - t0))
    print("worst error / bound:", {"/".join(k): round(v, 3) for k, v in sorted(WORST.items())})


# ---------------------------------------------------------------------------------------------------------------------
# inputs
# ---------------------------------------------------------------------------------------------------------------------
def params(C, seed=41):
    t = {n: trunk_value(n, shape, seed).cuda() for n, shape, _ in trunk_specs(C)}
    return t, torch.cat([v.reshape(-1) for v in t.values()]).contiguous()


def plan_masks(B, size, seed):
    """[B, 1, size, size] binary floor plans (synthetic.floor_plan_mask, as bench_floorplan.py feeds them)."""
    from diffuscene_b200.synthetic import floor_plan_mask
    g = torch.Generator().manual_seed(seed)
    return torch.stack([floor_plan_mask(g, size) for _ in range(B)]).cuda()


def continuous_masks(B, C, H, W, seed):
    """[B, C, H, W]: a room of a per-channel level in [0.3, 1.7] (not a bf16 value), with Gaussian noise over a
    quarter of it.  The flat part keeps exact max-pool ties; the rest makes the pack rounding and the channel order
    of every tap matter."""
    g = torch.Generator().manual_seed(seed)
    m = torch.zeros(B, C, H, W)
    r = lambda lo, hi: int(torch.randint(lo, hi, (1,), generator=g))
    for i in range(B):
        y0, y1, x0, x1 = r(1, H // 4), r(3 * H // 4, H), r(1, W // 4), r(3 * W // 4, W)
        m[i, :, y0:y1, x0:x1] = (0.3 + 1.4 * torch.rand(C, generator=g))[:, None, None]
        ym, xm = (y0 + y1) // 2, (x0 + x1) // 2
        m[i, :, y0:ym, x0:xm] += 0.5 * torch.randn(C, ym - y0, xm - x0, generator=g)
    return m.cuda()


def geometry(C, H, W):
    """The convs in expected-weight order (stem, then per block conv1, conv2 (, downsample)) and per block the conv
    indices (conv1, conv2, downsample or None), as ds_room_enc_create lays them out."""
    convs = []

    def add(name, bn, cin, cout, k, stride, pad, hin, win):
        convs.append(dict(name=name, bn=bn, cin=cin, cout=cout, k=k, stride=stride, pad=pad, hin=hin, win=win,
                          hout=(hin + 2 * pad - k) // stride + 1, wout=(win + 2 * pad - k) // stride + 1,
                          Kp=(k * k * cin + 63) // 64 * 64))
        return len(convs) - 1

    add("conv1", "bn1", C, 64, 7, 2, 3, H, W)
    blocks = []
    hin, win, cin = H // 4, W // 4, 64
    for L in range(4):
        cout = 64 << L
        for j in range(2):
            stride = 2 if (L > 0 and j == 0) else 1
            pre = "layer%d.%d." % (L + 1, j)
            c1 = add(pre + "conv1", pre + "bn1", cin, cout, 3, stride, 1, hin, win)
            g1 = convs[c1]
            c2 = add(pre + "conv2", pre + "bn2", cout, cout, 3, 1, 1, g1["hout"], g1["wout"])
            cd = None
            if stride != 1 or cin != cout:
                cd = add(pre + "downsample.0", pre + "downsample.1", cin, cout, 1, stride, 0, hin, win)
            blocks.append((c1, c2, cd))
            hin, win, cin = g1["hout"], g1["wout"], cout
    return convs, blocks


# ---------------------------------------------------------------------------------------------------------------------
# float64 building blocks: im2col / col2im in the kernels' column order, per chunk of scenes
# ---------------------------------------------------------------------------------------------------------------------
def _chunks(B, per_scene):
    n = max(1, (1 << 25) // per_scene)
    return [(s, min(B, s + n)) for s in range(0, B, n)]


def _sl(t, per, s0, s1):
    return t[s0 * per:s1 * per]


def _cols(x, g, s0, s1):
    """im2col of scenes s0 .. s1 of NHWC rows x: [b hout wout, Kp], columns (ky, kx, cin), zero-padded."""
    b = s1 - s0
    x4 = _sl(x, g["hin"] * g["win"], s0, s1).reshape(b, g["hin"], g["win"], g["cin"]).permute(0, 3, 1, 2)
    u = F.unfold(x4, g["k"], padding=g["pad"], stride=g["stride"])      # [b, (cin, ky, kx), L]
    L = u.shape[-1]
    u = u.reshape(b, g["cin"], g["k"] * g["k"], L).permute(0, 3, 2, 1).reshape(b * L, -1)
    return F.pad(u, (0, g["Kp"] - u.shape[1]))


def _fold(dcols, g, b):
    """col2im of [b hout wout, Kp] (columns (ky, kx, cin)) -> NHWC rows [b hin win, cin]."""
    k, cin, L = g["k"], g["cin"], g["hout"] * g["wout"]
    t = dcols[:, :k * k * cin].reshape(b, L, k * k, cin).permute(0, 3, 2, 1).reshape(b, cin * k * k, L)
    y = F.fold(t, (g["hin"], g["win"]), k, padding=g["pad"], stride=g["stride"])
    return y.permute(0, 2, 3, 1).reshape(b * g["hin"] * g["win"], cin)


def _nchw(x, b, h, w):
    return x.reshape(b, h, w, -1).permute(0, 3, 1, 2)


def _rows(x4):
    return x4.permute(0, 2, 3, 1).reshape(-1, x4.shape[1])


def colsum_depth(M):
    return 256 + math.ceil(M / 256) + 2


def count_pool_ties(a1, B, H2, W2):
    """Max-pool windows whose positive maximum is held by two or more of its inputs."""
    n = 0
    for s0, s1 in _chunks(B, H2 * W2 * 64 * 9 // 4):
        u = F.unfold(_nchw(_sl(a1, H2 * W2, s0, s1), s1 - s0, H2, W2), 3, padding=1, stride=2)
        u = u.reshape(s1 - s0, 64, 9, -1)
        mx = u.amax(dim=2, keepdim=True)
        n += int((((u == mx).sum(dim=2) >= 2) & (mx[:, :, 0] > 0)).sum())
    return n


# ---------------------------------------------------------------------------------------------------------------------
# the checker
# ---------------------------------------------------------------------------------------------------------------------
def check_encoder(enc, t, mask, prec, feat, dfeat=None, grads=None):
    """Every op of the last forward (and of the backward after it, with dfeat / grads) against float64; returns the
    list of (what, worst ratio) over 1."""
    bf = prec == "bf16"
    B, C, H, W = mask.shape
    convs, blocks = geometry(C, H, W)
    H2, W2, H4, W4 = H // 2, W // 2, H // 4, W // 4
    fails = []
    dev = mask.device
    T = {k: v.double() for k, v in t.items()}
    rd = lambda kind, i=0: enc.read(kind, i).double()
    ulp = bf16_ulp if bf else torch.zeros_like

    def note(what, key, got, ref, bound):
        err = (got - ref).abs()
        r = (err / bound.clamp_min(1e-300)).max().item() if err.numel() else 0.0
        if not math.isfinite(r):
            r = float("inf")
        key = (prec,) + key
        WORST[key] = max(WORST.get(key, 0.0), r)
        if r > 1.0:
            fails.append((what, round(r, 3)))

    def exact(what, key, got, ref):
        ok = torch.equal(got, ref)
        WORST[(prec,) + key] = max(WORST.get((prec,) + key, 0.0), 0.0 if ok else float("inf"))
        if not ok:
            fails.append((what, float("inf")))

    # ---- BatchNorm fold: W' and the bias as the kernels read them
    wp, bias = [], []
    for c, g in enumerate(convs):
        got_w, got_b = rd("wp", c), rd("bias", c)[0]
        bw, bb, rm, rv = (T["%s.%s" % (g["bn"], k)] for k in BN_KEYS)
        s = bw / rv.sqrt()
        kin = g["k"] ** 2 * g["cin"]
        ref = (T[g["name"] + ".weight"] * s[:, None, None, None]).permute(0, 2, 3, 1).reshape(g["cout"], kin)
        note("fold W' %s" % g["name"], ("FOLD", "W'"), got_w[:, :kin], ref, ulp(ref) + 8 * U * ref.abs())
        exact("fold W' padding %s" % g["name"], ("FOLD", "pad"), got_w[:, kin:], torch.zeros_like(got_w[:, kin:]))
        note("fold bias %s" % g["name"], ("FOLD", "bias"), got_b, bb - rm * s, 8 * U * (bb.abs() + (rm * s).abs()))
        wp.append(got_w)
        bias.append(got_b)

    def conv_pre(c, x, s0, s1):
        """fp64 conv + bias of scenes s0 .. s1 from the native input and W', and its fp32 accumulation bound."""
        g = convs[c]
        cols = _cols(x, g, s0, s1)
        pre = torch.addmm(bias[c], cols, wp[c].t())
        terms = torch.addmm(bias[c].abs(), cols.abs(), wp[c].abs().t())
        depth = g["Kp"] / 16 + 2 if (bf and g["cout"] % 128 == 0) else g["Kp"] + 2
        return pre, depth * 2 * U * terms

    # ---- mask pack, stem, max pool
    x0 = rd("x0")
    ref = mask.permute(0, 2, 3, 1).reshape(-1, C)
    exact("pack", ("PACK", "x0"), x0, (ref.to(torch.bfloat16) if bf else ref).double())
    a1 = rd("a1")
    for s0, s1 in _chunks(B, H2 * W2 * convs[0]["Kp"]):
        pre, D = conv_pre(0, x0, s0, s1)
        note("stem", ("STEM", "a1"), _sl(a1, H2 * W2, s0, s1), pre.clamp_min(0), ulp(pre) + D * SLACK)
    p = rd("p")
    exact("max pool", ("MAXPOOL", "p"), p, _rows(F.max_pool2d(_nchw(a1, B, H2, W2), 3, 2, 1)))
    ties = count_pool_ties(a1, B, H2, W2)
    assert ties > 0, "no max-pool window with a tied positive maximum: the tie routing is not exercised"

    # ---- blocks
    x = p
    outs, hs = [], []
    for b, (c1, c2, cd) in enumerate(blocks):
        g1, g2 = convs[c1], convs[c2]
        pin, pout = g1["hin"] * g1["win"], g1["hout"] * g1["wout"]
        h, o = rd("h", b), rd("o", b)
        for s0, s1 in _chunks(B, pout * max(g1["Kp"], g2["Kp"])):
            pre, D = conv_pre(c1, x, s0, s1)
            note("conv1 block %d" % b, ("CONV1", "h"), _sl(h, pout, s0, s1), pre.clamp_min(0), ulp(pre) + D * SLACK)
            z, Dz = conv_pre(c2, h, s0, s1)
            if cd is not None:
                r, Dr = conv_pre(cd, x, s0, s1)
                Dr = ulp(r) + Dr * SLACK
            else:
                r, Dr = _sl(x, pin, s0, s1), 0.0
            ref = z + r
            bound = ulp(z) + Dz * SLACK + Dr + ulp(ref) + 2 * U * (z.abs() + r.abs()) * (not bf)
            note("tail block %d" % b, ("TAIL", "o"), _sl(o, pout, s0, s1), ref.clamp_min(0), bound * SLACK)
        outs.append(o)
        hs.append(h)
        x = o
    hw = convs[blocks[7][1]]["hout"] * convs[blocks[7][1]]["wout"]
    o7 = outs[7].reshape(B, hw, 512)
    note("average pool", ("AVGPOOL", "feat"), feat.double(), o7.mean(dim=1), (hw + 2) * 2 * U * o7.abs().mean(dim=1))
    if dfeat is None:
        return fails

    # ---- backward
    dfeat = dfeat.double()
    dz7 = rd("dz", 7)
    ref = ((o7 > 0) * (dfeat[:, None, :] / hw)).reshape(-1, 512)
    note("average-pool adjoint", ("AVGPOOL", "dz7"), dz7, ref, ulp(ref) + 2 * U * ref.abs())

    def check_dw(c, x, dy):
        g = convs[c]
        pin, pout = g["hin"] * g["win"], g["hout"] * g["wout"]
        M = B * pout
        ref = torch.zeros(g["cout"], g["Kp"], dtype=torch.float64, device=dev)
        mag = torch.zeros_like(ref)
        for s0, s1 in _chunks(B, pout * g["Kp"]):
            cols = _cols(x, g, s0, s1)
            d = _sl(dy, pout, s0, s1)
            ref += d.t() @ cols
            mag += d.abs().t() @ cols.abs()
        note("dW' %s" % g["name"], ("CONV", "dW'"), rd("dwp", c), ref, simt_dw_depth(M, g["cout"], g["Kp"]) * 2 * U * mag)
        note("dbias %s" % g["name"], ("CONV", "dbias"), rd("dbias", c)[0], dy.sum(dim=0),
             colsum_depth(M) * 2 * U * dy.abs().sum(dim=0))

    def dcols_fold(c, dy, s0, s1):
        """col2im(dY W') of scenes s0 .. s1 and its bound: per tap the k_gemm_nn term and one rounding of dcols,
        then the fp32 tap sum (before any final rounding)."""
        g = convs[c]
        d = _sl(dy, g["hout"] * g["wout"], s0, s1)
        dc = d @ wp[c]
        e = (g["cout"] + 2) * 2 * U * (d.abs() @ wp[c].abs()) + ulp(dc)
        val = _fold(dc, g, s1 - s0)
        return val, (_fold(e, g, s1 - s0) + g["k"] ** 2 * 2 * U * _fold(dc.abs(), g, s1 - s0)) * SLACK

    for b in range(7, -1, -1):
        c1, c2, cd = blocks[b]
        g1 = convs[c1]
        pin, pout = g1["hin"] * g1["win"], g1["hout"] * g1["wout"]
        x = outs[b - 1] if b > 0 else p
        dz, dh = rd("dz", b), rd("dh", b)
        dx = rd("dz", b - 1) if b > 0 else rd("dp")
        for s0, s1 in _chunks(B, pout * max(convs[c1]["Kp"], convs[c2]["Kp"])):
            val, bnd = dcols_fold(c2, dz, s0, s1)
            m = _sl(hs[b], pout, s0, s1) > 0
            note("dh block %d" % b, ("CONV2", "dh"), _sl(dh, pout, s0, s1), val * m, (bnd + ulp(val)) * m)
            A, bA = dcols_fold(c1, dh, s0, s1)
            if cd is not None:
                Cv, bC = dcols_fold(cd, dz, s0, s1)
                ref = A + Cv
                bound = bA + bC + ulp(A) + ulp(ref) + 2 * U * (A.abs() + Cv.abs())
            else:
                r = _sl(dz, pin, s0, s1)
                ref = A + r
                bound = bA + ulp(ref) + 2 * U * (A.abs() + r.abs())
            m = (_sl(x, pin, s0, s1) > 0) if b > 0 else torch.ones_like(ref, dtype=torch.bool)
            note("dx block %d" % b, ("BLOCK", "dx"), _sl(dx, pin, s0, s1), ref * m, bound * SLACK * m)
        check_dw(c2, hs[b], dz)
        check_dw(c1, x, dh)
        if cd is not None:
            check_dw(cd, x, dz)
    dp, da1 = rd("dp"), rd("da1")
    for s0, s1 in _chunks(B, H2 * W2 * 64 * 4):
        a = _nchw(_sl(a1, H2 * W2, s0, s1), s1 - s0, H2, W2).clone().requires_grad_(True)
        d4 = _nchw(_sl(dp, H4 * W4, s0, s1), s1 - s0, H4, W4)
        with torch.enable_grad():
            y = F.max_pool2d(a, 3, 2, 1)
            (gv,) = torch.autograd.grad(y, a, d4, retain_graph=True)
            (ga,) = torch.autograd.grad(y, a, d4.abs())
        m = a.detach() > 0
        ref, mag = _rows(gv * m), _rows(ga * m)
        note("max-pool adjoint", ("MAXPOOL", "da1"), _sl(da1, H2 * W2, s0, s1), ref, ulp(ref) + 8 * U * mag)
    check_dw(0, x0, da1)

    # ---- the fold adjoint into the named flat gradients, from the native dW' and d(bias)
    off, G = 0, {}
    for n, shape, _ in trunk_specs(C):
        k = math.prod(shape)
        G[n] = grads[off:off + k].double().reshape(shape)
        off += k
    for c, g in enumerate(convs):
        dwp, db = rd("dwp", c), rd("dbias", c)[0]
        bw, bb, rm, rv = (T["%s.%s" % (g["bn"], k)] for k in BN_KEYS)
        r = 1 / rv.sqrt()
        kin = g["k"] ** 2 * g["cin"]
        d = dwp[:, :kin]
        ref = d.reshape(g["cout"], g["k"], g["k"], g["cin"]).permute(0, 3, 1, 2) * (bw * r)[:, None, None, None]
        note("fold adjoint %s.weight" % g["name"], ("FOLD_BWD", "dW"), G[g["name"] + ".weight"], ref,
             8 * U * ref.abs())
        prod = d * T[g["name"] + ".weight"].permute(0, 2, 3, 1).reshape(g["cout"], kin)
        ref = (prod.sum(dim=1) - rm * db) * r
        depth = math.ceil(kin / 256) + 5 + 8 + 4
        note("fold adjoint %s.weight" % g["bn"], ("FOLD_BWD", "dweight"), G[g["bn"] + ".weight"], ref,
             depth * 2 * U * (prod.abs().sum(dim=1) + (rm * db).abs()) * r + 4 * U * ref.abs())
        exact("fold adjoint %s.bias" % g["bn"], ("FOLD_BWD", "dbias"), G[g["bn"] + ".bias"], db)
        for k in ("running_mean", "running_var"):
            exact("%s.%s gradient" % (g["bn"], k), ("FOLD_BWD", "running"), G["%s.%s" % (g["bn"], k)],
                  torch.zeros_like(rm))
    return fails


def run(enc, t, flat, mask, prec, backward=True, seed=0):
    feat = enc.forward(flat, mask, keep=backward)
    dfeat = grads = None
    if backward:
        dfeat = torch.randn(mask.shape[0], 512, generator=torch.Generator().manual_seed(seed)).cuda()
        grads = torch.full_like(flat, float("nan"))
        enc.backward(dfeat, grads)
    torch.cuda.synchronize()
    return check_encoder(enc, t, mask, prec, feat, dfeat, grads)


# ---------------------------------------------------------------------------------------------------------------------
# cases
# ---------------------------------------------------------------------------------------------------------------------
CASES = {
    # name: precision, channels, height, width, batch, masks
    "bench": ("bf16", 1, 64, 64, 1024, "plan"),          # the training batch of bench_floorplan.py
    "bench32": ("fp32", 1, 64, 64, 1024, "plan"),        # the parity mode at the same batch
    "chunk_mid": ("bf16", 1, 96, 96, 1003, "plan"),      # 2304 stem rows per scene: the row split inside scene 910
    "chunk_mid32": ("fp32", 1, 96, 96, 1003, "plan"),
    "rect": ("bf16", 3, 96, 64, 37, "cont"),             # H != W, C = 3, stem Kp 192, layer4 3 x 2
    "rect32": ("fp32", 3, 96, 64, 37, "cont"),
    "small": ("bf16", 8, 32, 32, 5, "cont"),             # layer4 at 1 x 1, stem Kp 448
    "small32": ("fp32", 8, 32, 32, 5, "cont"),
}


def case_masks(C, H, W, B, kind, seed):
    return plan_masks(B, H, seed) if kind == "plan" else continuous_masks(B, C, H, W, seed)


def test_chunk_mid_splits_inside_a_scene():
    """The chunk_mid geometry: 1003 scenes of 48 x 48 stem rows pass RE_ROW_CHUNK, inside scene 910 at its row 512."""
    assert 1003 * 48 * 48 > ROW_CHUNK
    assert divmod(ROW_CHUNK, 48 * 48) == (910, 512)


@pytest.mark.parametrize("case", list(CASES))
def test_encoder_op_by_op(case):
    prec, C, H, W, B, kind = CASES[case]
    t0 = time.time()
    t, flat = params(C)
    mask = case_masks(C, H, W, B, kind, seed=B + C)
    enc = RoomMaskEncoder(C, H, W, precision=prec)
    fails = run(enc, t, flat, mask, prec, seed=B)
    enc.close()
    print("%s: %.1f s" % (case, time.time() - t0))
    assert not fails, fails[:10]


def test_sample_batch_then_training_step_on_one_handle():
    """The model's order: sample() encodes 4096 scenes (the stem's 4M rows split in two), then train_on_batch runs
    1024 scenes forward and backward on the same handle, whose tensor-core plans were built at 4096 and whose cols
    rows past the smaller batch hold the larger batch's values."""
    t0 = time.time()
    t, flat = params(1)
    enc = RoomMaskEncoder(1, 64, 64, precision="bf16")
    big = plan_masks(4096, 64, seed=4096)
    assert 4096 * 32 * 32 > ROW_CHUNK
    fails = run(enc, t, flat, big, "bf16", backward=False)
    fails += run(enc, t, flat, plan_masks(1024, 64, seed=1025), "bf16", seed=1024)
    enc.close()
    print("sample: %.1f s" % (time.time() - t0))
    assert not fails, fails[:10]


# ---------------------------------------------------------------------------------------------------------------------
# scene isolation and stale rows
# ---------------------------------------------------------------------------------------------------------------------
ISO = {"64": (64, 1024, (0, 511, 1023)), "chunk_mid": (96, 1003, (0, 909, 910, 911, 1002))}


@pytest.mark.parametrize("where", list(ISO))
@pytest.mark.parametrize("prec", ["bf16", "fp32"])
def test_scene_isolation(prec, where):
    """Replacing one scene's mask by NaN, +Inf or 1e30 changes no other scene's features by a single bit, and a NaN
    mask gives 512 NaN features, as the autograd twin (functional.room_trunk) does."""
    from diffuscene_b200.networks.functional import room_trunk
    size, B, positions = ISO[where]
    t, flat = params(1)
    masks = plan_masks(B, size, seed=7)
    enc = RoomMaskEncoder(1, size, size, precision=prec)
    base = enc.forward(flat, masks).clone()
    assert torch.isfinite(base).all()
    bad = []
    for j in positions:
        for val in (float("nan"), float("inf"), 1e30):
            mj = masks.clone()
            mj[j] = val
            out = enc.forward(flat, mj)
            keep = torch.ones(B, dtype=torch.bool, device=out.device)
            keep[j] = False
            if not torch.equal(out[keep], base[keep]):
                bad.append((j, val, (out != base).any(dim=1).nonzero().flatten().tolist()[:5]))
            if val != val and not torch.isnan(out[j]).all():
                bad.append((j, "NaN mask gives %d finite features" % int(torch.isfinite(out[j]).sum())))
    with torch.no_grad():
        twin = room_trunk(t, torch.full((1, 1, size, size), float("nan"), device="cuda"))
    assert torch.isnan(twin).all()
    enc.close()
    assert not bad, bad


@pytest.mark.parametrize("where", list(ISO))
@pytest.mark.parametrize("prec", ["bf16", "fp32"])
def test_stale_rows_of_a_larger_nan_batch(prec, where):
    """One handle: 1003 scenes whose scenes from 500 on are NaN, then 500 finite scenes forward and backward.  The
    features equal a fresh handle's bit for bit, the gradients are finite and every op holds its bound."""
    size = ISO[where][0]
    t, flat = params(1)
    masks = plan_masks(1003, size, seed=11)
    enc = RoomMaskEncoder(1, size, size, precision=prec)
    dirty = masks.clone()
    dirty[500:] = float("nan")
    enc.forward(flat, dirty)
    small = masks[:500].contiguous()
    feat = enc.forward(flat, small, keep=True)
    dfeat = torch.randn(500, 512, generator=torch.Generator().manual_seed(500)).cuda()
    grads = torch.full_like(flat, float("nan"))
    enc.backward(dfeat, grads)
    torch.cuda.synchronize()
    fresh = RoomMaskEncoder(1, size, size, precision=prec)
    ref = fresh.forward(flat, small)
    fresh.close()
    assert torch.equal(feat, ref), (feat != ref).any(dim=1).nonzero().flatten().tolist()[:5]
    assert torch.isfinite(grads).all()
    fails = check_encoder(enc, t, small, prec, feat, dfeat, grads)
    enc.close()
    assert not fails, fails[:10]


# ---------------------------------------------------------------------------------------------------------------------
# ds_room_enc_read itself
# ---------------------------------------------------------------------------------------------------------------------
def test_read_errors_and_shapes():
    """No forward yet, gradients before a backward or after a new forward (DS_ERR_STATE); a bad kind, block or conv
    index, too small a capacity (DS_ERR_INVALID); a size query sets the shape only."""
    import ctypes as C
    from diffuscene_b200 import capi
    t, flat = params(1)
    enc = RoomMaskEncoder(1, 32, 32, precision="bf16")
    lib, h = enc.lib, enc.h
    r, w = C.c_int32(), C.c_int32()
    out = torch.empty(1 << 20, device="cuda")
    S = capi.ROOM_ENC_STATE
    call = lambda kind, idx, cap, ptr=C.c_void_p(out.data_ptr()): lib.ds_room_enc_read(h, kind, idx, ptr, cap,
                                                                                      C.byref(r), C.byref(w), None)
    assert call(S["x0"], 0, out.numel()) == -4                       # DS_ERR_STATE: no forward yet
    mask = plan_masks(3, 32, seed=3)
    enc.forward(flat, mask)
    assert call(S["x0"], 0, out.numel()) == 0 and (r.value, w.value) == (3 * 32 * 32, 1)
    assert call(S["dwp"], 0, out.numel()) == -4                      # no backward yet
    enc.forward(flat, mask, keep=True)
    enc.backward(torch.ones(3, 512, device="cuda"), torch.empty_like(flat))
    r.value = w.value = 0
    assert call(S["dwp"], 0, 0, None) == 0 and (r.value, w.value) == (64, 64)      # size query: the stem's [64, Kp]
    assert call(S["dwp"], 0, 64 * 64 - 1) == -1                                   # capacity too small
    assert call(S["dz"], 7, out.numel()) == 0 and (r.value, w.value) == (3, 512)  # layer4 at 1 x 1
    assert call(S["h"], 4, out.numel()) == 0 and (r.value, w.value) == (3 * 2 * 2, 256)
    assert call(S["bias"], 19, out.numel()) == 0 and (r.value, w.value) == (1, 512)
    for kind, bad in ((S["h"], 8), (S["dh"], -1), (S["wp"], 20), (S["dbias"], -1), (len(S), 0), (-1, 0)):
        assert call(kind, bad, out.numel()) == -1, (kind, bad)
    assert enc.read("wp", 0).shape == (64, 64)
    enc.forward(flat, mask)
    assert call(S["da1"], 0, out.numel()) == -4                      # a forward since the backward
    assert enc.read("a1").shape == (3 * 16 * 16, 64)
    enc.close()
