"""GPU, op by op: the frozen BERT text encoder (ds_text_enc_*, csrc/text_encoder.cu) against float64, in both
precisions, at the batches scripts/bench_text_encoder.py times (128 and 1024 sequences of 16 .. 64 tokens), across the
attention kernels' key tiles and query blocks (L = 129 and 512), with near one-hot attention, and at a small geometry.

One native forward runs per tapped layer (ds_text_enc_set_tap); then every op of that layer is re-evaluated on the GPU
in float64 from the exact values its kernel read, taken with ds_text_enc_read, so errors do not compound.  The weights
are restated from the fp32 state dict: in bf16 mode the packed matrices are its round-to-nearest-even bf16 values
(q | k | v rows fused), biases and LayerNorm parameters stay fp32.  Every element is compared, padded query rows
included: the text projection and the denoiser's cross-attention consume all L positions.

Bounds, per element (never on a mean).  u = 2^-24; ulp(v) is the bf16 spacing at |v| (test_gpu_bf16_ops.bf16_ulp).
D is the longest chain of fp32 roundings a result sees, from the kernel code and the launch geometry, times 2u
sum|terms| (fp64).  bf16 mode: a value rounded to bf16 once from a pre-value within e of the reference is within
ulp(ref) + e (1 + 2^-7).  fp32 mode has no such term (its final rounding is the last link of D).
- Embeddings: v = (word[id] + type[0]) + position[r % L] is formed in fp32 exactly as the kernel forms it (two
  additions, nothing to contract), then LayerNorm in fp64.
- LayerNorm (k_te_embed_ln, k_te_layernorm; one warp per row, lane-strided sums then a 5-level shuffle tree, two
  passes): the mean is off by dmu = (H / 32 + 5) 2u mean|v| + u |mean|; the centred sum of squares is a sum of
  positive terms, so rstd is off by rel = ((H / 32 + 6) 2u + dmu^2 / var + 2u) / 2 + 2u; the output
  (v - mean) rstd g + b by |y - b| (rel + 4u) + dmu rstd |g| + 2u |y|.
- GEMMs: k_gemm_wg (bf16) adds one k16 MMA step at a time, D = K / 16, then the bias (+1) and the residual (+1) in
  fp32 before the one bf16 rounding.  The SIMT GEMM (fp32) is one fmaf per k: D = K, + 1 bias, + 1 residual.  The
  terms are |A| |W|^T + |bias| (+ |residual|).
- Intermediate GEMM + GELU.  The reference is HF's erf GELU of the fp64 pre-activation x.  The pre-activation error
  passes through a slope of at most 1.13.  bf16: the epilogue is the tanh form through tanh.approx.f32 (relative
  error 2^-10.987, times 0.5 |x|), plus 8u |x| for its fp32 polynomial and 2u |ref|; the tanh-vs-erf deviation
  |gelu_tanh(x) - gelu_erf(x)| is allowed per element in fp64, and its share of the worst ratio is printed.  fp32:
  gelu_erf through erff (2 ulp) and three roundings: 3u |x| + 4u |ref|.
- Masked self-attention, per (query, key): a = sum_d |q_d k_d| / 8, z = s / 8 - max (natural-log units).  The
  softmax is invariant to the running max and to the rescale factors (o and l are multiplied by the same corr), so a
  key's weight is off by the relative delta = 2u ((Ds + 1) a + |z|) + 4u: Ds the logit's accumulation depth (+1 for the
  scale, or the bf16 kernel's log2(e) / 8 product), |z| for the rounding of s - m and of the scale constant, 4u for
  exp2f / expf (2 ulp).  That moves o by sum_j p_j delta_j |v_j - o| / l <= (P delta) |V| + |o| sum_j P delta.  Then
  the P V and l sums: D sum_j p_j |v_j| / l.
  bf16 (k_te_attn_bf16, mma.sync m16n8k16, 64-key tiles): Ds = 64 / 16; per tile 4 k16 MMA steps and the rescale
  for o, 16 additions and the rescale for l, then 2 shuffle additions, 1 / l and the product: D = 22 ceil(len / 64)
  + 5.  P is rounded to bf16 for P V while l sums the unrounded p: + 2^-8 sum_j p_j |v_j| / l.
  fp32 (k_te_attn_f32, 32-key tiles, 16-key chunks): Ds = 64 (fmaf chain; the 1/8 is exact); one addition / fmaf
  per key and one rescale per chunk, for o and for l, then 1 / l and the product: D = 2 (len + ceil(len / 16)) + 2.
WORST[(precision, op)] collects the worst |err| / bound and is printed with the module's wall time.
"""
import ctypes as C
import math
import time

import pytest
import torch
import torch.nn.functional as F

from diffuscene_b200 import capi
from diffuscene_b200.text_encoder import BertTextEncoder
from tests.test_gpu_bf16_ops import bf16_ulp
from tests.test_gpu_text_encoder import batch, perturbed_bert

pytestmark = pytest.mark.gpu

U = 2.0 ** -24
SLACK = 1 + 2.0 ** -7           # one bf16 rounding of a pre-value that carries an fp32 error (docstring)
TANH_APPROX = 2.0 ** -10.987    # relative error of tanh.approx.f32
GELU_SLOPE = 1.13               # max |GELU'|
LN_EPS = 1e-12
ROWS = 16384                    # rows per float64 evaluation chunk
BERT_BASE = dict(vocab_size=28996)
SMALL = dict(vocab_size=1000, hidden_size=256, num_hidden_layers=2, num_attention_heads=4, intermediate_size=512,
             max_position_embeddings=160)
WORST = {}                      # (precision, op) -> worst |err| / bound
GELU_SHARE = {}                 # precision -> (worst GELU ratio, the tanh-vs-erf allowance's share of its bound)


@pytest.fixture(scope="module", autouse=True)
def _wall_time():
    t0 = time.time()
    yield
    print("\ntest_gpu_text_encoder_ops: wall time %.1f s" % (time.time() - t0))
    print("worst error / bound:", {"/".join(k): round(v, 3) for k, v in sorted(WORST.items())})
    for prec, (r, share) in sorted(GELU_SHARE.items()):
        print("%s GELU: worst ratio %.3f, of which the tanh-vs-erf allowance is %.1f %% of the bound" % (
            prec, r, 100 * share))


@pytest.fixture(scope="module")
def bert_base():
    """The perturbed bert-base of test_gpu_text_encoder (seed 11)."""
    m = perturbed_bert(11, **BERT_BASE)
    return m.config, {k: v.detach().clone() for k, v in m.state_dict().items()}


def bench_batch(B, L, vocab, seed):
    """Lengths as scripts/bench_text_encoder.make_batch draws them: uniform in 16 .. L, the first sequence full."""
    g = torch.Generator().manual_seed(seed)
    lengths = torch.randint(16, L + 1, (B,), generator=g)
    lengths[0] = L
    return batch(lengths.tolist(), L, vocab, seed)


# ---------------------------------------------------------------------------------------------------------------------
# float64 references with their bounds
# ---------------------------------------------------------------------------------------------------------------------
def layernorm(v, g, b):
    """LayerNorm of rows v and its bound before any final rounding (docstring)."""
    H = v.shape[-1]
    mu = v.mean(-1, keepdim=True)
    d = v - mu
    var = (d * d).mean(-1, keepdim=True)
    r = 1 / (var + LN_EPS).sqrt()
    y = d * r * g + b
    dmu = (H / 32 + 5) * 2 * U * v.abs().mean(-1, keepdim=True) + U * mu.abs()
    rel = ((H / 32 + 6) * 2 * U + dmu ** 2 / var + 2 * U) / 2 + 2 * U
    return y, (y - b).abs() * (rel + 4 * U) + dmu * r * g.abs() + 2 * U * y.abs()


def linear(a, w, b, res=None, bf=True):
    """a w^T + b (+ res) and its fp32 accumulation bound."""
    K = a.shape[1]
    ref = torch.addmm(b, a, w.t())
    mag = torch.addmm(b.abs(), a.abs(), w.abs().t())
    depth = (K / 16 if bf else K) + 1
    if res is not None:
        ref, mag, depth = ref + res, mag + res.abs(), depth + 1
    return ref, depth * 2 * U * mag


def gelu_tanh(x):
    return 0.5 * x * (1 + torch.tanh(math.sqrt(2 / math.pi) * (x + 0.044715 * x ** 3)))


def attention(qkv, lengths, heads, bf):
    """Masked softmax(q k^T / 8) v of [b, L, 3 H] rows and its bound before the final rounding (docstring)."""
    b, L, _ = qkv.shape
    q, k, v = (t.reshape(b, L, heads, 64).transpose(1, 2) for t in qkv.chunk(3, dim=-1))
    s = q @ k.transpose(-1, -2) / 8
    a = q.abs() @ k.abs().transpose(-1, -2) / 8
    keep = (torch.arange(L, device=qkv.device)[None] < lengths[:, None])[:, None, None, :]
    s = s.masked_fill(~keep, -math.inf)
    P = torch.softmax(s, dim=-1)
    o = P @ v
    z = (s - s.amax(-1, keepdim=True)).masked_fill(~keep, 0)
    n = lengths.double()[:, None, None, None]
    if bf:
        ds, depth, p_round = 64 / 16, 22 * torch.ceil(n / 64) + 5, 2.0 ** -8
    else:
        ds, depth, p_round = 64, 2 * (n + torch.ceil(n / 16)) + 2, 0.0
    Pd = P * (2 * U * ((ds + 1) * a + z.abs()) + 4 * U)
    av = P @ v.abs()
    err = Pd @ v.abs() + o.abs() * Pd.sum(-1, keepdim=True) + (p_round + depth * 2 * U) * av
    flat = lambda t: t.transpose(1, 2).reshape(b * L, heads * 64)
    return flat(o), flat(err)


# ---------------------------------------------------------------------------------------------------------------------
# the checker
# ---------------------------------------------------------------------------------------------------------------------
class Checker:
    def __init__(self, prec):
        self.prec, self.bf, self.fails = prec, prec == "bf16", []

    def note(self, what, op, got, ref, err, final_bf16=True):
        """|got - ref| <= bound elementwise, bound = ulp(ref) (one bf16 rounding) + err (1 + 2^-7), or err."""
        bound = bf16_ulp(ref) + err * SLACK if (self.bf and final_bf16) else err
        ratio = ((got - ref).abs() / bound.clamp_min(1e-300))
        r = ratio.max().item() if ratio.numel() else 0.0
        if not math.isfinite(r):
            r = float("inf")
        key = (self.prec, op)
        WORST[key] = max(WORST.get(key, 0.0), r)
        if r > 1.0:
            self.fails.append((what, round(r, 3)))
        return ratio, bound


def layer_weights(sd, l, bf):
    pre = "encoder.layer.%d." % l
    mat = (lambda t: t.cuda().to(torch.bfloat16).double()) if bf else (lambda t: t.cuda().double())
    vec = lambda n: sd[pre + n].cuda().double()
    return dict(
        wqkv=mat(torch.cat([sd[pre + "attention.self.%s.weight" % n] for n in ("query", "key", "value")])),
        bqkv=torch.cat([vec("attention.self.%s.bias" % n) for n in ("query", "key", "value")]),
        wo=mat(sd[pre + "attention.output.dense.weight"]), bo=vec("attention.output.dense.bias"),
        g1=vec("attention.output.LayerNorm.weight"), b1n=vec("attention.output.LayerNorm.bias"),
        wi=mat(sd[pre + "intermediate.dense.weight"]), bi=vec("intermediate.dense.bias"),
        w2=mat(sd[pre + "output.dense.weight"]), b2=vec("output.dense.bias"),
        g2=vec("output.LayerNorm.weight"), b2n=vec("output.LayerNorm.bias"))


def check_layer(ck, enc, sd, l, layers, heads, ids, lengths, out):
    """Every op of tapped layer l of the last forward against float64."""
    B, L = ids.shape
    bf = ck.bf
    W = layer_weights(sd, l, bf)
    tap = {k: enc.read(k) for k in ("x", "qkv", "ctx", "y1", "h1", "inter", "y2")}
    last = l == layers - 1
    tap["out"] = out.reshape(B * L, -1) if last else enc.read("out")
    lens = lengths.cuda().long()
    if l == 0:
        word = sd["embeddings.word_embeddings.weight"].cuda()
        pos = sd["embeddings.position_embeddings.weight"].cuda()
        typ = sd["embeddings.token_type_embeddings.weight"].cuda()
        g, b = sd["embeddings.LayerNorm.weight"].cuda().double(), sd["embeddings.LayerNorm.bias"].cuda().double()
        flat_ids = ids.reshape(-1).cuda().long()
    seqs = max(1, ROWS // L)
    for s0 in range(0, B, seqs):
        s1 = min(B, s0 + seqs)
        r0, r1 = s0 * L, s1 * L
        T = {k: v[r0:r1].double() for k, v in tap.items()}
        if l == 0:
            v = (word[flat_ids[r0:r1]] + typ[0]) + pos[torch.arange(r0, r1, device="cuda") % L]
            ref, err = layernorm(v.double(), g, b)
            ck.note("embedding LayerNorm", "EMBED_LN", T["x"], ref, err)
        ref, err = linear(T["x"], W["wqkv"], W["bqkv"], bf=bf)
        ck.note("QKV GEMM layer %d" % l, "QKV", T["qkv"], ref, err)
        ref, err = attention(T["qkv"].reshape(s1 - s0, L, -1), lens[s0:s1], heads, bf)
        ck.note("attention layer %d" % l, "ATTN", T["ctx"], ref, err)
        ref, err = linear(T["ctx"], W["wo"], W["bo"], T["x"], bf=bf)
        ck.note("output GEMM + residual layer %d" % l, "OUT_RES", T["y1"], ref, err)
        ref, err = layernorm(T["y1"], W["g1"], W["b1n"])
        ck.note("LayerNorm 1 layer %d" % l, "LN1", T["h1"], ref, err)
        pre, err = linear(T["h1"], W["wi"], W["bi"], bf=bf)
        ref = F.gelu(pre)
        if bf:
            allow = (gelu_tanh(pre) - ref).abs()
            err = GELU_SLOPE * err + allow + 0.5 * pre.abs() * (TANH_APPROX + 8 * U) + 2 * U * ref.abs()
        else:
            err = GELU_SLOPE * err + 3 * U * pre.abs() + 4 * U * ref.abs()
        ratio, bound = ck.note("intermediate GEMM + GELU layer %d" % l, "INTER_GELU", T["inter"], ref, err)
        if bf:
            i = int(ratio.argmax())
            r = ratio.reshape(-1)[i].item()
            if r >= GELU_SHARE.get(ck.prec, (-1.0, 0.0))[0]:
                GELU_SHARE[ck.prec] = (r, (allow.reshape(-1)[i] * SLACK / bound.reshape(-1)[i]).item())
        ref, err = linear(T["inter"], W["w2"], W["b2"], T["h1"], bf=bf)
        ck.note("FFN GEMM + residual layer %d" % l, "FFN_RES", T["y2"], ref, err)
        ref, err = layernorm(T["y2"], W["g2"], W["b2n"])
        ck.note("LayerNorm 2 layer %d" % l, "LN2_OUT" if last else "LN2", T["out"], ref, err, final_bf16=not last)
        del T


def run_case(config, sd, prec, ids, mask, layers_to_tap):
    lengths = mask.sum(1).to(torch.int32)
    B, L = ids.shape
    enc = BertTextEncoder(config=config, state_dict=sd, precision=prec, capacity=B * L)
    ck = Checker(prec)
    for l in layers_to_tap:
        enc.set_tap(l)
        out = enc(input_ids=ids, attention_mask=mask)
        torch.cuda.synchronize()
        check_layer(ck, enc, sd, l, config.num_hidden_layers, config.num_attention_heads, ids, lengths, out)
    enc.close()
    return ck.fails


# ---------------------------------------------------------------------------------------------------------------------
# cases
# ---------------------------------------------------------------------------------------------------------------------
RAGGED = [1, 2, 15, 16, 17, 31, 32, 33, 63, 64, 65, 127, 128, 129]
CASES = {
    # name: batch (sequences, L, lengths or None for the benchmark's draw), layers tapped (None: all)
    "b128": (128, 64, None, None),
    "b1024": (1024, 64, None, (0, 6, 11)),
    "ragged129": (len(RAGGED), 129, RAGGED, None),       # key tiles / chunks and 64-query blocks; 1806 GEMM rows
    "len512": (3, 512, [512, 200, 1], None),
}


@pytest.mark.parametrize("prec", ["bf16", "fp32"])
@pytest.mark.parametrize("case", list(CASES))
def test_bert_base_op_by_op(bert_base, case, prec):
    config, sd = bert_base
    B, L, lengths, taps = CASES[case]
    t0 = time.time()
    if lengths is None:
        ids, mask = bench_batch(B, L, config.vocab_size, seed=B)
    else:
        ids, mask = batch(lengths, L, config.vocab_size, seed=L)
    fails = run_case(config, sd, prec, ids, mask, taps or range(config.num_hidden_layers))
    print("%s %s: %.1f s" % (case, prec, time.time() - t0))
    assert not fails, fails[:10]


@pytest.mark.parametrize("prec", ["bf16", "fp32"])
def test_sharp_attention(bert_base, prec):
    """The query weights and biases of the last two layers scaled so that layer 10's largest logit q k / 8 is 100:
    P nearly one-hot and the running max moving across key tiles, on the L = 129 batch."""
    config, sd = bert_base
    ids, mask = batch(RAGGED, 129, config.vocab_size, seed=129)
    lengths = mask.sum(1).cuda()
    heads, layers = config.num_attention_heads, config.num_hidden_layers

    def max_logit(state, enc_prec):
        enc = BertTextEncoder(config=config, state_dict=state, precision=enc_prec, capacity=ids.numel())
        enc.set_tap(layers - 2)
        enc(input_ids=ids, attention_mask=mask)
        qkv = enc.read("qkv").double().reshape(len(RAGGED), 129, -1)
        enc.close()
        q, k, _ = (t.reshape(len(RAGGED), 129, heads, 64).transpose(1, 2) for t in qkv.chunk(3, dim=-1))
        s = (q @ k.transpose(-1, -2) / 8).abs()
        keep = (torch.arange(129, device="cuda")[None] < lengths[:, None])[:, None, None, :]
        return s.masked_fill(~keep, 0).amax().item()

    f = 100 / max_logit(sd, "fp32")
    sharp = dict(sd)
    for l in (layers - 2, layers - 1):
        for n in ("weight", "bias"):
            key = "encoder.layer.%d.attention.self.query.%s" % (l, n)
            sharp[key] = sd[key] * f
    reached = max_logit(sharp, prec)
    print("sharp %s: query scale %.1f, largest |logit| %.1f" % (prec, f, reached))
    assert reached > 80
    fails = run_case(config, sharp, prec, ids, mask, (layers - 2, layers - 1))
    assert not fails, fails[:10]


@pytest.mark.parametrize("prec", ["bf16", "fp32"])
def test_small_geometry_op_by_op(prec):
    """H 256, 4 heads, I 512, 2 layers: other N tile counts (768 / 256 / 512) and K (256 / 512)."""
    model = perturbed_bert(3, **SMALL)
    sd = {k: v.detach().clone() for k, v in model.state_dict().items()}
    ids, mask = batch([70, 1, 33, 64, 65, 17, 2], 70, SMALL["vocab_size"], seed=5)
    fails = run_case(model.config, sd, prec, ids, mask, (0, 1))
    assert not fails, fails[:10]


# ---------------------------------------------------------------------------------------------------------------------
# the tap itself
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("prec", ["bf16", "fp32"])
def test_tap_changes_no_output_bit(prec):
    """A forward with a tap set gives the same output, bit for bit, as one without; so does one after the tap is
    turned off again."""
    model = perturbed_bert(3, **SMALL)
    ids, mask = batch([70, 1, 33, 64, 65, 17, 2], 70, SMALL["vocab_size"], seed=6)
    enc = BertTextEncoder(model, precision=prec)
    ref = enc(input_ids=ids, attention_mask=mask).clone()
    for layer in (0, 1, -1):
        enc.set_tap(layer)
        out = enc(input_ids=ids, attention_mask=mask)
        assert torch.equal(out, ref), (prec, layer)
    enc.close()


def test_tap_abi_errors():
    """A tap layer outside [-1, layers) and a null handle (DS_ERR_INVALID); a read before any forward with a tap, or
    after a forward without one (DS_ERR_STATE); a bad kind, DS_TE_OUT of the last layer or too small a capacity
    (DS_ERR_INVALID); a size query sets the shape only."""
    model = perturbed_bert(3, **SMALL)
    ids, mask = batch([70, 1, 33], 70, SMALL["vocab_size"], seed=7)
    enc = BertTextEncoder(model, precision="bf16", capacity=512)
    lib, h = enc.lib, enc.h
    r, w = C.c_int32(), C.c_int32()
    out = torch.empty(1 << 20, device="cuda")
    S = capi.TEXT_ENC_TAP
    call = lambda kind, cap, ptr=C.c_void_p(out.data_ptr()): lib.ds_text_enc_read(h, kind, ptr, cap, C.byref(r),
                                                                                   C.byref(w), None)
    assert lib.ds_text_enc_set_tap(None, 0) == -1
    assert lib.ds_text_enc_read(None, S["x"], None, 0, C.byref(r), C.byref(w), None) == -1
    for bad in (-2, 2, 1 << 20):
        assert lib.ds_text_enc_set_tap(h, bad) == -1, bad
    assert call(S["x"], out.numel()) == -4                       # no forward yet
    enc(input_ids=ids, attention_mask=mask)
    assert call(S["x"], out.numel()) == -4                       # a forward without a tap
    enc.set_tap(1)
    assert call(S["x"], out.numel()) == -4                       # set, but no forward since
    enc(input_ids=ids, attention_mask=mask)
    r.value = w.value = 0
    assert call(S["inter"], 0, None) == 0 and (r.value, w.value) == (3 * 70, 512)      # size query
    assert call(S["qkv"], 3 * 70 * 768 - 1) == -1                                      # capacity too small
    assert call(S["qkv"], 3 * 70 * 768) == 0 and (r.value, w.value) == (3 * 70, 768)
    for kind in (-1, len(S), S["out"]):                          # DS_TE_OUT: layer 1 is the last layer
        assert call(kind, out.numel()) == -1, kind
    enc.set_tap(0)
    enc(input_ids=ids, attention_mask=mask)
    assert call(S["out"], out.numel()) == 0 and (r.value, w.value) == (3 * 70, 256)
    assert enc.read("y2").shape == (3 * 70, 256)
    enc.set_tap(-1)
    enc(input_ids=ids, attention_mask=mask)
    assert call(S["x"], out.numel()) == -4                       # the last forward ran without a tap
    enc.close()
