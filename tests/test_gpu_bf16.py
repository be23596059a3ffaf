"""GPU, bf16 throughput mode: tensor-core (wgmma; backend id "tcgen05" kept from the C ABI) GEMM unit tests, SIMT cross-check, error bounds against the golden
vectors (the bound the CPU bf16 emulation in tests/test_plan_cpu.py predicts), and size-independent
properties at BASELINE batch sizes."""
import ctypes as C

import numpy as np
import pytest
import torch

from diffuscene_b200 import capi
from tests.cases import CASES, noise_stream
from tests.gpu_common import cuda, get_engine, gold

pytestmark = pytest.mark.gpu

# bf16 throughput-mode gates against the fp32 goldens of the unmodified reference: bf16 storage and weights put the
# separate-head networks near max 2e-3 / mean 4e-4 (the stated north-star figure "within 1e-3" is met by the fp32
# parity mode only, SURVEY 0.6); bench.py prints the measured value of the benched precision (`parity_max_abs`).
# The weights are random-init, so class scores are near ties and a 1e-3 perturbation flips a few argmaxes.
# The 5-channel arrangement head (arr5) produces O(1) outputs: its own gate.
BF16_MAX, BF16_MEAN, BF16_ARGMAX = 5e-3, 1e-3, 0.97
BF16_GATE = {"arr5": (2.5e-2, 6e-3)}


def _gemm(backend, a, w, bias, act=0):
    lib = capi.load()
    M, K = a.shape
    N = w.shape[0]
    d = torch.empty(M, N, device="cuda", dtype=torch.bfloat16)
    torch.cuda.synchronize()
    capi.check(lib.ds_test_gemm_bf16(backend, a.data_ptr(), w.data_ptr(), None if bias is None else bias.data_ptr(),
                                     d.data_ptr(), M, N, K, act, None))
    return d


@pytest.mark.parametrize("backend", [capi.DS_GEMM_SIMT, capi.DS_GEMM_TCGEN05], ids=["simt", "tcgen05"])
@pytest.mark.parametrize("shape", [(128, 128, 64), (256, 256, 128), (1000, 512, 512), (3001, 384, 512),
                                   (5000, 1536, 64), (777, 512, 3072), (40000, 1024, 512)])
def test_gemm_matches_torch(backend, shape):
    M, N, K = shape
    g = torch.Generator(device="cpu").manual_seed(M + N + K)
    a = (torch.randn(M, K, generator=g) * 0.5).to(torch.bfloat16).cuda()
    w = (torch.randn(N, K, generator=g) / K ** 0.5).to(torch.bfloat16).cuda()
    bias = torch.randn(N, generator=g).cuda()
    ref = a.float() @ w.float().t() + bias
    for act, fn in ((0, lambda z: z), (1, torch.nn.functional.gelu)):
        d = _gemm(backend, a, w, bias, act).float()
        r = fn(ref)
        err = (d - r).abs().max().item()
        assert err <= 2e-2 * max(1.0, r.abs().max().item()), (shape, act, err)
        # bf16 output rounding only: relative error of a bf16 ulp
        assert ((d - r).abs() <= 8e-3 * r.abs() + 2e-3).all()


@pytest.mark.parametrize("backend", ["simt", "tcgen05"])
@pytest.mark.parametrize("name", ["bed62", "bed97", "liv65", "text62", "arr5", "obj29"])
def test_forward_error_bound(name, backend, golden_dir):
    eng, case, spec, inp = get_engine(name, "bf16", backend)
    g = torch.from_numpy(gold(golden_dir, name)["fwd"])
    out = eng.forward(cuda(inp["x"]), cuda(inp["t"])).cpu()
    err = (out - g).abs()
    # bf16 storage + bf16 weights, fp32 accumulate: the reference probe (SURVEY 0.6) saw max 1.8e-3
    print("bf16 forward error %s/%s: max %.3g mean %.3g" % (name, backend, err.max().item(), err.mean().item()))
    gmax, gmean = BF16_GATE.get(name, (BF16_MAX, BF16_MEAN))
    assert err.max() < gmax and err.mean() < gmean, (err.max().item(), err.mean().item())
    if spec.seperate_all:
        b0 = spec.bbox_dim
        agree = (out[..., b0:b0 + spec.class_dim - 1].argmax(-1) == g[..., b0:b0 + spec.class_dim - 1].argmax(-1))
        assert agree.float().mean() >= BF16_ARGMAX


@pytest.mark.parametrize("name", ["bed62", "liv65", "arr5"])
def test_fused_groupnorm_epilogue_matches_unfused(name, golden_dir):
    """fuse_level 1 (Block = one GEMM with the GroupNorm epilogue) against fuse_level 0 (GEMM, then GroupNorm
    kernel): same math, the fused path skips one bf16 rounding of the conv output."""
    ef, case, spec, inp = get_engine(name, "bf16", "tcgen05", fuse=1)
    eu, _, _, _ = get_engine(name, "bf16", "tcgen05", fuse=0)
    a = ef.forward(cuda(inp["x"]), cuda(inp["t"])).cpu()
    b = eu.forward(cuda(inp["x"]), cuda(inp["t"])).cpu()
    g = torch.from_numpy(gold(golden_dir, name)["fwd"])
    assert (a - b).abs().max().item() < 4e-2
    assert (a - g).abs().mean() <= (b - g).abs().mean() * 1.5 + 1e-4


@pytest.mark.parametrize("fuse", [0, 2, 3, 4, 5])
@pytest.mark.parametrize("name", ["bed62", "bed97", "text62", "arr5", "obj29", "bed62_loop", "liv65", "text62_loop"])
def test_channels_on_lanes_groupnorm_gemm(name, fuse, golden_dir):
    """Every fuse level against the golden forward and against fuse_level 1.
    fuse_level 0 runs one kernel per op (GEMM, then GroupNorm / LayerNorm / attention kernels); 4 also fuses to_out +
    LayerNorm + residual of every (cross-)attention wrapper into k_gemm_ln; 5 also fuses LayerNorm + to_qkv + the
    linear-attention core into k_ln_qkv_attn (N = 12 or 21 objects; other object counts keep the separate ops).
    Levels 2 and 3 selected the sm_100a GEMM with the output channels on the tensor-memory lanes; sm_90a has no
    tensor memory and these levels are declared to run the level-1 program, which is what is checked for them: the
    engine reports level 1 and its output equals level 1's bit for bit.  Covers per-scene FiLM (forward with per-scene
    t), the per-object FiLM of the context blocks, the two-operand skip convs, cross-attention and the residual path."""
    e2, case, spec, inp = get_engine(name, "bf16", "tcgen05", fuse=fuse)
    e1, _, _, _ = get_engine(name, "bf16", "tcgen05", fuse=1)
    g = torch.from_numpy(gold(golden_dir, name)["fwd"])
    a = e2.forward(cuda(inp["x"]), cuda(inp["t"])).cpu()
    b = e1.forward(cuda(inp["x"]), cuda(inp["t"])).cpu()
    err = (a - g).abs()
    gmax, gmean = BF16_GATE.get(name, (BF16_MAX, BF16_MEAN))
    assert err.max() < gmax and err.mean() < gmean, (err.max().item(), err.mean().item())
    if fuse in (2, 3):
        assert e2.fuse_level == 1 and torch.equal(a, b)
    assert (a - b).abs().max().item() < 2 * gmax
    assert (a - g).abs().mean() <= (b - g).abs().mean() * 1.5 + 1e-4


@pytest.mark.parametrize("fuse", [2, 3, 4, 5])
def test_channels_on_lanes_sampling_and_batch_independence(fuse, golden_dir):
    """The sampling loop (batch-uniform t) at a batch with a ragged last tile, against the fp32 golden loop; scenes
    are independent of the batch they are in.  Levels 4 and 5 run the fused attention-wrapper kernels; levels 2 and 3
    (the sm_100a tensor-memory variants) are declared to run the level-1 program on sm_90a."""
    eng, case, spec, inp = get_engine("bed62_loop", "bf16", "tcgen05", fuse=fuse)
    assert eng.fuse_level == (1 if fuse in (2, 3) else fuse)
    g = gold(golden_dir, "bed62_loop")
    T = case["diffusion_kwargs"]["time_num"]
    shape = tuple(inp["x"].shape)
    nz = noise_stream(case["seed"] + 100)
    x_T = nz(shape)
    noise = torch.stack([nz(shape) for _ in range(T)])
    out = eng.sample(shape[0], clip_denoised=True, x_init=x_T, noise=noise).cpu().numpy()
    assert np.abs(out - g["loop"]).max() < 5e-2
    B = 1003                                    # 100 full 10-scene tiles + 3 scenes
    gen = torch.Generator(device="cpu").manual_seed(5)
    x = torch.randn(B, case["N"], spec.point_dim, generator=gen).cuda()
    t = torch.randint(0, T, (B,), generator=gen).cuda()
    big = eng.forward(x, t)
    assert torch.isfinite(big).all()
    assert torch.equal(big[:5], eng.forward(x[:5].contiguous(), t[:5].contiguous()))
    assert torch.equal(big[-3:], eng.forward(x[-3:].contiguous(), t[-3:].contiguous()))
    s1 = eng.sample(40, seed=4)
    s2 = eng.sample(13, seed=4, scene_offset=27)
    assert torch.equal(s1[27:], s2)


def test_tcgen05_agrees_with_simt_bf16():
    """Same bf16 inputs, fp32 accumulation in both: only the summation order differs."""
    e1, case, spec, inp = get_engine("bed62", "bf16", "tcgen05")
    e2, _, _, _ = get_engine("bed62", "bf16", "simt")
    a = e1.forward(cuda(inp["x"]), cuda(inp["t"]))
    b = e2.forward(cuda(inp["x"]), cuda(inp["t"]))
    assert (a - b).abs().max().item() < 3e-3


def test_sampling_loop_bf16_close_to_fp32_reference(golden_dir):
    eng, case, spec, inp = get_engine("bed62_loop", "bf16", "tcgen05")
    g = gold(golden_dir, "bed62_loop")
    T = case["diffusion_kwargs"]["time_num"]
    shape = tuple(inp["x"].shape)
    nz = noise_stream(case["seed"] + 100)
    x_T = nz(shape)
    noise = torch.stack([nz(shape) for _ in range(T)])
    out = eng.sample(shape[0], clip_denoised=True, x_init=x_T, noise=noise).cpu().numpy()
    assert np.abs(out - g["loop"]).max() < 5e-2


def test_batch_independence_at_full_size():
    """Size-independent property at BASELINE batch (4096 scenes): a scene's result does not depend on what
    else is in the batch (tiles never mix scenes), so the first rows of a big batch equal a small batch."""
    eng, case, spec, inp = get_engine("bed62", "bf16", "tcgen05")
    B = 4096
    g = torch.Generator(device="cpu").manual_seed(5)
    x = torch.randn(B, case["N"], spec.point_dim, generator=g).cuda()
    t = torch.randint(0, 1000, (B,), generator=g).cuda()
    big = eng.forward(x, t)
    small = eng.forward(x[:5].contiguous(), t[:5].contiguous())
    assert torch.isfinite(big).all()
    assert torch.equal(big[:5], small)
    # permuting scenes permutes outputs
    perm = torch.randperm(B, generator=g).cuda()
    assert torch.equal(eng.forward(x[perm].contiguous(), t[perm].contiguous()), big[perm])


def test_batch_independence_living_room_shape():
    """N = 21 objects (odd scenes): the fused GroupNorm GEMM tiles 6 scenes = 126 of 128 rows, per-object FiLM loaded
    per element; x0-prediction, fixedlarge
    variance."""
    eng, case, spec, inp = get_engine("liv65", "bf16", "tcgen05")
    B = 1500
    g = torch.Generator(device="cpu").manual_seed(9)
    x = torch.randn(B, case["N"], spec.point_dim, generator=g).cuda()
    t = torch.randint(0, 1000, (B,), generator=g).cuda()
    big = eng.forward(x, t)
    assert torch.isfinite(big).all()
    small = eng.forward(x[:7].contiguous(), t[:7].contiguous())
    assert torch.equal(big[:7], small)
    s1 = eng.sample(40, seed=4, num_steps=6)
    s2 = eng.sample(13, seed=4, num_steps=6, scene_offset=27)
    assert torch.equal(s1[27:], s2)            # sharding by scene does not change any scene's sample


def test_chunked_sampling_is_identical():
    """Sub-batching (L2-resident chunks run one after the other) must not change any scene's result."""
    eng, case, spec, inp = get_engine("bed62_loop", "bf16", "tcgen05")
    a = eng.sample(70, seed=21)
    b = eng.sample(70, seed=21, chunk_scenes=24)
    assert torch.equal(a, b)


def test_full_sample_smoke_bf16():
    eng, case, spec, inp = get_engine("bed62_loop", "bf16", "tcgen05")
    out = eng.sample(256, seed=11)
    assert torch.isfinite(out).all()
    out_h = eng.sample(256, seed=11, host_output=True)
    assert torch.equal(out_h, out.cpu())


@pytest.mark.parametrize("prec", ["fp32", "bf16"])
def test_large_batch_against_oracle(prec):
    """Oracle comparison at a batch with a ragged last tile (B = 1003 scenes: 62 full 16-scene tiles + 11): every
    scene is checked against the CPU oracle, per-scene timesteps, in both precisions."""
    from oracle.unet1d_ref import unet1d_forward
    from diffuscene_b200.weights import seeded_state_dict, unet1d_param_specs
    eng, case, spec, inp = get_engine("bed62", prec)
    B, N = 1003, case["N"]
    gen = torch.Generator(device="cpu").manual_seed(9)
    x = torch.randn(B, N, spec.point_dim, generator=gen)
    t = torch.randint(0, case["diffusion_kwargs"]["time_num"], (B,), generator=gen)
    sd = seeded_state_dict(unet1d_param_specs(spec), seed=case["seed"])
    ctx = inp["context"][0][None].expand(B, N, spec.cond_dim).contiguous()
    with torch.no_grad():
        ref = unet1d_forward(sd, spec, x, t, ctx, None)
    out = eng.forward(x.cuda(), t.cuda()).cpu()
    err = (out - ref).abs()
    b0 = spec.bbox_dim
    agree = (out[..., b0:b0 + spec.class_dim - 1].argmax(-1) == ref[..., b0:b0 + spec.class_dim - 1].argmax(-1)).float().mean()
    print("B=1003 %s: max %.3g mean %.3g argmax agreement %.5f" % (prec, err.max().item(), err.mean().item(), agree.item()))
    if prec == "fp32":
        assert torch.allclose(out, ref, rtol=1e-3, atol=1e-4)
        assert agree == 1.0
    else:
        assert err.max() < 2 * BF16_MAX and err.mean() < BF16_MEAN and agree >= BF16_ARGMAX      # max over 750k outputs
