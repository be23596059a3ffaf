"""CPU: the engine's step program (exported from the C++ plan builder), interpreted with torch on the CPU,
reproduces the reference's golden denoiser outputs -- i.e. op order, buffer reuse, weight packing recipes and
the hoisted FiLM tables are right before a single kernel runs."""
import os

import numpy as np
import pytest
import torch

from diffuscene_b200 import capi
from diffuscene_b200.weights import NetSpec, seeded_state_dict, unet1d_param_specs
from oracle.plan_interp import run_plan
from tests.cases import CASES, make_inputs


def _run(name, no_reuse, bf16=False, fuse=0):
    case = CASES[name]
    spec = NetSpec.from_net_kwargs(case["net_kwargs"])
    cfg = capi.make_config(spec, case["N"], case["diffusion_kwargs"]["time_num"], fuse_level=fuse)
    plan = capi.plan_export(cfg, no_reuse=no_reuse)
    sd = {k[len("diffusion.model."):]: v for k, v in
          seeded_state_dict(unet1d_param_specs(spec), seed=case["seed"]).items()}
    inp = make_inputs(case, spec)
    return run_plan(plan, sd, inp["x"], inp["t"], inp["context"], inp["context_cross"], emulate_bf16=bf16)


@pytest.mark.parametrize("name", list(CASES))
def test_plan_reproduces_golden(name, golden_dir):
    torch.set_grad_enabled(False)
    gold = np.load(os.path.join(golden_dir, name + ".npz"))["fwd"]
    out = _run(name, no_reuse=False)
    np.testing.assert_allclose(out.numpy(), gold, rtol=1e-3, atol=1e-4)    # the north-star tolerance
    np.testing.assert_allclose(out.numpy(), gold, rtol=2e-4, atol=3e-5)    # and much tighter in practice


@pytest.mark.parametrize("name", ["bed62", "liv65", "text62", "arr5"])
def test_fused_plan_reproduces_golden(name, golden_dir):
    """fuse_level 1: every Block (conv+GroupNorm+FiLM+SiLU) is one GEMM_GN op."""
    torch.set_grad_enabled(False)
    gold = np.load(os.path.join(golden_dir, name + ".npz"))["fwd"]
    out = _run(name, no_reuse=False, fuse=1)
    np.testing.assert_allclose(out.numpy(), gold, rtol=2e-4, atol=3e-5)
    case = CASES[name]
    cfg = capi.make_config(NetSpec.from_net_kwargs(case["net_kwargs"]), case["N"], 1000, fuse_level=1)
    txt = capi.plan_describe(cfg)
    assert " GN " not in txt and txt.count(" GEMM_GN ") == 56


@pytest.mark.parametrize("name", ["bed62", "text62"])
def test_fuse_level_4_plan_reproduces_golden(name, golden_dir):
    """fuse_level 4: to_out + LayerNorm + residual of the attention wrappers is one GEMM_LN op."""
    torch.set_grad_enabled(False)
    gold = np.load(os.path.join(golden_dir, name + ".npz"))["fwd"]
    out = _run(name, no_reuse=False, fuse=4)
    np.testing.assert_allclose(out.numpy(), gold, rtol=2e-4, atol=3e-5)
    case = CASES[name]
    spec = NetSpec.from_net_kwargs(case["net_kwargs"])
    txt = capi.plan_describe(capi.make_config(spec, case["N"], 1000, fuse_level=4))
    assert txt.count(" GEMM_LN ") == (17 if spec.text_condition else 8) and txt.count(" LN ") == (18 if spec.text_condition else 9)


@pytest.mark.parametrize("name", ["bed62", "text62", "liv65"])
def test_fuse_level_5_plan_reproduces_golden(name, golden_dir):
    """fuse_level 5: LayerNorm + to_qkv + linear-attention core is one LN_QKV_ATTN op (N = 12 or 21), the LayerNorm
    gain travels inside the packed weights."""
    torch.set_grad_enabled(False)
    gold = np.load(os.path.join(golden_dir, name + ".npz"))["fwd"]
    out = _run(name, no_reuse=False, fuse=5)
    np.testing.assert_allclose(out.numpy(), gold, rtol=2e-4, atol=3e-5)
    case = CASES[name]
    spec = NetSpec.from_net_kwargs(case["net_kwargs"])
    txt = capi.plan_describe(capi.make_config(spec, case["N"], 1000, fuse_level=5))
    assert txt.count(" LN_QKV_ATTN ") == 8


def test_buffer_reuse_does_not_change_results():
    torch.set_grad_enabled(False)
    a = _run("bed62", no_reuse=False)
    b = _run("bed62", no_reuse=True)
    assert torch.equal(a, b)


def test_bf16_emulation_error_is_bounded(golden_dir):
    """Predicts the throughput-mode error (bf16 storage + bf16 weights, fp32 accumulate); the GPU test
    asserts the same bound on the real kernels."""
    torch.set_grad_enabled(False)
    gold = torch.from_numpy(np.load(os.path.join(golden_dir, "bed62.npz"))["fwd"])
    out = _run("bed62", no_reuse=False, bf16=True)
    err = (out - gold).abs()
    assert err.max() < 0.05 and err.mean() < 0.01, (err.max(), err.mean())


def _reads(op):
    """(buffer, first column, last column + 1) of every buffer slice an op reads."""
    from oracle.plan_interp import OP_PACK
    if op["kind"] == OP_PACK:
        return []
    r = [(s["buf"], s["col"], s["col"] + s["k"]) for s in (op["in0"], op["in1"]) if s["buf"] >= 0]
    if op.get("res", -1) >= 0:
        r.append((op["res"], 0, None))
    return r


@pytest.mark.parametrize("fuse", [0, 1, 4, 5])
@pytest.mark.parametrize("name", ["bed62", "liv65", "text62", "arr5"])
def test_no_reuse_plan_taps_are_op_inputs(name, fuse):
    """In the program exported with no_reuse (the one the engine runs with taps on), no op reads a buffer that a
    later op writes, and no op writes a buffer it reads.  So after one forward, the buffers an op read still hold
    exactly what it read: the per-op GPU test evaluates each op from those taps."""
    case = CASES[name]
    spec = NetSpec.from_net_kwargs(case["net_kwargs"])
    plan = capi.plan_export(capi.make_config(spec, case["N"], 1000, fuse_level=fuse), no_reuse=True)
    ops = plan["ops"]
    for i, op in enumerate(ops):
        read = {b for b, _, _ in _reads(op)}
        assert op["out"] not in read, op["name"]
        for later in ops[i + 1:]:
            assert later["out"] not in read, (op["name"], later["name"])
