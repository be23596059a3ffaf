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


def _run(name, no_reuse, bf16=False, fuse=0, train=False):
    case = CASES[name]
    spec = NetSpec.from_net_kwargs(case["net_kwargs"])
    cfg = capi.make_config(spec, case["N"], case["diffusion_kwargs"]["time_num"], fuse_level=fuse, train=train)
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


@pytest.mark.parametrize("name", ["bed62", "liv65", "bed97", "obj29", "arr5", "text62"])
def test_train_plan_reproduces_golden(name, golden_dir):
    """The training step program (every activated GEMM split into `<name>.pre` + an ACT op, one buffer per op output,
    as ds_train_step builds it) computes the reference's forward."""
    torch.set_grad_enabled(False)
    gold = np.load(os.path.join(golden_dir, name + ".npz"))["fwd"]
    out = _run(name, no_reuse=True, train=True)
    np.testing.assert_allclose(out.numpy(), gold, rtol=2e-4, atol=3e-5)


def _fwd_write(op):
    """(buffer, first column, last column + 1) an op's forward writes."""
    return op["out"], op["out_col"], op["out_col"] + op["N"]


def _bwd_reads(op):
    """Activation slices the op's backward reads: GEMM operands (dW), the pre-activation of ACT, the input of
    GN / LN / the attention cores."""
    from oracle.plan_interp import OP_PACK
    if op["kind"] == OP_PACK:
        return []
    return [(s["buf"], s["col"], s["col"] + s["k"]) for s in (op["in0"], op["in1"]) if s["buf"] >= 0]


def _bwd_writes(op, plan, pack_buf):
    """Gradient slices the op's backward writes: d(inputs) except the packed network input, d(residual)."""
    w = [r for r in _bwd_reads(op) if r[0] != pack_buf]
    if op.get("res", -1) >= 0:
        w.append((op["res"], 0, plan["buf_width"][op["res"]]))
    return w


def _overlap(a, b):
    return a[0] == b[0] and a[1] < b[2] and b[1] < a[2]


@pytest.mark.parametrize("name", ["bed62", "liv65", "text62", "arr5", "obj29"])
def test_train_plan_state_after_the_step_is_what_each_backward_read(name):
    """ds_train_step runs the backward of the train program op by op in reverse.  So that the buffers read after the
    step (ds_train_read) equal what each op's backward kernels read:
    - the gradient slice an op's backward reads (its output slice) gets no writer later in the backward pass, i.e. no
      earlier op of the program has it among its inputs or as its residual;
    - no activation an op's backward reads is written by that op or by any later op of the forward program."""
    from oracle.plan_interp import OP_ACT, OP_PACK
    case = CASES[name]
    spec = NetSpec.from_net_kwargs(case["net_kwargs"])
    plan = capi.plan_export(capi.make_config(spec, case["N"], 1000, train=True), no_reuse=True)
    ops = plan["ops"]
    pack_buf = next(op["out"] for op in ops if op["kind"] == OP_PACK)
    for i, op in enumerate(ops):
        if op["kind"] == OP_PACK:
            continue
        if op["kind"] == OP_ACT:      # the engine's ACT kernels take no residual (the oracle's OP_ACT would add one)
            assert op["res"] < 0, op["name"]
        g = _fwd_write(op)
        for earlier in ops[:i]:
            for w in _bwd_writes(earlier, plan, pack_buf):
                assert not _overlap(g, w), (op["name"], earlier["name"])
        for r in _bwd_reads(op):
            for later in ops[i:]:
                assert not _overlap(r, _fwd_write(later)), (op["name"], later["name"])
