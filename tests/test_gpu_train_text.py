"""GPU: native training of the text-conditioned denoiser (ds_train_step_cross: the LinearAttentionCross layers in the
forward and backward pass of the training step) against torch autograd over the CPU oracle with `context_cross`
requiring grad: losses, the 9 dict entries, every parameter gradient (the 9 to_kv weights included), d(context) and
d(cross) in fp32 parity mode; bf16 mode against the same gradients; the forward-only value against the sampling
engine's p_losses; the drop-in class's train_on_batch against its autograd twin; argument checks of the ABI."""
import ctypes as C

import numpy as np
import pytest
import torch

from diffuscene_b200 import capi
from diffuscene_b200.engine import DenoiserEngine
from diffuscene_b200.weights import NetSpec, seeded_state_dict, unet1d_param_specs
from oracle import diffusion_ref as D
from oracle.unet1d_ref import unet1d_forward
from tests.cases import CASES, STATS, make_inputs
from tests.gpu_common import case_tables

pytestmark = pytest.mark.gpu

# text62 with more scenes, a text longer than one warp of tokens, eps-prediction and the IoU regulariser
TEXT_CASES = {
    "text62": CASES["text62"],
    "text62_b5_l33": dict(CASES["text62"], seed=19, B=5, L=33,
                          diffusion_kwargs=dict(CASES["text62"]["diffusion_kwargs"], model_mean_type="eps",
                                                loss_iou=True)),
}
BOUNDS = STATS["bounds_translations"] + STATS["bounds_sizes"]
DS_ERR_INVALID = -1


def _setup(name):
    case = TEXT_CASES[name]
    spec = NetSpec.from_net_kwargs(case["net_kwargs"])
    sd = seeded_state_dict(unet1d_param_specs(spec), seed=case["seed"])
    inp = make_inputs(case, spec)
    return case, spec, sd, inp, inp["context"][0], inp["context_cross"]


def _oracle_grads(case, spec, sd, inp, ctx, cross):
    """autograd through the oracle: loss = p_losses(...).mean(); (losses, dict, grads by name, d(context), d(cross))."""
    dk = case["diffusion_kwargs"]
    sched = D.make_schedule(D.make_betas(dk["schedule_type"], dk["beta_start"], dk["beta_end"], dk["time_num"]),
                            dk["model_mean_type"], dk["model_var_type"])
    cfg = case["net_cfg"]
    ls = D.LossSpec(class_dim=cfg["class_dim"], angle_dim=cfg["angle_dim"], objfeat_dim=cfg["objfeat_dim"],
                    objectness_dim=cfg["objectness_dim"], loss_separate=dk["loss_separate"], loss_iou=dk["loss_iou"],
                    bounds_translations=STATS["bounds_translations"], bounds_sizes=STATS["bounds_sizes"])
    sdg = {k: v.clone().requires_grad_(True) for k, v in sd.items()}
    c = ctx.clone().requires_grad_(True)
    xc = cross.clone().requires_grad_(True)
    B, N = case["B"], case["N"]
    with torch.enable_grad():
        den = lambda xx, tt: unet1d_forward(sdg, spec, xx, tt, c[None].expand(B, N, -1), xc)
        losses, ld = D.p_losses(sched, ls, den, inp["x0"], inp["t_loss"], inp["noise_loss"])
        losses.mean().backward()
    return losses.detach(), ld, {k: v.grad for k, v in sdg.items()}, c.grad, xc.grad


def _engine(case, spec, prec):
    eng = DenoiserEngine(spec, case["N"], case["diffusion_kwargs"]["time_num"], precision=prec)
    eng.set_schedule(case_tables(case))
    return eng


def _flat(eng, sd):
    layout = eng.flat_layout()
    flat = torch.empty(sum(n for _, n in layout.values()), device="cuda")
    for k, (off, n) in layout.items():
        flat[off:off + n] = sd[k].reshape(-1).cuda()
    return flat, layout


def _native(case, spec, sd, inp, ctx, cross, prec):
    eng = _engine(case, spec, prec)
    flat, layout = _flat(eng, sd)
    grads = torch.full_like(flat, float("nan"))
    dk = case["diffusion_kwargs"]
    losses, ld, dctx, dcross = eng.train_step(flat, inp["x0"].cuda(), inp["t_loss"].cuda(), inp["noise_loss"].cuda(),
                                              ctx.cuda(), True, dk["loss_separate"], dk["loss_iou"], BOUNDS,
                                              flat_grads=grads, cross=cross.cuda())
    torch.cuda.synchronize()
    out = {k: grads[off:off + n].reshape(sd[k].shape).cpu() for k, (off, n) in layout.items()}
    eng.close()
    return losses.cpu(), {k: float(v) for k, v in ld.items()}, out, dctx.cpu(), dcross.cpu()


@pytest.mark.parametrize("name", list(TEXT_CASES))
def test_text_gradients_match_oracle_autograd_fp32(name):
    case, spec, sd, inp, ctx, cross = _setup(name)
    ref_losses, ref_ld, ref_g, ref_dc, ref_dx = _oracle_grads(case, spec, sd, inp, ctx, cross)
    losses, ld, g, dc, dx = _native(case, spec, sd, inp, ctx, cross, "fp32")
    np.testing.assert_allclose(losses.numpy(), ref_losses.numpy(), rtol=1e-3, atol=1e-4)
    assert len(ref_ld) == 9
    for k, v in ref_ld.items():
        np.testing.assert_allclose(ld[k], float(torch.as_tensor(v).detach()), rtol=1e-3, atol=1e-4, err_msg=k)
    assert set(g) == set(ref_g)
    kv = [k for k in g if k.endswith(".fn.fn.to_kv.weight")]
    assert len(kv) == 9
    for k in kv:
        assert torch.isfinite(g[k]).all() and g[k].abs().max() > 0, k
    worst = []
    for k in sorted(g):
        a, b = g[k], ref_g[k]
        assert torch.isfinite(a).all(), k
        scale = max(b.abs().max().item(), 1e-6)
        worst.append(((a - b).abs().max().item() / scale, k))
    worst.sort(reverse=True)
    print("worst relative gradient errors:", worst[:5])
    assert worst[0][0] < 2e-3, worst[:8]
    np.testing.assert_allclose(dc.numpy(), ref_dc.numpy(), rtol=2e-3, atol=2e-3 * ref_dc.abs().max().item())
    np.testing.assert_allclose(dx.numpy(), ref_dx.numpy(), rtol=2e-3, atol=2e-3 * ref_dx.abs().max().item())


def test_text_gradients_bf16_close_to_fp32_oracle():
    """bf16 storage of activations and their gradients, fp32 text side and parameter gradients: the cosine of every
    parameter gradient and of d(cross) with the oracle's, lowest > 0.97 and mean > 0.995."""
    case, spec, sd, inp, ctx, cross = _setup("text62")
    _, _, ref_g, _, ref_dx = _oracle_grads(case, spec, sd, inp, ctx, cross)
    _, _, g, _, dx = _native(case, spec, sd, inp, ctx, cross, "bf16")
    pairs = [(g[k], ref_g[k], k) for k in sorted(g)] + [(dx, ref_dx, "d(cross)")]
    cos = []
    for a, b, k in pairs:
        a, b = a.flatten().double(), b.flatten().double()
        if b.norm() < 1e-10:
            continue
        cos.append((float(a @ b / (a.norm() * b.norm() + 1e-30)), k))
    cos.sort()
    print("lowest gradient cosines (bf16 mode):", cos[:5])
    assert any(k == "d(cross)" for _, k in cos)
    assert cos[0][0] > 0.97 and np.mean([c for c, _ in cos]) > 0.995


@pytest.mark.parametrize("prec,rtol", [("fp32", 1e-4), ("bf16", 1e-3)])
def test_text_forward_only_matches_p_losses(prec, rtol):
    """ds_train_step_cross without gradients = the sampling engine's p_losses after set_context_cross (both run the
    one-kernel-per-op program: fuse level 0)."""
    case, spec, sd, inp, ctx, cross = _setup("text62_b5_l33")
    dk = case["diffusion_kwargs"]
    x0, t, noise = inp["x0"].cuda(), inp["t_loss"].cuda(), inp["noise_loss"].cuda()
    ref = DenoiserEngine(spec, case["N"], dk["time_num"], precision=prec, fuse_level=0)
    ref.load_state_dict(sd)
    ref.set_schedule(case_tables(case))
    ref.set_context(ctx.cuda(), shared=True)
    ref.set_context_cross(cross.cuda())
    ref_losses, ref_ld = ref.p_losses(x0, t, noise, dk["loss_separate"], dk["loss_iou"], BOUNDS)
    eng = _engine(case, spec, prec)
    flat, _ = _flat(eng, sd)
    out = eng.train_step(flat, x0, t, noise, ctx.cuda(), True, dk["loss_separate"], dk["loss_iou"], BOUNDS,
                         flat_grads=None, cross=cross.cuda())
    torch.cuda.synchronize()
    losses, ld, dctx, dcross = out
    assert dctx is None and dcross is None
    np.testing.assert_allclose(losses.cpu().numpy(), ref_losses.cpu().numpy(), rtol=rtol, atol=1e-6)
    for k in ld:
        np.testing.assert_allclose(float(ld[k]), float(ref_ld[k]), rtol=rtol, atol=1e-6, err_msg=k)
    ref.close()
    eng.close()


def test_text_train_on_batch_native_matches_autograd(tmp_path):
    """Two optimizer iterations of the shipped text config through the drop-in API: native backward (with the
    cross-attention layers and d(cross) into fc_text_f) + fused Adam + device-side clip against torch autograd over
    functional.DenoiserFn + torch.optim.Adam + clip_grad_norm_ on a twin model (fp32 mode, same t / noise draws)."""
    import copy
    import json
    import os
    import yaml
    from scene_synthesis.networks import build_network, optimizer_factory
    from diffuscene_b200.optim import NativeAdam
    from tests.cases_class import fake_bert_hidden
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    cfg = yaml.safe_load(open(os.path.join(root, "config", "text/diffusion_bedrooms_instancond_lat32_v_bert.yaml")))
    stats = tmp_path / "stats.json"
    stats.write_text(json.dumps(STATS))
    cfg["network"]["diffusion_kwargs"]["train_stats_file"] = str(stats)
    cfg["training"]["max_grad_norm"] = 0.05          # small enough that the clip is active
    torch.manual_seed(3)
    net_a, train_on_batch, _ = build_network(30, 23, cfg, None, device="cuda", precision="fp32")
    net_b, _, _ = build_network(30, 23, cfg, None, device="cuda", precision="fp32")
    net_b.load_state_dict(copy.deepcopy(net_a.state_dict()))
    net_b.native_backward = False
    assert net_a.native_training_supported()
    opt_a = optimizer_factory(cfg["training"], net_a.parameters())
    assert isinstance(opt_a, NativeAdam)
    opt_b = torch.optim.Adam(net_b.parameters(), lr=cfg["training"]["lr"], weight_decay=0.0)
    g = torch.Generator().manual_seed(0)
    B = 4
    cls = torch.randint(0, 22, (B, 12), generator=g)
    desc = fake_bert_hidden(["a bedroom with a double bed and two nightstands", "wardrobe next to the desk",
                             "a single bed under the window", "a desk, a chair and a tall wardrobe"])
    sp = dict(translations=torch.rand(B, 12, 3, generator=g) * 2 - 1, sizes=torch.rand(B, 12, 3, generator=g) * 2 - 1,
              angles=torch.nn.functional.normalize(torch.randn(B, 12, 2, generator=g), dim=-1),
              class_labels=torch.nn.functional.one_hot(cls, 22).float() * 2 - 1,
              objfeats_32=torch.rand(B, 12, 32, generator=g) * 2 - 1, room_layout=torch.zeros(B, 1, 64, 64),
              description=desc)
    sp = {k: v.cuda() for k, v in sp.items()}
    text0 = net_a.fc_text_f.weight.detach().clone()
    for it in range(2):
        torch.manual_seed(100 + it)
        la = train_on_batch(net_a, opt_a, sp, cfg)
        assert net_a._native_grads_ready and net_a.fc_text_f.weight.grad is not None
        torch.manual_seed(100 + it)
        lb = train_on_batch(net_b, opt_b, sp, cfg)
        assert abs(la - lb) < 1e-3 * max(1.0, abs(lb)), (it, la, lb)
    sa, sb = net_a.state_dict(), net_b.state_dict()
    assert "fc_text_f.weight" in sa
    assert (sa["fc_text_f.weight"] - text0).abs().max() > 0
    worst = max(((sa[k] - sb[k]).abs().max().item(), k) for k in sa)
    print("largest parameter difference after 2 iterations:", worst,
          "fc_text_f.weight:", (sa["fc_text_f.weight"] - sb["fc_text_f.weight"]).abs().max().item())
    assert worst[0] < 3 * cfg["training"]["lr"], worst
    mean_diff = np.mean([(sa[k] - sb[k]).abs().mean().item() for k in sa])
    assert mean_diff < 0.05 * cfg["training"]["lr"], mean_diff
    room = torch.zeros(2, 1, 64, 64, device="cuda")
    s = net_a.sample(room, 12, 62, batch_size=2, text=desc[:2].cuda(), clip_denoised=True, ddim=True, ddim_steps=3, seed=1)
    assert torch.isfinite(s).all()


def test_text_train_argument_errors():
    """Wrong entry point for the network, a NULL text and a text longer than DS_TRAIN_CROSS_MAX_L are refused before
    anything is launched; the handles keep working afterwards."""
    max_l = 200      # DS_TRAIN_CROSS_MAX_L
    lib = capi.load()
    P = lambda t: None if t is None else C.c_void_p(t.data_ptr())

    def call(eng, flat, inp, ctx, dk, cross=None, L=0, text_entry=True):
        B = inp["x0"].shape[0]
        losses = torch.empty(B, device="cuda")
        ld = torch.empty(9, device="cuda")
        barr = (C.c_float * 12)(*BOUNDS)
        args = (eng.h, P(flat), P(inp["x0"]), P(inp["t_loss"]), P(inp["noise_loss"]), P(ctx), 0, 1,
                int(dk["loss_separate"]), int(dk["loss_iou"]), barr, C.c_float(1.0), P(losses), P(ld), None, None)
        if text_entry:
            rc = lib.ds_train_step_cross(*args, P(cross), L, None, B, eng._stream())
        else:
            rc = lib.ds_train_step(*args, B, eng._stream())
        torch.cuda.synchronize()
        return rc, lib.ds_last_error().decode(), losses

    engines = {}
    for name in ("text62", "bed62"):
        case = CASES[name]
        spec = NetSpec.from_net_kwargs(case["net_kwargs"])
        sd = seeded_state_dict(unet1d_param_specs(spec), seed=case["seed"])
        inp = {k: (v.cuda() if torch.is_tensor(v) else v) for k, v in make_inputs(case, spec).items()}
        eng = _engine(case, spec, "fp32")
        engines[name] = (eng, _flat(eng, sd)[0], inp, inp["context"][0].contiguous(), case["diffusion_kwargs"])
    et, ft, it_, ct, dkt = engines["text62"]
    eb, fb, ib, cb, dkb = engines["bed62"]
    cross = it_["context_cross"].contiguous()
    bad = [call(et, ft, it_, ct, dkt, text_entry=False),                      # text network through ds_train_step
           call(eb, fb, ib, cb, dkb, cross=cross, L=cross.shape[1]),          # ds_train_step_cross without text condition
           call(et, ft, it_, ct, dkt, cross=None, L=cross.shape[1]),          # NULL text
           call(et, ft, it_, ct, dkt, cross=cross, L=max_l + 1),              # text too long
           call(et, ft, it_, ct, dkt, cross=cross, L=0)]
    for rc, msg, _ in bad:
        assert rc == DS_ERR_INVALID and msg, (rc, msg)
    assert "ds_train_step_cross" in bad[0][1]
    # both handles still train
    rc, msg, lt = call(et, ft, it_, ct, dkt, cross=cross, L=cross.shape[1])
    assert rc == 0 and torch.isfinite(lt).all(), msg
    rc, msg, lb = call(eb, fb, ib, cb, dkb, text_entry=False)
    assert rc == 0 and torch.isfinite(lb).all(), msg
    for e in engines.values():
        e[0].close()
