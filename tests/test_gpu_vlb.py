"""GPU: the variational bound (ds_vlb_loop, DenoiserEngine.vlb, DiffusionSceneLayout_DDPM.diffusion.all_kl /
prior_kl) against the golden vectors of the unmodified reference, in fp32 with the reference's q_sample draws injected;
bf16 against fp32; the Philox path; batch independence; isolation from the sampling graph; argument and state
errors."""
import ctypes as C

import numpy as np
import pytest
import torch

from diffuscene_b200 import capi
from diffuscene_b200.engine import DenoiserEngine
from diffuscene_b200.weights import NetSpec, seeded_state_dict, unet1d_param_specs
from oracle import diffusion_ref as D
from tests import vlb_oracle as V
from tests.cases import _clean_scene, make_inputs
from tests.cases_vlb import VLB_CASES
from tests.gpu_common import case_tables, gold

pytestmark = pytest.mark.gpu
TOL = dict(rtol=1e-3, atol=1e-4)      # t >= 1 terms, mse, prior
REL = 1e-3                            # t = 0 term and the totals it dominates

_ENGINES = {}


def _engine(name, precision="fp32"):
    key = (name, precision)
    if key not in _ENGINES:
        while len(_ENGINES) >= 3:
            _ENGINES.pop(next(iter(_ENGINES)))[0].close()
        case = VLB_CASES[name]
        spec = NetSpec.from_net_kwargs(case["net_kwargs"])
        eng = DenoiserEngine(spec, case["N"], case["diffusion_kwargs"]["time_num"], precision=precision)
        eng.load_state_dict(seeded_state_dict(unet1d_param_specs(spec), seed=case["seed"]))
        eng.set_schedule(case_tables(case))
        _ENGINES[key] = (eng, case, spec, make_inputs(case, spec))
    eng, case, spec, inp = _ENGINES[key]
    # conditioning of the case's own batch (tests below may set another batch)
    shared = case.get("shared_context", True)
    eng.set_context(inp["context"][0] if shared else inp["context"], shared=shared)
    if spec.text_condition:
        eng.set_context_cross(inp["context_cross"])
    return eng, case, spec, inp


def _rel(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return float(np.max(np.abs(a - b) / np.maximum(np.abs(b), 1e-30)))


def _check_terms(vb, mse, g_vb, g_mse):
    np.testing.assert_allclose(vb[:, 1:], g_vb[:, 1:], **TOL)
    assert _rel(vb[:, 0], g_vb[:, 0]) < REL
    np.testing.assert_allclose(mse, g_mse, **TOL)


def _model(name):
    """DiffusionSceneLayout_DDPM (fp32) carrying the case's network, schedule and seeded weights."""
    from diffuscene_b200.networks.diffusion_scene_layout_ddpm import DiffusionSceneLayout_DDPM
    case = VLB_CASES[name]
    spec = NetSpec.from_net_kwargs(case["net_kwargs"])
    cfg = dict(case["net_cfg"], net_type="unet1d", room_mask_condition=False, net_kwargs=case["net_kwargs"],
               diffusion_kwargs=case["diffusion_kwargs"], point_dim=spec.point_dim, sample_num_points=case["N"],
               text_condition=spec.text_condition, text_embed_dim=spec.text_dim)
    net = DiffusionSceneLayout_DDPM(23, None, cfg, precision="fp32")
    net.load_state_dict(seeded_state_dict(unet1d_param_specs(spec), seed=case["seed"]), strict=False)
    return net.cuda()


@pytest.mark.parametrize("name", list(VLB_CASES))
def test_fp32_parity_with_reference(name, golden_dir):
    eng, case, spec, inp = _engine(name)
    g = gold(golden_dir, name)
    x0, noise = inp["x0"].cuda(), torch.from_numpy(g["noise"]).cuda()
    for clip in (0, 1):
        res = {}
        for use_graph in (True, False):
            res[use_graph] = [r.cpu() for r in eng.vlb(x0, clip_denoised=bool(clip), noise=noise, use_graph=use_graph)]
        for a, b in zip(res[True], res[False]):
            assert torch.equal(a, b)                  # graph replay == plain launches, bit for bit
        vb, mse, prior = [r.numpy() for r in res[True]]
        _check_terms(vb, mse, g["vb_clip%d" % clip], g["mse_clip%d" % clip])
        np.testing.assert_allclose(prior, g["prior"], **TOL)
        assert _rel((vb.sum(1) + prior).mean(), g["total_bpd_b_clip%d" % clip]) < REL
    # the drop-in surface: the reference's dict of four means, and prior_kl
    net = _model(name)
    cross = None if inp["context_cross"] is None else inp["context_cross"].cuda()
    for clip in (0, 1):
        d = net.diffusion.all_kl(x0, inp["context"].cuda(), cross, clip_denoised=bool(clip), noise=noise)
        assert sorted(d) == ["mse_bt", "prior_bpd_b", "terms_bpd", "total_bpd_b"]
        for k in ("total_bpd_b", "terms_bpd"):
            assert d[k].dim() == 0 and _rel(float(d[k]), g["%s_clip%d" % (k, clip)]) < REL, k
        for k in ("prior_bpd_b", "mse_bt"):
            np.testing.assert_allclose(float(d[k]), float(g["%s_clip%d" % (k, clip)]), **TOL)
    np.testing.assert_allclose(net.diffusion.prior_kl(x0).cpu().numpy(), g["prior"], **TOL)
    net._engine.close()


# bf16 (wgmma tensor cores, bf16 activations) against fp32 on 256 scenes, same injected draws: t >= 1 terms and mse
# relative to their batch-mean magnitude at that t, t = 0 relative per scene.  Measured on an H100: 1.43e-4, 1.43e-4
# and 1.14e-4 (DESIGN.md section 4); the bounds leave a margin of about 14x.
BF16_T1_BOUND = 2e-3
BF16_MSE_BOUND = 2e-3
BF16_T0_BOUND = 2e-3


def _bf16_errors(B=256):
    name = "vlb_bed62"
    out = {}
    g = torch.Generator().manual_seed(5)
    case = VLB_CASES[name]
    spec = NetSpec.from_net_kwargs(case["net_kwargs"])
    x0 = _clean_scene(g, B, case["N"], spec).cuda()
    T = case["diffusion_kwargs"]["time_num"]
    noise = torch.randn(T, B, case["N"], spec.point_dim, generator=g).cuda()
    for prec in ("fp32", "bf16"):
        eng, _, _, inp = _engine(name, prec)
        out[prec] = [r.cpu().double() for r in eng.vlb(x0, noise=noise)]
    (vb32, mse32, p32), (vb16, mse16, p16) = out["fp32"], out["bf16"]
    t1 = ((vb16[:, 1:] - vb32[:, 1:]).abs() / vb32[:, 1:].abs().mean(dim=0)).max().item()
    ms = ((mse16 - mse32).abs() / mse32.abs().mean(dim=0)).max().item()
    t0 = ((vb16[:, 0] - vb32[:, 0]).abs() / vb32[:, 0].abs()).max().item()
    return dict(t1=t1, mse=ms, t0=t0, prior=(p16 - p32).abs().max().item(),
                finite=bool(torch.isfinite(vb16).all() and torch.isfinite(mse16).all()))


def test_bf16_against_fp32():
    e = _bf16_errors()
    print("bf16 vs fp32 VLB errors:", e)
    assert e["finite"]
    assert e["t1"] < BF16_T1_BOUND and e["mse"] < BF16_MSE_BOUND and e["t0"] < BF16_T0_BOUND, e
    assert e["prior"] == 0.0          # no denoiser in the prior: identical kernels on identical inputs


def test_philox_path():
    eng, case, spec, inp = _engine("vlb_bed62")
    g = torch.Generator().manual_seed(9)
    x0 = _clean_scene(g, 4, case["N"], spec).cuda()
    a = [r.cpu() for r in eng.vlb(x0, seed=7)]
    b = [r.cpu() for r in eng.vlb(x0, seed=7)]
    for u, v in zip(a, b):
        assert torch.equal(u, v)
    c = [r.cpu() for r in eng.vlb(x0, seed=8)]
    assert not torch.equal(a[0], c[0]) and not torch.equal(a[1], c[1])
    assert all(torch.isfinite(r).all() for r in a)
    # scenes 2, 3 run as their own shard reproduce their rows of the unsharded run
    s = [r.cpu() for r in eng.vlb(x0[2:], seed=7, scene_offset=2)]
    for u, v in zip(s, a):
        np.testing.assert_allclose(u.numpy(), v[2:].numpy(), rtol=1e-5, atol=1e-6)
    # the prior has no noise: the oracle's value
    dk = case["diffusion_kwargs"]
    sched = D.make_schedule(D.make_betas(dk["schedule_type"], dk["beta_start"], dk["beta_end"], dk["time_num"]),
                            dk["model_mean_type"], dk["model_var_type"])
    np.testing.assert_allclose(a[2].numpy(), V.prior_bpd(sched, x0.cpu()).numpy(), rtol=1e-5, atol=1e-6)
    _, _, p = eng.vlb(x0, prior_only=True)
    assert torch.equal(p.cpu(), a[2])


@pytest.mark.parametrize("name", ["vlb_bed62", "vlb_text62"])
def test_batch_independence(name, golden_dir):
    eng, case, spec, inp = _engine(name)
    noise = torch.from_numpy(gold(golden_dir, name)["noise"]).cuda()
    full = [r.cpu() for r in eng.vlb(inp["x0"].cuda(), noise=noise)]
    if spec.text_condition:
        eng.set_context_cross(inp["context_cross"][1:2])
    one = [r.cpu() for r in eng.vlb(inp["x0"][1:2].cuda(), noise=noise[:, 1:2])]
    for u, v in zip(one, full):
        np.testing.assert_allclose(u.numpy(), v[1:2].numpy(), rtol=1e-5, atol=1e-6)


def test_vlb_does_not_disturb_the_sampling_graph():
    eng, case, spec, inp = _engine("vlb_bed62")
    B = case["B"]
    s1 = eng.sample(B, seed=3)
    n1 = eng.graph_build_count()
    eng.vlb(inp["x0"].cuda(), seed=4)
    eng.vlb(inp["x0"].cuda(), seed=4, use_graph=False)
    assert eng.graph_build_count() == n1
    s2 = eng.sample(B, seed=3)
    assert eng.graph_build_count() == n1
    assert torch.equal(s1, s2)


def _code(fn):
    with pytest.raises(capi.DsError) as e:
        fn()
    return e.value.code


def test_argument_and_state_errors():
    eng, case, spec, inp = _engine("vlb_arr5")         # per-scene context of batch 2
    lib, B, T = eng.lib, case["B"], case["diffusion_kwargs"]["time_num"]
    x0 = inp["x0"].cuda()
    vb, mse, prior = (torch.empty(B, T, device="cuda"), torch.empty(B, T, device="cuda"), torch.empty(B, device="cuda"))
    p = lambda t: C.c_void_p(t.data_ptr())

    def call(x0_ptr, vb_ptr, mse_ptr, prior_ptr, batch=B):
        a = capi.DsVlbArgs()
        a.batch, a.clip_denoised, a.x0_dev, a.use_graph = batch, 1, x0_ptr, 1
        return lambda: capi.check(lib.ds_vlb_loop(eng.h, C.byref(a), vb_ptr, mse_ptr, prior_ptr, None))

    assert _code(call(None, p(vb), p(mse), p(prior))) == capi_invalid()
    assert _code(call(x0.data_ptr(), p(vb), p(mse), None)) == capi_invalid()
    assert _code(call(x0.data_ptr(), p(vb), None, p(prior))) == capi_invalid()
    assert _code(call(x0.data_ptr(), p(vb), p(mse), p(prior), batch=0)) == capi_invalid()
    assert _code(lambda: eng.vlb(torch.cat([inp["x0"], inp["x0"][:1]]).cuda())) == capi_state()   # context batch 2
    call(x0.data_ptr(), p(vb), p(mse), p(prior))()                                                   # and it runs
    assert _code(lambda: capi.check(lib.ds_set_vlb_schedule(eng.h, T + 1, p(prior), p(prior), p(prior)))) == capi_invalid()
    assert _code(lambda: capi.check(lib.ds_set_vlb_schedule(eng.h, T, None, None, None))) == capi_invalid()
    # a fresh handle: no schedule, then a schedule without the VLB tables
    fresh = DenoiserEngine(spec, case["N"], T, precision="fp32")
    try:
        fresh.load_state_dict(seeded_state_dict(unet1d_param_specs(spec), seed=case["seed"]))
        fresh.set_context(inp["context"], shared=False)
        assert _code(lambda: fresh.vlb(x0)) == capi_state()
        tb = case_tables(case)
        s = capi.DsSchedule()
        s.T, s.mean_type = T, capi.MEAN_TYPES[tb.mean_type]
        keep = []
        for f in ("sqrt_ac", "sqrt_1mac", "sqrt_recip_ac", "sqrt_recipm1_ac", "coef1", "coef2", "sigma",
                  "alphas_cumprod", "loss_weight"):
            keep.append(tb[f].contiguous())
            setattr(s, f, C.cast(C.c_void_p(keep[-1].data_ptr()), C.POINTER(C.c_float)))
        capi.check(fresh.lib.ds_set_schedule(fresh.h, C.byref(s)))
        assert _code(lambda: fresh.vlb(x0)) == capi_state()
        assert _code(lambda: fresh.vlb(x0, prior_only=True)) == capi_state()
        fresh.set_schedule(tb)
        fresh.vlb(x0)
    finally:
        fresh.close()


def capi_invalid():
    return -1       # DS_ERR_INVALID


def capi_state():
    return -4       # DS_ERR_STATE
