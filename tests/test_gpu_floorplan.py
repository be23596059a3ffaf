"""GPU: the native floor-plan encoder (ds_room_enc_*) and the floor-plan model class.  The trunk in fp32 against the
functional restatement (functional.room_trunk) and the reference goldens, every trunk parameter gradient against
torch autograd of the restatement on binary masks (max-pool ties included), bf16 against fp32, batch independence,
the class-level get_loss / sample / train_on_batch against goldens and the autograd twin, and the ABI's errors."""
import ctypes as C

import numpy as np
import pytest
import torch

from tests.cases_floorplan import FP_CASES, TRUNK, class_config, fp_batch, fp_masks, fp_state_dict, trunk_value

pytestmark = pytest.mark.gpu
RTOL, ATOL = 1e-3, 1e-4
GRAD_REL = 1e-4


def _trunk(seed, device="cuda"):
    from diffuscene_b200.room_encoder import trunk_specs
    t = {n: trunk_value(n, shape, seed).to(device) for n, shape, _ in trunk_specs(1)}
    flat = torch.cat([v.reshape(-1) for v in t.values()]).contiguous()
    return t, flat


def _binary_masks(B, seed):
    g = torch.Generator().manual_seed(seed)
    from diffuscene_b200.synthetic import floor_plan_mask
    return torch.stack([floor_plan_mask(g) for _ in range(B)]).cuda()


def _ref_trunk(t, mask):
    from diffuscene_b200.networks.functional import room_trunk
    return room_trunk(t, mask)


@pytest.fixture
def fp32_twin():
    """The autograd twin's convolutions and GEMMs in true fp32 (no TF32) for one test, settings restored after."""
    saved = torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
    yield
    torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = saved


def test_expected_weights_match_python_layout():
    from diffuscene_b200.room_encoder import RoomMaskEncoder, trunk_specs
    enc = RoomMaskEncoder(1, 64, 64, precision="fp32")
    exp = enc.expected_weights()
    assert [n for n, _ in exp] == [n for n, _, _ in trunk_specs(1)]
    assert [k for _, k in exp] == [int(np.prod(s)) for _, s, _ in trunk_specs(1)]
    assert len(exp) == 100
    enc.close()


@pytest.mark.parametrize("B", [3, 1003])
def test_fp32_trunk_matches_restatement(B, golden_dir, fp32_twin):
    from diffuscene_b200.room_encoder import RoomMaskEncoder
    t, flat = _trunk(41)
    mask = fp_masks(B).cuda() if B == 3 else _binary_masks(B, 5)
    enc = RoomMaskEncoder(1, 64, 64, precision="fp32")
    out = enc.forward(flat, mask)
    with torch.no_grad():
        ref = _ref_trunk(t, mask)
    torch.testing.assert_close(out, ref, rtol=RTOL, atol=ATOL)
    if B == 3:      # the golden trunk of the same weights and masks (fp_bed: seed 41, B = 4)
        g = np.load("%s/fp_bed.npz" % golden_dir)
        np.testing.assert_allclose(out.cpu().numpy(), g["trunk"][:3], rtol=RTOL, atol=ATOL)
    enc.close()


def _native_and_ref_grads(precision, B, seed):
    from diffuscene_b200.room_encoder import RoomMaskEncoder, trunk_specs
    t, flat = _trunk(seed)
    mask = _binary_masks(B, seed)
    probe = torch.randn(B, 512, generator=torch.Generator().manual_seed(seed)).cuda()
    enc = RoomMaskEncoder(1, 64, 64, precision=precision)
    feat = enc.forward(flat, mask, keep=True)
    grads = torch.full_like(flat, float("nan"))
    enc.backward(probe, grads)
    tr = {k: v.clone().requires_grad_(not k.endswith(("running_mean", "running_var"))) for k, v in t.items()}
    ref = _ref_trunk(tr, mask)
    (ref * probe).sum().backward()
    out, off = {}, 0
    for name, shape, is_buf in trunk_specs(1):
        n = int(np.prod(shape))
        g = grads[off:off + n].view(shape)
        off += n
        if is_buf:
            assert torch.count_nonzero(g) == 0, name
        else:
            out[name] = (g, tr[name].grad)
    enc.close()
    return feat, ref.detach(), out


def test_fp32_gradients_match_autograd_on_binary_masks(fp32_twin):
    feat, ref, grads = _native_and_ref_grads("fp32", 8, 11)
    torch.testing.assert_close(feat, ref, rtol=RTOL, atol=ATOL)
    worst, worst_name = 0.0, None
    for name, (g, r) in grads.items():
        rel = ((g - r).norm() / r.norm().clamp_min(1e-30)).item()
        if rel > worst:
            worst, worst_name = rel, name
    print("fp32 trunk gradients: worst relative error %.3g (%s)" % (worst, worst_name))
    assert worst <= GRAD_REL, (worst_name, worst)


def test_bf16_against_fp32(fp32_twin):
    f32, _, g32 = _native_and_ref_grads("fp32", 16, 12)
    bf, _, gbf = _native_and_ref_grads("bf16", 16, 12)
    fe = ((bf - f32).norm() / f32.norm()).item()
    ge, gk = max((((gbf[k][0] - g32[k][0]).norm() / g32[k][0].norm().clamp_min(1e-30)).item(), k) for k in g32)
    print("bf16 vs fp32: features %.3g, worst gradient tensor %.3g (%s) (relative norms)" % (fe, ge, gk))
    assert fe < 3e-2 and ge < 3.5e-1      # measured on an H100: 4.4e-3 and 1.8e-1


@pytest.mark.parametrize("precision", ["fp32", "bf16"])
def test_features_independent_of_batch(precision):
    from diffuscene_b200.room_encoder import RoomMaskEncoder
    _, flat = _trunk(13)
    masks = _binary_masks(257, 13)
    enc = RoomMaskEncoder(1, 64, 64, precision=precision)
    full = enc.forward(flat, masks).clone()
    for i in (0, 100, 256):
        one = enc.forward(flat, masks[i:i + 1])
        assert torch.equal(one[0], full[i]), i
    enc.close()


def test_abi_errors():
    from diffuscene_b200 import capi
    lib = capi.load()
    h = C.c_void_p()
    for prec, cin, H, W in [(0, 0, 64, 64), (0, 9, 64, 64), (0, 1, 48, 64), (0, 1, 64, 16), (1, 1, 0, 64)]:
        cfg = capi.DsRoomEncConfig(precision=prec, input_channels=cin, height=H, width=W, device=0)
        assert lib.ds_room_enc_create(C.byref(cfg), C.byref(h)) == -1
    cfg = capi.DsRoomEncConfig(precision=0, input_channels=1, height=64, width=64, device=0)
    assert lib.ds_room_enc_create(None, C.byref(h)) == -1
    assert lib.ds_room_enc_create(C.byref(cfg), C.byref(h)) == 0
    buf = torch.zeros(4096, device="cuda")
    p = C.c_void_p(buf.data_ptr())
    assert lib.ds_room_enc_backward(h, p, p, None) == -1          # no kept forward
    assert b"keep_for_backward" in lib.ds_last_error()
    assert lib.ds_room_enc_forward(h, None, p, 1, p, 0, None) == -1
    assert lib.ds_room_enc_forward(h, p, p, 0, p, 0, None) == -1
    assert lib.ds_room_enc_backward(h, None, p, None) == -1
    assert lib.ds_room_enc_expected_weight(h, 100, None, None) == -1
    assert lib.ds_room_enc_destroy(h) == 0


# ---- the model class --------------------------------------------------------------------------------------
def _net(name, tmp_path, precision="fp32"):
    from scene_synthesis.networks import build_network
    case = FP_CASES[name]
    cfg = class_config(case, str(tmp_path / "stats.json"))
    net, train_on_batch, _ = build_network(30, case["n_classes"], cfg, None, device="cuda", precision=precision)
    net.load_state_dict(fp_state_dict(net.state_dict(), case["seed"]), strict=True)
    return net, case, cfg, train_on_batch


def _sp(case):
    return {k: (v.cuda() if torch.is_tensor(v) else v) for k, v in fp_batch(case).items()}


@pytest.mark.parametrize("name", list(FP_CASES))
def test_class_get_loss_and_sample_match_reference(name, tmp_path, golden_dir):
    net, case, _, _ = _net(name, tmp_path)
    g = np.load("%s/%s.npz" % (golden_dir, name))
    sp = _sp(case)
    t, noise = torch.from_numpy(g["loss_t"]), torch.from_numpy(g["loss_noise"])
    with torch.no_grad():
        loss, ld = net.get_loss(sp, t=t, noise=noise)
    np.testing.assert_allclose(float(loss), float(g["loss"]), rtol=RTOL, atol=ATOL)
    for k in [k[3:] for k in g.files if k.startswith("ld.")]:
        np.testing.assert_allclose(float(ld[k]), float(g["ld." + k]), rtol=RTOL, atol=ATOL, err_msg=k)
    B, N = case["B"], case["N"]
    draws = torch.from_numpy(g["sample_draws"])
    kw = dict(clip_denoised=True, x_init=draws[0], noise=draws[1:])
    room = sp["room_layout"]
    if case["kind"] == "partial":
        out = net.sample(room, N, 62, batch_size=B, partial_boxes=torch.from_numpy(g["partial_boxes"]).cuda(),
                         partial_noise=torch.from_numpy(g["sample_draws_partial"]), **kw)
    else:
        out = net.sample(room, N, 62, batch_size=B, **kw)
    # get_loss ran first on the same model: sample() must not read a condition the encoder is still computing
    np.testing.assert_allclose(out.cpu().numpy(), g["sample"], rtol=RTOL, atol=5 * ATOL)
    with pytest.raises(ValueError):
        net.sample(room[:1], N, 62, batch_size=B)


@pytest.mark.parametrize("name", list(FP_CASES))
def test_class_training_gradients_match_autograd_twin(name, tmp_path, golden_dir, fp32_twin):
    net, case, _, _ = _net(name, tmp_path)
    g = np.load("%s/%s.npz" % (golden_dir, name))
    sp = _sp(case)
    t, noise = torch.from_numpy(g["loss_t"]), torch.from_numpy(g["loss_noise"])
    grads = {}
    for native in (True, False):
        net.native_backward = native
        net.zero_grad(set_to_none=True)
        loss, _ = net.get_loss(sp, t=t, noise=noise)
        loss.backward()
        np.testing.assert_allclose(float(loss), float(g["loss"]), rtol=RTOL, atol=ATOL)
        grads[native] = {k: p.grad.detach().clone() for k, p in net.named_parameters()
                         if k.startswith(("feature_extractor.", "fc_room_f."))}
    assert len(grads[True]) == 66
    worst = max(((grads[True][k] - grads[False][k]).norm() / grads[False][k].norm().clamp_min(1e-30)).item()
                for k in grads[False])
    print("%s: class-level floor-plan gradients, worst relative error %.3g" % (name, worst))
    assert worst < 2e-3


def test_gradients_accumulate_over_backward_passes_like_the_twin(tmp_path, fp32_twin):
    """Two backward passes into existing .grad tensors (zero_grad(set_to_none=False) between steps, then gradient
    accumulation): the trunk gradients must be the twin's, not aliases of the encoder's reused gradient buffer."""
    net, case, _, _ = _net("fp_bed", tmp_path)
    sp = _sp(case)
    B = case["B"]
    t = torch.randint(0, case["T"], (B,), generator=torch.Generator().manual_seed(0))
    noise = torch.randn(B, case["N"], 62, generator=torch.Generator().manual_seed(1))
    sp2 = dict(sp, room_layout=sp["room_layout"].flip(0).contiguous())
    res = {}
    for native in (True, False):
        net.native_backward = native
        net.zero_grad(set_to_none=True)
        out = []
        for batch in (sp, sp2):           # step: zero in place, one backward
            if out:
                net.zero_grad(set_to_none=False)
            loss, _ = net.get_loss(batch, t=t, noise=noise)
            loss.backward()
            out.append({k: p.grad.detach().clone() for k, p in net.named_parameters() if k.startswith(TRUNK)})
        loss, _ = net.get_loss(sp, t=t, noise=noise)      # accumulate a third backward onto the second
        loss.backward()
        out.append({k: p.grad.detach().clone() for k, p in net.named_parameters() if k.startswith(TRUNK)})
        res[native] = out
    for i in range(3):
        for k, ref in res[False][i].items():
            err = ((res[True][i][k] - ref).norm() / ref.norm().clamp_min(1e-30)).item()
            assert err < 2e-3, (i, k, err)


def test_train_on_batch_matches_autograd_twin_and_round_trips(tmp_path, fp32_twin):
    from diffuscene_b200.networks import optimizer_factory
    from diffuscene_b200.stats_logger import StatsLogger
    nets = []
    for native in (True, False):
        torch.manual_seed(0)
        net, case, cfg, train_on_batch = _net("fp_bed", tmp_path)
        net.native_backward = native
        opt = optimizer_factory(cfg["training"], net.parameters())
        sp = _sp(case)
        StatsLogger.instance()
        for step in range(2):
            torch.manual_seed(100 + step)
            train_on_batch(net, opt, sp, cfg)
        nets.append(net)
    a, b = nets[0].state_dict(), nets[1].state_dict()
    worst = max(((a[k] - b[k]).norm() / b[k].norm().clamp_min(1e-30)).item() for k in a
                if k.startswith(("feature_extractor.", "fc_room_f.")))
    print("train_on_batch: floor-plan parameters after 2 steps, worst relative difference %.3g" % worst)
    assert worst < 1e-3
    # state-dict round trip, strict, into a fresh model: the same features
    fresh, case, _, _ = _net("fp_bed", tmp_path)
    fresh.load_state_dict(a, strict=True)
    room = fp_masks(4).cuda()
    with torch.no_grad():
        torch.testing.assert_close(fresh._room_features(room), nets[0]._room_features(room), rtol=0, atol=0)
