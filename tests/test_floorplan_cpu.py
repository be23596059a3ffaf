"""CPU: the floor-plan model (room_mask_condition, ResNet-18 room-mask encoder) against goldens of the UNMODIFIED
reference (tests/golden/make_golden_floorplan.py).  On the CPU the model's autograd twin runs (native_backward =
False: functional.room_trunk + DenoiserFn): it must reproduce the reference's trunk output, feature_extractor output,
get_loss value and the gradients of every floor-plan parameter.  Also: the state-dict inventory, the configurations
that raise, and that the synthetic data of the existing configs is unchanged."""
import copy
import os

import numpy as np
import pytest
import torch
import yaml

from tests.cases_floorplan import FP_CASES, TRUNK, class_config, fp_batch, fp_state_dict, full_grad, probe

RTOL, ATOL = 2e-4, 2e-5
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _net(name, tmp_path):
    from scene_synthesis.networks import build_network
    case = FP_CASES[name]
    cfg = class_config(case, str(tmp_path / "stats.json"))
    net, _, _ = build_network(30, case["n_classes"], cfg, None, device="cpu", precision="fp32")
    net.load_state_dict(fp_state_dict(net.state_dict(), case["seed"]), strict=True)
    net.native_backward = False
    return net, case, cfg


@pytest.mark.parametrize("name", list(FP_CASES))
def test_state_dict_keys_match_reference(name, tmp_path, golden_dir):
    net, _, _ = _net(name, tmp_path)
    g = np.load("%s/%s.npz" % (golden_dir, name))
    assert sorted(net.state_dict().keys()) == sorted(str(k) for k in g["keys"])
    fp = [k for k in net.state_dict() if k.startswith(("feature_extractor.", "fc_room_f."))]
    assert len(fp) == 106
    from diffuscene_b200.room_encoder import trunk_specs
    trunk = [k[len(TRUNK):] for k in fp if k.startswith(TRUNK) and not k.startswith(TRUNK + "fc.")]
    assert trunk == [n for n, _, _ in trunk_specs(1)]      # the flat layout of ds_room_enc_expected_weight


@pytest.mark.parametrize("name", list(FP_CASES))
def test_trunk_and_feature_extractor_match_reference(name, tmp_path, golden_dir):
    from diffuscene_b200.networks.functional import room_trunk
    net, case, _ = _net(name, tmp_path)
    g = np.load("%s/%s.npz" % (golden_dir, name))
    room = torch.from_numpy(g["room_layout"])
    with torch.no_grad():
        trunk = room_trunk(net._room_tensors(), room)
        feat = net.feature_extractor._feature_extractor.fc(trunk)
    np.testing.assert_allclose(trunk.numpy(), g["trunk"], rtol=RTOL, atol=ATOL)
    np.testing.assert_allclose(feat.numpy(), g["feat"], rtol=RTOL, atol=ATOL)


@pytest.mark.parametrize("name", list(FP_CASES))
def test_get_loss_and_gradients_match_reference(name, tmp_path, golden_dir):
    net, case, _ = _net(name, tmp_path)
    g = np.load("%s/%s.npz" % (golden_dir, name))
    sp = fp_batch(case)
    loss, ld = net.get_loss(sp, t=torch.from_numpy(g["loss_t"]), noise=torch.from_numpy(g["loss_noise"]))
    np.testing.assert_allclose(float(loss), float(g["loss"]), rtol=RTOL, atol=ATOL)
    for k in [k[3:] for k in g.files if k.startswith("ld.")]:
        np.testing.assert_allclose(float(ld[k]), float(g["ld." + k]), rtol=RTOL, atol=ATOL, err_msg=k)
    loss.backward()
    n = 0
    for k, p in net.named_parameters():
        if not k.startswith(("feature_extractor.", "fc_room_f.")):
            continue
        n += 1
        gr = p.grad.detach()
        scale = float(g["gnorm." + k]) + 1e-12
        np.testing.assert_allclose(gr.norm().item(), float(g["gnorm." + k]), rtol=1e-3, atol=1e-9, err_msg=k)
        dot = (gr.double() * probe(k, gr.shape).double()).sum().item()
        # a unit-variance probe projects an error e to about |e|: this bounds the error at ~3e-3 of the gradient's norm
        assert abs(dot - float(g["gdot." + k])) <= 3e-3 * scale, k
        if full_grad(k):
            np.testing.assert_allclose(gr.numpy(), g["grad." + k], rtol=1e-3, atol=1e-5 * scale + 1e-9, err_msg=k)
    assert n == 66      # 20 convs + 40 BatchNorm affines, the fc head (4) and fc_room_f (2); buffers get none


def _cfg(tmp_path, **net_over):
    case = FP_CASES["fp_bed"]
    cfg = class_config(case, str(tmp_path / "stats.json"))
    cfg["network"].update(net_over)
    return case, cfg


@pytest.mark.parametrize("fe_over, net_over, match", [
    (dict(name="alexnet"), {}, "alexnet"),
    (dict(freeze_bn=False), {}, "freeze_bn"),
    ({}, dict(text_condition=True), "text_condition"),
])
def test_unsupported_floor_plan_configs_raise(tmp_path, fe_over, net_over, match):
    from scene_synthesis.networks import build_network
    case, cfg = _cfg(tmp_path, **net_over)
    cfg["feature_extractor"].update(fe_over)
    with pytest.raises(NotImplementedError, match=match):
        build_network(30, case["n_classes"], cfg, None, device="cpu", precision="fp32")


def test_sample_rejects_mask_batch_mismatch(tmp_path):
    net, case, _ = _net("fp_bed", tmp_path)
    with pytest.raises(ValueError, match="room_mask"):
        net.sample(torch.zeros(3, 1, 64, 64), 12, 62, batch_size=2)


def test_models_without_floor_plan_still_drop_its_keys(tmp_path):
    from scene_synthesis.networks import build_network
    case, cfg = _cfg(tmp_path, room_mask_condition=False, latent_dim=0)
    cfg["network"]["net_kwargs"]["context_dim"] = 0
    net, _, _ = build_network(30, case["n_classes"], cfg, None, device="cpu", precision="fp32")
    sd = net.state_dict()
    assert not any(k.startswith(("feature_extractor.", "fc_room_f.")) for k in sd)
    extra = dict(sd, **{"fc_room_f.weight": torch.zeros(64, 64), TRUNK + "conv1.weight": torch.zeros(64, 1, 7, 7)})
    net.load_state_dict(extra, strict=True)


def test_synthetic_data_of_existing_configs_unchanged():
    from diffuscene_b200.synthetic import SyntheticScenes
    for rel in ("uncond/diffusion_bedrooms_instancond_lat32_v.yaml", "uncond/diffusion_livingrooms_instancond_lat32_v.yaml",
                "rearrange/diffusion_bedrooms_instancond_lat32_v_rearrange.yaml",
                "text/diffusion_bedrooms_instancond_lat32_v_bert.yaml"):
        with open(os.path.join(ROOT, "config", rel)) as f:
            net_cfg = yaml.safe_load(f)["network"]
        assert net_cfg["room_mask_condition"] is False
        fp_cfg = dict(copy.deepcopy(net_cfg), room_mask_condition=True)
        a, b = SyntheticScenes(net_cfg, 8, seed=3), SyntheticScenes(fp_cfg, 8, seed=3)
        for i in range(8):
            x, y = a[i], b[i]
            assert torch.equal(x["room_layout"], torch.zeros(1, 64, 64))
            for k in x:
                if k != "room_layout":
                    assert (x[k] == y[k]) if not torch.is_tensor(x[k]) else torch.equal(x[k], y[k]), (rel, k)
            m = y["room_layout"]
            assert m.shape == (1, 64, 64) and set(m.unique().tolist()) == {0.0, 1.0}
