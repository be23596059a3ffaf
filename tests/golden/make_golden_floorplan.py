"""Floor-plan golden vectors: the UNMODIFIED reference `DiffusionSceneLayout_DDPM` with room_mask_condition and its
ResNet-18 feature extractor (build_network's construction, networks/__init__.py:50-55; feature_extractors.py:19-47,
frozen BatchNorm) run on CPU / fp32.

Run in the authoring container only (needs the reference checkout and torchvision):
    python tests/golden/make_golden_floorplan.py
Writes tests/golden/fp_*.npz: the state-dict key list, the trunk output [B, 512] and feature_extractor(room_layout),
get_loss and its dict (with the recorded t / noise draws), the gradients of that loss for every floor-plan parameter
(norm and dot product with a seeded probe; BatchNorm, conv1 and fc_room_f in full), and one short sampling loop.
Randomness and weights follow make_golden_class.py.
"""
import contextlib
import io
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
from tests.golden.make_golden_class import Recorder   # noqa: E402  (also puts the reference on sys.path)
from tests.cases_floorplan import FP_CASES, TRUNK, class_config, fp_batch, fp_state_dict, full_grad, probe  # noqa: E402


def build_reference(case):
    from scene_synthesis.networks.diffusion_scene_layout_ddpm import DiffusionSceneLayout_DDPM
    from scene_synthesis.networks.feature_extractors import get_feature_extractor
    cfg = class_config(case, "/tmp/ds_b200_fp_stats.json")
    fe = cfg["feature_extractor"]
    with contextlib.redirect_stdout(io.StringIO()):
        net = DiffusionSceneLayout_DDPM(case["n_classes"], get_feature_extractor(
            fe.get("name", "resnet18"), freeze_bn=fe.get("freeze_bn", True),
            input_channels=fe.get("input_channels", 1), feature_size=fe.get("feature_size", 256)), cfg["network"])
    net.load_state_dict(fp_state_dict(net.state_dict(), case["seed"]), strict=True)
    net.eval()
    return net


def main():
    torch.manual_seed(0)
    quiet = lambda: contextlib.redirect_stdout(io.StringIO())
    for name, case in FP_CASES.items():
        net = build_reference(case)
        out = {"keys": np.array(list(net.state_dict().keys()))}
        B, N, d = case["B"], case["N"], case["point_dim"]
        sp = fp_batch(case)
        room = sp["room_layout"]
        fe = net.feature_extractor._feature_extractor
        pooled = []
        hook = fe.avgpool.register_forward_hook(lambda m, i, o: pooled.append(o.flatten(1).detach().clone()))
        with torch.no_grad():
            out["feat"] = net.feature_extractor(room).numpy()
        hook.remove()
        out["trunk"] = pooled[0].numpy()
        out["room_layout"] = room.numpy()
        # ---- get_loss and its gradients ------------------------------------------------------------------
        net.zero_grad(set_to_none=True)
        with Recorder(case["seed"] + 1) as r, quiet():
            loss, ld = net.get_loss(sp)
        loss.backward()
        out["loss"] = np.asarray(loss.detach().numpy())
        for k, v in ld.items():
            out["ld." + k] = np.asarray(v.detach().numpy())
        out["loss_t"] = r.randint_draws[0].numpy()
        out["loss_noise"] = r.randn_draws[0].numpy()
        for k, p in net.named_parameters():
            if not k.startswith(("feature_extractor.", "fc_room_f.")):
                continue
            g = p.grad.detach()
            out["gnorm." + k] = np.asarray(g.norm().item(), np.float64)
            out["gdot." + k] = np.asarray((g.double() * probe(k, g.shape).double()).sum().item(), np.float64)
            if full_grad(k):
                out["grad." + k] = g.numpy()
        # ---- one short sampling loop ---------------------------------------------------------------------
        with torch.no_grad():
            if case["kind"] == "partial":
                full = torch.cat([sp["translations"], sp["sizes"], sp["angles"], sp["class_labels"], sp["objfeats_32"]], -1)
                partial = full[:, :case["partial_num_points"]].contiguous()
                with Recorder(case["seed"] + 2) as r, quiet():
                    s = net.sample(room, N, d, batch_size=B, partial_boxes=partial, clip_denoised=True)
                out["partial_boxes"] = partial.numpy()
                out["sample_draws_partial"] = np.stack([a.numpy() for a in r.randn_draws[1:]
                                                        if a.shape[1] == case["partial_num_points"]])
            else:
                with Recorder(case["seed"] + 2) as r, quiet():
                    s = net.sample(room, N, d, batch_size=B, clip_denoised=True)
        out["sample"] = s.numpy()
        out["sample_draws"] = np.stack([a.numpy() for a in r.randn_draws[1:] if tuple(a.shape) == (B, N, d)])
        np.savez(os.path.join(HERE, name + ".npz"), **out)
        print(name, len(out["keys"]), "keys;", {k: getattr(v, "shape", None) for k, v in out.items()
                                                if not k.startswith(("gnorm", "gdot", "grad"))})


if __name__ == "__main__":
    main()
