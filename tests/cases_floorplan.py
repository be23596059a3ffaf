"""Seeded floor-plan parity cases (the reference's `DiffusionSceneLayout_DDPM` with room_mask_condition and its
ResNet-18 room-mask encoder), shared by tests/golden/make_golden_floorplan.py (runs the unmodified reference) and the
CPU / GPU tests.  Everything is a function of the case seed; only outputs are stored."""
from __future__ import annotations

import zlib

import torch

from tests.cases_class import class_batch, class_config, class_state_dict

TRUNK = "feature_extractor._feature_extractor."
FP_YAML = "floorplan/diffusion_bedrooms_instancond_lat32_v_floorplan.yaml"

FP_CASES = {
    # the floor-plan bedroom config, v-prediction, short schedule
    "fp_bed": dict(seed=41, B=4, N=12, point_dim=62, n_classes=23, kind="uncond", T=6, yaml=FP_YAML),
    # + the partial-scene condition after the room feature and fc_instance_condition
    "fp_part": dict(seed=42, B=4, N=12, point_dim=62, n_classes=23, kind="partial", T=5, partial_num_points=3,
                    yaml=FP_YAML,
                    override=dict(learnable_embedding=False, room_partial_condition=True, partial_num_points=3,
                                  partial_emb_dim=64),
                    net_override=dict(instanclass_dim=192)),
}


def fp_masks(B: int, size: int = 64) -> torch.Tensor:
    """[B, 1, size, size] binary floor plans, cycling: empty room, full room, rectangle, L-shape."""
    out = []
    for i in range(B):
        m = torch.zeros(1, size, size)
        kind = i % 4
        if kind == 1:
            m[:] = 1.0
        elif kind == 2:
            m[:, 9:51, 14:47] = 1.0
        elif kind == 3:
            m[:, 6:58, 5:55] = 1.0
            m[:, 6:30, 31:55] = 0.0
        out.append(m)
    return torch.stack(out)


def _gen(name: str, seed: int) -> torch.Generator:
    return torch.Generator().manual_seed(zlib.crc32(name.encode()) * 7 + seed)


def trunk_value(name: str, shape, seed: int) -> torch.Tensor:
    """Seeded value of one trunk tensor: fan-in scaled convs, BatchNorm statistics away from (0, 1)."""
    g = _gen(name, seed)
    if len(shape) == 4:
        fan_in = shape[1] * shape[2] * shape[3]
        return torch.randn(shape, generator=g) * (1.0 / fan_in) ** 0.5
    u = torch.rand(shape, generator=g)
    if name.endswith("running_var"):
        return 0.5 + u
    if name.endswith("running_mean"):
        return 0.2 * (u - 0.5)
    if name.endswith("weight"):
        return 0.8 + 0.4 * u
    return 0.2 * (u - 0.5)


def fp_state_dict(like_sd, seed):
    out = class_state_dict(like_sd, seed)
    for k, v in like_sd.items():
        if k.startswith(TRUNK) and not k.startswith(TRUNK + "fc."):
            out[k] = trunk_value(k[len(TRUNK):], tuple(v.shape), seed)
    return out


def fp_batch(case):
    sp = class_batch(case)
    sp["room_layout"] = fp_masks(case["B"])
    return sp


def probe(name: str, shape) -> torch.Tensor:
    """The seeded tensor each parameter gradient is projected on (gradients are stored as norm + this dot)."""
    return torch.randn(tuple(shape), generator=_gen("probe:" + name, 0))


def full_grad(name: str) -> bool:
    """Gradients stored in full: every BatchNorm weight and bias, conv1 and fc_room_f."""
    return (".bn" in name or "downsample.1" in name or name.startswith(TRUNK + "bn1") or
            name.startswith(TRUNK + "conv1") or name.startswith("fc_room_f"))


__all__ = ["FP_CASES", "TRUNK", "class_config", "fp_masks", "fp_state_dict", "fp_batch", "probe", "full_grad",
           "trunk_value"]
