"""Synthetic stand-in for the reference's data layer (3D-FRONT is licensed and absent here).

Produces the `sample_params` contract of `Diffusion.__getitem__` after `Scale_CosinAngle_ObjfeatsNorm`
(reference scene_synthesis/datasets/threed_front_dataset.py:481-513, 888-925; SURVEY.md A.4) and its inverse
`post_process` (:515-535): +-1 class one-hots whose last channel is the 'empty' slot, translations / sizes /
objfeats in [-1, 1], angles as (cos, sin), and a room layout: a seeded binary floor plan (rectangle or L-shape) for
networks with room_mask_condition, zeros otherwise.
"""
from __future__ import annotations

import json

import numpy as np
import torch
from torch.utils.data import Dataset

DEFAULT_BOUNDS = {
    "translations": (np.array([-2.7, 0.04, -2.75], np.float32), np.array([2.8, 3.6, 2.9], np.float32)),
    "sizes": (np.array([0.04, 0.02, 0.01], np.float32), np.array([2.9, 1.8, 2.6], np.float32)),
    "angles": (np.array([-3.14159], np.float32), np.array([3.14159], np.float32)),
    "objfeats_32": (np.array([1.0], np.float32), np.array([-4.0], np.float32), np.array([4.0], np.float32)),
}


def write_stats_file(path, bounds=DEFAULT_BOUNDS):
    """The `train_stats_file` JSON that loss_iou reads (reference diffusion_ddpm.py:137-151)."""
    with open(path, "w") as f:
        json.dump({"bounds_translations": [float(v) for v in np.concatenate(bounds["translations"])],
                   "bounds_sizes": [float(v) for v in np.concatenate(bounds["sizes"])],
                   "bounds_angles": [float(bounds["angles"][0][0]), float(bounds["angles"][1][0])]}, f)
    return path


def floor_plan_mask(g: torch.Generator, size: int = 64) -> torch.Tensor:
    """A binary floor plan [1, size, size]: an axis-aligned rectangular room, half of the time with one corner cut
    away (an L-shape)."""
    r = lambda lo, hi: int(torch.randint(lo, hi, (1,), generator=g))
    y0, x0 = r(1, size // 3), r(1, size // 3)
    y1, x1 = r(2 * size // 3, size), r(2 * size // 3, size)
    m = torch.zeros(1, size, size)
    m[:, y0:y1, x0:x1] = 1.0
    if r(0, 2):
        cy, cx = r(y0 + 2, y1 - 1), r(x0 + 2, x1 - 1)
        ys = slice(y0, cy) if r(0, 2) else slice(cy, y1)
        xs = slice(x0, cx) if r(0, 2) else slice(cx, x1)
        m[:, ys, xs] = 0.0
    return m


class SyntheticScenes(Dataset):
    def __init__(self, net_cfg: dict, length: int = 4096, seed: int = 0, bounds=DEFAULT_BOUNDS):
        self.N = net_cfg.get("sample_num_points", 12)
        self.class_dim = net_cfg.get("class_dim", 21)
        self.angle_dim = net_cfg.get("angle_dim", 1)
        self.objfeat_dim = net_cfg.get("objfeat_dim", 0)
        self.objectness_dim = net_cfg.get("objectness_dim", 1)
        self.room_mask = net_cfg.get("room_mask_condition", True)
        self.length, self.seed, self.bounds = length, seed, bounds
        self.n_classes = self.class_dim + 1      # + start token, as the reference counts them
        self.feature_size = 8 + self.class_dim

    def __len__(self):
        return self.length

    def __getitem__(self, idx):
        g = torch.Generator().manual_seed(self.seed * 1000003 + idx)
        N = self.N
        n_real = int(torch.randint(2, N + 1, (1,), generator=g))
        cls = torch.randint(0, self.class_dim - 1, (N,), generator=g)
        cls[n_real:] = self.class_dim - 1                                   # padded slots carry the 'empty' class
        onehot = torch.nn.functional.one_hot(cls, self.class_dim).float() * 2 - 1
        real = (torch.arange(N) < n_real).float()[:, None]
        tr = (torch.rand(N, 3, generator=g) * 2 - 1) * real
        sz = (torch.rand(N, 3, generator=g) * 2 - 1) * real
        th = (torch.rand(N, 1, generator=g) * 2 - 1) * 3.14159
        if self.angle_dim == 2:
            ang = torch.cat([torch.cos(th), torch.sin(th)], dim=-1) * real
        else:
            ang = th.expand(N, self.angle_dim) / 3.14159 * real
        out = {"class_labels": onehot, "translations": tr, "sizes": sz, "angles": ang,
               "room_layout": torch.zeros(1, 64, 64), "length": n_real}
        if self.room_mask:      # a generator of its own: the other fields do not depend on whether masks are drawn
            out["room_layout"] = floor_plan_mask(torch.Generator().manual_seed(self.seed * 1000003 + idx + (1 << 40)))
        if self.objfeat_dim > 0:
            key = "objfeats_32" if self.objfeat_dim == 32 else "objfeats"
            out[key] = (torch.rand(N, self.objfeat_dim, generator=g) * 2 - 1) * real
        if self.objectness_dim > 0:
            out["objectness"] = 1 - 2 * real
        return out

    @staticmethod
    def descale(x, lo, hi):
        return (x + 1) / 2 * (hi - lo) + lo

    def post_process(self, s: dict) -> dict:
        """Inverse scaling of network samples (numpy arrays [B, n, k]); angles -> atan2(sin, cos)."""
        out = {}
        for k, v in s.items():
            v = np.asarray(v)
            if k in ("class_labels", "room_layout", "description", "desc_emb"):
                out[k] = v
            elif k == "angles":
                out[k] = np.arctan2(v[:, :, 1:2], v[:, :, 0:1]) if v.shape[-1] == 2 else v * 3.14159
            elif k in ("objfeats", "objfeats_32"):
                b = self.bounds["objfeats_32"]
                out[k] = self.descale(v, b[1], b[2])
            else:
                out[k] = self.descale(v, self.bounds[k][0], self.bounds[k][1])
        return out


class SyntheticShapes(Dataset):
    """Stand-in for the reference's object point-cloud dataset (threed_future_dataset.py:100-120, 3D-FUTURE is licensed
    and absent here): seeded boxes and ellipsoids with random proportions, surface-sampled densely, centred and scaled
    into the unit sphere, from which `num_points` points are drawn WITH replacement as the reference does, so a cloud
    holds exact duplicate points.  Items are {"points": [P, 3] fp32, "label": int, "size": [3] fp32}."""

    N_DENSE = 4096

    def __init__(self, length: int = 1024, num_points: int = 2048, seed: int = 0, n_classes: int = 2):
        self.length, self.num_points, self.seed, self.n_classes = length, num_points, seed, n_classes

    def __len__(self):
        return self.length

    def __getitem__(self, i):
        g = torch.Generator().manual_seed(self.seed * 1000003 + i)
        label = int(torch.randint(0, self.n_classes, (1,), generator=g))
        half = 0.2 + torch.rand(3, generator=g)
        u = torch.randn(self.N_DENSE, 3, generator=g)
        if label % 2 == 0:      # box: project onto the face of the largest normalised coordinate
            u = u / u.abs().amax(dim=1, keepdim=True)
        else:                   # ellipsoid
            u = u / u.norm(dim=1, keepdim=True)
        dense = u * half
        dense = dense - dense.mean(dim=0)
        dense = dense / dense.norm(dim=1).max()
        pick = torch.randint(0, self.N_DENSE, (self.num_points,), generator=g)
        return {"points": dense[pick].float().contiguous(), "label": label, "size": (2 * half).float()}


def write_reference_rooms(dataset_directory: str, annotation_file: str, n_rooms: int, max_objects: int = 12,
                          n_object_classes: int = 21, layout_size: int = 256, seed: int = 0,
                          splits=("train", "val", "test")) -> list:
    """Seeded rooms in the reference's preprocessed format, for tests and benchmarks of diffuscene_b200.scene_data:
    <dataset_directory>/<scene>_<room>/boxes.npz (class_labels one-hot over classes + start + end, translations,
    sizes, angles, objfeats [L, 64], objfeats_32 [L, 32], a [layout_size, layout_size, 1] uint8 room_layout), the
    dataset_stats.txt JSON and the splits CSV `annotation_file` (room id, split; room i takes splits[i % len]).
    Some values fall outside the stats' bounds, so scaling clips them.  Returns the room tags in sorted order."""
    import os
    rng = np.random.default_rng(seed)
    os.makedirs(dataset_directory, exist_ok=True)
    n_cols = n_object_classes + 2
    labels = ["class%02d" % c for c in range(n_object_classes)] + ["start", "end"]
    b = DEFAULT_BOUNDS
    stats = {"bounds_translations": [float(v) for v in np.concatenate(b["translations"])],
             "bounds_sizes": [float(v) for v in np.concatenate(b["sizes"])],
             "bounds_angles": [-3.141592653589793, 3.141592653589793],
             "bounds_objfeats": [1.25, -5.0, 5.0], "bounds_objfeats_32": [1.0, -4.0, 4.0],
             "class_labels": labels, "object_types": labels[:-2],
             "class_frequencies": {k: 1.0 / n_object_classes for k in labels[:-2]},
             "class_order": {k: i for i, k in enumerate(labels[:-2])}, "count_furniture": {k: 1 for k in labels[:-2]}}
    with open(os.path.join(dataset_directory, "dataset_stats.txt"), "w") as f:
        json.dump(stats, f)
    tags, rows = [], []
    g = torch.Generator().manual_seed(seed)
    for i in range(n_rooms):
        room = "Bedroom-%05d" % i
        tag = "%08x_%s" % (int(rng.integers(0, 2 ** 31)), room)
        L = int(rng.integers(1, max_objects + 1))
        onehot = np.zeros((L, n_cols), np.float32)
        onehot[np.arange(L), rng.integers(0, n_object_classes, L)] = 1
        lo_t, hi_t = b["translations"]
        lo_s, hi_s = b["sizes"]
        mask = floor_plan_mask(g, layout_size)[0].numpy()
        os.makedirs(os.path.join(dataset_directory, tag), exist_ok=True)
        np.savez_compressed(
            os.path.join(dataset_directory, tag, "boxes.npz"), scene_id=np.array(room), class_labels=onehot,
            translations=rng.uniform(lo_t * 1.1, hi_t * 1.1, (L, 3)).astype(np.float32),
            sizes=rng.uniform(lo_s * 0.5, hi_s * 1.05, (L, 3)).astype(np.float32),
            angles=rng.uniform(-np.pi, np.pi, (L, 1)).astype(np.float32),
            objfeats=rng.normal(0, 2.0, (L, 64)).astype(np.float32),
            objfeats_32=rng.normal(0, 1.6, (L, 32)).astype(np.float32),
            room_layout=(mask[:, :, None] * 255).astype(np.uint8),
            floor_plan_vertices=np.zeros((0, 3), np.float32), floor_plan_faces=np.zeros((0, 3), np.int32),
            floor_plan_centroid=np.zeros(3, np.float32))
        tags.append(tag)
        rows.append((room, splits[i % len(splits)]))
    with open(annotation_file, "w") as f:
        f.write("".join("%s,%s\n" % r for r in rows))
    return sorted(tags)
