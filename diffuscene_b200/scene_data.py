"""Training data from the reference's preprocessed 3D-FRONT rooms, kept on the device.

The reference builds every training sample on the CPU, one scene at a time: `CachedThreedFront.get_room_params`
loads a compressed npz per item and epoch (scene_synthesis/datasets/threed_front.py:349-373), then a chain of numpy
decorators augments, scales, permutes and pads it (threed_front_dataset.py:313-584, 888-1071).  Here the rooms of a
split are read once into a packed store on the device (`SceneStore`), and one kernel, `ds_scene_batch`
(csrc/scene_batch.cu), builds a whole batch from per-scene draws.  `SceneLoader` iterates epochs and draws those
numbers on a seeded device generator.

Room selection follows `CachedThreedFront.__init__` and `CSVSplitsBuilder` (splits_builder.py): the split ids are the
first CSV column of the rows whose second column is one of the splits, and a room is a directory of the dataset whose
tag.split("_")[1] is one of those ids, taken in sorted tag order.  Only directories holding boxes.npz count, so an
entry without "_" in its name is skipped where the reference fails on it.

One known difference: the permutation moves every per-object key, the objfeats included.  The reference permutes the
objfeats only when "objfeats" is part of the encoding name (threed_front_dataset.py:1037-1042), so its living-room
encoding cached_diffusion_cosin_angle_wocm shuffles the boxes but leaves their shape latents in file order.
"""
from __future__ import annotations

import csv
import ctypes
import json
import math
import os
from typing import Dict, List, Optional, Sequence

import numpy as np
import torch

from . import capi
from .postprocess import load_dataset_stats

DEFAULT_ENCODING = "cached_diffusion_cosin_angle_objfeatsnorm_lat32_wocm"
DEFAULT_AUGMENTATIONS = ("fixed_rotations",)
DEFAULT_STATS = "dataset_stats.txt"
AUGMENTATIONS = {"fixed_rotations": capi.DS_SCENE_AUG_FIXED_ROTATION, "rotations": capi.DS_SCENE_AUG_ROTATION,
                 "jitter": capi.DS_SCENE_AUG_JITTER}
MIN_RAD, MAX_RAD = 0.174533, 5.06145        # RotationAugmentation's continuous range
MAX_SLOTS = 32                              # one lane per object in ds_scene_batch


def split_ids(annotation_file: str, splits: Sequence[str]) -> set:
    """Scene ids of `splits` in the reference's splits CSV (first column, where the second is a wanted split)."""
    with open(annotation_file, newline="") as f:
        rows = [r for r in csv.reader(f)]
    return {r[0] for r in rows if len(r) > 1 and r[1] in set(splits)}


def select_rooms(dataset_directory: str, ids) -> List[str]:
    """Sorted room tags whose second "_"-separated field is one of `ids` and that hold boxes.npz."""
    tags = []
    for tag in os.listdir(dataset_directory):
        parts = tag.split("_")
        if len(parts) > 1 and parts[1] in ids and os.path.isfile(os.path.join(dataset_directory, tag, "boxes.npz")):
            tags.append(tag)
    return sorted(tags)


def room_layout(s, size):
    """The reference's room mask (threed_front.py:311-319): room_layout[:, :, 0] resized with PIL bilinear, / 255.
    `size` is PIL's (width, height)."""
    from PIL import Image
    img = Image.fromarray(np.asarray(s["room_layout"])[:, :, 0])
    img = img.resize(size, resample=Image.BILINEAR)
    return np.asarray(img).astype(np.float32) / np.float32(255)


def parse_encoding(name: str, angle_dim: int):
    """(scaling, permute) of a cached diffusion encoding name, as dataset_encoding_factory (:942-1071) reads it."""
    if "text" in name:
        raise ValueError("encoding %r adds text (Add_Text needs GloVe and nltk); text configs train on synthetic "
                         "scenes only" % name)
    if "cached" not in name or "diffusion" not in name or "eval" in name or "wocm" not in name:
        raise ValueError("encoding %r is not a cached_diffusion_*_wocm[_no_prm] training encoding" % name)
    cosin = "cosin_angle" in name or "objfeatsnorm" in name
    scaling = capi.DS_SCENE_SCALE_COSIN_OBJFEATSNORM if cosin else capi.DS_SCENE_SCALE
    if angle_dim != (2 if cosin else 1):
        raise ValueError("encoding %r gives angle_dim %d, the network has %d" % (name, 2 if cosin else 1, angle_dim))
    return scaling, "wocm_no_prm" not in name


def parse_augmentations(names, layouts: bool) -> List[int]:
    """ds_scene_batch codes of the reference's augmentation names, in order."""
    names = list(names or [])
    out = []
    for n in names:
        if n not in AUGMENTATIONS:
            raise ValueError("unknown augmentation %r (known: %s)" % (n, ", ".join(sorted(AUGMENTATIONS))))
        if names.count(n) > 1:
            raise ValueError("augmentation %r is listed twice" % n)
        out.append(AUGMENTATIONS[n])
    if "rotations" in names and "fixed_rotations" in names:
        raise ValueError("rotations and fixed_rotations together are not supported")
    if layouts and "rotations" in names:
        raise ValueError("continuous rotations of room layouts are not supported; use fixed_rotations")
    return out


def fixed_rotation_angles(u: torch.Tensor) -> torch.Tensor:
    """RotationAugmentation.fixed_rot_angle (:338-346) from three uniforms per scene u [B, 3] (fp64): 1.5 pi when
    u0 < 0.25, else pi when u1 < 0.5, else 0.5 pi when u2 < 0.75, else 0."""
    z = torch.zeros_like(u[:, 0])
    return torch.where(u[:, 0] < 0.25, z + math.pi * 1.5,
                       torch.where(u[:, 1] < 0.5, z + math.pi, torch.where(u[:, 2] < 0.75, z + math.pi * 0.5, z)))


def continuous_rotation_angles(u: torch.Tensor) -> torch.Tensor:
    """RotationAugmentation.rot_angle (:331-335): U(MIN_RAD, MAX_RAD) when u0 < 0.5, else 0."""
    return torch.where(u[:, 0] < 0.5, u[:, 1] * (MAX_RAD - MIN_RAD) + MIN_RAD, torch.zeros_like(u[:, 0]))


def _stats_bounds(stats_path: str) -> Dict[str, tuple]:
    """fp64 bounds as CachedThreedFront._parse_train_stats (:383-407) holds them; absent objfeat bounds are (1, -1, 1)."""
    b = load_dataset_stats(stats_path, np.float64)
    for k in ("objfeats", "objfeats_32"):
        if k not in b:
            b[k] = (np.array([1.0]), np.array([-1.0]), np.array([1.0]))
    return b


class SceneStore:
    """The rooms of some splits of a preprocessed dataset, packed on `device`.

    network_config is the config's `network` section: sample_num_points N (<= 32), class_dim, angle_dim,
    objfeat_dim and room_mask_condition decide what is stored and what a batch holds."""

    def __init__(self, dataset_directory: str, annotation_file: str, splits: Sequence[str], network_config: dict,
                 encoding_type: str = DEFAULT_ENCODING, train_stats: str = DEFAULT_STATS,
                 room_layout_size: str = "64,64", max_length: Optional[int] = None, device="cuda"):
        net = network_config
        self.N = int(net.get("sample_num_points", 12))
        self.class_dim = int(net.get("class_dim", 21))
        self.angle_dim = int(net.get("angle_dim", 1))
        self.objfeat_dim = int(net.get("objfeat_dim", 0))
        self.with_layouts = bool(net.get("room_mask_condition", False))
        if self.N > MAX_SLOTS:
            raise ValueError("sample_num_points %d > %d: ds_scene_batch holds a scene in one warp" % (self.N, MAX_SLOTS))
        if max_length is not None and int(max_length) != self.N:
            raise ValueError("data max_length %s disagrees with network sample_num_points %d" % (max_length, self.N))
        if int(net.get("objectness_dim", 0)) > 0:
            raise ValueError("objectness_dim > 0: the reference's Diffusion samples carry no objectness")
        if self.objfeat_dim not in (0, 32, 64):
            raise ValueError("objfeat_dim %d: the dataset holds objfeats_32 (32) or objfeats (64)" % self.objfeat_dim)
        self.objfeat_key = {0: None, 32: "objfeats_32", 64: "objfeats"}[self.objfeat_dim]
        self.encoding_type = encoding_type
        self.scaling, self.permute = parse_encoding(encoding_type, self.angle_dim)
        self.device = torch.device(device)

        self.stats_path = os.path.join(dataset_directory, train_stats)
        self.bounds = _stats_bounds(self.stats_path)
        with open(self.stats_path) as f:
            self.class_labels = list(json.load(f)["class_labels"])
        self.n_classes = len(self.class_labels)
        self.feature_size = 7 + self.n_classes          # Diffusion.bbox_dims + n_classes
        if self.class_dim != self.n_classes - 1:
            raise ValueError("network class_dim %d disagrees with %d class labels (class_dim = labels - 1)"
                             % (self.class_dim, self.n_classes))

        self.tags = select_rooms(dataset_directory, split_ids(annotation_file, splits))
        if not self.tags:
            raise ValueError("no room of splits %s under %s" % (list(splits), dataset_directory))
        size = tuple(int(v) for v in str(room_layout_size).split(","))
        lengths, cls, tr, sz, an, of, lay = [], [], [], [], [], [], []
        for tag in self.tags:
            D = np.load(os.path.join(dataset_directory, tag, "boxes.npz"), allow_pickle=True)
            onehot = np.asarray(D["class_labels"])
            L = onehot.shape[0]
            if onehot.ndim != 2 or onehot.shape[1] != self.n_classes:
                raise ValueError("room %s: class_labels %s, expected [L, %d]" % (tag, onehot.shape, self.n_classes))
            if L > self.N:
                raise ValueError("room %s holds %d objects, more than sample_num_points %d" % (tag, L, self.N))
            if not (np.all((onehot == 0) | (onehot == 1)) and np.all(onehot.sum(axis=1) == 1)):
                raise ValueError("room %s: a class_labels row is not one-hot" % tag)
            lengths.append(L)
            cls.append(onehot.argmax(axis=1).astype(np.int32))
            tr.append(np.asarray(D["translations"], np.float32).reshape(L, 3))
            sz.append(np.asarray(D["sizes"], np.float32).reshape(L, 3))
            an.append(np.asarray(D["angles"], np.float32).reshape(L))
            if self.objfeat_key is not None:
                if self.objfeat_key not in D.files:
                    raise ValueError("room %s has no %s (objfeat_dim %d)" % (tag, self.objfeat_key, self.objfeat_dim))
                of.append(np.asarray(D[self.objfeat_key], np.float32).reshape(L, self.objfeat_dim))
            if self.with_layouts:
                lay.append(room_layout(D, size))
        lengths = np.asarray(lengths, np.int32)
        offsets = np.concatenate([[0], np.cumsum(lengths)[:-1]]).astype(np.int32)
        put = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(self.device)
        self.lengths, self.offsets = put(lengths), put(offsets)
        self.class_index = put(np.concatenate(cls))
        self.translations = put(np.concatenate(tr).reshape(-1, 3))
        self.sizes = put(np.concatenate(sz).reshape(-1, 3))
        self.angles = put(np.concatenate(an))
        self.objfeats = put(np.concatenate(of).reshape(-1, self.objfeat_dim)) if self.objfeat_key else None
        self.layouts = put(np.stack(lay)[:, None]) if self.with_layouts else None

    def __len__(self):
        return len(self.tags)

    @property
    def num_objects(self) -> int:
        return int(self.class_index.numel())

    def batch(self, indices, rot_angle=None, jitter=None, perm_key=None, augmentations=(), permute=None) -> dict:
        """One batch of the scenes `indices` with explicit draws: rot_angle [B] and jitter [B, 3] fp64 for the
        augmentations that are on, perm_key [B, N] fp32 when permuting (the encoding decides unless `permute` is
        given).  Indices are checked against the store on the host."""
        idx = torch.as_tensor(indices, dtype=torch.int64).reshape(-1)
        if idx.numel() and (int(idx.min()) < 0 or int(idx.max()) >= len(self)):
            raise IndexError("scene index outside [0, %d)" % len(self))
        return self._launch(idx.to(self.device), parse_augmentations(augmentations, self.with_layouts),
                            self.permute if permute is None else bool(permute), rot_angle, jitter, perm_key)

    def _launch(self, idx, augs, permute, rot_angle, jitter, perm_key) -> dict:
        dev = self.device
        B, N, C = int(idx.numel()), self.N, self.n_classes - 1
        f32 = dict(dtype=torch.float32, device=dev)
        out = {"class_labels": torch.empty(B, N, C, **f32), "translations": torch.empty(B, N, 3, **f32),
               "sizes": torch.empty(B, N, 3, **f32), "angles": torch.empty(B, N, self.angle_dim, **f32),
               "length": torch.empty(B, dtype=torch.int64, device=dev)}
        if self.objfeat_key:
            out[self.objfeat_key] = torch.empty(B, N, self.objfeat_dim, **f32)
        if self.with_layouts:
            out["room_layout"] = torch.empty((B,) + tuple(self.layouts.shape[1:]), **f32)
        keep = []

        def ptr(t, dtype, shape):
            if t is None:
                return None
            t = torch.as_tensor(t, dtype=dtype, device=dev).contiguous()
            if tuple(t.shape) != shape:
                raise ValueError("draws of shape %s, expected %s" % (tuple(t.shape), shape))
            keep.append(t)
            return t.data_ptr()

        a = capi.DsSceneBatchArgs()
        a.num_scenes, a.num_class_columns, a.objfeat_dim = len(self), self.n_classes, self.objfeat_dim
        if self.with_layouts:
            a.layout_h, a.layout_w = int(self.layouts.shape[2]), int(self.layouts.shape[3])
        a.scaling, a.angle_dim, a.permute = self.scaling, self.angle_dim, int(permute)
        a.num_augmentations = len(augs)
        for i, op in enumerate(augs):
            a.augmentations[i] = op
        a.batch, a.num_slots = B, N
        a.offsets_dev, a.lengths_dev, a.class_dev = (self.offsets.data_ptr(), self.lengths.data_ptr(),
                                                     self.class_index.data_ptr())
        a.translations_dev, a.sizes_dev, a.angles_dev = (self.translations.data_ptr(), self.sizes.data_ptr(),
                                                         self.angles.data_ptr())
        a.objfeats_dev = self.objfeats.data_ptr() if self.objfeats is not None else None
        a.layouts_dev = self.layouts.data_ptr() if self.layouts is not None else None
        bt, bs, ba = self.bounds["translations"], self.bounds["sizes"], self.bounds["angles"]
        a.bounds_translations[:] = [float(v) for v in np.concatenate([bt[0], bt[1]]).reshape(-1)]
        a.bounds_sizes[:] = [float(v) for v in np.concatenate([bs[0], bs[1]]).reshape(-1)]
        a.bounds_angles[:] = [float(np.asarray(ba[0]).reshape(-1)[0]), float(np.asarray(ba[1]).reshape(-1)[0])]
        bo = self.bounds[self.objfeat_key or "objfeats"]
        a.bounds_objfeats[:] = [float(np.asarray(bo[1]).reshape(-1)[0]), float(np.asarray(bo[2]).reshape(-1)[0])]
        a.scene_index_dev = ptr(idx, torch.int64, (B,))
        rot = capi.DS_SCENE_AUG_FIXED_ROTATION in augs or capi.DS_SCENE_AUG_ROTATION in augs
        a.rot_angle_dev = ptr(rot_angle, torch.float64, (B,)) if rot else None
        a.jitter_dev = ptr(jitter, torch.float64, (B, 3)) if capi.DS_SCENE_AUG_JITTER in augs else None
        a.perm_key_dev = ptr(perm_key, torch.float32, (B, N)) if permute else None
        a.class_labels_out_dev = out["class_labels"].data_ptr()
        a.translations_out_dev, a.sizes_out_dev = out["translations"].data_ptr(), out["sizes"].data_ptr()
        a.angles_out_dev, a.length_out_dev = out["angles"].data_ptr(), out["length"].data_ptr()
        a.objfeats_out_dev = out[self.objfeat_key].data_ptr() if self.objfeat_key else None
        a.room_layout_out_dev = out["room_layout"].data_ptr() if self.with_layouts else None
        stream = torch.cuda.current_stream(dev).cuda_stream if dev.type == "cuda" else None
        capi.check(capi.load().ds_scene_batch(ctypes.byref(a), stream))
        return out


class SceneLoader:
    """Epochs over a SceneStore: batches of `batch_size` scenes, the last one partial (the reference's DataLoader
    keeps it), in one torch.randperm order per epoch when shuffling.  Each batch draws its augmentation and
    permutation numbers with a few device ops on `generator` (seeded from `seed` when not given) and runs one
    ds_scene_batch.  Validation loaders pass no augmentations and keep the encoding's permutation, as the reference's
    validation dataset does."""

    def __init__(self, store: SceneStore, batch_size: int, shuffle: bool = True, augmentations=DEFAULT_AUGMENTATIONS,
                 permute: Optional[bool] = None, generator: Optional[torch.Generator] = None, seed: int = 0):
        if batch_size < 1:
            raise ValueError("batch_size %d < 1" % batch_size)
        self.store, self.batch_size, self.shuffle = store, int(batch_size), bool(shuffle)
        self.augmentations = list(augmentations or [])
        self.augs = parse_augmentations(self.augmentations, store.with_layouts)
        self.permute = store.permute if permute is None else bool(permute)
        if generator is None:
            generator = torch.Generator(device=store.device).manual_seed(seed)
        self.generator = generator

    def __len__(self):
        return (len(self.store) + self.batch_size - 1) // self.batch_size

    def epoch_indices(self) -> List[torch.Tensor]:
        """The scene indices of each batch of one epoch (device int64)."""
        S, dev = len(self.store), self.store.device
        order = torch.randperm(S, generator=self.generator, device=dev) if self.shuffle else \
            torch.arange(S, device=dev)
        return list(torch.split(order, self.batch_size))

    def draws(self, B: int):
        """(rot_angle [B] fp64 or None, jitter [B, 3] fp64 or None, perm_key [B, N] fp32 or None)."""
        g, dev = self.generator, self.store.device
        rot = jit = key = None
        if capi.DS_SCENE_AUG_FIXED_ROTATION in self.augs:
            rot = fixed_rotation_angles(torch.rand(B, 3, generator=g, device=dev, dtype=torch.float64))
        elif capi.DS_SCENE_AUG_ROTATION in self.augs:
            rot = continuous_rotation_angles(torch.rand(B, 2, generator=g, device=dev, dtype=torch.float64))
        if capi.DS_SCENE_AUG_JITTER in self.augs:
            jit = torch.randn(B, 3, generator=g, device=dev, dtype=torch.float64) * 0.01
        if self.permute:
            key = torch.rand(B, self.store.N, generator=g, device=dev, dtype=torch.float32)
        return rot, jit, key

    def __iter__(self):
        for idx in self.epoch_indices():
            yield self.store._launch(idx, self.augs, self.permute, *self.draws(int(idx.numel())))
