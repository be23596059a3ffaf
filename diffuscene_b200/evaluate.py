"""Batched scene evaluation of generated layouts: the statistics the reference's generation script writes to
`iou_states.txt` with `--compute_intersec` (scripts/generate_diffusion.py:394-430), for a whole batch on the device.

Per scene, over its kept objects placed with their retrieved models (scripts/utils.py:664-745):
  * the number of objects and of object pairs;
  * the pairwise 3D box IoU of the placed models' axis-aligned bounds: its sum over pairs and the pairs with IoU > 0;
  * the overlap ratio of the scene;
  * the number of symmetric pairs (same class and model, sizes and one centre coordinate within 0.1).

The reference loads every retrieved mesh with trimesh and takes the bounds of the placed vertices.  Here each
catalogue model is summarised once on the host (`model_footprint`): the placement is an anisotropic scale, a shift,
a rotation about y and a translation, and the maximum of a linear function over a mesh is reached at a vertex of its
convex hull, so the x / z bounds are exact over the xz hull and the y bounds need only the raw y range.  An object
without a footprint is evaluated as its own box.  Differences from the reference: the floor mesh the reference adds
to the scene unless --without_floor is not part of the statistics, and the mesh-level intersection test
(judge_mesh_intersec) is not built.
"""
from __future__ import annotations

from typing import Dict, List, Optional, Sequence

import numpy as np
import torch

from . import capi
from .postprocess import ObjectCatalog, post_process_batch
from .stats_logger import AverageAggregator

STAT_KEYS = ("num_objects", "num_pairs", "iou_sum", "insec_count", "overlap_ratio", "num_symmetry")


def _hull_xz(p: np.ndarray) -> np.ndarray:
    """Convex hull of 2-D points (Andrew's monotone chain), counter-clockwise, collinear points dropped."""
    p = np.unique(p, axis=0)                       # sorted by x, then z
    if len(p) <= 2:
        return p

    def chain(pts):
        out: List[np.ndarray] = []
        for q in pts:
            while len(out) >= 2 and ((out[-1][0] - out[-2][0]) * (q[1] - out[-2][1])
                                     - (out[-1][1] - out[-2][1]) * (q[0] - out[-2][0])) <= 0:
                out.pop()
            out.append(q)
        return out[:-1]
    return np.array(chain(p) + chain(p[::-1]))


def model_footprint(vertices, bbox_vertices):
    """(raw_half [3], raw_aabb [6], hull_xz [K, 2]) of one catalogue model, float64.

    vertices [V, 3] are the raw mesh vertices, bbox_vertices [8, 3] the model's stored bounding-box corners; the half
    sizes are taken from them exactly as scene_synthesis/utils.py:115-120 does."""
    v = np.asarray(vertices, dtype=np.float64).reshape(-1, 3)
    bv = np.asarray(bbox_vertices, dtype=np.float64)
    raw_half = np.array([np.sqrt(np.sum((bv[4] - bv[0]) ** 2)) / 2,
                         np.sqrt(np.sum((bv[2] - bv[0]) ** 2)) / 2,
                         np.sqrt(np.sum((bv[1] - bv[0]) ** 2)) / 2])
    raw_aabb = np.concatenate([v.min(0), v.max(0)])
    return raw_half, raw_aabb, _hull_xz(v[:, [0, 2]])


def footprint_table(footprints: Sequence) -> Dict[str, np.ndarray]:
    """The CSR table `ObjectCatalog(footprints=...)` takes, from one `model_footprint` result (or None: the model is
    evaluated as its own box) per catalogue model, in catalogue order."""
    M = len(footprints)
    offsets = np.zeros(M + 1, np.int32)
    half, aabb, hulls = np.zeros((M, 3)), np.zeros((M, 6)), []
    for m, fp in enumerate(footprints):
        n = 0
        if fp is not None:
            half[m], aabb[m] = fp[0], fp[1]
            hulls.append(np.asarray(fp[2], np.float64).reshape(-1, 2))
            n = len(hulls[-1])
        offsets[m + 1] = offsets[m] + n
    hull = np.concatenate(hulls) if hulls else np.zeros((0, 2))
    return {"hull_offsets": offsets, "hull_xz": hull, "raw_half": half, "raw_aabb": aabb}


def scene_boxes(translations: torch.Tensor, sizes: torch.Tensor, angles: torch.Tensor,
                model_index: Optional[torch.Tensor] = None, catalog: Optional[ObjectCatalog] = None) -> torch.Tensor:
    """World-space translations / sizes [..., 3] and angles [..., 1] (after post_process_batch), catalogue indices
    [...] (-1: none) -> fp64 bounds [..., 6] = (x1, y1, z1, x2, y2, z2) of the placed models (ds_scene_boxes).
    Without a catalogue footprint table, or for index -1, an object is its own box."""
    dev = translations.device
    shape = tuple(translations.shape[:-1])
    t = translations.to(dev, torch.float32).reshape(-1, 3).contiguous()
    s = sizes.to(dev, torch.float32).reshape(-1, 3).contiguous()
    a = angles.to(dev, torch.float32).reshape(-1).contiguous()
    Q = t.shape[0]
    if s.shape[0] != Q or a.shape[0] != Q:
        raise ValueError("translations, sizes and angles describe different objects: %s, %s, %s"
                         % (tuple(translations.shape), tuple(sizes.shape), tuple(angles.shape)))
    fp = catalog.footprints if catalog is not None else None
    idx = None
    if model_index is not None and fp is not None:
        idx = model_index.to(dev, torch.int64).reshape(-1).contiguous()
        if idx.shape[0] != Q:
            raise ValueError("model_index holds %d entries for %d objects" % (idx.shape[0], Q))
    out = torch.empty(Q, 6, dtype=torch.float64, device=dev)
    lib = capi.load()
    capi.check(lib.ds_scene_boxes(
        capi.ptr(t), capi.ptr(s), capi.ptr(a), capi.ptr(idx), Q, capi.ptr(fp and fp["hull_offsets"]),
        capi.ptr(fp and fp["hull_xz"]),
        0 if fp is None else fp["hull_xz"].shape[0], capi.ptr(fp and fp["raw_half"]), capi.ptr(fp and fp["raw_aabb"]),
        0 if fp is None else fp["raw_half"].shape[0], capi.ptr(out), capi.stream(dev)))
    return out.reshape(shape + (6,))


def scene_stats(bounds: torch.Tensor, class_index: torch.Tensor, keep: Optional[torch.Tensor] = None,
                model_ids: Optional[torch.Tensor] = None, pair_iou: bool = False) -> Dict[str, torch.Tensor]:
    """bounds [B, N, 6] fp64, class_index [B, N] int, keep [B, N] bool (None: all), model_ids [B, N] int (None: the
    symmetry test ignores models) -> per-scene device tensors STAT_KEYS (ds_scene_stats), plus "pair_iou" [B, N, N]
    when asked for.  N <= 64."""
    dev = bounds.device
    B, N = int(bounds.shape[0]), int(bounds.shape[1])
    bx = bounds.to(dev, torch.float64).contiguous()
    cl = class_index.to(dev, torch.int64).contiguous()
    kp = None if keep is None else keep.to(dev, torch.bool).contiguous().view(torch.uint8)
    mi = None if model_ids is None else model_ids.to(dev, torch.int64).contiguous()
    for name, x in (("class_index", cl), ("keep", kp), ("model_ids", mi)):
        if x is not None and tuple(x.shape) != (B, N):
            raise ValueError("%s has shape %s, expected %s" % (name, tuple(x.shape), (B, N)))
    i32 = lambda: torch.empty(B, dtype=torch.int32, device=dev)
    out = {"num_objects": i32(), "num_pairs": i32(), "iou_sum": torch.empty(B, device=dev), "insec_count": i32(),
           "overlap_ratio": torch.empty(B, device=dev), "num_symmetry": i32()}
    if pair_iou:
        out["pair_iou"] = torch.empty(B, N, N, device=dev)
    lib = capi.load()
    capi.check(lib.ds_scene_stats(
        capi.ptr(bx), capi.ptr(kp), capi.ptr(cl), capi.ptr(mi), B, N, *[capi.ptr(out[k]) for k in STAT_KEYS],
        capi.ptr(out.get("pair_iou")), capi.stream(dev)))
    return out


def place_samples(network, samples: torch.Tensor, bounds, catalog: Optional[ObjectCatalog] = None,
                  mode: str = "objfeats"):
    """The placed objects of a batch of network samples [B, N, d] on the device: the keep mask of
    `delete_empty_batched`, the class index (argmax over all class channels), the world-space attributes of
    `post_process_batch` and the catalogue indices retrieved from `catalog` in `mode` ("objfeats",
    "objfeats_and_size" or "box"; None without a catalogue) -> (world, keep, class_index, model_index)."""
    td, sd, bb, cd = network.translation_dim, network.size_dim, network.bbox_dim, network.class_dim
    keep = ~(samples[:, :, bb + cd - 1] >= 0)
    cls = samples[:, :, bb:bb + cd - 1].argmax(dim=-1)
    params = {"translations": samples[:, :, :td], "sizes": samples[:, :, td:td + sd], "angles": samples[:, :, td + sd:bb]}
    if catalog is not None and mode != "box":
        if network.objfeat_dim <= 0:
            raise ValueError("retrieval mode %r needs a network with objfeats" % mode)
        params["objfeats"] = samples[:, :, bb + cd:bb + cd + network.objfeat_dim]
        if "objfeats" not in bounds and "objfeats_32" in bounds:
            bounds = dict(bounds, objfeats=bounds["objfeats_32"])
    world = post_process_batch(params, bounds)
    model_index = None
    if catalog is not None:
        model_index = catalog.retrieve(cls, world.get("objfeats"), world["sizes"], mode)
    return world, keep, cls, model_index


def evaluate_samples(network, samples: torch.Tensor, bounds, catalog: Optional[ObjectCatalog] = None,
                     mode: str = "objfeats", pair_iou: bool = False) -> Dict[str, torch.Tensor]:
    """Scene statistics of a batch of network samples [B, N, d] on the device, with no per-scene host loop: the placed
    objects of `place_samples`, their bounds and the statistics.  Without a catalogue every object is its own box and
    symmetry ignores models.  Returns STAT_KEYS plus "bounds", "keep", "class_index" and "model_index" (None without a
    catalogue)."""
    world, keep, cls, model_index = place_samples(network, samples, bounds, catalog, mode)
    model_ids = None
    if catalog is not None:
        model_ids = torch.where(model_index >= 0, catalog.model_ids[model_index.clamp(min=0)], -1)
    boxes = scene_boxes(world["translations"], world["sizes"], world["angles"], model_index, catalog)
    out = scene_stats(boxes, cls, keep, model_ids, pair_iou=pair_iou)
    out.update(bounds=boxes, keep=keep, class_index=cls, model_index=model_index)
    return out


class PlausibilityAggregator:
    """Running totals over evaluated scenes and the reference's `iou_states.txt` line for each
    (scripts/generate_diffusion.py:396-430): means of the object count, pairs, average IoU, intersecting share and
    overlap ratio, the std of the object counts, and the symmetry and pair totals.  `suffix` is the reference's tail
    of the line: SUFFIX_OBJFEATS for the retrieved models, SUFFIX_ONLYSIZE for the size-retrieved ones."""

    SUFFIX_OBJFEATS = "retrive objfeats  "
    SUFFIX_ONLYSIZE = "retrive only size"
    FORMAT = ("num scenes: {:d} - num objects avg: {:f} - std: {:f} - num pairs: {:f} - box iou: {:f} - "
              "box intersec: {:f} - overlap ratio: {:f} - total num symmetries: {:d} - total num pairs: {:d} ")

    def __init__(self, suffix: str = SUFFIX_OBJFEATS):
        self.suffix = suffix
        self.num_scenes = 0
        self.num_objects_counter: List[int] = []
        self.total_num_symmetry = self.total_num_pairs = 0
        self.num_obj, self.num_pairs, self.box_iou = AverageAggregator(), AverageAggregator(), AverageAggregator()
        self.box_insec, self.overlap_ratio = AverageAggregator(), AverageAggregator()

    def update(self, stats: Dict[str, torch.Tensor]) -> List[str]:
        """Adds every scene of one `scene_stats` / `evaluate_samples` result, in batch order; returns their lines."""
        host = {k: stats[k].cpu().numpy() for k in STAT_KEYS}
        lines = []
        for b in range(len(host["num_objects"])):
            n, pairs = int(host["num_objects"][b]), int(host["num_pairs"][b])
            self.num_scenes += 1
            self.num_objects_counter.append(n)
            self.num_obj.value = n
            self.num_pairs.value = pairs
            self.box_iou.value = float(host["iou_sum"][b]) / pairs
            self.box_insec.value = float(host["insec_count"][b]) / pairs
            self.overlap_ratio.value = float(host["overlap_ratio"][b])
            self.total_num_symmetry += int(host["num_symmetry"][b])
            self.total_num_pairs += pairs
            lines.append(self.FORMAT.format(
                self.num_scenes, self.num_obj.value, np.array(self.num_objects_counter).std(), self.num_pairs.value,
                self.box_iou.value, self.box_insec.value, self.overlap_ratio.value, self.total_num_symmetry,
                self.total_num_pairs) + self.suffix)
        return lines


def categorical_kl(p, q):
    """KL(p || q) of two class distributions as the reference computes it (scripts/generate_diffusion.py:44-45)."""
    p, q = np.asarray(p), np.asarray(q)
    return (p * (np.log(p + 1e-6) - np.log(q + 1e-6))).sum()


def class_frequencies(class_index: torch.Tensor, keep: torch.Tensor, n_classes: int) -> torch.Tensor:
    """Share of each class among the kept objects of a batch, on the device ([n_classes] fp64, zeros when nothing
    is kept); with training-set frequencies it gives the batch's category KL through `categorical_kl`."""
    counts = torch.bincount(class_index[keep].reshape(-1), minlength=n_classes)[:n_classes].to(torch.float64)
    return counts / counts.sum().clamp(min=1)
