"""Batched attribute scaling around the sampler (SURVEY 8f row 3), on whatever device the tensors live on.

The reference encodes / decodes scene attributes on the CPU with numpy, one scene at a time
(scene_synthesis/datasets/threed_front_dataset.py: `Scale_CosinAngle_ObjfeatsNorm.scale` :483-489, `.descale`
:491-495, `__getitem__` :497-513, `post_process` :515-535).  Here the same arithmetic runs on the whole [B, N, .]
batch that `network.sample()` returns, so finished scenes never leave the GPU between the sampler and retrieval:

  encode   translations / sizes: clip to [lo, hi], map to [-1, 1];  angles: theta -> (cos, sin);
           objfeats: bounds entries 1 and 2 are (lo, hi) (entry 0 is the std the reference ignores here)
  decode   the inverse: angles = atan2(sin, cos); class labels, layouts and text pass through.

`bounds[k]` is a sequence of array-likes exactly as the reference's dataset objects hold them.
"""
from __future__ import annotations

from typing import Dict, Mapping, Sequence

import torch

_PASS_THROUGH = ("room_layout", "class_labels", "relations", "description", "desc_emb")
_OBJFEAT_KEYS = ("objfeats", "objfeats_32")


def _lo_hi(bounds: Mapping[str, Sequence], key: str, like: torch.Tensor):
    b = bounds[key]
    lo, hi = (b[1], b[2]) if key in _OBJFEAT_KEYS else (b[0], b[1])
    as_t = lambda v: torch.as_tensor(v, dtype=torch.float32, device=like.device)
    return as_t(lo), as_t(hi)


def scale(x: torch.Tensor, lo: torch.Tensor, hi: torch.Tensor) -> torch.Tensor:
    """clip to [lo, hi] then affine map onto [-1, 1] (reference :483-489)."""
    x = torch.minimum(torch.maximum(x.float(), lo), hi)
    return 2.0 * ((x - lo) / (hi - lo)) - 1.0


def descale(x: torch.Tensor, lo: torch.Tensor, hi: torch.Tensor) -> torch.Tensor:
    """inverse of `scale` without the clip (reference :491-495)."""
    return (x + 1.0) / 2.0 * (hi - lo) + lo


def encode_batch(params: Mapping[str, torch.Tensor], bounds: Mapping[str, Sequence]) -> Dict[str, torch.Tensor]:
    """World-space attributes -> network space for a whole batch (reference `__getitem__` :497-513)."""
    out: Dict[str, torch.Tensor] = {}
    for k, v in params.items():
        if k == "angles":
            out[k] = torch.cat([torch.cos(v), torch.sin(v)], dim=-1)
        elif k in _OBJFEAT_KEYS or k in bounds:
            out[k] = scale(v, *_lo_hi(bounds, k, v))
        else:
            out[k] = v
    return out


def load_dataset_stats(path: str, dtype=None) -> Dict[str, tuple]:
    """`bounds` for encode_batch / post_process_batch from the reference's dataset_stats.txt JSON: bounds_translations
    / bounds_sizes are 6 floats (lo xyz, hi xyz), bounds_angles 2 (lo, hi), bounds_objfeats[_32] 3 (std, lo, hi).
    Arrays are float32, or `dtype` (the training data layer keeps the reference's float64)."""
    import json

    import numpy as np
    with open(path) as f:
        stats = json.load(f)
    out: Dict[str, tuple] = {}
    for key, n in (("translations", 6), ("sizes", 6), ("angles", 2), ("objfeats", 3), ("objfeats_32", 3)):
        if "bounds_" + key not in stats:
            continue
        v = np.asarray(stats["bounds_" + key], np.float32 if dtype is None else dtype).reshape(-1)
        if v.size != n:
            raise ValueError("%s: bounds_%s holds %d values, expected %d" % (path, key, v.size, n))
        out[key] = tuple(np.split(v, n // (3 if n == 6 else 1)))
    missing = [k for k in ("translations", "sizes", "angles") if k not in out]
    if missing:
        raise ValueError("%s lacks bounds_%s" % (path, ", bounds_".join(missing)))
    return out


def post_process_batch(params: Mapping[str, torch.Tensor], bounds: Mapping[str, Sequence]) -> Dict[str, torch.Tensor]:
    """Network-space samples -> world-space attributes for a whole batch (reference `post_process` :515-535)."""
    out: Dict[str, torch.Tensor] = {}
    for k, v in params.items():
        if k in _PASS_THROUGH:
            out[k] = v
        elif k == "angles":
            out[k] = torch.atan2(v[..., 1:2], v[..., 0:1])
        else:
            out[k] = descale(v, *_lo_hi(bounds, k, v))
    return out


class ObjectCatalog:
    """Device-resident furniture catalogue for batched nearest-model retrieval (the last step of the reference's
    generation scripts: `ThreedFutureDataset.get_closest_furniture_to_objfeats_and_size` & co,
    scene_synthesis/datasets/threed_future_dataset.py:28-77, called once per generated object on the CPU).

    labels [M] int class index per catalogue model, feats [M, F] latent shape codes, sizes [M, 3].  The entries are
    grouped by class once (stable, so catalogue order inside a class -- the reference's tie-break -- is kept);
    `retrieve` answers a whole [B, N] batch of generated objects with ONE kernel launch (one warp per object) and
    returns indices into the ORIGINAL catalogue order (-1: class has no model).  Indices are bit-exact with the
    reference's per-object numpy code (the kernel accumulates in numpy's float32 summation order).

    For scene evaluation (diffuscene_b200.evaluate) two optional keyword arguments, both in original catalogue order:
    `footprints`, the dict `evaluate.footprint_table` builds (one CSR table of xz hull polygons, raw half sizes and
    raw AABBs, kept on the device; a model with an empty hull row is evaluated as its own box), and `model_ids` [M]
    int, which stand in for the reference's model jids in the symmetry test (default: the catalogue index)."""

    MODES = {"objfeats_and_size": 0, "objfeats": 1, "box": 2}
    FOOTPRINT_KEYS = ("hull_offsets", "hull_xz", "raw_half", "raw_aabb")

    def __init__(self, labels, feats, sizes, n_classes=None, device="cuda", footprints=None, model_ids=None):
        import ctypes as C
        from . import capi
        self._C, self._capi = C, capi
        self.lib = capi.load()
        labels = torch.as_tensor(labels, dtype=torch.int64).cpu()
        self.n_classes = int(n_classes if n_classes is not None else (int(labels.max()) + 1 if labels.numel() else 1))
        order = torch.argsort(labels, stable=True)
        counts = torch.bincount(labels, minlength=self.n_classes)
        start = torch.zeros(self.n_classes + 1, dtype=torch.int32)
        start[1:] = torch.cumsum(counts, 0).to(torch.int32)
        dev = torch.device(device)
        self.device = dev
        self.order = order.to(dev)
        self.class_start = start.to(dev)
        self.feats = None if feats is None else torch.as_tensor(feats, dtype=torch.float32)[order].contiguous().to(dev)
        self.sizes = None if sizes is None else torch.as_tensor(sizes, dtype=torch.float32)[order].contiguous().to(dev)
        M = labels.numel()
        ids = torch.arange(M) if model_ids is None else torch.as_tensor(model_ids, dtype=torch.int64).reshape(-1)
        if ids.numel() != M:
            raise ValueError("model_ids holds %d entries for %d catalogue models" % (ids.numel(), M))
        self.model_ids = ids.to(dev)
        self.footprints = None
        if footprints is not None:
            fp = {k: torch.as_tensor(footprints[k]) for k in self.FOOTPRINT_KEYS}
            H = fp["hull_xz"].reshape(-1, 2).shape[0]
            if fp["hull_offsets"].shape != (M + 1,) or fp["raw_half"].numel() != 3 * M or fp["raw_aabb"].numel() != 6 * M:
                raise ValueError("footprint table does not describe %d models" % M)
            self.footprints = {
                "hull_offsets": fp["hull_offsets"].to(torch.int32).contiguous().to(dev),
                "hull_xz": fp["hull_xz"].to(torch.float64).reshape(H, 2).contiguous().to(dev),
                "raw_half": fp["raw_half"].to(torch.float64).reshape(M, 3).contiguous().to(dev),
                "raw_aabb": fp["raw_aabb"].to(torch.float64).reshape(M, 6).contiguous().to(dev)}

    def retrieve(self, class_index, objfeats=None, sizes=None, mode="objfeats_and_size"):
        """class_index [...] int64, objfeats [..., F], sizes [..., 3] (world-space, i.e. after post_process_batch) ->
        catalogue indices [...] int64 on the device."""
        m = self.MODES[mode]
        C = self._C
        shape = tuple(class_index.shape)
        ql = class_index.to(self.device, torch.int64).reshape(-1).contiguous()
        Q = ql.numel()
        qf = None if objfeats is None else objfeats.to(self.device, torch.float32).reshape(Q, -1).contiguous()
        qs = None if sizes is None else sizes.to(self.device, torch.float32).reshape(Q, -1).contiguous()
        out = torch.empty(Q, dtype=torch.int64, device=self.device)
        p = lambda t: None if t is None else C.c_void_p(t.data_ptr())
        self._capi.check(self.lib.ds_retrieve_objects(
            p(self.class_start), self.n_classes, p(self.feats), p(self.sizes),
            0 if self.feats is None else self.feats.shape[1], 0 if self.sizes is None else self.sizes.shape[1],
            p(ql), p(qf), p(qs), Q, m, p(out), C.c_void_p(torch.cuda.current_stream(self.device).cuda_stream)))
        hit = out >= 0
        res = torch.where(hit, self.order[out.clamp(min=0)], out)
        return res.reshape(shape)
