"""ORACLE (test infrastructure only -- never imported by the product): numpy restatement of the reference's scene
evaluation, the `--compute_intersec` statistics of scripts/generate_diffusion.py:394-430.

  * `place_bounds`: the placement of scene_synthesis/utils.py:114-163 applied to a FULL vertex set in float64, as
    trimesh applies it (vertices *= query_size / raw_sizes; -= centroid; .dot(R) + translation), then the AABB.
  * `intersection`: computer_intersection / axis_aligned_bbox_overlaps_3d (scripts/utils.py:560-701) on the bounds
    rounded to float32, elementwise in torch's order; the IoU sum over pairs i < j accumulated in float32 like the
    reference's sum() over numpy float32 scalars.
  * `symmetry`: computer_symmetry / judge_if_symmetry (:703-745) on the float64 bounds.
Pinned by tests/test_scene_eval_cpu.py against tests/golden/scene_eval.npz (the unmodified reference functions).
"""
from __future__ import annotations

import numpy as np


def raw_half_sizes(bbox_vertices) -> np.ndarray:
    bv = np.asarray(bbox_vertices, np.float64)
    return np.array([np.sqrt(np.sum((bv[4] - bv[0]) ** 2)) / 2, np.sqrt(np.sum((bv[2] - bv[0]) ** 2)) / 2,
                     np.sqrt(np.sum((bv[1] - bv[0]) ** 2)) / 2])


def box_vertices(half) -> np.ndarray:
    """The 8 corners of a centred box with half sizes `half` (the layout-only stand-in for a model)."""
    s = np.array([[x, y, z] for x in (-1, 1) for y in (-1, 1) for z in (-1, 1)], np.float64)
    return s * np.asarray(half, np.float64)


def place_bounds(vertices, raw_half, size, translation, angle) -> np.ndarray:
    """[x1, y1, z1, x2, y2, z2] of the placed mesh; raw_half None: the mesh is used unscaled (its own box)."""
    size = np.asarray(size, np.float32)
    v = np.array(vertices, np.float64)
    if raw_half is not None:
        v *= size / np.asarray(raw_half, np.float64)
    centroid = (v.min(0) + v.max(0)) / 2
    theta = np.float32(angle)
    R = np.zeros((3, 3))
    R[0, 0] = np.cos(theta)
    R[0, 2] = -np.sin(theta)
    R[2, 0] = np.sin(theta)
    R[2, 2] = np.cos(theta)
    R[1, 1] = 1.
    v -= centroid
    v = v.dot(R) + np.asarray(translation, np.float32)
    return np.concatenate([v.min(0), v.max(0)])


def iou_matrix(bounds):
    """(ious [n, n], overlaps [n, n], areas [n]) in float32, torch's elementwise order."""
    b = np.asarray(bounds, np.float64).astype(np.float32).reshape(-1, 6)
    area = ((b[:, 3] - b[:, 0]) * (b[:, 4] - b[:, 1])) * (b[:, 5] - b[:, 2])
    lt = np.maximum(b[:, None, :3], b[None, :, :3])
    rb = np.minimum(b[:, None, 3:], b[None, :, 3:])
    wh = np.maximum(rb - lt, np.float32(0))
    overlap = (wh[..., 0] * wh[..., 1]) * wh[..., 2]
    union = np.maximum((area[:, None] + area[None, :]) - overlap, np.float32(1e-6))
    return overlap / union, overlap, area


def intersection(bounds):
    """(num_objects, num_pairs, iou_sum float32, insec_count, overlap_ratio float32) of one scene."""
    n = len(bounds)
    if n <= 1:
        return n, 1, np.float32(0), 0, np.float32(0)
    iou, overlap, area = iou_matrix(bounds)
    s, cnt = np.float32(0), 0
    for i in range(n):
        for j in range(i + 1, n):
            if iou[i, j] > 0:
                s = np.float32(s + iou[i, j])
                cnt += 1
    # the two sums in float64, rounded once: they differ from torch's float32 reductions (whose order is not
    # reproduced) by those reductions' own rounding only; the rest is the reference's float32 arithmetic
    ov = np.float32(np.triu(overlap, 1).sum(dtype=np.float64))
    area_total = np.float32(area.sum(dtype=np.float64))
    with np.errstate(invalid="ignore", divide="ignore"):
        ratio = np.float32(ov / (np.float32(area_total + area_total) / np.float32(2) - ov))
    return n, n * (n - 1) // 2, s, cnt, ratio


def judge_if_symmetry(box1, box2, size_diff=0.1, pos_diff=0.1) -> bool:
    center1, size1 = (box1[3:6] + box1[0:3]) / 2.0, (box1[3:6] - box1[0:3]) / 2.0
    center2, size2 = (box2[3:6] + box2[0:3]) / 2.0, (box2[3:6] - box2[0:3]) / 2.0
    if np.abs(size1 - size2).max() < size_diff:
        return bool(abs(center1[0] - center2[0]) < pos_diff or abs(center1[2] - center2[2]) < pos_diff)
    return False


def symmetry(bounds, classes, model_ids=None) -> int:
    """Symmetric pairs; model_ids None: models are not compared (every object counts as the same model)."""
    b = np.asarray(bounds, np.float64).reshape(-1, 6)
    n, count = len(b), 0
    for i in range(n):
        for j in range(i + 1, n):
            if classes[i] == classes[j] and (model_ids is None or model_ids[i] == model_ids[j]):
                count += judge_if_symmetry(b[i], b[j])
    return count


def evaluate_scene(bounds, classes, model_ids=None):
    """(num_objects, num_pairs, iou_sum, insec_count, overlap_ratio, num_symmetry) of one scene's kept objects."""
    return intersection(bounds) + (symmetry(bounds, classes, model_ids),)
