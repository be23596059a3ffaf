"""Seeded synthetic furniture meshes, mesh catalogues and scenes for the renderer's tests and benchmark.

Models are subdivided boxes, cylinders, sloped wedges and composites of overlapping parts (a table: a top and four
legs), with per-corner planar UVs (some faces without), random windings, and smooth random textures.  Scenes place
them on non-convex floors (unions of rectangles) with the reference's conventions: world-space translations, half
sizes and angles about y, floors centred on their centroid.
"""
from __future__ import annotations

from typing import Dict, Tuple

import numpy as np


def _grid(n: int):
    """Unit square [0, 1]^2 split into n x n quads: (points [P, 2], triangles [2 n^2, 3])."""
    u = np.linspace(0, 1, n + 1)
    P = np.stack(np.meshgrid(u, u, indexing="ij"), -1).reshape(-1, 2)
    i, j = np.meshgrid(np.arange(n), np.arange(n), indexing="ij")
    a = (i * (n + 1) + j).reshape(-1)
    b, c, d = a + 1, a + n + 1, a + n + 2
    return P, np.concatenate([np.stack([a, c, b], 1), np.stack([b, c, d], 1)])


def box(n: int = 2, lo=(-1, -1, -1), hi=(1, 1, 1)):
    """Closed axis-aligned box with every side an n x n grid: (vertices [V, 3], faces [F, 3])."""
    P, T = _grid(n)
    lo, hi = np.asarray(lo, np.float64), np.asarray(hi, np.float64)
    vs, fs = [], []
    for axis in range(3):
        for side in (0, 1):
            v = np.zeros((len(P), 3))
            a1, a2 = [k for k in range(3) if k != axis]
            v[:, axis] = hi[axis] if side else lo[axis]
            v[:, a1] = lo[a1] + P[:, 0] * (hi[a1] - lo[a1])
            v[:, a2] = lo[a2] + P[:, 1] * (hi[a2] - lo[a2])
            fs.append(T + sum(len(x) for x in vs))
            vs.append(v)
    return np.concatenate(vs), np.concatenate(fs)


def cylinder(segments: int = 24, rings: int = 2, radius: float = 1.0, height: float = 2.0):
    """Closed y-axis cylinder centred at the origin."""
    th = np.linspace(0, 2 * np.pi, segments, endpoint=False)
    ys = np.linspace(-height / 2, height / 2, rings + 1)
    side = np.array([[radius * np.cos(t), y, radius * np.sin(t)] for y in ys for t in th])
    faces = []
    for r in range(rings):
        for s in range(segments):
            a, b = r * segments + s, r * segments + (s + 1) % segments
            faces += [[a, b + segments, b], [a, a + segments, b + segments]]
    c0, c1 = len(side), len(side) + 1
    verts = np.concatenate([side, [[0, -height / 2, 0], [0, height / 2, 0]]])
    top = rings * segments
    for s in range(segments):
        faces += [[c0, (s + 1) % segments, s], [c1, top + s, top + (s + 1) % segments]]
    return verts, np.asarray(faces)


def wedge(n: int = 2):
    """A box whose top slopes from y = 1 at x = -1 down to y = -0.2 at x = 1."""
    v, f = box(n)
    top = v[:, 1] > 0
    v[top, 1] = 1 - 0.6 * (v[top, 0] + 1)
    return v, f


def merge(*parts):
    vs, fs, off = [], [], 0
    for v, f in parts:
        vs.append(v); fs.append(f + off); off += len(v)
    return np.concatenate(vs), np.concatenate(fs)


def table(n: int = 2):
    """A top slab over four legs that pass into it (overlapping parts)."""
    parts = [box(n, (-1, 0.7, -1), (1, 1, 1))]
    for sx in (-0.85, 0.75):
        for sz in (-0.85, 0.75):
            parts.append(box(max(1, n // 2), (sx, -1, sz), (sx + 0.1, 0.8, sz + 0.1)))
    return merge(*parts)


def texture(rng: np.random.Generator, size: int) -> np.ndarray:
    """A smooth random uint8 RGB texture: a few sinusoids per channel."""
    y, x = np.mgrid[0:size, 0:size] / size
    img = np.zeros((size, size, 3))
    for c in range(3):
        for _ in range(3):
            fx, fy, ph = rng.integers(1, 6), rng.integers(1, 6), rng.uniform(0, 2 * np.pi)
            img[..., c] += np.sin(2 * np.pi * (fx * x + fy * y) + ph)
    img = (img - img.min()) / max(np.ptp(img), 1e-9)
    return (40 + 200 * img).astype(np.uint8)


def _uvs(rng, v, f, with_uv: bool):
    """Per-corner UVs: planar xz projection scaled to [0, 2] (so textures repeat), NaN for ~10 % of the faces."""
    uv = np.full((len(f), 3, 2), np.nan, np.float32)
    if with_uv:
        lo, hi = v.min(0), v.max(0)
        p = (v[:, [0, 2]] - lo[[0, 2]]) / np.maximum(hi[[0, 2]] - lo[[0, 2]], 1e-9) * 2
        uv[:] = p[f]
        uv[rng.random(len(f)) < 0.1] = np.nan
    return uv


def catalogue(seed: int = 0, num_models: int = 12, detail: int = 2, texture_size: int = 64) -> Dict[str, np.ndarray]:
    """A mesh_catalogue.npz-shaped dict of `num_models` seeded models; `detail` scales the face counts (box sides are
    (2 detail)^2 quads, cylinders 12 detail segments)."""
    from .evaluate import model_footprint
    rng = np.random.default_rng(seed)
    kinds = [lambda: box(2 * detail), lambda: cylinder(12 * detail, detail), lambda: wedge(2 * detail),
             lambda: table(2 * detail)]
    vo, fo = [0], [0]
    vs, fs, uvs, half, aabb, kd, tex = [], [], [], [], [], [], []
    for m in range(num_models):
        v, f = kinds[m % len(kinds)]()
        v = v * rng.uniform(0.3, 1.5, 3) + rng.normal(0, 0.2, 3)        # off-centre raw frames
        flip = rng.random(len(f)) < 0.3                                   # inconsistent windings
        f = np.where(flip[:, None], f[:, ::-1], f).astype(np.int32)
        lo, hi = v.min(0), v.max(0)
        corners = np.array([[lo[0], lo[1], lo[2]], [lo[0], lo[1], hi[2]], [lo[0], hi[1], lo[2]], [lo[0], hi[1], hi[2]],
                            [hi[0], lo[1], lo[2]], [hi[0], lo[1], hi[2]], [hi[0], hi[1], lo[2]], [hi[0], hi[1], hi[2]]])
        h, bb, _ = model_footprint(v.astype(np.float32), corners)
        vs.append(v.astype(np.float32)); fs.append(f); uvs.append(_uvs(rng, v, f, m % 5 != 4))
        vo.append(vo[-1] + len(v)); fo.append(fo[-1] + len(f))
        half.append(h); aabb.append(bb); kd.append(rng.uniform(0.5, 1.0, 3))
        tex.append(texture(rng, texture_size))
    return {"vertex_offsets": np.asarray(vo, np.int32), "vertices": np.concatenate(vs),
            "face_offsets": np.asarray(fo, np.int32), "faces": np.concatenate(fs), "uvs": np.concatenate(uvs),
            "raw_half": np.asarray(half), "raw_aabb": np.asarray(aabb), "kd": np.asarray(kd, np.float32),
            "textures": np.stack(tex), "jids": np.array(["model-%04d" % m for m in range(num_models)])}


def floor_plan(rng: np.random.Generator) -> Tuple[np.ndarray, np.ndarray]:
    """A non-convex floor (an L or a U of rectangles, 4 or 6 triangles), centred on its vertex centroid as the
    reference centres floor_plan_vertices."""
    w, d = rng.uniform(2.0, 3.0), rng.uniform(2.0, 3.0)
    rects = [(-w, -d, w, -d + 1.2), (-w, -d + 1.2, -w + 1.2, d)]        # disjoint, sharing edges
    if rng.random() < 0.5:
        rects.append((w - 1.2, -d + 1.2, w, d))
    vs, fs = [], []
    for x0, z0, x1, z1 in rects:
        b = len(vs)
        vs += [[x0, 0, z0], [x1, 0, z0], [x1, 0, z1], [x0, 0, z1]]
        fs += [[b, b + 1, b + 2], [b, b + 2, b + 3]]
    v = np.asarray(vs, np.float64)
    return (v - v.mean(0)).astype(np.float32), np.asarray(fs, np.int32)


def scenes(num_scenes: int, num_objects: int, num_models: int, seed: int = 0, empty: float = 0.25,
           num_classes: int = 21):
    """Seeded scene batch: translations / sizes [B, N, 3], angles [B, N, 1] fp32, model_index / class_index [B, N]
    int64 (-1: empty slot, a share `empty` of the slots) and one floor (vertices, faces) per scene."""
    rng = np.random.default_rng(seed)
    B, N = num_scenes, num_objects
    sizes = rng.uniform(0.15, 0.9, (B, N, 3)).astype(np.float32)
    sizes[..., 1] = rng.uniform(0.2, 1.0, (B, N)).astype(np.float32)
    trans = np.stack([rng.uniform(-2.4, 2.4, (B, N)), sizes[..., 1], rng.uniform(-2.4, 2.4, (B, N))],
                     -1).astype(np.float32)
    angles = rng.uniform(-np.pi, np.pi, (B, N, 1)).astype(np.float32)
    model = rng.integers(0, num_models, (B, N))
    model[rng.random((B, N)) < empty] = -1
    cls = rng.integers(0, num_classes, (B, N))
    floors = [floor_plan(rng) for _ in range(B)]
    return {"translations": trans, "sizes": sizes, "angles": angles, "model_index": model, "class_index": cls,
            "floors": floors}
