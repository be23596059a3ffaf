"""Top-down and perspective rendering of scenes on the device, and renders fed to FID / KID and precision-recall without the host.

The reference renders every scene top-down with simple-3dviz / OpenGL (scripts/utils.py:220-254,
scripts/generate_diffusion.py:251-264, scripts/preprocess_data.py:297-350).  Here:

  * `pack_catalogue` / `parse_obj` turn 3D-FUTURE model directories into one `mesh_catalogue.npz`, and
    `MeshCatalog` uploads it once (ds_mesh_catalog_*);
  * `render_scenes` rasterises the placed catalogue meshes (and the floor) of a whole batch of scenes into uint8
    [B, H, W, 3] device images with the reference's orthographic top-down camera or its perspective view
    (REFERENCE_PERSPECTIVE) (ds_render_scenes);
  * `clean_resize` / `ipr_resize` are Pillow's resizes of the two metrics on the device, bit-exact with PIL
    (ds_resize_f32 / ds_resize_u8), from the coefficient tables `pillow_coeffs` computes on the host;
  * `inception_features` / `vgg16_features` / `evaluate_renders` take device renders to features and metrics.

The geometry, placement and camera are the reference's; the shading constants are this project's (simple-3dviz is
not available to compare against).  FID / KID / precision-recall of native renders therefore compare only with
native renders of the real scenes (scripts/render_scenes.py), never with images rendered by the reference.
"""
from __future__ import annotations

import colorsys
import ctypes as C
import math
import os
import re
from dataclasses import dataclass
from typing import Dict, List, Optional, Sequence, Tuple

import numpy as np
import torch

from . import capi

CATALOGUE_KEYS = ("vertex_offsets", "vertices", "face_offsets", "faces", "uvs", "raw_half", "raw_aabb", "kd",
                  "textures", "jids")
TEXTURE_SIZE = 256            # default cap of the packed textures (PIL bilinear resize to T x T)
ROOM_SIDE = 3.1               # the reference's orthographic half extent (args.room_side)


# ---- catalogue --------------------------------------------------------------------------------------------------

def parse_mtl(path: str) -> Dict[str, Dict[str, object]]:
    """{material: {"Kd": [3] floats, "map_Kd": file or None}} of a .mtl file."""
    mats: Dict[str, Dict[str, object]] = {}
    cur = None
    with open(path, "r", errors="replace") as f:
        for line in f:
            tok = line.split()
            if not tok:
                continue
            if tok[0] == "newmtl":
                cur = mats.setdefault(" ".join(tok[1:]), {"Kd": None, "map_Kd": None})
            elif cur is not None and tok[0] == "Kd" and len(tok) >= 4:
                cur["Kd"] = [float(t) for t in tok[1:4]]
            elif cur is not None and tok[0] == "map_Kd" and len(tok) >= 2:
                cur["map_Kd"] = tok[-1]
    return mats


def _index(tok: str, n: int) -> int:
    i = int(tok)
    return i - 1 if i > 0 else n + i           # OBJ indices are 1-based; negative ones count back from the end


def parse_obj(path: str):
    """(vertices [V, 3] float64, faces [F, 3] int32, uvs [F, 3, 2] float32 with NaN where a face has none, Kd [3])
    of a Wavefront OBJ: `v`, `vt`, `f` with v, v/vt, v//vn or v/vt/vn corners, negative indices, polygons fanned into
    triangles (0, i, i + 1).  Kd is that of the first material of its `mtllib` that has one (1, 1, 1 without)."""
    verts: List[List[float]] = []
    tex: List[List[float]] = []
    faces: List[Tuple[int, int, int]] = []
    uvi: List[Tuple[int, int, int]] = []
    mtllibs: List[str] = []
    with open(path, "r", errors="replace") as f:
        for line in f:
            tok = line.split()
            if not tok:
                continue
            if tok[0] == "v":
                verts.append([float(t) for t in tok[1:4]])
            elif tok[0] == "vt":
                tex.append([float(t) for t in tok[1:3]] + [0.0] * (2 - len(tok[1:3])))
            elif tok[0] == "f":
                vi, ti = [], []
                for c in tok[1:]:
                    parts = c.split("/")
                    vi.append(_index(parts[0], len(verts)))
                    ti.append(_index(parts[1], len(tex)) if len(parts) > 1 and parts[1] else -1)
                for k in range(1, len(vi) - 1):
                    faces.append((vi[0], vi[k], vi[k + 1]))
                    uvi.append((ti[0], ti[k], ti[k + 1]))
            elif tok[0] == "mtllib":
                mtllibs.append(" ".join(tok[1:]))
    v = np.asarray(verts, np.float64).reshape(-1, 3)
    fa = np.asarray(faces, np.int64).reshape(-1, 3)
    if fa.size and (fa.min() < 0 or fa.max() >= len(v)):
        raise ValueError("%s: a face refers to a vertex outside [1, %d]" % (path, len(v)))
    t = np.asarray(tex, np.float64).reshape(-1, 2)
    ti = np.asarray(uvi, np.int64).reshape(-1, 3)
    uv = np.full((len(fa), 3, 2), np.nan, np.float32)
    has = (ti >= 0).all(axis=1)
    if has.any():
        if ti[has].max() >= len(t):
            raise ValueError("%s: a face refers to a texture coordinate outside [1, %d]" % (path, len(t)))
        uv[has] = t[ti[has]]
    kd = np.ones(3)
    for lib in mtllibs:
        mp = os.path.join(os.path.dirname(path), lib)
        if os.path.isfile(mp):
            found = [m["Kd"] for m in parse_mtl(mp).values() if m["Kd"] is not None]
            if found:
                kd = np.asarray(found[0], np.float64)
                break
    return v, fa.astype(np.int32), uv, kd


def load_texture(path: Optional[str], size: int = TEXTURE_SIZE) -> np.ndarray:
    """uint8 [size, size, 3]: the RGB image resized with PIL bilinear (which widens its support when shrinking, so
    it averages); white when there is no texture."""
    from PIL import Image
    if path is None or not os.path.isfile(path):
        return np.full((size, size, 3), 255, np.uint8)
    with Image.open(path) as im:
        im = im.convert("RGB")
        if im.size != (size, size):
            im = im.resize((size, size), Image.BILINEAR)
        return np.asarray(im, np.uint8).copy()


def pack_catalogue(model_dirs: Sequence[str], jids: Sequence[str], texture_size: int = TEXTURE_SIZE) -> dict:
    """The arrays of mesh_catalogue.npz from 3D-FUTURE model directories (raw_model.obj, texture.png,
    bbox_vertices.npy) in catalogue order.  raw_half / raw_aabb are evaluate.model_footprint's."""
    from .evaluate import model_footprint
    if len(model_dirs) != len(jids):
        raise ValueError("%d model directories for %d jids" % (len(model_dirs), len(jids)))
    M = len(model_dirs)
    vo, fo = np.zeros(M + 1, np.int32), np.zeros(M + 1, np.int32)
    vs, fs, uvs = [], [], []
    half, aabb, kd = np.zeros((M, 3)), np.zeros((M, 6)), np.zeros((M, 3), np.float32)
    tex = np.zeros((M, texture_size, texture_size, 3), np.uint8)
    for m, d in enumerate(model_dirs):
        v, f, uv, k = parse_obj(os.path.join(d, "raw_model.obj"))
        h, bb, _ = model_footprint(v, np.load(os.path.join(d, "bbox_vertices.npy")))
        vs.append(v.astype(np.float32)); fs.append(f); uvs.append(uv)
        vo[m + 1], fo[m + 1] = vo[m] + len(v), fo[m] + len(f)
        half[m], aabb[m], kd[m] = h, bb, k
        tex[m] = load_texture(os.path.join(d, "texture.png"), texture_size)
    cat = lambda xs, shape, dt: np.concatenate(xs).astype(dt) if xs else np.zeros(shape, dt)
    return {"vertex_offsets": vo, "vertices": cat(vs, (0, 3), np.float32), "face_offsets": fo,
            "faces": cat(fs, (0, 3), np.int32), "uvs": cat(uvs, (0, 3, 2), np.float32), "raw_half": half,
            "raw_aabb": aabb, "kd": kd, "textures": tex, "jids": np.asarray(list(jids), dtype=str)}


def _c(a: np.ndarray, dt) -> np.ndarray:
    return np.ascontiguousarray(np.asarray(a, dt))


class MeshCatalog:
    """The packed mesh catalogue on the device (ds_mesh_catalog_create).  `src` is a mesh_catalogue.npz path or the
    dict `pack_catalogue` returns."""

    def __init__(self, src, device: int = 0):
        data = np.load(src) if isinstance(src, (str, os.PathLike)) else src
        missing = [k for k in CATALOGUE_KEYS if k not in data]
        if missing:
            raise KeyError("mesh catalogue lacks %s" % ", ".join(missing))
        self.jids = [str(j) for j in data["jids"]]
        self.arrays = {k: data[k] for k in CATALOGUE_KEYS if k != "jids"}
        a = self.arrays
        self.num_models = len(a["vertex_offsets"]) - 1
        tex = _c(a["textures"], np.uint8)
        if tex.ndim != 4 or tex.shape[0] != self.num_models or tex.shape[1] != tex.shape[2] or tex.shape[3] != 3:
            raise ValueError("textures must be [M, T, T, 3], got %s" % (tex.shape,))
        self.texture_size = tex.shape[1]
        self.face_counts = np.diff(np.asarray(a["face_offsets"], np.int64))
        self.lib = capi.load()
        self.device = device
        arrs = [_c(a["vertex_offsets"], np.int32), _c(a["vertices"], np.float32), _c(a["face_offsets"], np.int32),
                _c(a["faces"], np.int32), _c(a["uvs"], np.float32), _c(a["raw_half"], np.float64),
                _c(a["raw_aabb"], np.float64), _c(a["kd"], np.float32), tex]
        self._h = C.c_void_p()
        ptr = lambda x: C.c_void_p(x.ctypes.data) if x.size else None
        capi.check(self.lib.ds_mesh_catalog_create(self.num_models, *[ptr(x) for x in arrs], self.texture_size,
                                                   device, C.byref(self._h)))

    def index_of(self, jids: Sequence[str]) -> np.ndarray:
        """Catalogue indices of model jids (-1 where a jid is not in the catalogue)."""
        pos = {j: i for i, j in enumerate(self.jids)}
        return np.array([pos.get(str(j), -1) for j in jids], np.int64)

    def close(self):
        if getattr(self, "_h", None) and self._h.value:
            self.lib.ds_mesh_catalog_destroy(self._h)
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


# ---- camera, palette, floors ------------------------------------------------------------------------------------

PROJECTIONS = {"orthographic": capi.DS_RENDER_ORTHOGRAPHIC, "perspective": capi.DS_RENDER_PERSPECTIVE}


@dataclass
class Camera:
    """The reference's top-down camera (generate_diffusion.py:251-264): eye (0, 4, 0) looking at the origin with up
    (0, 0, -1), Matrix44.orthogonal_projection(left=-s, right=s, bottom=s, top=-s, near=0.1, far=6), s = 3.1, 256^2.

    With projection "perspective", left / right / bottom / top are the frustum bounds on the near plane (pyrr's
    create_perspective_projection_from_bounds) and depth is the view depth -z_view; `Camera.perspective` builds one
    from a vertical field of view."""
    eye: Tuple[float, float, float] = (0.0, 4.0, 0.0)
    target: Tuple[float, float, float] = (0.0, 0.0, 0.0)
    up: Tuple[float, float, float] = (0.0, 0.0, -1.0)
    left: float = -ROOM_SIDE
    right: float = ROOM_SIDE
    bottom: float = ROOM_SIDE
    top: float = -ROOM_SIDE
    near: float = 0.1
    far: float = 6.0
    width: int = 256
    height: int = 256
    projection: str = "orthographic"

    @classmethod
    def perspective(cls, eye, target=(0.0, 0.0, 0.0), up=(0.0, 1.0, 0.0), fovy: float = 45.0, width: int = 512,
                    height: int = 512, near: float = 0.1, far: float = 1000.0) -> "Camera":
        """A perspective camera with pyrr's perspective_projection(fovy, width / height, near, far) bounds: ymax =
        near tan(fovy pi / 360), xmax = ymax width / height.  bottom = ymax, top = -ymax keeps the image upright
        (array row 0 is the top of the view), as the top-down camera's swapped bounds do.

        45 degrees, 0.1 and 1000 are, as far as we know, simple-3dviz Scene's default projection, which the
        reference's perspective renders use; simple-3dviz is not available to check this, and the shading is this
        project's own either way."""
        ymax = near * math.tan(fovy * math.pi / 360.0)
        xmax = ymax * width / height
        return cls(eye=tuple(float(v) for v in eye), target=tuple(float(v) for v in target),
                   up=tuple(float(v) for v in up), left=-xmax, right=xmax, bottom=ymax, top=-ymax, near=near,
                   far=far, width=width, height=height, projection="perspective")

    def struct(self) -> capi.DsRenderCamera:
        if self.projection not in PROJECTIONS:
            raise ValueError("unknown projection %r (one of %s)" % (self.projection, ", ".join(PROJECTIONS)))
        c = capi.DsRenderCamera()
        c.eye[:], c.target[:], c.up[:] = self.eye, self.target, self.up
        c.left, c.right, c.bottom, c.top = self.left, self.right, self.bottom, self.top
        c.near_plane, c.far_plane, c.width, c.height = self.near, self.far, self.width, self.height
        c.projection = PROJECTIONS[self.projection]
        return c


# the reference driver's perspective view (scripts/completion_rearrange.py defaults, scripts/utils.py:431-458)
REFERENCE_PERSPECTIVE = Camera.perspective(eye=(-0.10923499, 1.9325259, -7.19009), target=(0.0, 0.0, 0.0),
                                           up=(0.0, 1.0, 0.0), width=512, height=512)


def hls_palette(n_colors: int, h: float = 0.01, l: float = 0.6, s: float = 0.65) -> np.ndarray:
    """seaborn's color_palette('hls', n_colors) (hls_palette): n evenly spaced hues from h, lightness 0.6, saturation
    0.65 -> float64 [n, 3] RGB in [0, 1]."""
    hues = np.linspace(0, 1, n_colors + 1)[:-1]
    hues += h
    hues %= 1
    hues -= hues.astype(int)
    return np.array([colorsys.hls_to_rgb(hu, l, s) for hu in hues]).reshape(-1, 3)


def floor_triangles(floors: Sequence[Optional[Tuple[np.ndarray, np.ndarray]]]) -> Tuple[np.ndarray, np.ndarray]:
    """The CSR floor list ds_render_scenes takes from per-scene (vertices [V, 3], faces [F, 3]) pairs, the vertices
    already centred (floor_plan_vertices - floor_plan_centroid); None: no floor -> (offsets [B + 1] int32,
    triangles [T, 3, 3] float32)."""
    offsets = np.zeros(len(floors) + 1, np.int32)
    tris = []
    for b, fl in enumerate(floors):
        n = 0
        if fl is not None:
            v, f = np.asarray(fl[0], np.float32).reshape(-1, 3), np.asarray(fl[1], np.int64).reshape(-1, 3)
            tris.append(v[f])
            n = len(f)
        offsets[b + 1] = offsets[b] + n
    return offsets, (np.concatenate(tris) if tris else np.zeros((0, 3, 3), np.float32)).astype(np.float32)


def load_floor_textures(folder: str, size: int = TEXTURE_SIZE) -> np.ndarray:
    """uint8 [F, size, size, 3] of every image in `folder`, sorted by name."""
    names = sorted(n for n in os.listdir(folder) if re.search(r"\.(png|jpe?g|bmp)$", n, re.I))
    if not names:
        raise FileNotFoundError("no floor textures in %s" % folder)
    return np.stack([load_texture(os.path.join(folder, n), size) for n in names])


def choose_floor_textures(num_scenes: int, num_textures: int, seed: int = 0) -> np.ndarray:
    """One floor texture per scene, drawn uniformly with a seeded generator (the reference draws np.random.choice)."""
    return np.random.default_rng(seed).integers(0, num_textures, num_scenes).astype(np.int32)


# ---- rendering --------------------------------------------------------------------------------------------------

def _ptr(t: Optional[torch.Tensor]):
    return None if t is None else C.c_void_p(t.data_ptr())


def render_scenes(catalog: MeshCatalog, translations, sizes, angles, model_index, class_index=None,
                  floors: Optional[Tuple[np.ndarray, np.ndarray]] = None, no_texture: bool = False,
                  white_background: bool = False, camera: Optional[Camera] = None, palette=None,
                  floor_textures=None, floor_texture_index=None, return_ids: bool = False):
    """uint8 [B, H, W, 3] renders on the catalogue's device (top-down unless `camera` says otherwise).

    translations / sizes [B, N, 3] and angles [B, N] or [B, N, 1] are world-space (after post_process_batch);
    model_index [B, N] indexes the catalogue (-1: empty slot); class_index [B, N] picks the flat colour of each object
    from `palette` ([P, 3] in [0, 1]) when no_texture is set.  floors is `floor_triangles`'s (offsets, triangles) or
    None for no floor; floor_textures [F, S, S, 3] uint8 with floor_texture_index [B] (-1: white) textures it.
    white_background is the reference's --without_floor background.  With return_ids, also the int64 [B, H, W] ids
    slot << 32 | face of the visible triangles (slot N: the floor, -1: background)."""
    camera = camera or Camera()
    dev = torch.device("cuda", catalog.device)
    t = torch.as_tensor(translations).to(dev, torch.float32).contiguous()
    B, N = int(t.shape[0]), int(t.shape[1])
    s = torch.as_tensor(sizes).to(dev, torch.float32).reshape(B, N, 3).contiguous()
    a = torch.as_tensor(angles).to(dev, torch.float32).reshape(B, N).contiguous()
    mi = torch.as_tensor(model_index).to(dev, torch.int64).reshape(B, N).contiguous()
    args = capi.DsRenderArgs()
    args.batch, args.num_objects = B, N
    keep = [t, s, a, mi]
    args.translation_dev, args.size_dev, args.angle_dev, args.model_index_dev = [x.data_ptr() for x in keep]
    if no_texture:
        if class_index is None or palette is None:
            raise ValueError("no_texture rendering needs class_index and a palette")
        ci = torch.as_tensor(class_index).to(dev, torch.int64).reshape(B, N).contiguous()
        pal = torch.as_tensor(np.asarray(palette, np.float32)).reshape(-1, 3).to(dev).contiguous()
        keep += [ci, pal]
        args.class_index_dev, args.palette_dev, args.num_colors = ci.data_ptr(), pal.data_ptr(), pal.shape[0]
        args.flags |= capi.DS_RENDER_NO_TEXTURE
    if white_background:
        args.flags |= capi.DS_RENDER_WHITE_BACKGROUND
    if floors is not None:
        off = torch.as_tensor(np.asarray(floors[0], np.int32)).to(dev).contiguous()
        tri = torch.as_tensor(np.asarray(floors[1], np.float32)).reshape(-1, 9).to(dev).contiguous()
        if off.numel() != B + 1:
            raise ValueError("floor offsets hold %d entries for %d scenes" % (off.numel(), B))
        keep += [off, tri]
        args.floor_offsets_dev, args.num_floor_tris = off.data_ptr(), tri.shape[0]
        args.floor_tris_dev = tri.data_ptr() if tri.numel() else None
        if floor_texture_index is not None:
            ft = torch.as_tensor(np.asarray(floor_textures, np.uint8)).to(dev).contiguous()
            fi = torch.as_tensor(np.asarray(floor_texture_index, np.int32)).reshape(B).to(dev).contiguous()
            keep += [ft, fi]
            args.floor_textures_dev, args.num_floor_textures = ft.data_ptr(), ft.shape[0]
            args.floor_texture_size, args.floor_texture_index_dev = ft.shape[1], fi.data_ptr()
    img = torch.empty(B, camera.height, camera.width, 3, dtype=torch.uint8, device=dev)
    ids = torch.empty(B, camera.height, camera.width, dtype=torch.int64, device=dev) if return_ids else None
    if B == 0:
        return (img, ids) if return_ids else img
    args.image_dev = img.data_ptr()
    args.id_dev = None if ids is None else ids.data_ptr()
    cam = camera.struct()
    capi.check(catalog.lib.ds_render_scenes(catalog._h, C.byref(cam), C.byref(args),
                                            C.c_void_p(torch.cuda.current_stream(dev).cuda_stream)))
    return (img, ids) if return_ids else img


# ---- Pillow's resize coefficients -------------------------------------------------------------------------------

def _bicubic(x: float) -> float:
    a = -0.5
    if x < 0.0:
        x = -x
    if x < 1.0:
        return ((a + 2.0) * x - (a + 3.0)) * x * x + 1
    if x < 2.0:
        return (((x - 5) * x + 8) * x - 4) * a
    return 0.0


def _bilinear(x: float) -> float:
    if x < 0.0:
        x = -x
    if x < 1.0:
        return 1.0 - x
    return 0.0


FILTERS = {"bicubic": (_bicubic, 2.0), "bilinear": (_bilinear, 1.0)}
PRECISION_BITS = 32 - 8 - 2


def pillow_coeffs(in_size: int, out_size: int, filt: str) -> Tuple[np.ndarray, np.ndarray]:
    """Pillow's precompute_coeffs (libImaging/Resample.c) for the box (0, in_size): bounds [out, 2] int32 (first
    input index, count) and float64 weights [out, ksize], in the same double operations."""
    fn, base = FILTERS[filt]
    filterscale = scale = float(in_size) / out_size
    if filterscale < 1.0:
        filterscale = 1.0
    support = base * filterscale
    ksize = int(math.ceil(support)) * 2 + 1
    bounds = np.zeros((out_size, 2), np.int32)
    kk = np.zeros((out_size, ksize), np.float64)
    for xx in range(out_size):
        center = 0.0 + (xx + 0.5) * scale
        ww = 0.0
        ss = 1.0 / filterscale
        xmin = int(center - support + 0.5)
        if xmin < 0:
            xmin = 0
        xmax = int(center + support + 0.5)
        if xmax > in_size:
            xmax = in_size
        xmax -= xmin
        k = [0.0] * ksize
        for x in range(xmax):
            w = fn((x + xmin - center + 0.5) * ss)
            k[x] = w
            ww += w
        for x in range(xmax):
            if ww != 0.0:
                k[x] /= ww
        kk[xx] = k
        bounds[xx] = (xmin, xmax)
    return bounds, kk


def coeffs_8bpc(kk: np.ndarray) -> np.ndarray:
    """Pillow's normalize_coeffs_8bpc: round half away from zero to 22 fraction bits, truncated to int32."""
    one = float(1 << PRECISION_BITS)
    return np.array([int(-0.5 + k * one) if k < 0 else int(0.5 + k * one) for k in kk.reshape(-1)],
                    np.int32).reshape(kk.shape)


def resize_f32_host(img: np.ndarray, out_h: int, out_w: int, filt: str = "bicubic") -> np.ndarray:
    """Pillow's 'F'-mode resize of each channel of uint8 [H, W, 3] applied in numpy from the restated tables ->
    float32 [3, out_h, out_w] (not clipped)."""
    H, W, _ = img.shape
    hb, hk = pillow_coeffs(W, out_w, filt)
    vb, vk = pillow_coeffs(H, out_h, filt)
    x = img.astype(np.float32).astype(np.float64)
    tmp = np.zeros((H, out_w, 3), np.float64)
    for k in range(hk.shape[1]):
        idx = np.minimum(hb[:, 0] + k, W - 1)
        tmp = tmp + x[:, idx, :] * np.where(k < hb[:, 1], hk[:, k], 0.0)[None, :, None]
    tmp = tmp.astype(np.float32).astype(np.float64)
    out = np.zeros((out_h, out_w, 3), np.float64)
    for k in range(vk.shape[1]):
        idx = np.minimum(vb[:, 0] + k, H - 1)
        out = out + tmp[idx, :, :] * np.where(k < vb[:, 1], vk[:, k], 0.0)[:, None, None]
    return out.astype(np.float32).transpose(2, 0, 1)


def resize_u8_host(img: np.ndarray, out_h: int, out_w: int, filt: str = "bilinear") -> np.ndarray:
    """Pillow's 8-bpc resize of uint8 [H, W, 3] applied in numpy from the restated fixed-point tables -> uint8
    [out_h, out_w, 3]."""
    H, W, _ = img.shape
    hb, hk = pillow_coeffs(W, out_w, filt)
    vb, vk = pillow_coeffs(H, out_h, filt)
    hk, vk = coeffs_8bpc(hk).astype(np.int64), coeffs_8bpc(vk).astype(np.int64)
    clip8 = lambda s: np.clip(s >> PRECISION_BITS, 0, 255).astype(np.uint8)
    x = img.astype(np.int64)
    acc = np.full((H, out_w, 3), 1 << (PRECISION_BITS - 1), np.int64)
    for k in range(hk.shape[1]):
        idx = np.minimum(hb[:, 0] + k, W - 1)
        acc += x[:, idx, :] * np.where(k < hb[:, 1], hk[:, k], 0)[None, :, None]
    tmp = clip8(acc).astype(np.int64)
    acc = np.full((out_h, out_w, 3), 1 << (PRECISION_BITS - 1), np.int64)
    for k in range(vk.shape[1]):
        idx = np.minimum(vb[:, 0] + k, H - 1)
        acc += tmp[idx, :, :] * np.where(k < vb[:, 1], vk[:, k], 0)[:, None, None]
    return clip8(acc)


_TABLES: Dict[tuple, tuple] = {}


def _tables(H: int, W: int, oh: int, ow: int, filt: str, fixed: bool, dev: torch.device):
    key = (H, W, oh, ow, filt, fixed, str(dev))
    if key not in _TABLES:
        out = []
        for n, o in ((W, ow), (H, oh)):
            b, k = pillow_coeffs(n, o, filt)
            k = coeffs_8bpc(k) if fixed else k
            out += [torch.as_tensor(b).to(dev).contiguous(), torch.as_tensor(k).to(dev).contiguous()]
        _TABLES[key] = tuple(out)
    return _TABLES[key]


def _check_renders(renders: torch.Tensor) -> torch.Tensor:
    if renders.dim() != 4 or renders.shape[3] != 3 or renders.dtype != torch.uint8 or not renders.is_cuda:
        raise ValueError("renders must be a uint8 CUDA tensor [B, H, W, 3], got %s %s"
                         % (renders.dtype, tuple(renders.shape)))
    return renders.contiguous()


def clean_resize(renders: torch.Tensor, size: int = 299) -> torch.Tensor:
    """fid.clean_resize of device uint8 renders [B, H, W, 3] on the device -> float32 [B, 3, size, size], bit-exact."""
    x = _check_renders(renders)
    B, H, W, _ = x.shape
    hb, hk, vb, vk = _tables(H, W, size, size, "bicubic", False, x.device)
    out = torch.empty(B, 3, size, size, device=x.device, dtype=torch.float32)
    capi.check(capi.load().ds_resize_f32(_ptr(x), B, H, W, size, size, _ptr(hb), _ptr(hk), hk.shape[1], _ptr(vb),
                                         _ptr(vk), vk.shape[1], _ptr(out),
                                         C.c_void_p(torch.cuda.current_stream(x.device).cuda_stream)))
    return out


def ipr_resize(renders: torch.Tensor, size: int = 224) -> torch.Tensor:
    """ipr.load_image of device uint8 renders [B, H, W, 3] on the device (PIL bilinear to size^2, ToTensor, ImageNet
    Normalize) -> float32 [B, 3, size, size], bit-exact."""
    from .ipr import IMAGENET_MEAN, IMAGENET_STD
    x = _check_renders(renders)
    B, H, W, _ = x.shape
    hb, hk, vb, vk = _tables(H, W, size, size, "bilinear", True, x.device)
    ms = (C.c_float * 6)(*IMAGENET_MEAN, *IMAGENET_STD)
    out = torch.empty(B, 3, size, size, device=x.device, dtype=torch.float32)
    capi.check(capi.load().ds_resize_u8(_ptr(x), B, H, W, size, size, _ptr(hb), _ptr(hk), hk.shape[1], _ptr(vb),
                                        _ptr(vk), vk.shape[1], ms, _ptr(out),
                                        C.c_void_p(torch.cuda.current_stream(x.device).cuda_stream)))
    return out


# ---- features and metrics of device renders ---------------------------------------------------------------------

def inception_features(model, renders: torch.Tensor, batch_size: int = 64) -> torch.Tensor:
    """FID pool3 features [B, 2048] (device) of device renders, resized on the device as fid.clean_resize does."""
    out = [model(clean_resize(renders[i:i + batch_size])) for i in range(0, renders.shape[0], batch_size)]
    return torch.cat(out) if out else torch.zeros(0, 2048, device=renders.device)


def vgg16_features(model, renders: torch.Tensor, batch_size: int = 64) -> torch.Tensor:
    """VGG16 fc2 features [B, 4096] (device) of device renders, transformed on the device as ipr.load_image does."""
    out = [model(ipr_resize(renders[i:i + batch_size])) for i in range(0, renders.shape[0], batch_size)]
    return torch.cat(out) if out else torch.zeros(0, 4096, device=renders.device)


def evaluate_renders(real: torch.Tensor, fake: torch.Tensor, inception=None, vgg16=None, k: int = 3,
                     num_subsets: int = 100, max_subset_size: int = 1000, batch_size: int = 64) -> Dict[str, float]:
    """FID and KID (with an InceptionFeatures `inception`) and improved precision and recall (with a VGG16Features
    `vgg16`, k-NN radius k) of fake against real device renders, with no image leaving the device.  KID subsets are
    drawn from the global np.random as clean-fid draws them."""
    from . import fid, ipr
    out: Dict[str, float] = {}
    if inception is not None:
        fr = inception_features(inception, real, batch_size).cpu().numpy()
        ff = inception_features(inception, fake, batch_size).cpu().numpy()
        out["fid"] = fid.fid_from_features(fr, ff)
        out["kid"] = fid.kernel_distance(fr, ff, num_subsets, max_subset_size)
    if vgg16 is not None:
        vr = vgg16_features(vgg16, real, batch_size).cpu().numpy()
        vf = vgg16_features(vgg16, fake, batch_size).cpu().numpy()
        ref = ipr.Manifold(vr, ipr.manifold_radii(vr, k))
        prec, rec, _ = ipr.manifold_cover(ref, vf, ipr.manifold_radii(vf, k))
        out["precision"], out["recall"] = float(prec.mean()), float(rec.mean())
    return out
