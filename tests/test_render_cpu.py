"""CPU: the top-down renderer's host side and its fp64 oracle (oracle.render_ref): the camera map on hand-placed
squares, placed-vertex bounds against oracle.scene_eval_ref, the OBJ / MTL parser on hand-written files, the packer
round trip, the seaborn 'hls' palette against hand-computed colorsys values, Pillow's resize coefficients restated on
the host against PIL itself, and the catalogue checks that run before any device is touched."""
import colorsys
import ctypes as C
import os

import numpy as np
import pytest
from PIL import Image

from diffuscene_b200 import capi, fid
from diffuscene_b200 import render as R
from diffuscene_b200 import synthetic_meshes as SM
from diffuscene_b200.evaluate import model_footprint
from oracle import render_ref as RR
from oracle import scene_eval_ref as SE
from tests.cases_fid import render_like as render_like_fid
from tests.cases_ipr import render_like as render_like_ipr

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def unit_box_catalogue():
    v, f = SM.box(1)
    return {"vertex_offsets": np.array([0, len(v)], np.int32), "vertices": v.astype(np.float32),
            "face_offsets": np.array([0, len(f)], np.int32), "faces": f.astype(np.int32),
            "uvs": np.full((len(f), 3, 2), np.nan, np.float32), "raw_half": np.ones((1, 3)),
            "raw_aabb": np.array([[-1.0, -1, -1, 1, 1, 1]]), "kd": np.ones((1, 3), np.float32),
            "textures": np.full((1, 4, 4, 3), 255, np.uint8), "jids": np.array(["box"])}


def test_camera_map_formula():
    m = RR.pixel_map(R.Camera())
    k = 256 / 6.2
    want = np.array([[k, 0, 0, 128], [0, 0, k, 128], [0, -1, 0, 4]])   # x -> column, z -> row, depth = 4 - y
    np.testing.assert_allclose(m, want, rtol=0, atol=1e-12)


@pytest.mark.parametrize("block", [(100, 119, 30, 59), (0, 255, 200, 201), (7, 7, 128, 140)])
def test_camera_map_places_squares(block):
    """A flat box whose sides lie on pixel boundaries covers exactly the predicted pixel block."""
    c0, c1, r0, r1 = block
    s, k = 3.1, 256 / 6.2
    x0, x1 = (c0 - 128) / k, (c1 + 1 - 128) / k
    z0, z1 = (r0 - 128) / k, (r1 + 1 - 128) / k
    trans = np.array([[[(x0 + x1) / 2, 0.5, (z0 + z1) / 2]]], np.float32)
    size = np.array([[[(x1 - x0) / 2, 0.05, (z1 - z0) / 2]]], np.float32)
    img, ids, amb = RR.render(unit_box_catalogue(), trans, size, np.zeros((1, 1)), np.zeros((1, 1)), R.Camera())
    want = np.zeros((256, 256), bool)
    want[r0:r1 + 1, c0:c1 + 1] = True
    assert not (amb[0] & ~want).any()            # only the top's diagonal may pass through a pixel centre
    assert np.array_equal(ids[0] >= 0, want)
    assert s == R.ROOM_SIDE


def test_depth_range_is_clipped_per_pixel():
    """Objects beyond far (depth 6) or nearer than near (0.1) leave the background."""
    cat = unit_box_catalogue()
    size = np.full((1, 3, 3), 0.2, np.float32)
    trans = np.array([[[0, -2.5, 0], [1, 4.5, 1], [-1, 0.5, -1]]], np.float32)   # depths 6.5, -0.5, 3.5
    _, ids, _ = RR.render(cat, trans, size, np.zeros((1, 3)), np.zeros((1, 3)), R.Camera())
    assert set(np.unique(ids[0] >> 32)) == {-1, 2}


def test_placed_bounds_match_scene_eval_ref():
    rng = np.random.default_rng(4)
    for _ in range(20):
        v = rng.normal(size=(50, 3)) * rng.uniform(0.2, 2, 3) + rng.normal(size=3)
        half, aabb, _ = model_footprint(v, SE.box_vertices(np.ptp(v, 0) / 2) + v.min(0) + np.ptp(v, 0) / 2)
        size = rng.uniform(0.1, 1.5, 3).astype(np.float32)
        trans = rng.normal(size=3).astype(np.float32)
        ang = np.float32(rng.uniform(-np.pi, np.pi))
        placed = RR.place(v, size, trans, ang, half, aabb)
        got = np.concatenate([placed.min(0), placed.max(0)])
        want = SE.place_bounds(v, half, size, trans, ang)
        assert np.array_equal(got, want), (got, want)


OBJ = """# hand-written test model
mtllib test.mtl
v 0 0 0
v 1 0 0
v 1 1 0
v 0 1 0
v 0 0 1
vt 0 0
vt 1 0
vt 1 1
vt 0 1
vn 0 0 1
usemtl wood
f 1/1/1 2/2/1 3/3/1 4/4/1
f -5/-4 -3/-2 -1/-1
f 1//1 2//1 5//1
f 5 4 3 2 1
"""

MTL = """newmtl empty
Ka 1 1 1
newmtl wood
Kd 0.25 0.5 0.75
map_Kd texture.png
"""


def test_obj_mtl_parser(tmp_path):
    (tmp_path / "m.obj").write_text(OBJ)
    (tmp_path / "test.mtl").write_text(MTL)
    v, f, uv, kd = R.parse_obj(str(tmp_path / "m.obj"))
    assert v.shape == (5, 3) and v.dtype == np.float64
    # quad fanned (0, 1, 2), (0, 2, 3); negative indices -5, -3, -1 -> 0, 2, 4; no-UV triangle; pentagon -> 3 triangles
    assert f.tolist() == [[0, 1, 2], [0, 2, 3], [0, 2, 4], [0, 1, 4], [4, 3, 2], [4, 2, 1], [4, 1, 0]]
    assert uv[0].tolist() == [[0, 0], [1, 0], [1, 1]] and uv[1].tolist() == [[0, 0], [1, 1], [0, 1]]
    assert uv[2].tolist() == [[0, 0], [1, 1], [0, 1]]                     # -4, -2, -1 of 4 texture coordinates
    assert np.isnan(uv[3:]).all()
    assert kd.tolist() == [0.25, 0.5, 0.75]
    mats = R.parse_mtl(str(tmp_path / "test.mtl"))
    assert mats["wood"]["map_Kd"] == "texture.png" and mats["empty"]["Kd"] is None
    (tmp_path / "bad.obj").write_text("v 0 0 0\nf 1 2 3\n")
    with pytest.raises(ValueError):
        R.parse_obj(str(tmp_path / "bad.obj"))


def _write_model(d, rng, with_texture):
    d.mkdir(parents=True)
    v, f = SM.cylinder(7, 1) if with_texture else SM.box(2)
    v = v * rng.uniform(0.5, 2, 3)
    lines = ["v %r %r %r" % tuple(float(x) for x in p) for p in v]
    lines += ["vt %r %r" % tuple(float(x) for x in t) for t in rng.uniform(0, 1, (len(v), 2))]
    lines += ["f %d/%d %d/%d %d/%d" % (a + 1, a + 1, b + 1, b + 1, c + 1, c + 1) for a, b, c in f]
    (d / "raw_model.obj").write_text("\n".join(lines) + "\n")
    lo, hi = v.min(0), v.max(0)
    np.save(str(d / "bbox_vertices.npy"), SE.box_vertices((hi - lo) / 2) + (lo + hi) / 2)
    if with_texture:
        Image.fromarray(rng.integers(0, 256, (40, 70, 3), dtype=np.uint8)).save(str(d / "texture.png"))
    return v, f


def test_packer_round_trip(tmp_path):
    import importlib.util
    rng = np.random.default_rng(2)
    jids = ["a-1", "b-2", "c-3"]
    models = [_write_model(tmp_path / "models" / j, rng, i != 1) for i, j in enumerate(jids)]
    (tmp_path / "jids.txt").write_text("\n".join(jids) + "\n")
    spec = importlib.util.spec_from_file_location("pmc", os.path.join(ROOT, "scripts", "pack_mesh_catalogue.py"))
    S = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(S)
    out = str(tmp_path / "mesh_catalogue.npz")
    S.main([str(tmp_path / "models"), str(tmp_path / "jids.txt"), out, "--texture_size", "16"])
    cat = np.load(out)
    assert [str(j) for j in cat["jids"]] == jids
    assert cat["textures"].shape == (3, 16, 16, 3) and (cat["textures"][1] == 255).all()
    for m, (v, f) in enumerate(models):
        vo, fo = cat["vertex_offsets"][m:m + 2], cat["face_offsets"][m:m + 2]
        assert np.array_equal(cat["vertices"][vo[0]:vo[1]], v.astype(np.float32))
        assert np.array_equal(cat["faces"][fo[0]:fo[1]], f)
        half, aabb, _ = model_footprint(v, np.load(str(tmp_path / "models" / jids[m] / "bbox_vertices.npy")))
        assert np.array_equal(cat["raw_half"][m], half) and np.array_equal(cat["raw_aabb"][m], aabb)
    tex = np.asarray(Image.open(str(tmp_path / "models" / "a-1" / "texture.png")).resize((16, 16), Image.BILINEAR))
    assert np.array_equal(cat["textures"][0], tex)


def test_palette_matches_hand_computed_hls():
    # colorsys.hls_to_rgb(h, 0.6, 0.65) by hand: m2 = 0.6 + 0.65 - 0.39 = 0.86, m1 = 1.2 - 0.86 = 0.34, hues 0.01 + i / 4
    want = np.array([[0.86, 0.3712, 0.34], [0.5688, 0.86, 0.34], [0.34, 0.8288, 0.86], [0.6312, 0.34, 0.86]])
    np.testing.assert_allclose(R.hls_palette(4), want, rtol=0, atol=1e-12)
    p = R.hls_palette(21)
    assert p.shape == (21, 3) and np.allclose(p[0], colorsys.hls_to_rgb(0.01, 0.6, 0.65))


IMAGE_CASES = [("random", 256, 256), ("random", 137, 300), ("random", 512, 96), ("random", 17, 23),
               ("random", 299, 224), ("render", 256, 256), ("render", 224, 224)]


def _image(kind, h, w, seed):
    if kind == "random":
        return np.random.default_rng(seed).integers(0, 256, (h, w, 3), dtype=np.uint8)
    img = np.asarray(render_like_fid(seed, size=h).convert("RGB")) if seed % 2 else render_like_ipr(1, h, seed)[0]
    return np.ascontiguousarray(img[:, :w])


@pytest.mark.parametrize("kind,h,w", IMAGE_CASES)
def test_host_coefficients_bit_identical_to_pil(kind, h, w):
    for seed in (1, 2):
        img = _image(kind, h, w, seed)
        got = R.resize_f32_host(img, 299, 299).clip(0, 255)
        want = fid.clean_resize(Image.fromarray(img))
        assert np.array_equal(got.view(np.uint32), want.view(np.uint32))
        got8 = R.resize_u8_host(img, 224, 224)
        want8 = np.asarray(Image.fromarray(img).resize((224, 224), Image.BILINEAR))
        assert np.array_equal(got8, want8)


def test_pillow_coeff_tables():
    b, k = R.pillow_coeffs(256, 299, "bicubic")
    assert k.shape == (299, 5) and b[0].tolist() == [0, 2] and b[-1].tolist() == [254, 2]
    np.testing.assert_allclose(k.sum(1), 1.0, rtol=0, atol=1e-15)
    b, k = R.pillow_coeffs(256, 224, "bilinear")
    k8 = R.coeffs_8bpc(k)
    assert k8.dtype == np.int32 and np.abs(k8.sum(1) - (1 << 22)).max() <= 2


def test_floor_triangles_csr():
    off, tris = R.floor_triangles([None, SM.floor_plan(np.random.default_rng(0)), None])
    assert off[0] == off[1] == 0 and off[2] == off[3] == len(tris) and tris.shape[1:] == (3, 3)


def test_catalogue_checks_run_before_the_device():
    """Malformed catalogues are refused with DS_ERR_INVALID before any device is touched."""
    lib = capi.load()
    cat = unit_box_catalogue()
    arr = lambda k, dt: np.ascontiguousarray(cat[k], dt)
    base = dict(vo=arr("vertex_offsets", np.int32), v=arr("vertices", np.float32), fo=arr("face_offsets", np.int32),
                f=arr("faces", np.int32), uv=arr("uvs", np.float32), h=arr("raw_half", np.float64),
                bb=arr("raw_aabb", np.float64), kd=arr("kd", np.float32), t=arr("textures", np.uint8))

    def create(ts=4, **over):
        a = dict(base, **over)
        h = C.c_void_p()
        ptr = lambda x: None if x is None else C.c_void_p(x.ctypes.data)
        rc = lib.ds_mesh_catalog_create(1, *[ptr(a[k]) for k in ("vo", "v", "fo", "f", "uv", "h", "bb", "kd", "t")],
                                        ts, 0, C.byref(h))
        return rc, lib.ds_last_error().decode()

    bad_faces = base["f"].copy()
    bad_faces[3, 1] = 99
    assert create(f=bad_faces)[0] == -1 and "vertex index 99" in create(f=bad_faces)[1]
    neg = base["f"].copy()
    neg[0, 0] = -1
    assert create(f=neg)[0] == -1
    assert create(ts=0)[0] == -1 and create(ts=5000)[0] == -1
    assert create(vo=np.array([1, 8], np.int32))[0] == -1
    assert create(h=np.array([[1.0, 0.0, 1.0]]))[0] == -1
    assert create(kd=None)[0] == -1
    assert lib.ds_mesh_catalog_create(1, *[None] * 9, 4, 0, None) == -1
    assert lib.ds_mesh_catalog_destroy(C.c_void_p(12345)) == -1
    assert "not a live mesh catalogue" in lib.ds_last_error().decode()
