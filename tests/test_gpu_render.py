"""GPU: the top-down renderer (ds_render_scenes) against the fp64 oracle (oracle.render_ref), its determinism and
batch independence, culling, watertight shared edges, the device resizes against PIL, renders -> features on the
device against the PNG folder path, the generation / real-scene scripts end to end, and every ABI error."""
import contextlib
import ctypes as C
import importlib.util
import io
import os
import shutil
import subprocess
import sys

import numpy as np
import pytest
import torch
from PIL import Image

from diffuscene_b200 import capi, fid as F, ipr as I
from diffuscene_b200 import render as R
from diffuscene_b200 import synthetic_meshes as SM
from oracle import inception_ref as IR
from oracle import render_ref as RR
from tests.cases_ipr import he_state_dict

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PALETTE = R.hls_palette(21)


@pytest.fixture(scope="module")
def cat_np():
    return SM.catalogue(seed=3, num_models=12, detail=2, texture_size=64)


@pytest.fixture(scope="module")
def cat(cat_np):
    c = R.MeshCatalog(cat_np)
    yield c
    c.close()


@pytest.fixture(scope="module")
def fine_np():
    return SM.catalogue(seed=4, num_models=8, detail=8, texture_size=32)


def _both(cat_obj, cat_arrays, sc, floors=True, **kw):
    fl = R.floor_triangles(sc["floors"]) if floors else None
    img, ids = R.render_scenes(cat_obj, sc["translations"], sc["sizes"], sc["angles"], sc["model_index"],
                               sc["class_index"], floors=fl, palette=PALETTE, return_ids=True, **kw)
    want = RR.render(cat_arrays, sc["translations"], sc["sizes"], sc["angles"], sc["model_index"], R.Camera(),
                     class_index=sc["class_index"], floors=fl, palette=PALETTE, **kw)
    return img.cpu().numpy(), ids.cpu().numpy(), want


def _check(got_img, got_ids, want, label):
    w_img, w_ids, amb = want
    ok = ~amb
    n_amb = int(amb.sum())
    print("%s: %d of %d pixels ambiguous (%.4f %%), %d drawn" % (label, n_amb, amb.size, 100 * amb.mean(),
                                                                  int((w_ids >= 0).sum())))
    assert amb.mean() < 1e-3
    bad = ok & (got_ids != w_ids)
    assert not bad.any(), (label, np.argwhere(bad)[:5], got_ids[bad][:5], w_ids[bad][:5])
    diff = np.abs(got_img.astype(int) - w_img.astype(int)).max(-1)
    assert diff[ok].max() <= 1, (label, np.argwhere(ok & (diff > 1))[:5])


MODES = {"textured_floor": dict(), "flat_floor": dict(no_texture=True),
         "textured_white": dict(floors=False, white_background=True),
         "flat_white": dict(floors=False, no_texture=True, white_background=True),
         "textured_black_no_floor": dict(floors=False)}


@pytest.mark.parametrize("mode", list(MODES))
def test_against_oracle(cat, cat_np, mode):
    sc = SM.scenes(6, 12, 12, seed=10)
    img, ids, want = _both(cat, cat_np, sc, **MODES[mode])
    _check(img, ids, want, mode)
    assert (ids >= 0).mean() > 0.1


def test_floor_textures_against_oracle(cat, cat_np):
    sc = SM.scenes(4, 8, 12, seed=11)
    tex = np.stack([SM.texture(np.random.default_rng(s), 32) for s in range(3)])
    fi = np.array([0, -1, 2, 1], np.int32)
    img, ids, want = _both(cat, cat_np, sc, floor_textures=tex, floor_texture_index=fi)
    _check(img, ids, want, "floor textures")


def test_fine_meshes_against_oracle(fine_np):
    """Sub-pixel triangles (8 x 8 subdivided sides, 96-segment cylinders) on small objects."""
    c = R.MeshCatalog(fine_np)
    sc = SM.scenes(4, 16, 8, seed=12)
    sc["sizes"] = sc["sizes"] * np.float32(0.4)
    for nt in (False, True):
        img, ids, want = _both(c, fine_np, sc, no_texture=nt)
        _check(img, ids, want, "fine no_texture=%s" % nt)
    c.close()


def test_deterministic_and_batch_independent(cat):
    sc = SM.scenes(4096, 12, 12, seed=13)
    fl = R.floor_triangles(sc["floors"])
    args = [sc[k] for k in ("translations", "sizes", "angles", "model_index", "class_index")]
    a = R.render_scenes(cat, *args, floors=fl, palette=PALETTE)
    b = R.render_scenes(cat, *args, floors=fl, palette=PALETTE)
    assert torch.equal(a, b)
    for k in (0, 1234, 4095):
        one = {key: sc[key][k:k + 1] for key in ("translations", "sizes", "angles", "model_index", "class_index")}
        alone = R.render_scenes(cat, *[one[key] for key in ("translations", "sizes", "angles", "model_index",
                                                             "class_index")],
                                floors=R.floor_triangles(sc["floors"][k:k + 1]), palette=PALETTE)
        assert torch.equal(alone[0], a[k]), k
    flat = R.render_scenes(cat, *args, floors=fl, palette=PALETTE, no_texture=True)
    assert torch.equal(flat[7], R.render_scenes(cat, *[x[7:8] for x in args], floors=R.floor_triangles(
        sc["floors"][7:8]), palette=PALETTE, no_texture=True)[0])


def test_empty_and_culled_objects_render_background(cat):
    """Empty slots, all-empty scenes, objects out of the view, behind far and in front of near leave only the
    background and the floor."""
    rng = np.random.default_rng(5)
    floor = [SM.floor_plan(rng)] * 3
    trans = np.array([[[20, 0.5, 0], [0, -3.0, 0], [0, 4.6, 0.5]], [[0, 0.5, 0]] * 3, [[0, 0.5, 0]] * 3], np.float32)
    size = np.full((3, 3, 3), 0.3, np.float32)
    model = np.array([[0, 1, 2], [-1, -1, -1], [-1, -1, -1]])
    ang = np.zeros((3, 3), np.float32)
    for white in (False, True):
        fl = None if white else R.floor_triangles(floor)
        img, ids = R.render_scenes(cat, trans, size, ang, model, floors=fl, white_background=white, return_ids=True)
        ids = ids.cpu().numpy()
        assert ((ids >> 32) == 3).sum() == ((ids >= 0)).sum()      # only the floor (slot N = 3), if any
        assert torch.equal(img[0], img[1]) and torch.equal(img[1], img[2])
        if white:
            assert (img == 255).all()
    img, ids = R.render_scenes(cat, trans[:0], size[:0], ang[:0], model[:0], return_ids=True)
    assert img.shape == (0, 256, 256, 3)


def test_shared_edges_are_watertight(cat):
    """A floor fanned into thin triangles whose shared edges run through pixel centres: every pixel centre inside
    the outline is covered by exactly one of them (no holes), so the floor is one solid block."""
    k = 256 / 6.2
    xs = (np.array([40.0, 200.0]) - 128) / k
    zs = (np.array([60.0, 180.0]) - 128) / k
    # the fan's centre sits on a pixel centre, so every shared edge passes through one
    c = np.array([(120.5 - 128) / k, 0, (100.5 - 128) / k])
    rim = []
    for t in np.linspace(0, 1, 33)[:-1]:
        rim.append([xs[0] + (xs[1] - xs[0]) * t, 0, zs[0]])
    for t in np.linspace(0, 1, 33)[:-1]:
        rim.append([xs[1], 0, zs[0] + (zs[1] - zs[0]) * t])
    for t in np.linspace(0, 1, 33)[:-1]:
        rim.append([xs[1] - (xs[1] - xs[0]) * t, 0, zs[1]])
    for t in np.linspace(0, 1, 33)[:-1]:
        rim.append([xs[0], 0, zs[1] - (zs[1] - zs[0]) * t])
    v = np.array([c] + rim, np.float32)
    n = len(rim)
    f = np.array([[0, 1 + i, 1 + (i + 1) % n] for i in range(n)])
    f[::2] = f[::2, ::-1]                                         # mixed windings
    fl = R.floor_triangles([(v, f)])
    _, ids = R.render_scenes(cat, np.zeros((1, 1, 3)), np.ones((1, 1, 3)), np.zeros((1, 1)),
                             -np.ones((1, 1), np.int64), floors=fl, return_ids=True)
    ids = ids[0].cpu().numpy()
    want = np.zeros((256, 256), bool)
    want[60:180, 40:200] = True
    assert np.array_equal(ids >= 0, want)


def _pil_rgb(img):
    return Image.fromarray(img)


@pytest.mark.parametrize("hw", [(256, 256), (137, 300), (96, 512)])
def test_device_resizes_bit_exact(hw, tmp_path):
    rng = np.random.default_rng(hw[0])
    imgs = rng.integers(0, 256, (5,) + hw + (3,), dtype=np.uint8)
    imgs[2] = 255
    imgs[3, :, : hw[1] // 2] = rng.integers(0, 256, 3)                     # flat regions, as renders have
    dev = torch.from_numpy(imgs).cuda()
    got = R.clean_resize(dev).cpu().numpy()
    got8 = R.ipr_resize(dev).cpu().numpy()
    for i, im in enumerate(imgs):
        want = F.clean_resize(_pil_rgb(im))
        assert np.array_equal(got[i].view(np.uint32), want.view(np.uint32)), i
        path = str(tmp_path / ("%d.png" % i))
        _pil_rgb(im).save(path)
        assert np.array_equal(got8[i].view(np.uint32), I.load_image(path).view(np.uint32)), i


@pytest.fixture(scope="module")
def extractors():
    inc = F.InceptionFeatures(IR.random_state_dict(seed=5))
    vgg = I.VGG16Features(he_state_dict(1))
    yield inc, vgg
    inc.close()
    vgg.close()


def test_features_in_memory_equal_png_path(cat, extractors, tmp_path):
    inc, vgg = extractors
    real_sc, fake_sc = SM.scenes(10, 10, 12, seed=20), SM.scenes(9, 10, 12, seed=21)
    renders = []
    for sc, name in ((real_sc, "real"), (fake_sc, "fake")):
        img = R.render_scenes(cat, sc["translations"], sc["sizes"], sc["angles"], sc["model_index"],
                              floors=R.floor_triangles(sc["floors"]))
        renders.append(img)
        os.makedirs(str(tmp_path / name))
        for i, im in enumerate(img.cpu().numpy()):
            Image.fromarray(im).save(str(tmp_path / name / ("scene_%05d_render.png" % i)))
    files = [sorted(str(tmp_path / n / f) for f in os.listdir(str(tmp_path / n))) for n in ("real", "fake")]
    bs = 4
    for r, fl in zip(renders, files):
        a = R.inception_features(inc, r, batch_size=bs).cpu().numpy()
        b = F.folder_features(fl, inc, batch_size=bs, num_workers=2)
        assert np.array_equal(a.view(np.uint32), b.view(np.uint32))
        ipr = I.IPR(batch_size=bs, num_samples=len(fl), model=vgg)
        c = R.vgg16_features(vgg, r, batch_size=bs).cpu().numpy()
        d = ipr.extract_features_from_files(fl)
        assert np.array_equal(c.view(np.uint32), d.view(np.uint32))
    np.random.seed(3)
    got = R.evaluate_renders(renders[0], renders[1], inception=inc, vgg16=vgg, num_subsets=10, batch_size=bs)
    fr, ff = (F.folder_features(fl, inc, batch_size=bs, num_workers=2) for fl in files)
    np.random.seed(3)
    assert got["fid"] == F.fid_from_features(fr, ff)
    assert got["kid"] == F.kernel_distance(fr, ff, num_subsets=10)
    ipr = I.IPR(batch_size=bs, num_samples=0, model=vgg)
    ipr.compute_manifold_ref(files[0])
    pr = ipr.precision_and_recall(files[1])
    assert (got["precision"], got["recall"]) == (pr.precision, pr.recall)
    print("in-memory metrics:", got)


def _load(name):
    spec = importlib.util.spec_from_file_location(name, os.path.join(ROOT, "scripts", name + ".py"))
    m = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(m)
    return m


def test_scripts_end_to_end(extractors, tmp_path):
    inc, vgg = extractors
    M = 42
    big = SM.catalogue(seed=6, num_models=M, detail=2, texture_size=32)
    np.savez(str(tmp_path / "mesh_catalogue.npz"), **big)
    rng = np.random.default_rng(8)
    np.savez(str(tmp_path / "catalogue.npz"), latents=rng.normal(size=(M, 32)).astype(np.float32),
             labels=np.arange(M) % 21, sizes=rng.uniform(0.2, 0.8, (M, 3)).astype(np.float32))
    # real scenes in the reference's preprocessed layout
    rooms, rows = tmp_path / "rooms", []
    sc = SM.scenes(6, 7, M, seed=30, empty=0.0)
    for b in range(6):
        n = 4 + b % 3
        cl = np.zeros((n, 23), np.float32)
        cl[np.arange(n), sc["class_index"][b, :n]] = 1
        fv, ff = sc["floors"][b]
        centroid = np.array([0.3, 0.0, -0.2], np.float32)
        d = rooms / ("Bedroom_s%d" % b)
        d.mkdir(parents=True)
        np.savez_compressed(str(d / "boxes.npz"), jids=big["jids"][sc["model_index"][b, :n]], class_labels=cl,
                            translations=sc["translations"][b, :n], sizes=sc["sizes"][b, :n],
                            angles=sc["angles"][b, :n], floor_plan_vertices=fv + centroid, floor_plan_faces=ff,
                            floor_plan_centroid=centroid)
        rows.append("s%d,train\n" % b)
    (tmp_path / "splits.csv").write_text("".join(rows))
    out = tmp_path / "real"
    _load("render_scenes").main([str(rooms), str(out), "--mesh_catalogue", str(tmp_path / "mesh_catalogue.npz")])
    real_files = sorted(str(out / ("Bedroom_s%d" % b) / "rendered_scene_256.png") for b in range(6))
    first = np.asarray(Image.open(real_files[0]))
    assert first.shape == (256, 256, 3) and (first != 0).any()
    # the same scene rendered through the API
    s0 = np.load(str(rooms / "Bedroom_s0" / "boxes.npz"))
    big_cat = R.MeshCatalog(big)
    api = R.render_scenes(big_cat, s0["translations"][None], s0["sizes"][None], s0["angles"][None],
                          sc["model_index"][:1, :4], floors=R.floor_triangles(
                              [(s0["floor_plan_vertices"] - s0["floor_plan_centroid"], s0["floor_plan_faces"])]))
    big_cat.close()
    assert np.array_equal(api[0].cpu().numpy(), first)
    # generated scenes with --render_top2down
    gen = tmp_path / "gen"
    cfg = os.path.join(ROOT, "config", "uncond", "diffusion_bedrooms_instancond_lat32_v.yaml")
    env = dict(os.environ, PYTHONNOUSERSITE="1")
    r = subprocess.run([sys.executable, os.path.join(ROOT, "scripts", "generate_diffusion.py"), cfg, str(gen),
                        "--n_sequences", "6", "--batch_size", "3", "--ddim", "--ddim_steps", "5", "--render_top2down",
                        "--catalogue", str(tmp_path / "catalogue.npz"), "--mesh_catalogue",
                        str(tmp_path / "mesh_catalogue.npz")], cwd=ROOT, env=env, capture_output=True, text=True,
                       timeout=900)
    assert r.returncode == 0, r.stderr[-3000:]
    pngs = sorted(f for f in os.listdir(str(gen)) if f.endswith("_render.png"))
    assert pngs == ["scene_%05d_render.png" % i for i in range(6)]
    npz = np.load(str(gen / "scene_00000.npz"))
    assert npz["model_index"].shape == npz["class_index"].shape
    # the metric scripts accept both sets
    wi, wv = str(tmp_path / "inc.pth"), str(tmp_path / "vgg.pth")
    torch.save(IR.random_state_dict(seed=5), wi)
    torch.save(he_state_dict(1), wv)
    buf = io.StringIO()
    with contextlib.redirect_stdout(buf):
        _load("compute_fid_scores").main([str(out), str(gen), str(tmp_path / "splits.csv"), "--inception_weights", wi,
                                          "--num_workers", "2"])
        # random-weight features of 6 + 6 unrelated scenes need not overlap, and the script's F-score divides by
        # precision + recall: the generated folder also gets copies of the real renders
        for i, f in enumerate(real_files):
            shutil.copy(f, str(gen / ("real_copy_%d.png" % i)))
        _load("improved_precision_recall").main([str(out), str(gen), str(tmp_path / "splits.csv"), "--vgg16_weights",
                                                 wv, "--num_samples", "12", "--batch_size", "4"])
        _load("render_scenes").main([str(rooms), "--mesh_catalogue", str(tmp_path / "mesh_catalogue.npz"),
                                     "--generated", str(gen), "--fid", "--ipr", "--inception_weights", wi,
                                     "--vgg16_weights", wv])
    text = buf.getvalue()
    print(text)
    for key in ("fid score:", "kid score:", "precision:", "recall:", "fid: ", "kid: "):
        assert key in text, key


def test_abi_errors(cat):
    lib = capi.load()
    sc = SM.scenes(2, 4, 12, seed=40)
    base = dict(translations=sc["translations"], sizes=sc["sizes"], angles=sc["angles"])

    def err(**kw):
        args = dict(base, model_index=sc["model_index"])
        args.update(kw)
        with pytest.raises(capi.DsError) as e:
            R.render_scenes(cat, args.pop("translations"), args.pop("sizes"), args.pop("angles"),
                            args.pop("model_index"), **args)
        return str(e.value)

    bad = sc["model_index"].copy()
    bad[1, 2] = 12
    assert "model index outside [-1, 12)" in err(model_index=bad)
    bad[1, 2] = -2
    assert "model index" in err(model_index=bad)
    cls = sc["class_index"].copy()
    cls[0, 0] = 21
    assert "palette" in err(class_index=cls, no_texture=True, palette=PALETTE, model_index=np.zeros((2, 4)))
    assert "image size" in err(camera=R.Camera(width=0))
    assert "image size" in err(camera=R.Camera(width=5000))
    assert "view volume" in err(camera=R.Camera(near=2.0, far=1.0))
    assert "objects per scene" in err(translations=np.zeros((1, 65, 3)), sizes=np.ones((1, 65, 3)),
                                      angles=np.zeros((1, 65)), model_index=-np.ones((1, 65)))
    off, tris = R.floor_triangles(sc["floors"])
    assert "floor offsets" in err(floors=(np.array([0, 4, 2]), tris))
    assert "floor offsets" in err(floors=(np.array([0, 2, len(tris) + 1]), tris))
    tex = np.zeros((2, 8, 8, 3), np.uint8)
    assert "floor texture index" in err(floors=(off, tris), floor_textures=tex, floor_texture_index=np.array([0, 2]))
    # NULL pointers and foreign handles through the raw ABI
    cam = R.Camera().struct()
    a = capi.DsRenderArgs()
    a.batch, a.num_objects = 1, 1
    s = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    assert lib.ds_render_scenes(cat._h, C.byref(cam), C.byref(a), s) == -1
    assert b"NULL image" in lib.ds_last_error()
    img = torch.empty(1, 256, 256, 3, dtype=torch.uint8, device="cuda")
    a.image_dev = img.data_ptr()
    assert lib.ds_render_scenes(cat._h, C.byref(cam), C.byref(a), s) == -1
    assert b"NULL translation" in lib.ds_last_error()
    assert lib.ds_render_scenes(cat._h, None, C.byref(a), s) == -1
    other = R.MeshCatalog(SM.catalogue(seed=1, num_models=2))
    h = other._h
    other.close()
    assert lib.ds_render_scenes(h, C.byref(cam), C.byref(a), s) == -1
    assert b"not a live mesh catalogue" in lib.ds_last_error()
    assert lib.ds_mesh_catalog_destroy(h) == -1
    vgg_like = C.c_void_p(img.data_ptr())
    assert lib.ds_render_scenes(vgg_like, C.byref(cam), C.byref(a), s) == -1
    # resize tables
    x = torch.zeros(1, 16, 16, 3, dtype=torch.uint8, device="cuda")
    out = torch.empty(1, 3, 8, 8, device="cuda")
    hb, hk = (torch.as_tensor(t).cuda() for t in R.pillow_coeffs(16, 8, "bicubic"))
    ptr = lambda t: C.c_void_p(t.data_ptr())
    hb_bad = hb.clone()
    hb_bad[3, 0] = 15
    assert lib.ds_resize_f32(ptr(x), 1, 16, 16, 8, 8, ptr(hb_bad), ptr(hk), hk.shape[1], ptr(hb), ptr(hk),
                             hk.shape[1], ptr(out), s) == -1
    assert b"horizontal coefficient bound" in lib.ds_last_error()
    assert lib.ds_resize_f32(ptr(x), 1, 16, 16, 8, 8, ptr(hb), ptr(hk), 0, ptr(hb), ptr(hk), hk.shape[1], ptr(out),
                             s) == -1
    assert lib.ds_resize_f32(ptr(x), 1, 16, 16, 8, 8000, ptr(hb), ptr(hk), hk.shape[1], ptr(hb), ptr(hk),
                             hk.shape[1], ptr(out), s) == -1
    assert lib.ds_resize_f32(None, 1, 16, 16, 8, 8, ptr(hb), ptr(hk), hk.shape[1], ptr(hb), ptr(hk), hk.shape[1],
                             ptr(out), s) == -1
    assert lib.ds_resize_u8(ptr(x), 1, 16, 16, 8, 8, ptr(hb), ptr(hk), hk.shape[1], ptr(hb), ptr(hk), hk.shape[1],
                            None, ptr(out), s) == -1
    with pytest.raises(ValueError):
        R.clean_resize(torch.zeros(1, 8, 8, 3, device="cuda"))
