"""GPU: perspective rendering (ds_render_scenes with DS_RENDER_PERSPECTIVE) against the fp64 perspective reference
(tests.render_perspective_ref) with the reference driver's camera, a camera inside the room whose near plane cuts
the floor and the furniture, orientation, determinism and batch independence, and the new ABI errors."""
import ctypes as C

import numpy as np
import pytest
import torch

from diffuscene_b200 import capi
from diffuscene_b200 import render as R
from diffuscene_b200 import synthetic_meshes as SM
from tests import render_perspective_ref as PR
from tests.test_gpu_render import MODES, PALETTE

pytestmark = pytest.mark.gpu
CAM = R.REFERENCE_PERSPECTIVE
# Seen from the side, the synthetic furniture shows coplanar faces (parts flush with each other) and grazing
# silhouettes, whose pixels are depth ties the top-down view never meets: they are flagged ambiguous, so the share
# of ambiguous pixels is bounded looser than top-down's 0.1 %.
MAX_AMBIGUOUS = 5e-3


def _check(got_img, got_ids, want, label, max_ambiguous=MAX_AMBIGUOUS):
    w_img, w_ids, amb = want
    ok = ~amb
    print("%s: %d of %d pixels ambiguous (%.4f %%), %d drawn" % (label, int(amb.sum()), amb.size, 100 * amb.mean(),
                                                                  int((w_ids >= 0).sum())))
    assert amb.mean() < max_ambiguous
    bad = ok & (got_ids != w_ids)
    assert not bad.any(), (label, int(bad.sum()), np.argwhere(bad)[:5], got_ids[bad][:5], w_ids[bad][:5])
    diff = np.abs(got_img.astype(int) - w_img.astype(int)).max(-1)
    assert diff[ok].max() <= 1, (label, int((ok & (diff > 1)).sum()), np.argwhere(ok & (diff > 1))[:5])


@pytest.fixture(scope="module")
def cat_np():
    return SM.catalogue(seed=3, num_models=12, detail=2, texture_size=64)


@pytest.fixture(scope="module")
def cat(cat_np):
    c = R.MeshCatalog(cat_np)
    yield c
    c.close()


def _both(cat_obj, cat_arrays, sc, camera, floors=True, **kw):
    fl = R.floor_triangles(sc["floors"]) if floors else None
    img, ids = R.render_scenes(cat_obj, sc["translations"], sc["sizes"], sc["angles"], sc["model_index"],
                               sc["class_index"], floors=fl, palette=PALETTE, return_ids=True, camera=camera, **kw)
    want = PR.render(cat_arrays, sc["translations"], sc["sizes"], sc["angles"], sc["model_index"], camera,
                     class_index=sc["class_index"], floors=fl, palette=PALETTE, **kw)
    return img.cpu().numpy(), ids.cpu().numpy(), want


@pytest.mark.parametrize("mode", list(MODES))
def test_against_oracle(cat, cat_np, mode):
    sc = SM.scenes(4, 12, 12, seed=10)
    img, ids, want = _both(cat, cat_np, sc, CAM, **MODES[mode])
    _check(img, ids, want, "perspective " + mode)
    assert img.shape == (4, 512, 512, 3) and (ids >= 0).mean() > 0.05


def test_floor_textures_against_oracle(cat, cat_np):
    sc = SM.scenes(4, 8, 12, seed=11)
    tex = np.stack([SM.texture(np.random.default_rng(s), 32) for s in range(3)])
    fi = np.array([0, -1, 2, 1], np.int32)
    img, ids, want = _both(cat, cat_np, sc, CAM, floor_textures=tex, floor_texture_index=fi)
    _check(img, ids, want, "perspective floor textures")


def test_near_plane_cuts_floor_and_objects(cat, cat_np):
    """A camera inside the room, near = 1.5: floor and furniture faces cross the near plane.  A table right in front
    of the camera shows its flush parts over about 1 % of the pixels, all flagged ambiguous."""
    cam = R.Camera.perspective((0.3, 1.2, 0.4), (-0.5, 0.2, -2.0), near=1.5, far=50.0)
    sc = SM.scenes(3, 12, 12, seed=14)
    h = PR.pixel_map(cam)
    crossing = 0
    for b in range(3):
        fv, ff = sc["floors"][b]
        d = np.asarray(fv, np.float64)[ff] @ h[2, :3] + h[2, 3]
        crossing += int(((d.min(1) < 1.5) & (d.max(1) >= 1.5)).sum())
    assert crossing > 0
    for nt in (False, True):
        img, ids, want = _both(cat, cat_np, sc, cam, no_texture=nt)
        _check(img, ids, want, "near plane no_texture=%s" % nt, max_ambiguous=2e-2)
        assert (ids >= 0).mean() > 0.05


def test_higher_objects_appear_higher(cat):
    tr = np.array([[[0.0, 0.4, 0.0]], [[0.0, 1.4, 0.0]]], np.float32)
    sz = np.full((2, 1, 3), 0.3, np.float32)
    _, ids = R.render_scenes(cat, tr, sz, np.zeros((2, 1)), np.zeros((2, 1), np.int64), camera=CAM,
                             return_ids=True)
    rows = [np.flatnonzero((i >= 0).any(1)).mean() for i in ids.cpu().numpy()]
    assert rows[1] < rows[0] - 10


def test_deterministic_and_batch_independent(cat):
    sc = SM.scenes(4096, 12, 12, seed=13)
    fl = R.floor_triangles(sc["floors"])
    keys = ("translations", "sizes", "angles", "model_index", "class_index")
    args = [sc[k] for k in keys]
    a = R.render_scenes(cat, *args, floors=fl, palette=PALETTE, camera=CAM)
    b = R.render_scenes(cat, *args, floors=fl, palette=PALETTE, camera=CAM)
    assert torch.equal(a, b)
    for k in (0, 1234, 4095):
        alone = R.render_scenes(cat, *[x[k:k + 1] for x in args], floors=R.floor_triangles(sc["floors"][k:k + 1]),
                                palette=PALETTE, camera=CAM)
        assert torch.equal(alone[0], a[k]), k


def test_abi_errors(cat):
    sc = SM.scenes(2, 4, 12, seed=40)

    def err(camera):
        with pytest.raises(capi.DsError) as e:
            R.render_scenes(cat, sc["translations"], sc["sizes"], sc["angles"], sc["model_index"], camera=camera)
        return str(e.value)

    zero = R.Camera.perspective((0, 1, 5))
    zero.near = 0.0
    assert "near > 0" in err(zero)
    assert "view volume" in err(R.Camera.perspective((0, 1, 5), near=-1.0))
    flat = R.Camera.perspective((0, 1, 5))
    flat.left = flat.right
    assert "view volume" in err(flat)
    flat = R.Camera.perspective((0, 1, 5))
    flat.top = flat.bottom
    assert "view volume" in err(flat)
    # an unknown projection value through the raw ABI
    cam = CAM.struct()
    cam.projection = 2
    a = capi.DsRenderArgs()
    img = torch.empty(1, 512, 512, 3, dtype=torch.uint8, device="cuda")
    a.batch, a.num_objects, a.image_dev = 1, 0, img.data_ptr()
    lib = capi.load()
    assert lib.ds_render_scenes(cat._h, C.byref(cam), C.byref(a), C.c_void_p(torch.cuda.current_stream()
                                                                               .cuda_stream)) == -1
    assert b"unknown projection 2" in lib.ds_last_error()
    cam.projection = 0                                                # the zeroed field keeps the orthographic path
    assert lib.ds_render_scenes(cat._h, C.byref(cam), C.byref(a), C.c_void_p(torch.cuda.current_stream()
                                                                               .cuda_stream)) == 0
