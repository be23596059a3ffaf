"""CPU: the perspective camera (diffuscene_b200.render.Camera.perspective, its C struct) and the fp64 perspective
reference (tests.render_perspective_ref): pyrr's matrices, known pixels, near-plane clipping, orientation."""
import math

import numpy as np
import pytest

from diffuscene_b200 import capi
from diffuscene_b200 import render as R
from tests import render_perspective_ref as PR


def _pyrr_look_at(eye, target, up):
    # pyrr.matrix44.create_look_at, written out
    eye, target, up = (np.asarray(v, np.float64) for v in (eye, target, up))
    forward = target - eye
    forward = forward / np.linalg.norm(forward)
    side = np.cross(forward, up)
    side = side / np.linalg.norm(side)
    up = np.cross(side, forward)
    up = up / np.linalg.norm(up)
    return np.array(((side[0], up[0], -forward[0], 0.), (side[1], up[1], -forward[1], 0.),
                     (side[2], up[2], -forward[2], 0.),
                     (-np.dot(side, eye), -np.dot(up, eye), np.dot(forward, eye), 1.0)))


def _pyrr_from_bounds(left, right, bottom, top, near, far):
    # pyrr.matrix44.create_perspective_projection_from_bounds, written out
    A = (right + left) / (right - left)
    B = (top + bottom) / (top - bottom)
    C = -(far + near) / (far - near)
    D = -2. * far * near / (far - near)
    E = 2. * near / (right - left)
    F = 2. * near / (top - bottom)
    return np.array(((E, 0., 0., 0.), (0., F, 0., 0.), (A, B, C, -1.), (0., 0., D, 0.)))


def test_reference_camera():
    c = R.REFERENCE_PERSPECTIVE
    assert c.projection == "perspective" and (c.width, c.height) == (512, 512)
    assert c.eye == (-0.10923499, 1.9325259, -7.19009) and c.target == (0, 0, 0) and c.up == (0, 1, 0)
    ymax = 0.1 * math.tan(45.0 * math.pi / 360.0)
    assert c.bottom == pytest.approx(ymax) and c.top == pytest.approx(-ymax) and c.right == pytest.approx(ymax)
    assert (c.near, c.far) == (0.1, 1000.0)
    w = R.Camera.perspective((0, 1, 5), width=640, height=320)
    assert w.right == pytest.approx(2 * w.bottom)
    s = c.struct()
    assert s.projection == capi.DS_RENDER_PERSPECTIVE == 1
    assert R.Camera().struct().projection == capi.DS_RENDER_ORTHOGRAPHIC == 0
    with pytest.raises(ValueError):
        R.Camera(projection="fisheye").struct()


def test_struct_layout_unchanged():
    # projection took the place of reserved[0]: size and offsets stay as they were
    import ctypes as C
    assert C.sizeof(capi.DsRenderCamera) == 4 * (9 + 6 + 2 + 4)
    assert capi.DsRenderCamera.projection.offset == 4 * (9 + 6 + 2)


@pytest.mark.parametrize("cam", [R.REFERENCE_PERSPECTIVE, R.Camera.perspective((1.0, 3.0, 2.0), (0.2, 0.0, -0.5),
                                                                               fovy=60, width=300, height=200,
                                                                               near=0.5, far=20.0)])
def test_pixel_map_equals_pyrr(cam):
    rng = np.random.default_rng(0)
    p = rng.uniform(-3, 3, (100, 3))
    clip = np.c_[p, np.ones(100)] @ _pyrr_look_at(cam.eye, cam.target, cam.up) @ _pyrr_from_bounds(
        cam.left, cam.right, cam.bottom, cam.top, cam.near, cam.far)
    ndc = clip[:, :3] / clip[:, 3:]
    want = np.c_[(ndc[:, 0] + 1) * cam.width / 2, (ndc[:, 1] + 1) * cam.height / 2, clip[:, 3]]
    M = PR.pixel_map(cam)
    h = p @ M[:, :3].T + M[:, 3]
    got = np.c_[h[:, :2] / h[:, 2:], h[:, 2]]
    np.testing.assert_allclose(got, want, rtol=1e-12, atol=1e-9)
    # depth is the distance along the view direction
    f = np.subtract(cam.target, cam.eye)
    np.testing.assert_allclose(h[:, 2], (p - cam.eye) @ (f / np.linalg.norm(f)), atol=1e-12)


def _floor_only(tris, cam, **kw):
    tris = np.asarray(tris, np.float32).reshape(-1, 3, 3)
    floors = (np.array([0, len(tris)], np.int32), tris)
    cat = {k: np.zeros((0,) + s, dt) for k, s, dt in (("vertices", (3,), np.float32), ("faces", (3,), np.int32),
                                                      ("uvs", (3, 2), np.float32))}
    cat.update(vertex_offsets=np.zeros(1, np.int32), face_offsets=np.zeros(1, np.int32))
    return PR.render(cat, np.zeros((1, 0, 3)), np.zeros((1, 0, 3)), np.zeros((1, 0)), np.zeros((1, 0), np.int64),
                     cam, floors=floors, **kw)


def test_square_at_known_depth_lands_on_predicted_pixels():
    # 90 degrees: x_ndc = x / depth.  The square [0, 1] x [0, 1] at depth 2 covers x_ndc, y_ndc in [0, 0.5]: columns
    # 32..47 and, the image being upright (row 0 at the top), rows 16..31
    cam = R.Camera.perspective((0, 0, 0), (0, 0, -1), (0, 1, 0), fovy=90.0, width=64, height=64)
    sq = [[[0, 0, -2], [1, 0, -2], [1, 1, -2]], [[0, 0, -2], [1, 1, -2], [0, 1, -2]]]
    img, ids, amb = _floor_only(sq, cam)
    want = np.zeros((64, 64), bool)
    want[16:32, 32:48] = True
    assert np.array_equal(ids[0] >= 0, want)
    assert amb[0].sum() <= 16                          # only the diagonal shared by both halves runs through centres
    # flat face towards the eye: the pixel straight ahead is fully lit
    img2, _, _ = _floor_only([[[-1, -1, -2], [1, -1, -2], [0, 1, -2]]], cam)
    assert (img2[0, 32, 32] == 255).all()


def test_face_crossing_near_is_cut_at_near():
    near = 1.5
    h = np.array([[[0.0, 0.0, 3.0], [2.0, 0.0, 0.5], [0.0, 2.0, -1.0]],      # one corner in front
                  [[0.0, 0.0, 3.0], [2.0, 0.0, 2.0], [0.0, 2.0, -1.0]],      # two corners in front
                  [[0.0, 0.0, 1.0], [2.0, 0.0, 0.5], [0.0, 2.0, -1.0]],      # none
                  [[0.0, 0.0, 3.0], [2.0, 0.0, 2.0], [0.0, 2.0, 1.6]]])      # all
    par, scr, inv, bar, kind = PR.clip_faces(h, near)
    assert par.tolist() == [3, 0, 1, 1]
    for s in range(len(par)):
        dep = bar[s] @ h[par[s], :, 2]                                       # corner depths in the original face
        np.testing.assert_allclose(1.0 / inv[s], dep, rtol=1e-12)
        assert (dep >= near - 1e-12).all()
        clipped = np.abs(bar[s] - np.eye(3)[:, None, :]).sum(-1).min(0) > 0  # corners that are no original corner
        np.testing.assert_allclose(dep[clipped], near, rtol=1e-12)
        hom = bar[s] @ h[par[s]]
        np.testing.assert_allclose(scr[s], hom[:, :2] / hom[:, 2:], rtol=1e-12)
    # the two halves of the clipped quad cover its area once
    area = lambda p: 0.5 * abs((p[1, 0] - p[0, 0]) * (p[2, 1] - p[0, 1]) - (p[2, 0] - p[0, 0]) * (p[1, 1] - p[0, 1]))
    assert (kind[2:] == PR.INNER).sum() == 2 and area(scr[2]) > 0 and area(scr[3]) > 0


def test_floor_crossing_near_plane_draws_only_depth_above_near():
    # camera 1 above a large floor, looking along -z; the floor reaches behind the eye.  A pixel centre on row r
    # sees the floor at depth 1 / -ty, ty = 1 - (2 r + 1) / H (90 degrees): drawn exactly where near <= depth
    near, H = 1.5, 64
    cam = R.Camera.perspective((0, 1, 0), (0, 1, -1), (0, 1, 0), fovy=90.0, width=H, height=H, near=near,
                               far=1000.0)
    fl = [[[-200, 0, 10], [200, 0, 10], [200, 0, -40]], [[-200, 0, 10], [200, 0, -40], [-200, 0, -40]]]
    img, ids, amb = _floor_only(fl, cam)
    r = np.arange(H)
    ty = 1 - (2 * r + 1) / H
    with np.errstate(divide="ignore"):
        depth = np.where(ty < 0, -1 / ty, np.inf)
    want_rows = (depth >= near) & (depth <= 40)
    drawn = ids[0] >= 0
    ok = ~amb[0]
    assert np.array_equal(drawn[ok], np.broadcast_to(want_rows[:, None], (H, H))[ok])
    assert want_rows.sum() > 10 and amb[0].mean() < 0.05


def test_higher_objects_land_on_smaller_rows():
    cam = R.REFERENCE_PERSPECTIVE
    M = PR.pixel_map(cam)
    p = np.array([[0.0, 0.0, 0.0], [0.0, 1.0, 0.0]])
    h = p @ M[:, :3].T + M[:, 3]
    rows = h[:, 1] / h[:, 2]
    assert rows[1] < rows[0]
