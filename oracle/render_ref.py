"""fp64 numpy rasterizer of the rules diffuscene_b200.render follows (the tests' reference for ds_render_scenes).

Camera: pyrr's create_look_at(eye, target, up) and orthogonal_projection(left, right, bottom, top, near, far), the
OpenGL viewport, and array row r = framebuffer row r counted from y_ndc = -1.  Placement: scene_synthesis/utils.py:
114-142 (scale = size / raw_half, centre on the scaled raw AABB, v . R + t with float32-rounded cos / sin).
Visibility: pixel centres, top-left fill rule, no culling, nearest depth in [near, far], ties to the lower
(slot, face).  Shading: ambient + diffuse * |n . l| with a point light at the eye.

Every pixel also gets an `ambiguous` flag: its centre lies within `edge_tol` pixels of an edge of a triangle that
could be visible there, within `depth_tol` of the clip range, or two different triangles are within `depth_tol` of
the nearest depth.  Only there may an fp32 rasterizer legitimately pick another triangle.
"""
from __future__ import annotations

import numpy as np

AMBIENT, DIFFUSE = 0.35, 0.65
FACE_SHIFT = 32


def look_at(eye, target, up) -> np.ndarray:
    """pyrr.matrix44.create_look_at (row-vector convention: p_view = [p, 1] @ M)."""
    eye, target, up = (np.asarray(v, np.float64) for v in (eye, target, up))
    f = target - eye
    f /= np.linalg.norm(f)
    s = np.cross(f, up)
    s /= np.linalg.norm(s)
    u = np.cross(s, f)
    u /= np.linalg.norm(u)
    return np.array([[s[0], u[0], -f[0], 0.0], [s[1], u[1], -f[1], 0.0], [s[2], u[2], -f[2], 0.0],
                     [-s.dot(eye), -u.dot(eye), f.dot(eye), 1.0]])


def orthogonal_projection(left, right, bottom, top, near, far) -> np.ndarray:
    """pyrr.matrix44.create_orthogonal_projection (row-vector convention)."""
    rml, tmb, fmn = right - left, top - bottom, far - near
    return np.array([[2.0 / rml, 0, 0, 0], [0, 2.0 / tmb, 0, 0], [0, 0, -2.0 / fmn, 0],
                     [-(right + left) / rml, -(top + bottom) / tmb, -(far + near) / fmn, 1.0]])


def pixel_map(cam) -> np.ndarray:
    """3 x 4 fp64 map world -> (pixel x, array row, depth along the view direction)."""
    V = look_at(cam.eye, cam.target, cam.up)
    P = orthogonal_projection(cam.left, cam.right, cam.bottom, cam.top, cam.near, cam.far)
    VP = V @ P                                     # [x y z 1] @ VP = clip coordinates (w = 1)
    out = np.zeros((3, 4))
    out[0] = np.r_[VP[:3, 0], VP[3, 0]] * (cam.width / 2.0)
    out[0, 3] += cam.width / 2.0
    out[1] = np.r_[VP[:3, 1], VP[3, 1]] * (cam.height / 2.0)
    out[1, 3] += cam.height / 2.0
    out[2] = -np.r_[V[:3, 2], V[3, 2]]             # depth = -z_view
    return out


def place(vertices, size, trans, angle, raw_half, raw_aabb) -> np.ndarray:
    """World vertices [V, 3] of a model placed as scene_synthesis/utils.py:114-142 places it."""
    v = np.asarray(vertices, np.float64)
    k = np.asarray(size, np.float32).astype(np.float64) / np.asarray(raw_half, np.float64)
    bb = np.asarray(raw_aabb, np.float64)
    centroid = (bb[:3] * k + bb[3:] * k) / 2
    th = np.float32(angle)
    c, s = np.float64(np.cos(th)), np.float64(np.sin(th))
    R = np.array([[c, 0, -s], [0, 1, 0], [s, 0, c]])
    return (v * k - centroid).dot(R) + np.asarray(trans, np.float32).astype(np.float64)


def _bilinear(tex, u, v):
    T = tex.shape[0]
    tx, ty = u * T - 0.5, (1.0 - v) * T - 0.5
    x0, y0 = np.floor(tx), np.floor(ty)
    ax, ay = (tx - x0)[..., None], (ty - y0)[..., None]
    x0, y0 = x0.astype(np.int64) % T, y0.astype(np.int64) % T
    x1, y1 = (x0 + 1) % T, (y0 + 1) % T
    t = tex.astype(np.float64)
    top = t[y0, x0] + ax * (t[y0, x1] - t[y0, x0])
    bot = t[y1, x0] + ax * (t[y1, x1] - t[y1, x0])
    return (top + ay * (bot - top)) / 255.0


def render(cat, translations, sizes, angles, model_index, cam, class_index=None, floors=None, no_texture=False,
           white_background=False, palette=None, floor_textures=None, floor_texture_index=None, edge_tol=1e-3,
           depth_tol=1e-4):
    """(image uint8 [B, H, W, 3], ids int64 [B, H, W], ambiguous bool [B, H, W]) of a batch; `cat` is the dict of
    mesh_catalogue.npz arrays, the other arguments as diffuscene_b200.render.render_scenes takes them."""
    translations = np.asarray(translations, np.float32)
    B, N = translations.shape[:2]
    sizes = np.asarray(sizes, np.float32).reshape(B, N, 3)
    angles = np.asarray(angles, np.float32).reshape(B, N)
    model_index = np.asarray(model_index, np.int64).reshape(B, N)
    Mp = pixel_map(cam)
    H, W = cam.height, cam.width
    img = np.zeros((B, H, W, 3), np.uint8)
    ids = np.full((B, H, W), -1, np.int64)
    amb = np.zeros((B, H, W), bool)
    vo, fo = np.asarray(cat["vertex_offsets"]), np.asarray(cat["face_offsets"])
    for b in range(B):
        world, tri_id, tri_slot, tri_face, tri_model = [], [], [], [], []
        for n in range(N):
            m = int(model_index[b, n])
            if m < 0:
                continue
            v = np.asarray(cat["vertices"][vo[m]:vo[m + 1]], np.float64)
            f = np.asarray(cat["faces"][fo[m]:fo[m + 1]], np.int64)
            wv = place(v, sizes[b, n], translations[b, n], angles[b, n], cat["raw_half"][m], cat["raw_aabb"][m])
            world.append(wv[f])
            nf = len(f)
            tri_slot.append(np.full(nf, n)); tri_face.append(np.arange(nf)); tri_model.append(np.full(nf, m))
        fl_min = None
        if floors is not None:
            off, tris = floors
            ft = np.asarray(tris, np.float64).reshape(-1, 3, 3)[off[b]:off[b + 1]]
            if len(ft):
                world.append(ft)
                tri_slot.append(np.full(len(ft), N)); tri_face.append(np.arange(len(ft)))
                tri_model.append(np.full(len(ft), -1))
                fl_min = ft.reshape(-1, 3).min(0)
        bg = 255 if white_background else 0
        img[b] = bg
        if not world:
            continue
        wt = np.concatenate(world)                                   # [T, 3 corners, 3]
        slot, face, model = np.concatenate(tri_slot), np.concatenate(tri_face), np.concatenate(tri_model)
        tid = (slot.astype(np.int64) << FACE_SHIFT) | face
        sc = wt @ Mp[:, :3].T + Mp[:, 3]                             # [T, 3, (x, y, d)]
        x, y, d = sc[..., 0], sc[..., 1], sc[..., 2]
        area = (x[:, 2] - x[:, 0]) * (y[:, 1] - y[:, 0]) - (y[:, 2] - y[:, 0]) * (x[:, 1] - x[:, 0])   # edge 0->1 at v2
        # candidate pixels: centres within edge_tol of each triangle's bounding box
        x0 = np.clip(np.ceil(x.min(1) - 0.5 - edge_tol), 0, W).astype(np.int64)
        x1 = np.clip(np.floor(x.max(1) - 0.5 + edge_tol), -1, W - 1).astype(np.int64)
        y0 = np.clip(np.ceil(y.min(1) - 0.5 - edge_tol), 0, H).astype(np.int64)
        y1 = np.clip(np.floor(y.max(1) - 0.5 + edge_tol), -1, H - 1).astype(np.int64)
        cw, ch = np.maximum(x1 - x0 + 1, 0), np.maximum(y1 - y0 + 1, 0)
        cnt = cw * ch
        T = np.repeat(np.arange(len(wt)), cnt)
        if T.size == 0:
            continue
        loc = np.arange(T.size) - np.repeat(np.cumsum(cnt) - cnt, cnt)
        px = x0[T] + loc % cw[T]
        py = y0[T] + loc // cw[T]
        cx, cy = px + 0.5, py + 0.5
        sg = np.where(area[T] >= 0, 1.0, -1.0)
        e = np.zeros((T.size, 3))
        dist = np.zeros((T.size, 3))
        owns = np.zeros((T.size, 3), bool)
        for k in range(3):
            a_, b_ = (k + 1) % 3, (k + 2) % 3
            ax_, ay_, bx_, by_ = x[T, a_], y[T, a_], x[T, b_], y[T, b_]
            e[:, k] = sg * ((cx - ax_) * (by_ - ay_) - (cy - ay_) * (bx_ - ax_))
            ln = np.hypot(bx_ - ax_, by_ - ay_)
            dist[:, k] = np.where(ln > 0, e[:, k] / np.where(ln > 0, ln, 1), 0.0)
            dx, dy = sg * (bx_ - ax_), sg * (by_ - ay_)
            owns[:, k] = (dy > 0) | ((dy == 0) & (dx < 0))
        degen = np.abs(area[T]) < 1e-6
        inside = ((e > 0) | ((e == 0) & owns)).all(1) & ~degen
        near_edge = (dist > -edge_tol).all(1) & ((np.abs(dist) < edge_tol).any(1) | degen)
        w = e / np.where(degen, 1.0, np.abs(area[T]))[:, None]
        dep = (w * d[T]).sum(1)
        clip_near = (np.abs(dep - cam.near) < depth_tol) | (np.abs(dep - cam.far) < depth_tol)
        in_range = (dep >= cam.near) & (dep <= cam.far)
        win_c = inside & in_range
        pix = py * W + px
        best_d = np.full(H * W, np.inf)
        best_i = np.full(H * W, -1, np.int64)
        best_t = np.full(H * W, -1, np.int64)
        if win_c.any():
            order = np.lexsort((tid[T[win_c]], dep[win_c], pix[win_c]))
            P = pix[win_c][order]
            first = np.r_[True, P[1:] != P[:-1]]
            sel = np.flatnonzero(win_c)[order][first]
            best_d[pix[sel]], best_i[pix[sel]], best_t[pix[sel]] = dep[sel], tid[T[sel]], T[sel]
        bd = best_d[pix]
        could = dep <= bd + depth_tol
        flag = could & (near_edge | (clip_near & inside))
        flag |= win_c & could & (tid[T] != best_i[pix])
        a = np.zeros(H * W, bool)
        a[pix[flag]] = True
        amb[b] = a.reshape(H, W)
        ids[b] = best_i.reshape(H, W)
        # shading of the winners
        hit = np.flatnonzero(best_t >= 0)
        t_ = best_t[hit]
        hy, hx = hit // W + 0.5, hit % W + 0.5
        ww = np.zeros((hit.size, 3))
        sgh = np.where(area[t_] >= 0, 1.0, -1.0)
        for k in range(3):
            a_, b_ = (k + 1) % 3, (k + 2) % 3
            ww[:, k] = sgh * ((hx - x[t_, a_]) * (y[t_, b_] - y[t_, a_]) - (hy - y[t_, a_]) * (x[t_, b_] - x[t_, a_]))
        ww /= np.abs(area[t_])[:, None]
        pw = (ww[:, :, None] * wt[t_]).sum(1)
        nrm = np.cross(wt[t_, 1] - wt[t_, 0], wt[t_, 2] - wt[t_, 0])
        l = np.asarray(cam.eye, np.float64) - pw
        den = np.linalg.norm(nrm, axis=1) * np.linalg.norm(l, axis=1)
        cosang = np.where(den > 0, np.minimum(np.abs((nrm * l).sum(1)) / np.where(den > 0, den, 1), 1.0), 0.0)
        shade = AMBIENT + DIFFUSE * cosang
        base = np.ones((hit.size, 3))
        obj = slot[t_] < N
        if no_texture:
            ci = np.asarray(class_index, np.int64).reshape(B, N)[b, slot[t_][obj]]
            base[obj] = np.asarray(palette, np.float32).astype(np.float64)[ci]
        else:
            for j in np.flatnonzero(obj):
                m, f = model[t_[j]], face[t_[j]]
                uv = np.asarray(cat["uvs"][fo[m] + f], np.float64)
                c = np.ones(3)
                if not np.isnan(uv[0, 0]):
                    c = _bilinear(np.asarray(cat["textures"][m]), ww[j] @ uv[:, 0], ww[j] @ uv[:, 1])
                base[j] = c * np.asarray(cat["kd"][m], np.float32).astype(np.float64)
        if floor_texture_index is not None and floor_texture_index[b] >= 0 and fl_min is not None:
            fl = ~obj
            u = (pw[fl, 0] - fl_min[0]) / 0.3
            v = (pw[fl, 2] - fl_min[2]) / 0.3
            base[fl] = _bilinear(np.asarray(floor_textures[floor_texture_index[b]]), u, v)
        col = np.rint(np.clip(base * shade[:, None], 0, 1) * 255).astype(np.uint8)
        flat = img[b].reshape(-1, 3)
        flat[hit] = col
    return img, ids, amb
