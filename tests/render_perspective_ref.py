"""fp64 numpy reference of ds_render_scenes with a perspective camera (the tests' oracle for that path).

It follows oracle.render_ref's rules and reuses its camera, placement and texture helpers; what differs:

  * pixel map: pyrr's create_look_at x create_perspective_projection_from_bounds, then the viewport.  `pixel_map`
    returns the homogeneous rows (pixel x * depth, pixel y * depth, depth), depth = -z_view;
  * near-plane clipping in view space: a face crossing depth = near becomes at most two triangles whose corners carry
    barycentrics of the original face (so ids and UVs refer to its corners); a face wholly behind draws nothing;
  * perspective-correct interpolation: 1 / depth is linear in screen space, and the face barycentrics of a pixel are
    the screen barycentrics weighted by 1 / depth.

`ambiguous` extends to this path: the edge distance is in pixels after the divide (clip edges included, the diagonal
that splits a clipped quad excluded), and the depth tolerance is relative to depth (1e-5 by default; the fp32 depth
of ds_render_scenes is good to about 1e-6 relative).
"""
from __future__ import annotations

import numpy as np

from oracle import render_ref as RR


def perspective_projection_from_bounds(left, right, bottom, top, near, far) -> np.ndarray:
    """pyrr.matrix44.create_perspective_projection_from_bounds (row-vector convention)."""
    A = (right + left) / (right - left)
    B = (top + bottom) / (top - bottom)
    C = -(far + near) / (far - near)
    D = -2.0 * far * near / (far - near)
    E = 2.0 * near / (right - left)
    F = 2.0 * near / (top - bottom)
    return np.array([[E, 0, 0, 0], [0, F, 0, 0], [A, B, C, -1.0], [0, 0, D, 0]], np.float64)


def pixel_map(cam) -> np.ndarray:
    """3 x 4 fp64 map world -> (pixel x * w, array row * w, w), w = clip w = depth along the view direction."""
    V = RR.look_at(cam.eye, cam.target, cam.up)
    P = perspective_projection_from_bounds(cam.left, cam.right, cam.bottom, cam.top, cam.near, cam.far)
    VP = V @ P
    col = lambda j: np.r_[VP[:3, j], VP[3, j]]
    w = col(3)
    return np.stack([(col(0) + w) * (cam.width / 2.0), (col(1) + w) * (cam.height / 2.0), w])


ORIG, CLIP, INNER = 0, 1, 2          # kinds of the edges of a clipped triangle (edge k is opposite corner k)


def clip_faces(h: np.ndarray, near: float):
    """Clip homogeneous faces h [T, 3, (X, Y, depth)] at depth = near.  Returns (parent [S], screen [S, 3, 2],
    inverse depth [S, 3], barycentrics [S, 3 corners, 3] in the parent face, edge kinds [S, 3])."""
    inside = h[..., 2] >= near
    nin = inside.sum(1)
    full = np.flatnonzero(nin == 3)
    par = [full]
    scr = [h[full, :, :2] / h[full, :, 2:3]]
    inv = [1.0 / h[full, :, 2]]
    bar = [np.broadcast_to(np.eye(3), (len(full), 3, 3))]
    kind = [np.full((len(full), 3), ORIG)]

    def cut(t_, a, b):
        """(screen point, barycentrics) on edge a -> b (a in front) at depth = near."""
        s = (near - h[t_, a, 2]) / (h[t_, b, 2] - h[t_, a, 2])
        p = (h[t_, a, :2] + s * (h[t_, b, :2] - h[t_, a, :2])) / near
        w = np.zeros(3)
        w[a], w[b] = 1.0 - s, s
        return p, w

    for t_ in np.flatnonzero((nin == 1) | (nin == 2)):
        e = np.eye(3)
        corner = lambda k: (h[t_, k, :2] / h[t_, k, 2], 1.0 / h[t_, k, 2], e[k])
        if nin[t_] == 1:
            i = int(np.flatnonzero(inside[t_])[0])
            j, k = (i + 1) % 3, (i + 2) % 3
            pi, ri, bi = corner(i)
            pj, bj = cut(t_, i, j)
            pk, bk = cut(t_, i, k)
            tris = [((pi, pj, pk), (ri, 1 / near, 1 / near), (bi, bj, bk), (CLIP, ORIG, ORIG))]
        else:
            k = int(np.flatnonzero(~inside[t_])[0])
            i, j = (k + 1) % 3, (k + 2) % 3
            pi, ri, bi = corner(i)
            pj, rj, bj = corner(j)
            pp, bp = cut(t_, j, k)
            pq, bq = cut(t_, i, k)
            tris = [((pi, pj, pp), (ri, rj, 1 / near), (bi, bj, bp), (ORIG, INNER, ORIG)),
                    ((pi, pp, pq), (ri, 1 / near, 1 / near), (bi, bp, bq), (CLIP, ORIG, INNER))]
        for p3, r3, b3, k3 in tris:
            par.append(np.array([t_]))
            scr.append(np.array(p3)[None])
            inv.append(np.array(r3)[None])
            bar.append(np.array(b3)[None])
            kind.append(np.array(k3)[None])
    return (np.concatenate(par).astype(np.int64), np.concatenate(scr).reshape(-1, 3, 2),
            np.concatenate(inv).reshape(-1, 3), np.concatenate(bar).reshape(-1, 3, 3),
            np.concatenate(kind).reshape(-1, 3))


def render(cat, translations, sizes, angles, model_index, cam, class_index=None, floors=None, no_texture=False,
           white_background=False, palette=None, floor_textures=None, floor_texture_index=None, edge_tol=1e-3,
           depth_tol=1e-5):
    """(image uint8 [B, H, W, 3], ids int64 [B, H, W], ambiguous bool [B, H, W]) of a batch seen by a perspective
    `cam`, arguments as oracle.render_ref.render takes them."""
    translations = np.asarray(translations, np.float32)
    B, N = translations.shape[:2]
    sizes = np.asarray(sizes, np.float32).reshape(B, N, 3)
    angles = np.asarray(angles, np.float32).reshape(B, N)
    model_index = np.asarray(model_index, np.int64).reshape(B, N)
    Mp = pixel_map(cam)
    H, W = cam.height, cam.width
    near, far = float(cam.near), float(cam.far)
    img = np.zeros((B, H, W, 3), np.uint8)
    ids = np.full((B, H, W), -1, np.int64)
    amb = np.zeros((B, H, W), bool)
    vo, fo = np.asarray(cat["vertex_offsets"]), np.asarray(cat["face_offsets"])
    for b in range(B):
        world, tri_slot, tri_face, tri_model = [], [], [], []
        for n in range(N):
            m = int(model_index[b, n])
            if m < 0:
                continue
            v = np.asarray(cat["vertices"][vo[m]:vo[m + 1]], np.float64)
            f = np.asarray(cat["faces"][fo[m]:fo[m + 1]], np.int64)
            wv = RR.place(v, sizes[b, n], translations[b, n], angles[b, n], cat["raw_half"][m], cat["raw_aabb"][m])
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
        img[b] = 255 if white_background else 0
        if not world:
            continue
        wt = np.concatenate(world)                                   # [T, 3 corners, 3]
        slot, face, model = np.concatenate(tri_slot), np.concatenate(tri_face), np.concatenate(tri_model)
        tid = (slot.astype(np.int64) << RR.FACE_SHIFT) | face
        h = wt @ Mp[:, :3].T + Mp[:, 3]                              # [T, 3, (X, Y, depth)]
        par, scr, inv, bar, kind = clip_faces(h, near)
        if par.size == 0:
            continue
        x, y = scr[..., 0], scr[..., 1]
        area = (x[:, 2] - x[:, 0]) * (y[:, 1] - y[:, 0]) - (y[:, 2] - y[:, 0]) * (x[:, 1] - x[:, 0])
        with np.errstate(invalid="ignore"):
            x0 = np.clip(np.ceil(x.min(1) - 0.5 - edge_tol), 0, W).astype(np.int64)
            x1 = np.clip(np.floor(x.max(1) - 0.5 + edge_tol), -1, W - 1).astype(np.int64)
            y0 = np.clip(np.ceil(y.min(1) - 0.5 - edge_tol), 0, H).astype(np.int64)
            y1 = np.clip(np.floor(y.max(1) - 0.5 + edge_tol), -1, H - 1).astype(np.int64)
        cw, ch = np.maximum(x1 - x0 + 1, 0), np.maximum(y1 - y0 + 1, 0)
        cnt = cw * ch
        T = np.repeat(np.arange(len(par)), cnt)
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
            # the split of a clipped quad is not an edge, nor is the zero-length edge of a sliver whose clip points
            # coincide
            dist[:, k] = np.where(ln > 0, e[:, k] / np.where(ln > 0, ln, 1), np.inf)
            dist[kind[T, k] == INNER, k] = np.inf
            dx, dy = sg * (bx_ - ax_), sg * (by_ - ay_)
            owns[:, k] = (dy > 0) | ((dy == 0) & (dx < 0))
        degen = np.abs(area[T]) < 1e-6
        inside = ((e > 0) | ((e == 0) & owns)).all(1) & ~degen
        # a degenerate triangle is a segment: only centres within edge_tol of its lines (inside its box) may be drawn
        near_edge = np.where(degen, (np.abs(dist) < edge_tol).any(1),
                             (dist > -edge_tol).all(1) & (np.abs(dist) < edge_tol).any(1))
        l = e / np.where(degen, 1.0, np.abs(area[T]))[:, None]
        with np.errstate(divide="ignore", invalid="ignore"):
            dep = 1.0 / (l * inv[T]).sum(1)
        clip_near = (np.abs(dep - near) < depth_tol * near) | (np.abs(dep - far) < depth_tol * far)
        in_range = (dep >= near) & (dep <= far)
        win_c = inside & in_range
        pix = py * W + px
        sid = tid[par[T]]
        best_d = np.full(H * W, np.inf)
        best_i = np.full(H * W, -1, np.int64)
        best_t = np.full(H * W, -1, np.int64)
        if win_c.any():
            order = np.lexsort((sid[win_c], dep[win_c], pix[win_c]))
            P = pix[win_c][order]
            first = np.r_[True, P[1:] != P[:-1]]
            sel = np.flatnonzero(win_c)[order][first]
            best_d[pix[sel]], best_i[pix[sel]], best_t[pix[sel]] = dep[sel], sid[sel], T[sel]
        bd = best_d[pix]
        could = dep <= bd * (1.0 + depth_tol)
        flag = could & (near_edge | (clip_near & inside))
        flag |= win_c & could & (sid != best_i[pix])
        a = np.zeros(H * W, bool)
        a[pix[flag]] = True
        amb[b] = a.reshape(H, W)
        ids[b] = best_i.reshape(H, W)
        # shading of the winners, at the perspective-correct barycentrics of the original face
        hit = np.flatnonzero(best_t >= 0)
        s_ = best_t[hit]
        t_ = par[s_]
        hy, hx = hit // W + 0.5, hit % W + 0.5
        ll = np.zeros((hit.size, 3))
        sgh = np.where(area[s_] >= 0, 1.0, -1.0)
        for k in range(3):
            a_, b_ = (k + 1) % 3, (k + 2) % 3
            ll[:, k] = sgh * ((hx - x[s_, a_]) * (y[s_, b_] - y[s_, a_]) - (hy - y[s_, a_]) * (x[s_, b_] - x[s_, a_]))
        pc = ll * inv[s_]
        pc /= pc.sum(1, keepdims=True)
        ww = np.einsum("nk,nkj->nj", pc, bar[s_])
        pw = (ww[:, :, None] * wt[t_]).sum(1)
        nrm = np.cross(wt[t_, 1] - wt[t_, 0], wt[t_, 2] - wt[t_, 0])
        lv = np.asarray(cam.eye, np.float64) - pw
        den = np.linalg.norm(nrm, axis=1) * np.linalg.norm(lv, axis=1)
        cosang = np.where(den > 0, np.minimum(np.abs((nrm * lv).sum(1)) / np.where(den > 0, den, 1), 1.0), 0.0)
        shade = RR.AMBIENT + RR.DIFFUSE * cosang
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
                    c = RR._bilinear(np.asarray(cat["textures"][m]), ww[j] @ uv[:, 0], ww[j] @ uv[:, 1])
                base[j] = c * np.asarray(cat["kd"][m], np.float32).astype(np.float64)
        if floor_texture_index is not None and floor_texture_index[b] >= 0 and fl_min is not None:
            fl = ~obj
            u = (pw[fl, 0] - fl_min[0]) / 0.3
            v = (pw[fl, 2] - fl_min[2]) / 0.3
            base[fl] = RR._bilinear(np.asarray(floor_textures[floor_texture_index[b]]), u, v)
        col = np.rint(np.clip(base * shade[:, None], 0, 1) * 255).astype(np.uint8)
        img[b].reshape(-1, 3)[hit] = col
    return img, ids, amb
