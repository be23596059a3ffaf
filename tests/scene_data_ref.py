"""numpy restatement of the reference's cached training chain with explicit draws, for tests of
diffuscene_b200.scene_data.

One sample follows scene_synthesis/datasets/threed_front_dataset.py in its order and with its numpy dtypes:
RotationAugmentation / Jitter in the configured order (:313-371, :559-567), then Scale (:375-401) or
Scale_CosinAngle_ObjfeatsNorm (:481-513), then Permutation (:570-584) and Diffusion's padding (:888-925).  Each step is
the same numpy expression the reference evaluates, so float64 and float32 roundings fall where they fall there.
The layout rotation is np.rot90, which scipy.ndimage.rotate(reshape=False) equals at right angles.
"""
import numpy as np

TWO_PI = 2 * np.pi


def _rotate(sp, theta, angle_lo):
    R = np.zeros((3, 3))
    R[0, 0] = np.cos(theta)
    R[0, 2] = -np.sin(theta)
    R[2, 0] = np.sin(theta)
    R[2, 2] = np.cos(theta)
    R[1, 1] = 1.
    for k, v in sp.items():
        if k == "translations":
            sp[k] = v.dot(R)
        elif k == "angles":
            sp[k] = (v + theta - angle_lo) % TWO_PI + angle_lo
        elif k == "room_layout":
            q = int(round(theta / (np.pi / 2))) % 4
            assert abs(theta - q * np.pi / 2) < 1e-12, "layouts rotate by right angles only: %r" % theta
            sp[k] = np.ascontiguousarray(np.rot90(v, q, axes=(1, 2)))


def _scale(x, lo, hi):
    X = x.astype(np.float32)
    X = np.clip(X, lo, hi)
    X = ((X - lo) / (hi - lo))
    return 2 * X - 1


def sample(room, encoding, augmentations, bounds, max_length, theta=0.0, jitter=(0.0, 0.0, 0.0), ordering=None,
           permute_objfeats=None):
    """The Diffusion sample of `room` (a dict as CachedThreedFront.get_room_params returns it: class_labels [L, C+2],
    translations, sizes, angles [L, 1], objfeat keys, optional room_layout [1, H, W] fp32) for `encoding` and
    `augmentations` (names, in order), with the draws made explicit: the rotation angle, the three jitter values
    (translations, sizes, angles) and the permutation `ordering` (new row j = old row ordering[j]).
    permute_objfeats=None follows the reference (objfeats move only when "objfeats" is in the encoding name); True
    moves them with the boxes.  bounds: fp64 (lo, hi) per key and (std, lo, hi) per objfeat key."""
    sp = {k: np.copy(v) for k, v in room.items()}
    for aug in augmentations:
        if aug in ("rotations", "fixed_rotations"):
            _rotate(sp, theta, bounds["angles"][0])
        elif aug == "jitter":
            j = iter(jitter)
            for k in list(sp):
                if k in ("translations", "sizes", "angles"):
                    sp[k] = sp[k] + float(next(j))      # a Python float, as np.random.normal returns
        else:
            raise ValueError(aug)
    cosin = "cosin_angle" in encoding or "objfeatsnorm" in encoding
    for k, v in sp.items():
        if k == "angles" and cosin:
            sp[k] = np.concatenate([np.cos(v), np.sin(v)], axis=-1)
        elif k in ("objfeats", "objfeats_32"):
            if cosin:
                sp[k] = _scale(v, bounds[k][1], bounds[k][2])
        elif k in ("translations", "sizes", "angles"):
            sp[k] = _scale(v, bounds[k][0], bounds[k][1])
    if "wocm_no_prm" not in encoding:
        keys = ["class_labels", "translations", "sizes", "angles"]
        if permute_objfeats or (permute_objfeats is None and "objfeats" in encoding):
            keys += [k for k in ("objfeats_32", "objfeats") if k in sp and
                     (permute_objfeats or ("lat32" in encoding) == (k == "objfeats_32"))]
        for k in keys:
            sp[k] = sp[k][ordering]
    out = {"length": sp["class_labels"].shape[0]}
    for k, v in sp.items():
        if k == "room_layout":
            out[k] = v
        elif k == "class_labels":
            c = np.concatenate([v[:, :-2], v[:, -1:]], axis=-1)
            L, C = c.shape
            out[k] = np.vstack([c, np.tile(np.eye(C)[-1][None, :], [max_length - L, 1])]).astype(np.float32) * 2.0 - 1.0
        else:
            L, C = v.shape
            out[k] = np.vstack([v, np.tile(np.zeros(C)[None, :], [max_length - L, 1])]).astype(np.float32)
    return out


def ordering_from_keys(keys, L):
    """The permutation ds_scene_batch applies for perm_key: slot j holds the object of rank j (ties by index)."""
    return np.argsort(np.asarray(keys[:L]), kind="stable")


def keys_from_ordering(ordering, N):
    """perm_key [N] fp32 under which ds_scene_batch applies `ordering`."""
    k = np.zeros(N, np.float32)
    k[np.asarray(ordering)] = np.arange(len(ordering), dtype=np.float32)
    return k


# ---- readers of tests/golden/scene_data.npz (tests/golden/make_golden_scene_data.py describes its layout) ----------

def golden_rooms(z, d, layout_size=None):
    """The rooms of golden dataset `d` as get_room_params returns them (objfeats_32 only); with `layout_size`, their
    room_layout resized to it as CachedThreedFront does, [1, H, W]."""
    from diffuscene_b200.scene_data import room_layout
    lengths = z[d + "/lengths"]
    off = np.concatenate([[0], np.cumsum(lengths)])
    rooms = []
    for r in range(len(lengths)):
        sl = slice(off[r], off[r + 1])
        room = {"room_layout": room_layout({"room_layout": z[d + "/room_layout"][r]}, layout_size)[None]} \
            if layout_size else {}
        room.update({k: z["%s/%s" % (d, k)][sl] for k in ("class_labels", "translations", "sizes", "angles",
                                                             "objfeats_32")})
        rooms.append(room)
    return rooms


def golden_draws(z, c, i):
    """(theta, jitter, ordering) of item i of golden case c: 0.0, zeros and None where nothing was drawn."""
    theta = float(z[c + "/theta"][i])
    jitter = z[c + "/normal"][i]
    perm = z[c + "/perm"][i]
    perm = perm[perm >= 0]
    return (0.0 if np.isnan(theta) else theta, np.zeros(3) if np.isnan(jitter).all() else jitter,
            perm if perm.size else None)


def golden_out(z, c, i):
    """The reference's sample i of golden case c; room_layout unpacked from its uint8 form."""
    pre = c + "/out/"
    out = {k[len(pre):]: z[k][i] for k in z.files if k.startswith(pre)}
    if "room_layout_u8" in out:
        out["room_layout"] = out.pop("room_layout_u8").astype(np.float32) / np.float32(255)
    return out
