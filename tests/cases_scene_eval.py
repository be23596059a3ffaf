"""Scenes of the scene-evaluation goldens (tests/golden/make_golden_scene_eval.py) and seeded meshes for the
placement tests.  A case is (bounds [n, 6] float64 as (x1, y1, z1, x2, y2, z2), classes [n] int, jids [n] int)."""
import numpy as np


def _case(boxes, classes, jids):
    return (np.asarray(boxes, np.float64).reshape(-1, 6), np.asarray(classes, np.int64).reshape(-1),
            np.asarray(jids, np.int64).reshape(-1))


def random_scene(rng, n, n_classes=6, room=(3.0, 1.5, 3.0), mirror=0.3):
    """n boxes in a room; a share of them copies an earlier object mirrored in x (same class and model), some with a
    small size jitter, so that symmetric pairs occur on both sides of the 0.1 thresholds."""
    half = rng.uniform(0.05, 0.9, (n, 3))
    centre = rng.uniform(-1, 1, (n, 3)) * np.asarray(room)
    centre[:, 1] = half[:, 1] + rng.uniform(0, 0.5, n)
    classes = rng.integers(0, n_classes, n)
    jids = rng.integers(0, 3, n) + 10 * classes
    for i in range(1, n):
        if rng.uniform() < mirror:
            j = int(rng.integers(0, i))
            half[i] = half[j] + rng.choice([0.0, 0.04, 0.12]) * rng.uniform(-1, 1, 3)
            centre[i] = centre[j] * [-1, 1, 1] + rng.choice([0.0, 0.05, 0.2]) * rng.uniform(-1, 1, 3)
            classes[i], jids[i] = classes[j], jids[j]
    half = np.abs(half)
    return _case(np.concatenate([centre - half, centre + half], 1), classes, jids)


def golden_cases():
    rng = np.random.default_rng(20261017)
    c = {}
    c["empty"] = _case(np.zeros((0, 6)), [], [])
    c["one"] = _case([[0, 0, 0, 1, 1, 1]], [3], [7])
    c["two"] = _case([[0, 0, 0, 1, 1, 1], [0.5, 0.25, 0.5, 1.5, 1.25, 1.5]], [1, 2], [1, 2])
    c["touching"] = _case([[0, 0, 0, 1, 1, 1], [1, 0, 0, 2, 1, 1], [0, 1, 0, 1, 2, 1], [2.5, 0, 0, 3, 1, 0.7]],
                          [0, 0, 0, 1], [5, 5, 5, 6])
    c["nested"] = _case([[0, 0, 0, 2, 2, 2], [0.5, 0.5, 0.5, 1.5, 1.5, 1.5], [0, 0, 0, 2, 2, 2],
                         [0.5, 0.5, 0.5, 1.5, 1.5, 1.5]], [4, 4, 4, 4], [9, 9, 9, 9])
    # sizes and centres differing by just under / just over 0.1 (half sizes: the threshold is on half extents)
    e = 1e-6
    c["sym_edge"] = _case([[0, 0, 0, 2, 1, 1], [0.1 - e, 0, 3, 2.1 - e, 1, 4], [0.1 + e, 0, 6, 2.1 + e, 1, 7],
                           [5, 0, 0, 6, 1, 1], [5, 0, 2, 6.2 - 2 * e, 1, 3], [5, 0, 5, 6.2 + 2 * e, 1, 6],
                           [9, 0, 0, 10, 1, 1], [11, 0, 0.1 - e, 12, 1, 1.1 - e]],
                          [2, 2, 2, 3, 3, 3, 5, 5], [4, 4, 4, 6, 6, 6, 8, 8])
    c["same_class_other_model"] = _case([[0, 0, 0, 1, 1, 1], [3, 0, 0, 4, 1, 1], [0, 0, 3, 1, 1, 4]],
                                        [1, 1, 1], [10, 11, 10])
    c["zero_volume"] = _case([[0, 0, 0, 1, 0, 1], [0, 0, 0, 1, 1, 1], [0.5, 0, 0.5, 0.5, 1, 0.5]], [0, 1, 2], [0, 1, 2])
    c["zero_area_pair"] = _case([[0, 0, 0, 1, 0, 1], [0, 0, 0, 1, 0, 1]], [0, 0], [0, 0])   # 0 / 0 overlap ratio
    for k in range(6):
        c["living21_%d" % k] = random_scene(rng, 21, n_classes=24, room=(4.0, 1.6, 4.0))
    for k, n in enumerate([2, 3, 5, 12, 12, 17, 33, 48, 64, 64]):
        c["random%d_%d" % (k, n)] = random_scene(rng, n)
    return c


def random_mesh(rng, n_vertices=300):
    """Raw mesh vertices (an off-centre blob with a flat side) and its 8 stored bbox corners in the reference's
    order (corner 4 - 0 spans x, 2 - 0 spans y, 1 - 0 spans z)."""
    v = rng.normal(size=(n_vertices, 3)) * rng.uniform(0.2, 1.5, 3) + rng.uniform(-0.3, 0.3, 3)
    v[v[:, 0] > 0.5, 0] = 0.5
    lo, hi = v.min(0), v.max(0)
    bbox = np.array([[x, y, z] for x in (lo[0], hi[0]) for y in (lo[1], hi[1]) for z in (lo[2], hi[2])])
    return v, bbox
